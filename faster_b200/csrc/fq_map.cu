// fq_map_* (include/faster_b200.h): the indexed map of the chained replan, uploaded and bucketed on the device (fq_map.h).
// An update copies U then O into one array, finds the grid (one CTA, which also rewrites the map's descriptor), keys every
// point by its cell, sorts each cloud's (cell, index) pairs with CUB's stable radix sort, gathers the sorted points and
// finds every cell's first point.
#include "fq_ctx.h"

#include <cub/device/device_radix_sort.cuh>

#include <cmath>

struct fq_map
{
  int device = 0;
  int n_occ = 0, n_unk = 0;
  long long cap = 0;                // points (U and O together) the arrays hold
  long long cell_cap = 0;           // cells one start array holds: fq_map_cell_limit(cap)
  bool valid = true;                // false after a failed update, until the next one succeeds
  FqMapDev* desc = nullptr;         // device: what submissions read (fq_map.h); one address for the map's life
  int* empty = nullptr;             // device: 2 zeros, the cell starts of the empty descriptor a failed update leaves
  double* raw = nullptr;            // cap x 3: U then O, as given
  double* xyz = nullptr;            // cap x 3: U sorted, then O sorted
  unsigned *key = nullptr, *key_s = nullptr;
  int *idx_in = nullptr, *idx = nullptr;
  int* start = nullptr;             // 2 x (cell_cap + 1): U's cell starts, then O's
  void* tmp = nullptr;
  size_t tmp_bytes = 0;
};

namespace
{
constexpr int kGridThreads = 512;

// origin, cell edge and dims of the map's finite points (bit-equal to the restatement of tests/test_pair_map_cpu.py),
// written with the update's clouds into the map's descriptor
__global__ void __launch_bounds__(kGridThreads) fq_map_grid_kernel(const double* p, int n, double edge, long long limit,
                                                                  const FqMapCloud unk, const FqMapCloud occ, FqMapDev* d)
{
  __shared__ double s_lo[3][kGridThreads], s_hi[3][kGridThreads];
  const int t = threadIdx.x;
  double lo[3] = { INFINITY, INFINITY, INFINITY }, hi[3] = { -INFINITY, -INFINITY, -INFINITY };
  for (int i = t; i < n; i += kGridThreads)
  {
    const double* q = p + 3 * (size_t)i;
    if (!(isfinite(q[0]) && isfinite(q[1]) && isfinite(q[2]))) continue;
    for (int k = 0; k < 3; k++) { lo[k] = fmin(lo[k], q[k]); hi[k] = fmax(hi[k], q[k]); }
  }
  for (int k = 0; k < 3; k++) { s_lo[k][t] = lo[k]; s_hi[k][t] = hi[k]; }
  __syncthreads();
  for (int s = kGridThreads / 2; s > 0; s >>= 1)
  {
    if (t < s)
      for (int k = 0; k < 3; k++) { s_lo[k][t] = fmin(s_lo[k][t], s_lo[k][t + s]); s_hi[k][t] = fmax(s_hi[k][t], s_hi[k][t + s]); }
    __syncthreads();
  }
  if (t != 0) return;
  FqMapGrid r;
  const bool any = s_lo[0][0] <= s_hi[0][0];
  double ext[3], dm[3];
  for (int k = 0; k < 3; k++) { r.origin[k] = any ? s_lo[0 + k][0] : 0.0; ext[k] = any ? s_hi[k][0] - r.origin[k] : 0.0; }
  double cell = edge;
  for (;;)
  {
    for (int k = 0; k < 3; k++) dm[k] = floor(ext[k] / cell) + 1;
    if (dm[0] * dm[1] * dm[2] <= (double)limit) break;
    cell *= 2;
  }
  r.cell = cell;
  for (int k = 0; k < 3; k++) r.dims[k] = (int)dm[k];
  r.n_cells = r.dims[0] * r.dims[1] * r.dims[2];
  d->grid = r;
  d->unk = unk;
  d->occ = occ;
}

// every point's cell (n_cells: not finite) and its index in its cloud (U: 0 .. n_unk-1, O: 0 .. n_occ-1)
__global__ void fq_map_key_kernel(const double* p, int n, int n_unk, const FqMapGrid* gp, unsigned* key, int* idx)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const FqMapGrid g = *gp;
  const double* q = p + 3 * (size_t)i;
  unsigned c = (unsigned)g.n_cells;
  if (isfinite(q[0]) && isfinite(q[1]) && isfinite(q[2]))
  {
    const int x = fq_map_axis(q[0], g.origin[0], g.cell, g.dims[0]), y = fq_map_axis(q[1], g.origin[1], g.cell, g.dims[1]);
    const int z = fq_map_axis(q[2], g.origin[2], g.cell, g.dims[2]);
    c = (unsigned)((z * g.dims[1] + y) * g.dims[0] + x);
  }
  key[i] = c;
  idx[i] = i < n_unk ? i : i - n_unk;
}

// the sorted points: position i of U (i < n_unk) or of O
__global__ void fq_map_gather_kernel(const double* p, int n, int n_unk, const int* idx, double* xyz)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t src = (size_t)idx[i] + (i < n_unk ? 0 : n_unk);
  for (int k = 0; k < 3; k++) xyz[3 * (size_t)i + k] = p[3 * src + k];
}

// start[c] = the first sorted position whose cell is >= c, for c = 0 .. n_cells
__global__ void fq_map_start_kernel(const unsigned* key, int n, const FqMapGrid* gp, long long cells, int* start)
{
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c > cells || c > gp->n_cells) return;
  int lo = 0, hi = n;
  while (lo < hi)
  {
    const int mid = lo + (hi - lo) / 2;
    if ((long long)key[mid] < c) lo = mid + 1; else hi = mid;
  }
  start[c] = lo;
}

int end_bit(long long limit)
{
  int b = 1;
  while ((1LL << b) <= limit) b++;
  return b;
}

void release(fq_map* m)
{
  for (void* p : { (void*)m->raw, (void*)m->xyz, (void*)m->key, (void*)m->key_s, (void*)m->idx_in, (void*)m->idx, (void*)m->start, m->tmp })
    if (p) cudaFree(p);
  m->raw = m->xyz = nullptr; m->key = m->key_s = nullptr; m->idx_in = m->idx = m->start = nullptr; m->tmp = nullptr;
  m->cap = m->cell_cap = 0; m->tmp_bytes = 0;
}

cudaError_t reserve(fq_map* m, long long n)
{
  if (m->start && n <= m->cap) return cudaSuccess;   // (a new map has no arrays yet, even for no points)
  release(m);
  const long long cap = n + n / 4 + 1024, cells = fq_map_cell_limit(cap);
  cudaError_t e = cudaSuccess;
  auto get = [&](auto** p, size_t count) { if (e == cudaSuccess) e = cudaMalloc((void**)p, sizeof(**p) * count); };
  get(&m->raw, 3 * cap); get(&m->xyz, 3 * cap); get(&m->key, cap); get(&m->key_s, cap); get(&m->idx_in, cap); get(&m->idx, cap);
  get(&m->start, 2 * (cells + 1));
  if (e == cudaSuccess)
    e = cub::DeviceRadixSort::SortPairs(nullptr, m->tmp_bytes, m->key, m->key_s, m->idx_in, m->idx, (int)cap, 0, end_bit(cells));
  if (e == cudaSuccess) e = cudaMalloc(&m->tmp, m->tmp_bytes);
  if (e != cudaSuccess) { release(m); return e; }
  m->cap = cap;
  m->cell_cap = cells;
  return cudaSuccess;
}

const char* check_counts(const fq_map* m, const void* occ, int n_occ, const void* unk, int n_unk)
{
  if (!m) return "map is NULL";
  if (n_occ < 0 || n_unk < 0) return "map: negative point count";
  if ((long long)n_occ + n_unk > (1LL << 30)) return "map: more than 2^30 points";
  if ((n_occ > 0 && !occ) || (n_unk > 0 && !unk)) return "map: NULL cloud with a positive count";
  return nullptr;
}

// the update itself; `kind`: where the clouds are
int build_index(fq_map* m, const double* occ, int n_occ, const double* unk, int n_unk, cudaMemcpyKind kind, cudaStream_t st)
{
  fq_ctx* ctx = nullptr;                        // errors go to fq_last_error(NULL)
  FQ_CUDA(cudaSetDevice(m->device));
  const int n = n_occ + n_unk;
  FQ_CUDA(reserve(m, n));
  if (n_unk) FQ_CUDA(cudaMemcpyAsync(m->raw, unk, sizeof(double) * 3 * (size_t)n_unk, kind, st));
  if (n_occ) FQ_CUDA(cudaMemcpyAsync(m->raw + 3 * (size_t)n_unk, occ, sizeof(double) * 3 * (size_t)n_occ, kind, st));
  const long long limit = fq_map_cell_limit(n);
  const FqMapCloud cu = { m->xyz, m->idx, m->start, n_unk };
  const FqMapCloud co = { m->xyz + 3 * (size_t)n_unk, m->idx + n_unk, m->start + m->cell_cap + 1, n_occ };
  fq_map_grid_kernel<<<1, kGridThreads, 0, st>>>(m->raw, n, FQ_MAP_CELL_EDGE, limit, cu, co, m->desc);
  FQ_CUDA(cudaGetLastError());
  const FqMapGrid* grid = &m->desc->grid;
  const int T = 256;
  if (n > 0)
  {
    fq_map_key_kernel<<<(n + T - 1) / T, T, 0, st>>>(m->raw, n, n_unk, grid, m->key, m->idx_in);
    FQ_CUDA(cudaGetLastError());
    const int bits = end_bit(limit);
    size_t bytes = m->tmp_bytes;
    if (n_unk) FQ_CUDA(cub::DeviceRadixSort::SortPairs(m->tmp, bytes, m->key, m->key_s, m->idx_in, m->idx, n_unk, 0, bits, st));
    bytes = m->tmp_bytes;
    if (n_occ)
      FQ_CUDA(cub::DeviceRadixSort::SortPairs(m->tmp, bytes, m->key + n_unk, m->key_s + n_unk, m->idx_in + n_unk, m->idx + n_unk,
                                              n_occ, 0, bits, st));
    fq_map_gather_kernel<<<(n + T - 1) / T, T, 0, st>>>(m->raw, n, n_unk, m->idx, m->xyz);
    FQ_CUDA(cudaGetLastError());
  }
  const unsigned blocks = (unsigned)((limit + 1 + T - 1) / T);
  fq_map_start_kernel<<<blocks, T, 0, st>>>(m->key_s, n_unk, grid, limit, m->start);
  fq_map_start_kernel<<<blocks, T, 0, st>>>(m->key_s + n_unk, n_occ, grid, limit, m->start + m->cell_cap + 1);
  FQ_CUDA(cudaGetLastError());
  m->n_occ = n_occ;
  m->n_unk = n_unk;
  return 0;
}

// an update; when it fails (an allocation, a launch) the map holds no points, its descriptor is the empty map's, so that
// nothing that still reads it can reach freed memory, and submissions refuse it until an update succeeds
int build(fq_map* m, const double* occ, int n_occ, const double* unk, int n_unk, cudaMemcpyKind kind, cudaStream_t st)
{
  const int rc = build_index(m, occ, n_occ, unk, n_unk, kind, st);
  m->valid = rc == 0;
  if (rc)
  {
    m->n_occ = m->n_unk = 0;
    FqMapDev d{};
    d.grid.cell = FQ_MAP_CELL_EDGE;
    d.grid.dims[0] = d.grid.dims[1] = d.grid.dims[2] = d.grid.n_cells = 1;
    d.unk = d.occ = { nullptr, nullptr, m->empty, 0 };
    cudaMemcpy(m->desc, &d, sizeof(d), cudaMemcpyHostToDevice);
  }
  return rc;
}
}  // namespace

const FqMapDev* fq_map_descriptor(const fq_map* m) { return m->desc; }
int fq_map_device(const fq_map* m) { return m->device; }
bool fq_map_valid(const fq_map* m) { return m->valid; }

extern "C" int fq_map_create(fq_map** out, int device)
{
  fq_ctx* ctx = nullptr;
  if (!out) return fq_fail(nullptr, FQ_E_ARG, "out is NULL");
  *out = nullptr;
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev <= 0) return fq_fail(nullptr, FQ_E_NOGPU, "no CUDA device");
  if (device < 0 || device >= n_dev) return fq_fail(nullptr, FQ_E_ARG, "device out of range");
  fq_map* m = new fq_map;
  m->device = device;
  FQ_CUDA(cudaSetDevice(device));
  cudaError_t e = cudaMalloc(&m->desc, sizeof(FqMapDev));
  if (e == cudaSuccess) e = cudaMalloc(&m->empty, 2 * sizeof(int));
  if (e == cudaSuccess) e = cudaMemset(m->empty, 0, 2 * sizeof(int));
  int rc = e == cudaSuccess ? build(m, nullptr, 0, nullptr, 0, cudaMemcpyHostToDevice, 0) : fq_cuda_fail(nullptr, e, "cudaMalloc");
  if (!rc && (e = cudaStreamSynchronize(0)) != cudaSuccess) rc = fq_cuda_fail(nullptr, e, "cudaStreamSynchronize");
  if (rc) { fq_map_destroy(m); return rc; }
  *out = m;
  return 0;
}

extern "C" void fq_map_destroy(fq_map* m)
{
  if (!m) return;
  cudaSetDevice(m->device);
  release(m);
  if (m->desc) cudaFree(m->desc);
  if (m->empty) cudaFree(m->empty);
  delete m;
}

extern "C" int fq_map_update(fq_map* m, const double* occ, int n_occ, const double* unk, int n_unk)
{
  fq_ctx* ctx = nullptr;
  if (const char* why = check_counts(m, occ, n_occ, unk, n_unk)) return fq_fail(nullptr, FQ_E_ARG, why);
  const struct { const double* p; int n; } clouds[2] = { { occ, n_occ }, { unk, n_unk } };
  for (const auto& c : clouds)
    for (size_t i = 0; i < 3 * (size_t)c.n; i++)
      if (!std::isfinite(c.p[i])) return fq_fail(nullptr, FQ_E_ARG, "map: non-finite coordinate");
  if (int rc = build(m, occ, n_occ, unk, n_unk, cudaMemcpyHostToDevice, 0)) return rc;
  FQ_CUDA(cudaStreamSynchronize(0));
  return 0;
}

extern "C" int fq_map_update_dev(fq_map* m, const double* d_occ, int n_occ, const double* d_unk, int n_unk, void* stream)
{
  if (const char* why = check_counts(m, d_occ, n_occ, d_unk, n_unk)) return fq_fail(nullptr, FQ_E_ARG, why);
  return build(m, d_occ, n_occ, d_unk, n_unk, cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
}

extern "C" int fq_map_size(const fq_map* m, int* n_occ, int* n_unk)
{
  if (!m) return fq_fail(nullptr, FQ_E_ARG, "map is NULL");
  if (n_occ) *n_occ = m->n_occ;
  if (n_unk) *n_unk = m->n_unk;
  return 0;
}
