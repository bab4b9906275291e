// fq_map_paths*, fq_paths_cloud and fq_jps_in (include/faster_b200.h): each corridor's whole and safe paths from its JPS_in,
// the safe one cropped where the path first nears the unknown space of its map (Faster::getFirstCollisionJPS,
// faster.cpp:767-921).  The arithmetic is fq_paths.h's, shared by the host twin over clouds and the device over maps.
//
// Device route: fq_paths_crop_kernel (one CTA per corridor: thread 0 marches the head, the CTA finds the nearest unknown
// point of each step in the map cells within range), then fq_paths_write_kernel (one CTA: the offsets of both paths and
// their rows).  Scratch -- each corridor's crop and the map table -- is stream-ordered memory, so the device entry never
// synchronises and a CUDA graph can capture it.
#include "fq_ctx.h"
#include "fq_paths.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

namespace
{
using fqpath::Crop;
constexpr int kThreads = 256;

struct CropArgs
{
  int n_prob, max_in, n_maps;
  const int* in_ofs;
  const double* in;
  const FqMapDev* const* maps;
  const int* map_index;
  double drone_radius;
  Crop* crop;
  int* status;
  uint8_t* crossed;
};

__global__ void __launch_bounds__(kThreads) fq_paths_crop_kernel(const CropArgs a)
{
  extern __shared__ double s_in[];                 // the corridor's JPS_in, max_in x 3
  __shared__ float s_q[3];
  __shared__ int s_c0[3], s_c1[3];
  __shared__ unsigned s_min;
  const int j = blockIdx.x, tid = threadIdx.x;
  if (j >= a.n_prob) return;
  const int b = a.in_ofs[j], n = a.in_ofs[j + 1] - b;
  const int map = a.map_index ? a.map_index[j] : 0;
  int st = n < 2 ? FQ_PATHS_SHORT : (b < 0 || n > a.max_in ? FQ_PATHS_INPUT : (map < 0 || map >= a.n_maps ? FQ_PATHS_MAP : FQ_PATHS_OK));
  if (st == FQ_PATHS_OK)
  {
    int bad = 0;
    for (int i = tid; i < 3 * n; i += kThreads)
    {
      const double v = a.in[3 * (size_t)b + i];
      s_in[i] = v;
      bad |= !isfinite(v);
    }
    if (__syncthreads_or(bad)) st = FQ_PATHS_INPUT;
  }
  Crop c{};
  if (st == FQ_PATHS_OK)
  {
    const FqMapDev* M = a.maps[map];
    const FqMapGrid g = M->grid;
    const FqMapCloud U = M->unk;
    fqpath::March mr(s_in);                        // thread 0's march; the CTA only scans
    const int warp = tid >> 5, lane = tid & 31;
    for (int it = 0;; it++)
    {
      if (it == fqpath::kMaxSteps) { st = FQ_PATHS_STALL; break; }
      if (tid == 0)
      { // the cells that can hold a point closer than R = max(drone_radius, farthest vertex left) to q, widened by a bound on
        // the float rounding of the point and of the distance ((|q| + R) 2^-20, far above it) and by one cell
        float q[3];
        mr.query(q);
        const double R = mr.need(s_in, n, a.drone_radius);
        double lo[3], hi[3];
        bool finite = true;
        for (int k = 0; k < 3; k++)
        {
          const double r = R + (fabs((double)q[k]) + R) * 0x1p-20;
          lo[k] = (double)q[k] - r; hi[k] = (double)q[k] + r;
          s_q[k] = q[k];
          finite = finite && isfinite(lo[k]) && isfinite(hi[k]);
        }
        int c0[3], c1[3];
        fq_map_range(g, lo, hi, c0, c1);
        for (int k = 0; k < 3; k++) { s_c0[k] = c0[k] > 0 ? c0[k] - 1 : 0; s_c1[k] = c1[k] < g.dims[k] - 1 ? c1[k] + 1 : g.dims[k] - 1; }
        // At large coordinates the reference's float intersection can put the head at NaN or infinity (a and b of the
        // quadratic round to 0).  Every distance from it is then NaN or infinite, so the step ends the crop whatever the
        // nearest point: no cells are read (the cell of a NaN coordinate is undefined).
        if (!finite) { s_c0[2] = 1; s_c1[2] = 0; }
        s_min = ~0u;
      }
      __syncthreads();
      if (U.n > 0)
      { // the smallest float d^2 as unsigned bits (non-negative floats order as their bits): one warp per row of cells
        const float q[3] = { s_q[0], s_q[1], s_q[2] };
        const int c0[3] = { s_c0[0], s_c0[1], s_c0[2] }, c1[3] = { s_c1[0], s_c1[1], s_c1[2] };
        const int rows = (c1[1] - c0[1] + 1) * (c1[2] - c0[2] + 1);
        unsigned m = ~0u;
        for (int r = warp; r < rows; r += kThreads / 32)
        {
          int pb, pe;
          fq_map_row(g, U, c0, c1, r, &pb, &pe);
          for (int p = pb + lane; p < pe; p += 32)
          {
            const unsigned v = __float_as_uint(fqp::flann_l2(q, U.xyz + 3 * (size_t)p));
            m = v < m ? v : m;
          }
        }
        m = __reduce_min_sync(0xffffffffu, m);
        if (lane == 0 && m != ~0u) atomicMin(&s_min, m);
      }
      __syncthreads();
      // no point in range: the nearest one is at least R away, which decides the step as no point at all would
      const bool done = tid == 0 && mr.step(s_in, n, a.drone_radius, s_min != ~0u, __uint_as_float(s_min), &c);
      if (__syncthreads_or(done)) break;           // also the barrier before thread 0 writes s_q again
    }
  }
  if (tid != 0) return;
  c.status = st;
  a.crop[j] = c;
  if (a.status) a.status[j] = st;
  if (a.crossed) a.crossed[j] = (uint8_t)(st == FQ_PATHS_OK && c.crossed);
}

struct WriteArgs
{
  int n_prob, max_poly_whole, max_poly_safe;
  const int* in_ofs;
  const double* in;
  const Crop* crop;
  int *ofs_whole, *ofs_safe;
  double *path_whole, *path_safe;
};

// the rows of one corridor's two paths, at the offsets poly_ofs[j] + j
FQ_HD void write_corridor(const WriteArgs& a, int j, int ow, int os)
{
  const Crop c = a.crop[j];
  const double* in = c.status ? nullptr : a.in + 3 * (size_t)a.in_ofs[j];
  const int pw = fqpath::whole_poly(c, c.status ? 0 : a.in_ofs[j + 1] - a.in_ofs[j], a.max_poly_whole);
  const int ps = fqpath::safe_poly(c, a.max_poly_safe);
  for (int i = 0; i <= pw; i++) fqpath::path_vertex(c, false, in, i, a.path_whole + 3 * ((size_t)ow + j + i));
  for (int i = 0; i <= ps; i++) fqpath::path_vertex(c, true, in, i, a.path_safe + 3 * ((size_t)os + j + i));
}

// poly_ofs_* = the exclusive scans of every corridor's polytope counts, then the rows.  One CTA (any size up to 1024):
// every thread takes a contiguous run of corridors, thread 0 scans the runs' sums.
__global__ void __launch_bounds__(1024) fq_paths_write_kernel(const WriteArgs a)
{
  __shared__ int s_w[1024], s_s[1024];
  const int T = blockDim.x, tid = threadIdx.x;
  const int per = (a.n_prob + T - 1) / T;
  const int j0 = min(a.n_prob, tid * per), j1 = min(a.n_prob, j0 + per);
  auto counts = [&](int j, int* pw, int* ps) {
    const Crop& c = a.crop[j];
    *pw = fqpath::whole_poly(c, c.status ? 0 : a.in_ofs[j + 1] - a.in_ofs[j], a.max_poly_whole);
    *ps = fqpath::safe_poly(c, a.max_poly_safe);
  };
  int sw = 0, ss = 0, pw, ps;
  for (int j = j0; j < j1; j++) { counts(j, &pw, &ps); sw += pw; ss += ps; }
  s_w[tid] = sw; s_s[tid] = ss;
  __syncthreads();
  if (tid == 0)
  {
    int rw = 0, rs = 0;
    for (int i = 0; i < T; i++)
    {
      const int xw = s_w[i], xs = s_s[i];
      s_w[i] = rw; s_s[i] = rs;
      rw += xw; rs += xs;
    }
    a.ofs_whole[a.n_prob] = rw; a.ofs_safe[a.n_prob] = rs;
  }
  __syncthreads();
  int ow = s_w[tid], os = s_s[tid];
  for (int j = j0; j < j1; j++)
  {
    counts(j, &pw, &ps);
    a.ofs_whole[j] = ow; a.ofs_safe[j] = os;
    write_corridor(a, j, ow, os);
    ow += pw; os += ps;
  }
}

// the checks of every entry that read no array: `maps` false for fq_paths_cloud
const char* check_struct(const fq_map_paths_args* p, bool maps)
{
  if (!p) return "map_paths: p is NULL";
  if (p->n_prob <= 0 || p->n_prob > (1 << 24)) return "map_paths: n_prob out of range (1..2^24)";
  if (!p->in_ofs || !p->in) return "map_paths: in_ofs / in must not be NULL";
  if (!p->poly_ofs_whole || !p->poly_ofs_safe || !p->path_whole || !p->path_safe)
    return "map_paths: poly_ofs_* / path_* must not be NULL";
  if (!std::isfinite(p->drone_radius) || !(p->drone_radius > 0)) return "map_paths: drone_radius must be finite and > 0";
  if (p->max_poly_whole < 1 || p->max_poly_whole > FQ_MAX_POLY || p->max_poly_safe < 1 || p->max_poly_safe > FQ_MAX_POLY)
    return "map_paths: max_poly_* out of range (1..FQ_MAX_POLY)";
  if (!maps) return nullptr;
  if (!p->maps || p->n_maps <= 0) return "map_paths: no maps";
  for (int i = 0; i < p->n_maps; i++)
  {
    if (!p->maps[i]) return "map_paths: a NULL map";
    if (fq_map_device(p->maps[i]) != fq_map_device(p->maps[0])) return "map_paths: maps on different devices";
    if (!fq_map_valid(p->maps[i])) return "map_paths: a map whose last update failed";
  }
  return nullptr;
}

// the host checks of the inputs (in_ofs, in); *longest: the longest JPS_in
const char* check_inputs(const fq_map_paths_args* p, int* longest)
{
  if (p->in_ofs[0] != 0) return "map_paths: in_ofs must start at 0";
  *longest = 0;
  for (int j = 0; j < p->n_prob; j++)
  {
    const int n = p->in_ofs[j + 1] - p->in_ofs[j];
    if (p->in_ofs[j + 1] < p->in_ofs[j]) return "map_paths: in_ofs decreasing";
    if (n < 2) return "map_paths: a JPS_in with fewer than 2 vertices";
    if (n > FQ_PATHS_MAX_IN) return "map_paths: a JPS_in with more than FQ_PATHS_MAX_IN vertices";
    *longest = std::max(*longest, n);
  }
  for (size_t i = 0; i < 3 * (size_t)p->in_ofs[p->n_prob]; i++)
    if (!std::isfinite(p->in[i])) return "map_paths: non-finite vertex";
  return nullptr;
}

// every launch of the device route on `st` (device pointers, every scalar checked, the maps' device current)
int enqueue(const fq_map_paths_args* p, cudaStream_t st)
{
  fq_ctx* ctx = nullptr;                           // errors go to fq_last_error(NULL)
  const size_t crop_bytes = fq_align16(sizeof(Crop) * (size_t)p->n_prob);
  char* scratch = nullptr;
  FQ_CUDA(cudaMallocAsync((void**)&scratch, crop_bytes + sizeof(FqMapDev*) * (size_t)p->n_maps, st));
  Crop* crop = (Crop*)scratch;
  const FqMapDev** table = (const FqMapDev**)(scratch + crop_bytes);
  cudaError_t e = cudaSuccess;
  for (int at = 0; at < p->n_maps && e == cudaSuccess; at += FqMapTableChunk::kCap)
  {
    FqMapTableChunk c{};
    c.n = std::min(FqMapTableChunk::kCap, p->n_maps - at); c.at = at; c.table = table;
    for (int i = 0; i < c.n; i++) c.m[i] = fq_map_descriptor(p->maps[at + i]);
    e = fq_launch_map_table(c, st);
  }
  const size_t smem = sizeof(double) * 3 * (size_t)p->max_in;
  if (e == cudaSuccess) e = cudaFuncSetAttribute(fq_paths_crop_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e == cudaSuccess)
  {
    const CropArgs ca = { p->n_prob, p->max_in, p->n_maps, p->in_ofs, p->in, table, p->map_index, p->drone_radius, crop,
                          p->status, p->crossed };
    fq_paths_crop_kernel<<<p->n_prob, kThreads, smem, st>>>(ca);
    const WriteArgs wa = { p->n_prob, p->max_poly_whole, p->max_poly_safe, p->in_ofs, p->in, crop, p->poly_ofs_whole,
                           p->poly_ofs_safe, p->path_whole, p->path_safe };
    fq_paths_write_kernel<<<1, 1024, 0, st>>>(wa);
    e = cudaGetLastError();
  }
  const cudaError_t ef = cudaFreeAsync(scratch, st);
  FQ_CUDA(e);
  FQ_CUDA(ef);
  return 0;
}

// runs f with the maps' device current, then restores the caller's
template <class F>
int on_device(int dev, F&& f)
{
  fq_ctx* ctx = nullptr;
  int cur = 0;
  FQ_CUDA(cudaGetDevice(&cur));
  FQ_CUDA(cudaSetDevice(dev));
  const int rc = f();
  cudaSetDevice(cur);
  return rc;
}

// device buffers of the host entry, freed on every return
struct DevBuf
{
  void* p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
};
}  // namespace

extern "C" int fq_map_paths_dev(const fq_map_paths_args* p, void* stream)
{
  if (const char* why = check_struct(p, true)) return fq_fail(nullptr, FQ_E_ARG, why);
  if (p->max_in < 2 || p->max_in > FQ_PATHS_MAX_IN) return fq_fail(nullptr, FQ_E_ARG, "map_paths: max_in out of range (2..FQ_PATHS_MAX_IN)");
  return on_device(fq_map_device(p->maps[0]), [&] { return enqueue(p, (cudaStream_t)stream); });
}

extern "C" int fq_map_paths(const fq_map_paths_args* p)
{
  if (const char* why = check_struct(p, true)) return fq_fail(nullptr, FQ_E_ARG, why);
  int longest = 0;
  if (const char* why = check_inputs(p, &longest)) return fq_fail(nullptr, FQ_E_ARG, why);
  for (int j = 0; p->map_index && j < p->n_prob; j++)
    if (p->map_index[j] < 0 || p->map_index[j] >= p->n_maps) return fq_fail(nullptr, FQ_E_ARG, "map_paths: map_index out of range");
  return on_device(fq_map_device(p->maps[0]), [&]() -> int {
    fq_ctx* ctx = nullptr;
    const size_t n = (size_t)p->n_prob, rows_in = (size_t)p->in_ofs[n];
    const size_t rw = n * (p->max_poly_whole + 1), rs = n * (p->max_poly_safe + 1);
    size_t at = 0;
    auto put = [&](size_t bytes) { const size_t o = at; at += fq_align16(bytes); return o; };
    const size_t o_in_ofs = put(sizeof(int) * (n + 1)), o_in = put(sizeof(double) * 3 * rows_in), o_idx = put(sizeof(int) * n);
    const size_t o_pw = put(sizeof(int) * (n + 1)), o_ps = put(sizeof(int) * (n + 1)), o_path_w = put(sizeof(double) * 3 * rw);
    const size_t o_path_s = put(sizeof(double) * 3 * rs), o_st = put(sizeof(int) * n), o_cr = put(n);
    DevBuf buf;
    FQ_CUDA(cudaMalloc(&buf.p, at));
    char* d = (char*)buf.p;
    fq_map_paths_args q = *p;
    q.in_ofs = (const int*)(d + o_in_ofs); q.in = (const double*)(d + o_in); q.map_index = p->map_index ? (const int*)(d + o_idx) : nullptr;
    q.max_in = longest;
    q.poly_ofs_whole = (int*)(d + o_pw); q.poly_ofs_safe = (int*)(d + o_ps);
    q.path_whole = (double*)(d + o_path_w); q.path_safe = (double*)(d + o_path_s);
    q.status = (int*)(d + o_st); q.crossed = (uint8_t*)(d + o_cr);
    FQ_CUDA(cudaMemcpy((void*)q.in_ofs, p->in_ofs, sizeof(int) * (n + 1), cudaMemcpyHostToDevice));
    FQ_CUDA(cudaMemcpy((void*)q.in, p->in, sizeof(double) * 3 * rows_in, cudaMemcpyHostToDevice));
    if (p->map_index) FQ_CUDA(cudaMemcpy((void*)q.map_index, p->map_index, sizeof(int) * n, cudaMemcpyHostToDevice));
    if (int rc = enqueue(&q, 0)) return rc;
    FQ_CUDA(cudaStreamSynchronize(0));
    FQ_CUDA(cudaMemcpy(p->poly_ofs_whole, q.poly_ofs_whole, sizeof(int) * (n + 1), cudaMemcpyDeviceToHost));
    FQ_CUDA(cudaMemcpy(p->poly_ofs_safe, q.poly_ofs_safe, sizeof(int) * (n + 1), cudaMemcpyDeviceToHost));
    FQ_CUDA(cudaMemcpy(p->path_whole, q.path_whole, sizeof(double) * 3 * (p->poly_ofs_whole[n] + n), cudaMemcpyDeviceToHost));
    FQ_CUDA(cudaMemcpy(p->path_safe, q.path_safe, sizeof(double) * 3 * (p->poly_ofs_safe[n] + n), cudaMemcpyDeviceToHost));
    if (p->status) FQ_CUDA(cudaMemcpy(p->status, q.status, sizeof(int) * n, cudaMemcpyDeviceToHost));
    if (p->crossed) FQ_CUDA(cudaMemcpy(p->crossed, q.crossed, n, cudaMemcpyDeviceToHost));
    return 0;
  });
}

extern "C" int fq_paths_cloud(const fq_map_paths_args* p, const int* unk_ofs, const double* unk)
{
  if (const char* why = check_struct(p, false)) return fq_fail(nullptr, FQ_E_ARG, why);
  int longest = 0;
  if (const char* why = check_inputs(p, &longest)) return fq_fail(nullptr, FQ_E_ARG, why);
  const int n_prob = p->n_prob;
  if (!unk_ofs) return fq_fail(nullptr, FQ_E_ARG, "map_paths: unk_ofs is NULL");
  if (unk_ofs[0] != 0) return fq_fail(nullptr, FQ_E_ARG, "map_paths: unk_ofs must start at 0");
  for (int j = 0; j < n_prob; j++)
    if (unk_ofs[j + 1] < unk_ofs[j]) return fq_fail(nullptr, FQ_E_ARG, "map_paths: unk_ofs decreasing");
  if (unk_ofs[n_prob] > 0 && !unk) return fq_fail(nullptr, FQ_E_ARG, "map_paths: unk is NULL");
  for (size_t i = 0; i < 3 * (size_t)unk_ofs[n_prob]; i++)
    if (!std::isfinite(unk[i])) return fq_fail(nullptr, FQ_E_ARG, "map_paths: non-finite unknown point");
  std::vector<Crop> crops((size_t)n_prob);
  for (int j = 0; j < n_prob; j++)
  {
    const double* in = p->in + 3 * (size_t)p->in_ofs[j];
    const int n = p->in_ofs[j + 1] - p->in_ofs[j];
    Crop& c = crops[(size_t)j];
    c = Crop{};
    fqpath::March mr(in);
    bool done = false;
    for (int it = 0; it < fqpath::kMaxSteps && !done; it++)
    {
      float q[3];
      mr.query(q);
      unsigned m = ~0u;
      for (int i = unk_ofs[j]; i < unk_ofs[j + 1]; i++)
      {
        const float d2 = fqp::flann_l2(q, unk + 3 * (size_t)i);
        unsigned v;
        std::memcpy(&v, &d2, 4);
        m = std::min(m, v);
      }
      float d2;
      std::memcpy(&d2, &m, 4);
      done = mr.step(in, n, p->drone_radius, unk_ofs[j + 1] > unk_ofs[j], d2, &c);
    }
    if (!done) c.status = FQ_PATHS_STALL;
  }
  WriteArgs a = { n_prob, p->max_poly_whole, p->max_poly_safe, p->in_ofs, p->in, crops.data(), p->poly_ofs_whole,
                  p->poly_ofs_safe, p->path_whole, p->path_safe };
  int ow = 0, os = 0;
  for (int j = 0; j < n_prob; j++)
  {
    const Crop& c = crops[(size_t)j];
    p->poly_ofs_whole[j] = ow; p->poly_ofs_safe[j] = os;
    write_corridor(a, j, ow, os);
    ow += fqpath::whole_poly(c, c.status ? 0 : p->in_ofs[j + 1] - p->in_ofs[j], p->max_poly_whole);
    os += fqpath::safe_poly(c, p->max_poly_safe);
    if (p->status) p->status[j] = c.status;
    if (p->crossed) p->crossed[j] = (uint8_t)(c.status == FQ_PATHS_OK && c.crossed);
  }
  p->poly_ofs_whole[n_prob] = ow; p->poly_ofs_safe[n_prob] = os;
  return 0;
}

extern "C" int fq_jps_in(const double* jps, int n, const double* start, const double* goal, double ra, double dist_max, double* out,
                         int cap)
{
  if (!jps || !start || !goal || n < 1) return fq_fail(nullptr, FQ_E_ARG, "jps_in: jps, start or goal NULL, or n < 1");
  if (cap < 0 || (!out && cap > 0)) return fq_fail(nullptr, FQ_E_ARG, "jps_in: cap < 0, or out NULL with cap > 0");
  for (size_t i = 0; i < 3 * (size_t)n; i++)
    if (!std::isfinite(jps[i])) return fq_fail(nullptr, FQ_E_ARG, "jps_in: non-finite vertex");
  for (int k = 0; k < 3; k++)
    if (!std::isfinite(start[k]) || !std::isfinite(goal[k])) return fq_fail(nullptr, FQ_E_ARG, "jps_in: non-finite start or goal");
  if (!std::isfinite(ra)) return fq_fail(nullptr, FQ_E_ARG, "jps_in: ra must be finite");
  if (!std::isfinite(dist_max) || !(dist_max > 0)) return fq_fail(nullptr, FQ_E_ARG, "jps_in: dist_max must be finite and > 0");
  const fqpath::JpsIn j(jps, n, start, goal, ra);
  if (j.count(dist_max) > (double)(1 << 30)) return fq_fail(nullptr, FQ_E_ARG, "jps_in: more than 2^30 vertices (dist_max too small)");
  return j.write(dist_max, out, cap);
}
