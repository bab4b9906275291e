// fq_jps_batch / fq_jps_batch_dev (include/faster_b200.h): every planner's JPS search from A to G and its JPS_in, on the
// device.  The kernels are fq_jps.cuh's; the search and the post-processing are fq_jps.h's and fq_jps_in's arithmetic is
// fq_paths.h's, both shared with the host entries fq_jps3d_plan_world and fq_jps_in.  Scratch is stream-ordered memory, so
// the device entry never synchronises and a CUDA graph can capture it.
#include "fq_ctx.h"
#include "fq_jps.cuh"

#include <cmath>
#include <cstring>
#include <vector>

namespace
{
constexpr int kWarpsPerCta = kFqJpsMaxWarps;

// the checks that read no array
const char* check_struct(const fq_jps_batch_args* a)
{
  if (!a) return "jps_batch: args is NULL";
  if (a->n_prob <= 0 || a->n_prob > (1 << 24)) return "jps_batch: n_prob out of range (1..2^24)";
  const fq_jps_grids& g = a->grids;
  if (!g.cells || !g.cell_ofs || !g.dims || !g.origin || !g.res) return "jps_batch: a NULL grid array";
  if (g.n_grids < 1) return "jps_batch: n_grids < 1";
  if (!a->x0 || !a->goal) return "jps_batch: x0 / goal must not be NULL";
  if (!a->in_ofs || !a->in || !a->status) return "jps_batch: in_ofs / in / status must not be NULL";
  if (!std::isfinite(a->Ra)) return "jps_batch: Ra must be finite";
  if (!std::isfinite(a->dist_max) || !(a->dist_max > 0)) return "jps_batch: dist_max must be finite and > 0";
  if (a->max_nodes < 1 || a->max_nodes > (1 << 26)) return "jps_batch: max_nodes out of range (1..2^26)";
  if (a->max_in < 2 || a->max_in > FQ_PATHS_MAX_IN) return "jps_batch: max_in out of range (2..FQ_PATHS_MAX_IN)";
  return nullptr;
}

// the host checks of the grids (host arrays); *cells: the cells the grids span
const char* check_grids(const fq_jps_grids& g, long long* cells)
{
  *cells = 0;
  for (int i = 0; i < g.n_grids; i++)
  {
    const long long xd = g.dims[3 * i], yd = g.dims[3 * i + 1], zd = g.dims[3 * i + 2];
    if (xd <= 0 || yd <= 0 || zd <= 0) return "jps_batch: a grid dimension <= 0";
    if (xd * yd * zd > (1ll << 31)) return "jps_batch: a grid with more than 2^31 cells";
    if (g.cell_ofs[i] < 0) return "jps_batch: a negative cell_ofs";
    if (!std::isfinite(g.res[i]) || !(g.res[i] > 0)) return "jps_batch: res must be finite and > 0";
    for (int k = 0; k < 3; k++)
      if (!std::isfinite(g.origin[3 * i + k])) return "jps_batch: non-finite origin";
    *cells = std::max(*cells, g.cell_ofs[i] + xd * yd * zd);
  }
  return nullptr;
}

// both kernels on `st` (device pointers, every scalar checked)
int enqueue(const fq_jps_batch_args* p, cudaStream_t st)
{
  fq_ctx* ctx = nullptr;                           // errors go to fq_last_error(NULL)
  const size_t n = (size_t)p->n_prob;
  const size_t per = fq_jps_scratch_layout(p->max_nodes, p->max_in).total;
  const size_t head = fq_align16(2 * sizeof(int) * n);
  char* scratch = nullptr;
  FQ_CUDA(cudaMallocAsync((void**)&scratch, head + per * n, st));
  FqJpsArgs a{};
  a.n_prob = p->n_prob; a.n_grids = p->grids.n_grids;
  a.cells = p->grids.cells; a.cell_ofs = p->grids.cell_ofs; a.dims = p->grids.dims; a.origin = p->grids.origin; a.res = p->grids.res;
  a.grid_index = p->grid_index; a.x0 = p->x0; a.goal = p->goal; a.pos = p->pos;
  a.Ra = p->Ra; a.dist_max = p->dist_max; a.use_jps = p->use_jps; a.max_nodes = p->max_nodes; a.max_in = p->max_in;
  a.cnt = (int*)scratch; a.st = a.cnt + n;
  a.scratch = scratch + head; a.per = per;
  a.in_ofs = p->in_ofs; a.in = p->in; a.status = p->status; a.k_end = p->k_end;
  const unsigned grid = (unsigned)((n + kWarpsPerCta - 1) / kWarpsPerCta);
  fq_jps_search_kernel<<<grid, 32 * kWarpsPerCta, 0, st>>>(a);
  fq_jps_write_kernel<<<1, 1024, 0, st>>>(a);
  const cudaError_t e = cudaGetLastError();
  const cudaError_t ef = cudaFreeAsync(scratch, st);
  FQ_CUDA(e);
  FQ_CUDA(ef);
  return 0;
}

struct DevBuf
{
  void* p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
};
}  // namespace

extern "C" int fq_jps_batch_dev(const fq_jps_batch_args* p, void* stream)
{
  if (const char* why = check_struct(p)) return fq_fail(nullptr, FQ_E_ARG, why);
  return enqueue(p, (cudaStream_t)stream);
}

extern "C" int fq_jps_batch(const fq_jps_batch_args* p)
{
  if (const char* why = check_struct(p)) return fq_fail(nullptr, FQ_E_ARG, why);
  long long cells = 0;
  if (const char* why = check_grids(p->grids, &cells)) return fq_fail(nullptr, FQ_E_ARG, why);
  const size_t n = (size_t)p->n_prob, ng = (size_t)p->grids.n_grids;
  for (size_t j = 0; j < n; j++)
  {
    if (p->grid_index && (p->grid_index[j] < 0 || p->grid_index[j] >= p->grids.n_grids))
      return fq_fail(nullptr, FQ_E_ARG, "jps_batch: grid_index out of range");
    for (int k = 0; k < 3; k++)
      if (!std::isfinite(p->x0[9 * j + k]) || !std::isfinite(p->goal[3 * j + k]) || (p->pos && !std::isfinite(p->pos[3 * j + k])))
        return fq_fail(nullptr, FQ_E_ARG, "jps_batch: non-finite A, G or pos");
  }
  fq_ctx* ctx = nullptr;
  size_t at = 0;
  auto put = [&](size_t bytes) { const size_t o = at; at += fq_align16(bytes); return o; };
  const size_t o_cells = put((size_t)cells), o_cofs = put(sizeof(long long) * ng), o_dims = put(sizeof(int) * 3 * ng);
  const size_t o_org = put(sizeof(double) * 3 * ng), o_res = put(sizeof(double) * ng), o_gi = put(sizeof(int) * n);
  const size_t o_x0 = put(sizeof(double) * 9 * n), o_goal = put(sizeof(double) * 3 * n), o_pos = put(sizeof(double) * 3 * n);
  const size_t o_iofs = put(sizeof(int) * (n + 1)), o_in = put(sizeof(double) * 3 * n * p->max_in), o_st = put(sizeof(int) * n);
  const size_t o_ke = put(sizeof(int) * n);
  DevBuf buf;
  FQ_CUDA(cudaMalloc(&buf.p, at));
  char* d = (char*)buf.p;
  fq_jps_batch_args q = *p;
  q.grids.cells = (const int8_t*)(d + o_cells); q.grids.cell_ofs = (const long long*)(d + o_cofs); q.grids.dims = (const int*)(d + o_dims);
  q.grids.origin = (const double*)(d + o_org); q.grids.res = (const double*)(d + o_res);
  q.grid_index = p->grid_index ? (const int*)(d + o_gi) : nullptr;
  q.x0 = (const double*)(d + o_x0); q.goal = (const double*)(d + o_goal); q.pos = p->pos ? (const double*)(d + o_pos) : nullptr;
  q.in_ofs = (int*)(d + o_iofs); q.in = (double*)(d + o_in); q.status = (int*)(d + o_st); q.k_end = p->k_end ? (int*)(d + o_ke) : nullptr;
  auto up = [&](const void* dst, const void* src, size_t bytes) { return cudaMemcpy((void*)dst, src, bytes, cudaMemcpyHostToDevice); };
  FQ_CUDA(up(q.grids.cells, p->grids.cells, (size_t)cells));
  FQ_CUDA(up(q.grids.cell_ofs, p->grids.cell_ofs, sizeof(long long) * ng));
  FQ_CUDA(up(q.grids.dims, p->grids.dims, sizeof(int) * 3 * ng));
  FQ_CUDA(up(q.grids.origin, p->grids.origin, sizeof(double) * 3 * ng));
  FQ_CUDA(up(q.grids.res, p->grids.res, sizeof(double) * ng));
  if (p->grid_index) FQ_CUDA(up(q.grid_index, p->grid_index, sizeof(int) * n));
  FQ_CUDA(up(q.x0, p->x0, sizeof(double) * 9 * n));
  FQ_CUDA(up(q.goal, p->goal, sizeof(double) * 3 * n));
  if (p->pos) FQ_CUDA(up(q.pos, p->pos, sizeof(double) * 3 * n));
  if (p->k_end) FQ_CUDA(up(q.k_end, p->k_end, sizeof(int) * n));
  if (int rc = enqueue(&q, 0)) return rc;
  FQ_CUDA(cudaStreamSynchronize(0));
  FQ_CUDA(cudaMemcpy(p->in_ofs, q.in_ofs, sizeof(int) * (n + 1), cudaMemcpyDeviceToHost));
  FQ_CUDA(cudaMemcpy(p->in, q.in, sizeof(double) * 3 * (size_t)p->in_ofs[n], cudaMemcpyDeviceToHost));
  FQ_CUDA(cudaMemcpy(p->status, q.status, sizeof(int) * n, cudaMemcpyDeviceToHost));
  if (p->k_end) FQ_CUDA(cudaMemcpy(p->k_end, q.k_end, sizeof(int) * n, cudaMemcpyDeviceToHost));
  return 0;
}
