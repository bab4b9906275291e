// TEST INFRASTRUCTURE ONLY -- the batch JPS kernels (faster_b200/csrc/fq_jps.cuh: fq_jps_search_kernel and
// fq_jps_write_kernel) compiled for the host and run under the block emulation of simt_emu/simt_emu.h, block by block, with
// 1 .. 4 warps per CTA (the results must not depend on it).  tests/test_jps_batch_cpu.py compares them with
// tests/jps_batch_oracle.py.  Not a CPU path.
#define FQ_EMULATE_ON_HOST 1
#define __shared__ static
#include "simt_emu/cuda_runtime.h"

using std::isfinite;

#include "fq_jps.cuh"

#include <vector>

namespace
{
template <class F>
struct Thunk
{
  F f;
  static void call(void* p) { static_cast<Thunk*>(p)->f(); }
};
template <class F>
void launch(unsigned grid, unsigned block, F f)
{
  Thunk<F> t{ f };
  for (unsigned b = 0; b < grid; b++) simt::run_block(dim3(grid), dim3(block), uint3{ b, 0, 0 }, Thunk<F>::call, &t, 256 * 1024);
}
}  // namespace

extern "C" {
// both kernels of fq_jps_batch_dev on host memory: `warps` warps per search CTA, `write_block` threads in the write CTA
void emu_jps_batch(int warps, int write_block, const fq_jps_batch_args* p)
{
  FqJpsArgs a{};
  const size_t n = (size_t)p->n_prob;
  a.n_prob = p->n_prob; a.n_grids = p->grids.n_grids;
  a.cells = p->grids.cells; a.cell_ofs = p->grids.cell_ofs; a.dims = p->grids.dims; a.origin = p->grids.origin; a.res = p->grids.res;
  a.grid_index = p->grid_index; a.x0 = p->x0; a.goal = p->goal; a.pos = p->pos;
  a.Ra = p->Ra; a.dist_max = p->dist_max; a.use_jps = p->use_jps; a.max_nodes = p->max_nodes; a.max_in = p->max_in;
  a.per = fq_jps_scratch_layout(p->max_nodes, p->max_in).total;
  std::vector<double> scratch((a.per * n + 7) / 8);
  std::vector<int> cnt(n, -7), st(n, -7);
  a.scratch = (char*)scratch.data(); a.cnt = cnt.data(); a.st = st.data();
  a.in_ofs = p->in_ofs; a.in = p->in; a.status = p->status; a.k_end = p->k_end;
  launch((unsigned)((n + warps - 1) / warps), (unsigned)(32 * warps), [=] { fq_jps_search_kernel(a); });
  launch(1u, (unsigned)write_block, [=] { fq_jps_write_kernel(a); });
}
}
