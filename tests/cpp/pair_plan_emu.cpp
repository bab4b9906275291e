// TEST INFRASTRUCTURE ONLY -- the plan kernels of the chained replan (faster_b200/csrc/fq_pair.cuh: fq_pair_plan_offsets_kernel
// and fq_pair_plan_sample_kernel) compiled for the host and run under the block emulation of simt_emu/simt_emu.h, block by
// block, with any block sizes (the results must not depend on them).  tests/test_pair_plan_cpu.py compares them with
// tests/pair_plan_oracle.py.  Not a CPU path.
#define FQ_EMULATE_ON_HOST 1
#define __shared__ static
#include "simt_emu/cuda_runtime.h"

#include "fq_kernels.cuh"
#include "fq_pair.cuh"

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
  for (unsigned b = 0; b < grid; b++) simt::run_block(dim3(grid), dim3(block), uint3{ b, 0, 0 }, Thunk<F>::call, &t, 64 * 1024);
}
}  // namespace

extern "C" {
// fq_launch_pair_plan with `block_ofs` threads for the offsets CTA and `block_rows` threads per corridor.  Ns: N_whole, N_safe;
// win_idx: whole then safe (2 x n_prob); win_dt likewise; need may be NULL; status may be NULL.
void emu_pair_plan(int block_ofs, int block_rows, int n_prob, const int* Ns, double DC, const int* win_idx, const double* win_dt,
                   const int* n_samples, const int* k_safe, const uint8_t* need, const double* coeffs_w, const double* coeffs_s,
                   long long cap, double* states, long long* plan_ofs, int* status)
{
  FqPairPlanArgs a;
  a.n_prob = n_prob; a.N_w = Ns[0]; a.N_s = Ns[1]; a.DC = DC;
  a.win_idx_w = win_idx; a.win_idx_s = win_idx + n_prob; a.win_dt_w = win_dt; a.win_dt_s = win_dt + n_prob;
  a.n_samples = n_samples; a.k_safe = k_safe; a.need = need; a.coeffs_w = coeffs_w; a.coeffs_s = coeffs_s;
  a.cap = cap; a.states = states; a.plan_ofs = plan_ofs; a.status = status;
  launch(1, (unsigned)block_ofs, [=] { fqp::fq_pair_plan_offsets_kernel(a); });
  launch((unsigned)n_prob, (unsigned)block_rows, [=] { fqp::fq_pair_plan_sample_kernel(a); });
}
}
