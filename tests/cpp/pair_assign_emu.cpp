// TEST INFRASTRUCTURE ONLY -- the per-corridor assignment-list kernels of the chained replan (faster_b200/csrc/fq_pair.cuh:
// candidate offsets, grid expansion with unranking, result records with per-corridor list lengths) compiled for the host and
// run under the block emulation of simt_emu/simt_emu.h, block by block with the launch shapes of fq_kernels.cu (the offsets
// kernel with a smaller CTA: it takes any block size).  tests/test_pair_assign_cpu.py checks them against enumerated lists
// and, together with kernel_emu.cpp and pair_emu.cpp, replays fq_replan_pairs_assign_dev's submission.  Not a CPU path.
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
long long emu_list_len(int N, int P, long long all_limit) { return fqa::list_len(N, P, all_limit); }

void emu_assign_offsets(int block, int n_prob, int N, int n_fac, long long all_limit, int max_poly, long long n_cand, const int* poly_ofs,
                        int* cand_ofs)
{ // fq_launch_assign_offsets (one CTA)
  launch(1, (unsigned)block, [=] { fqp::fq_assign_offsets_kernel(n_prob, N, n_fac, all_limit, max_poly, n_cand, poly_ofs, cand_ofs); });
}
void emu_expand_assign(int n_prob, int N, int n_fac, long long all_limit, const double* factors, const double* dt_base, const int* poly_ofs,
                       const int* cand_ofs, double* dt, uint8_t* sigma)
{ // fq_launch_expand_assign
  launch((unsigned)n_prob, 256, [=] { fqp::fq_expand_assign_kernel(n_prob, N, n_fac, all_limit, factors, dt_base, poly_ofs, cand_ofs, dt, sigma); });
}
void emu_pair_final_assign(int n_prob, int n_fac_w, int n_fac_s, int N_w, int N_s, const int* cand_ofs_w, const int* cand_ofs_s,
                           const int* win_idx_w, const int* win_idx_s, const int* n_samples, const int* k_safe, const double* win_cost_w,
                           const double* win_cost_s, const double* win_dt_w, const double* win_dt_s, const double* dt_base_w,
                           const double* dt_base_s, const double* x0_safe, const uint8_t* win_sig_w, const uint8_t* win_sig_s,
                           uint8_t* sigma_out_w, uint8_t* sigma_out_s, fq_pair_result* out)
{ // fq_launch_pair_final with per-corridor lists
  FqPairFinalArgs a;
  a.n_prob = n_prob; a.n_sig_w = 0; a.n_sig_s = 0; a.win_idx_w = win_idx_w; a.win_idx_s = win_idx_s; a.n_samples = n_samples;
  a.k_safe = k_safe; a.win_cost_w = win_cost_w; a.win_cost_s = win_cost_s; a.win_dt_w = win_dt_w; a.win_dt_s = win_dt_s;
  a.dt_base_w = dt_base_w; a.dt_base_s = dt_base_s; a.x0_safe = x0_safe; a.out = out;
  a.cand_ofs_w = cand_ofs_w; a.cand_ofs_s = cand_ofs_s; a.n_fac_w = n_fac_w; a.n_fac_s = n_fac_s; a.N_w = N_w; a.N_s = N_s;
  a.win_sig_w = win_sig_w; a.win_sig_s = win_sig_s; a.sigma_out_w = sigma_out_w; a.sigma_out_s = sigma_out_s;
  launch((unsigned)(n_prob + 127) / 128, 128, [=] { fqp::fq_pair_final_kernel(a); });
}
}
