// TEST INFRASTRUCTURE ONLY -- the per-corridor window kernels of the chained replan (faster_b200/csrc/fq_pair.cuh: factor
// rows, candidate offsets with per-corridor factor counts and a capacity, grid expansion from the factor rows, result records
// split by per-corridor counts, factor / trials / next windows) compiled for the host and run under the block emulation of
// simt_emu/simt_emu.h, block by block with the launch shapes of fq_kernels.cu (the offsets kernel with a smaller CTA: it
// takes any block size).  tests/test_pair_window_cpu.py checks them against fq_window.h's host build and, together with
// kernel_emu.cpp and pair_emu.cpp, replays fq_replan_pairs_window_dev's submission.  Not a CPU path.
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
void emu_window_factors(int n_prob, int max_fac, const double* init, const double* final_, double inc, double* fac, int* n_fac_j)
{ // fq_launch_window_factors
  launch((unsigned)(n_prob + 63) / 64, 64, [=] { fqp::fq_window_factors_kernel(n_prob, max_fac, init, final_, inc, fac, n_fac_j); });
}
void emu_window_offsets(int block, int n_prob, int N, int max_fac, long long all_limit, int max_poly, long long cap, const int* poly_ofs,
                        const int* n_fac_j, int* cand_ofs)
{ // fq_launch_window_offsets (one CTA)
  launch(1, (unsigned)block, [=] { fqp::fq_assign_offsets_kernel(n_prob, N, max_fac, all_limit, max_poly, cap, poly_ofs, cand_ofs, n_fac_j); });
}
void emu_expand_window(int n_prob, int N, int max_fac, long long all_limit, const double* fac, const int* n_fac_j, const double* dt_base,
                       const int* poly_ofs, const int* cand_ofs, double* dt, uint8_t* sigma)
{ // fq_launch_expand_window
  launch((unsigned)n_prob, 256,
         [=] { fqp::fq_expand_assign_kernel(n_prob, N, max_fac, all_limit, fac, dt_base, poly_ofs, cand_ofs, dt, sigma, n_fac_j); });
}
void emu_pair_final_window(int n_prob, int N_w, int N_s, const int* cand_ofs_w, const int* cand_ofs_s, const int* n_fac_j_w,
                           const int* n_fac_j_s, const int* win_idx_w, const int* win_idx_s, const int* n_samples, const int* k_safe,
                           const double* win_cost_w, const double* win_cost_s, const double* win_dt_w, const double* win_dt_s,
                           const double* dt_base_w, const double* dt_base_s, const double* x0_safe, const uint8_t* win_sig_w,
                           const uint8_t* win_sig_s, fq_pair_result* out)
{ // fq_launch_pair_final with per-corridor lists and windows
  FqPairFinalArgs a;
  a.n_prob = n_prob; a.n_sig_w = 0; a.n_sig_s = 0; a.win_idx_w = win_idx_w; a.win_idx_s = win_idx_s; a.n_samples = n_samples;
  a.k_safe = k_safe; a.win_cost_w = win_cost_w; a.win_cost_s = win_cost_s; a.win_dt_w = win_dt_w; a.win_dt_s = win_dt_s;
  a.dt_base_w = dt_base_w; a.dt_base_s = dt_base_s; a.x0_safe = x0_safe; a.out = out;
  a.cand_ofs_w = cand_ofs_w; a.cand_ofs_s = cand_ofs_s; a.N_w = N_w; a.N_s = N_s; a.win_sig_w = win_sig_w; a.win_sig_s = win_sig_s;
  a.n_fac_j_w = n_fac_j_w; a.n_fac_j_s = n_fac_j_s;
  launch((unsigned)(n_prob + 127) / 128, 128, [=] { fqp::fq_pair_final_kernel(a); });
}
// windows: [init_w, final_w, init_s, final_s] (n_prob each); gammas: [gamma_w, gammap_w, gamma_s, gammap_s]; factor: 2 n_prob;
// trials: 2 n_prob; next: 4 n_prob (may be `windows` itself)
void emu_pair_window(int n_prob, int max_fac_w, int max_fac_s, const fq_pair_result* rec, const int* cand_ofs_w, const int* cand_ofs_s,
                     const int* n_fac_w, const int* n_fac_s, const double* fac_w, const double* fac_s, const double* windows,
                     const double* gammas, double* factor, int* trials, double* next)
{ // fq_launch_pair_window
  FqPairWindowArgs a;
  a.n_prob = n_prob; a.max_fac_w = max_fac_w; a.max_fac_s = max_fac_s; a.rec = rec; a.cand_ofs_w = cand_ofs_w; a.cand_ofs_s = cand_ofs_s;
  a.n_fac_w = n_fac_w; a.n_fac_s = n_fac_s; a.fac_w = fac_w; a.fac_s = fac_s;
  a.init_w = windows; a.final_w = windows + n_prob; a.init_s = windows + 2 * n_prob; a.final_s = windows + 3 * n_prob;
  a.gamma_w = gammas[0]; a.gammap_w = gammas[1]; a.gamma_s = gammas[2]; a.gammap_s = gammas[3];
  a.factor_w = factor; a.factor_s = factor + n_prob; a.trials_w = trials; a.trials_s = trials + n_prob;
  a.next_init_w = next; a.next_final_w = next + n_prob; a.next_init_s = next + 2 * n_prob; a.next_final_s = next + 3 * n_prob;
  launch((unsigned)(n_prob + 127) / 128, 128, [=] { fqp::fq_pair_window_kernel(a); });
}
// the host build of fq_window.h
int emu_host_factors(double fi, double ff, double inc, double* out, int cap) { return fqw::factors(fi, ff, inc, out, cap); }
void emu_host_next_window(int both, double f_star, double gamma, double gammap, double init, double final_, double* out)
{
  fqw::next_window(both != 0, f_star, gamma, gammap, init, final_, out, out + 1);
}
}
