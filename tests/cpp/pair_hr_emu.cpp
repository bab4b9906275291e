// TEST INFRASTRUCTURE ONLY -- the H/R kernels of the chained replan (faster_b200/csrc/fq_pair.cuh: fq_pair_hr_kernel, and
// fq_pair_mid_kernel / fq_pair_window_kernel with its outputs) compiled for the host and run under the block emulation of
// simt_emu/simt_emu.h, block by block with the launch shapes of fq_kernels.cu (the H/R kernel with any block size: its
// results must not depend on it).  tests/test_pair_hr_cpu.py compares them with tests/pair_hr_oracle.py.  Not a CPU path.
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
// fq_launch_pair_hr with `block` threads per corridor; params: drone_radius, delta_a, delta_H
void emu_pair_hr(int block, int n_prob, int N, double DC, const double* params, const double* coeffs, const double* win_dt,
                 const int* win_idx, const double* lim, const int* unk_ofs, const double* unk, int* r_index, uint8_t* need, int* index_H)
{
  FqPairHrArgs a;
  a.n_prob = n_prob; a.N = N; a.DC = DC; a.drone_radius = params[0]; a.delta_a = params[1]; a.delta_H = params[2];
  a.coeffs = coeffs; a.win_dt = win_dt; a.win_idx = win_idx; a.lim = lim; a.unk_ofs = unk_ofs; a.unk = unk;
  a.r_index = r_index; a.need = need; a.need_out = nullptr; a.index_H = index_H;
  launch((unsigned)n_prob, (unsigned)block, [=] { fqp::fq_pair_hr_kernel(a); });
}
// fq_launch_pair_mid with R's index from the H/R kernel
void emu_pair_mid_hr(int n_prob, int N, double DC, const double* coeffs, const double* win_dt, const int* win_idx, const int* r_index,
                     double* x0_safe, int* n_samples, int* k_safe)
{
  FqPairMidArgs a;
  a.n_prob = n_prob; a.N = N; a.DC = DC; a.r_fraction = 0.5; a.coeffs = coeffs; a.win_dt = win_dt; a.win_idx = win_idx;
  a.x0_safe = x0_safe; a.n_samples = n_samples; a.k_safe = k_safe; a.r_index = r_index;
  launch((unsigned)(n_prob + 63) / 64, 64, [=] { fqp::fq_pair_mid_kernel(a); });
}
// fq_launch_pair_window with need_safe / last_factor_safe; the array layouts of pair_window_emu.cpp's emu_pair_window
void emu_pair_window_hr(int n_prob, int max_fac_w, int max_fac_s, const fq_pair_result* rec, const int* cand_ofs_w, const int* cand_ofs_s,
                        const int* n_fac_w, const int* n_fac_s, const double* fac_w, const double* fac_s, const double* windows,
                        const double* gammas, double* factor, int* trials, double* next, const uint8_t* need_safe, double* last_factor_safe)
{
  FqPairWindowArgs a;
  a.n_prob = n_prob; a.max_fac_w = max_fac_w; a.max_fac_s = max_fac_s; a.rec = rec; a.cand_ofs_w = cand_ofs_w; a.cand_ofs_s = cand_ofs_s;
  a.n_fac_w = n_fac_w; a.n_fac_s = n_fac_s; a.fac_w = fac_w; a.fac_s = fac_s;
  a.init_w = windows; a.final_w = windows + n_prob; a.init_s = windows + 2 * n_prob; a.final_s = windows + 3 * n_prob;
  a.gamma_w = gammas[0]; a.gammap_w = gammas[1]; a.gamma_s = gammas[2]; a.gammap_s = gammas[3];
  a.factor_w = factor; a.factor_s = factor + n_prob; a.trials_w = trials; a.trials_s = trials + n_prob;
  a.next_init_w = next; a.next_final_w = next + n_prob; a.next_init_s = next + 2 * n_prob; a.next_final_s = next + 3 * n_prob;
  a.need_safe = need_safe; a.last_factor_safe = last_factor_safe;
  launch((unsigned)(n_prob + 127) / 128, 128, [=] { fqp::fq_pair_window_kernel(a); });
}
}
