// TEST INFRASTRUCTURE ONLY -- the committed-plan kernels (faster_b200/csrc/fq_pair.cuh: fq_queue_reset_kernel,
// fq_queue_select_kernel, fq_queue_pop_kernel and the chain's append, fq_pair_queue_kernel) compiled for the host and run
// under the block emulation of simt_emu/simt_emu.h, block by block, with any block sizes (the results must not depend on
// them).  tests/test_pair_queue_cpu.py compares them with the host entries fq_queue_* and tests/plan_queue_oracle.py.
// Not a CPU path.
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

FqQueueArgs ring(int n, const int* rows, int n_rows, int cap, int delta_t, double* states, int* head, int* size)
{
  FqQueueArgs q{};
  q.n = n; q.rows = rows; q.n_rows = n_rows; q.cap = cap; q.delta_t = delta_t; q.states = states; q.head = head; q.size = size;
  return q;
}
}  // namespace

extern "C" {
// op 0 reset (pos), 1 select (x0, k_end), 2 pop (ticks, max_ticks, goals), with `block` threads per CTA
void emu_queue(int op, int block, int n, const int* rows, int n_rows, int cap, int delta_t, double* states, int* head, int* size,
               const double* pos, double* x0, int* k_end, const int* ticks, int max_ticks, double* goals)
{
  FqQueueArgs q = ring(n, rows, n_rows, cap, delta_t, states, head, size);
  q.pos = pos; q.x0 = x0; q.k_end = k_end; q.ticks = ticks; q.max_ticks = max_ticks; q.goals = goals;
  const unsigned grid = (unsigned)((n + block - 1) / block);
  if (op == 0) launch(grid, (unsigned)block, [=] { fqp::fq_queue_reset_kernel(q); });
  if (op == 1) launch(grid, (unsigned)block, [=] { fqp::fq_queue_select_kernel(q); });
  if (op == 2) launch(grid, (unsigned)block, [=] { fqp::fq_queue_pop_kernel(q); });
}

// fq_launch_pair_queue with `block` threads per corridor; the chain's intermediates as emu_pair_plan takes them
void emu_pair_queue(int block, int n_prob, const int* Ns, double DC, const int* win_idx, const double* win_dt, const int* n_samples,
                    const int* k_safe, const uint8_t* need, const double* coeffs_w, const double* coeffs_s, const int* rows, int n_rows,
                    int cap, double* states, int* head, int* size, int* k_end, const double* G_term, double goal_radius, int* status,
                    uint8_t* goal_seen)
{
  FqPairPlanArgs a{};
  a.n_prob = n_prob; a.N_w = Ns[0]; a.N_s = Ns[1]; a.DC = DC;
  a.win_idx_w = win_idx; a.win_idx_s = win_idx + n_prob; a.win_dt_w = win_dt; a.win_dt_s = win_dt + n_prob;
  a.n_samples = n_samples; a.k_safe = k_safe; a.need = need; a.coeffs_w = coeffs_w; a.coeffs_s = coeffs_s;
  FqQueueArgs q = ring(n_prob, rows, n_rows, cap, 1, states, head, size);
  q.k_end = k_end; q.G_term = G_term; q.goal_radius = goal_radius; q.status = status; q.goal_seen = goal_seen;
  launch((unsigned)n_prob, (unsigned)block, [=] { fqp::fq_pair_queue_kernel(a, q); });
}
}
