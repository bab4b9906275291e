// TEST INFRASTRUCTURE ONLY -- the product's kernel SOURCE (faster_b200/csrc/fq_kernels_t.cuh: fq_solve_kernel_t, the persistent
// warp-per-candidate dual active-set solver) compiled for the host and executed under the lock-step block emulation of
// simt_emu/simt_emu.h: 128 fibres = one CTA of four warps, claim counters, staging, item lists, the whole active-set iteration,
// run instruction for instruction as written for the GPU (the two MUFU seeds are replaced by a float-precision seed, the launch
// function is not compiled).  tests/test_kernel_emu_cpu.py compares its answers with the CPU restatement -- a check of the
// kernel's LOGIC that needs no GPU.  It is not a CPU path of the product and is far too slow to be one.
#define FQ_EMULATE_ON_HOST 1
#include "simt_emu/cuda_runtime.h"

#include "fq_kernels.cuh"
#include "fq_kernels_t.cuh"

#include <cstdio>

namespace fqt
{ // the kernel declares its dynamic shared array inside namespace fqt: this is that array (one block runs at a time)
alignas(16) unsigned char smem_raw[232 * 1024];
}


namespace
{
struct Call { FqKernelArgs a; int* counters; };
template <int N, bool WHOLE>
void entry(void* p)
{
  Call* c = static_cast<Call*>(p);
  fqt::fq_solve_kernel_t<N, WHOLE>(c->a, c->counters);
}
template <int N, bool WHOLE>
int run(Call& c)
{
  if (fqt::smem_bytes_t<N, WHOLE>(c.a.max_faces, c.a.item_cap) > sizeof(fqt::smem_raw)) return -2;
  simt::run_block(dim3(1), dim3(fqt::W * 32), uint3{ 0, 0, 0 }, entry<N, WHOLE>, &c);
  return 0;
}
}  // namespace

extern "C" {
int emu_solve_multi(int N, int force_final, const double* TZ, const double* T0, const double* FT, int n_prob, const double* x0,
                    const double* xf, const double* lim, const int* poly_ofs, const int* face_ofs, const double* Ab, int max_faces,
                    int max_poly_faces, const int* cand_ofs, const double* dt, const uint8_t* sigma, double row_tol, uint8_t* feasible,
                    double* cost, double* coeffs, int32_t* iters);
// options of the next emu_solve_multi call (the FqKernelArgs options the drop-in class's sweeps launch with, fq_capi.cu):
//   early_exit != 0: "first feasible factor wins" (first_feasible + sorted_dt: candidates whose dt exceeds the smallest feasible dt
//                    found so far are not evaluated, iters = -3);
//   sweep_n_sigma > 0: single-problem sweep, dt-major with that many assignments per time allocation: the warp that finishes the
//                    last candidate runs genNewTraj's selection inside the kernel and writes sweep_idx[2] / sweep_win[1 + 12 N].
static int g_early_exit = 0, g_sweep_n_sigma = 0;
static int* g_sweep_idx = nullptr;
static double* g_sweep_win = nullptr;
void emu_set_sweep(int early_exit, int sweep_n_sigma, int* sweep_idx, double* sweep_win)
{
  g_early_exit = early_exit; g_sweep_n_sigma = sweep_n_sigma; g_sweep_idx = sweep_idx; g_sweep_win = sweep_win;
}
// One CTA of the product kernel over a multi-problem batch laid out like fq_solve_multi (include/faster_b200.h); plan tables
// TZ / T0 / FT from fq_plan_tables.  Returns 0, -1 for an (N, mode) the harness does not instantiate, -2 if the batch needs more
// shared memory than a CTA has.
int emu_solve_multi(int N, int force_final, const double* TZ, const double* T0, const double* FT, int n_prob, const double* x0,
                    const double* xf, const double* lim, const int* poly_ofs, const int* face_ofs, const double* Ab, int max_faces,
                    int max_poly_faces, const int* cand_ofs, const double* dt, const uint8_t* sigma, double row_tol, uint8_t* feasible,
                    double* cost, double* coeffs, int32_t* iters)
{
  Call c;
  std::memset(&c.a, 0, sizeof(c.a));
  const int ne = force_final ? 3 : 2;
  c.a.N = N; c.a.force_final = force_final; c.a.ne = ne; c.a.nz = N - ne; c.a.nw = 3 * (N - ne); c.a.NY = 6 * N + 1;
  c.a.TZ = TZ; c.a.T0 = T0; c.a.FT = FT;
  c.a.n_prob = n_prob; c.a.x0 = x0; c.a.xf = xf; c.a.lim = lim; c.a.poly_ofs = poly_ofs; c.a.face_ofs = face_ofs; c.a.Ab = Ab;
  c.a.max_faces = max_faces > 0 ? max_faces : 1;
  c.a.item_cap = N * (max_poly_faces > 0 ? max_poly_faces : c.a.max_faces);
  c.a.cand_ofs = cand_ofs; c.a.dt = dt; c.a.sigma = sigma;
  c.a.feasible = feasible; c.a.cost = cost; c.a.coeffs = coeffs; c.a.iters = iters; c.a.row_tol = row_tol;
  std::vector<int> counters((size_t)n_prob + 1, 0);
  c.counters = counters.data();
  std::vector<unsigned long long> first((size_t)n_prob, ~0ull);
  if (g_early_exit) { c.a.first_feasible = first.data(); c.a.sorted_dt = 1; c.a.ee_width = g_sweep_n_sigma; }
  if (g_sweep_n_sigma > 0 && n_prob == 1 && coeffs)
  {
    c.a.sweep_done = counters.data() + n_prob; c.a.sweep_n_sigma = g_sweep_n_sigma; c.a.sweep_idx = g_sweep_idx; c.a.sweep_win = g_sweep_win;
  }
  g_early_exit = 0; g_sweep_n_sigma = 0;
  const int key = N * 2 + (force_final ? 1 : 0);
  switch (key)
  {
    case 4 * 2 + 0: return run<4, false>(c);
    case 5 * 2 + 1: return run<5, true>(c);
    case 6 * 2 + 1: return run<6, true>(c);
    case 10 * 2 + 1: return run<10, true>(c);
    case 10 * 2 + 0: return run<10, false>(c);
    case 11 * 2 + 0: return run<11, false>(c);
    case 12 * 2 + 0: return run<12, false>(c);
    case 13 * 2 + 1: return run<13, true>(c);
    case 13 * 2 + 0: return run<13, false>(c);
    case 14 * 2 + 1: return run<14, true>(c);
    case 15 * 2 + 1: return run<15, true>(c);
    case 16 * 2 + 0: return run<16, false>(c);
    default: return -1;
  }
}
}
