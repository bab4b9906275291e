// Device-side interface of the batched corridor-QP solver (sm_90a).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "../../include/faster_b200.h"

#define FQ_WARPS_PER_CTA 4
#ifndef FQ_MIN_CTAS_PER_SM
#define FQ_MIN_CTAS_PER_SM 4
#endif
#ifndef FQ_MIN_CTAS_WHOLE
#define FQ_MIN_CTAS_WHOLE 4   // whole-mode kernels for N <= 10; 5 needs <= 96 registers and spills
#endif
#ifndef FQ_MAX_N_3CTAS
#define FQ_MAX_N_3CTAS 15      // largest N whose kernels are compiled for 3 CTAs per SM (<= 168 registers); beyond: 2 CTAs.  N = 14, 15
                               // run 2 CTAs per SM anyway (shared memory), yet letting the compiler take 223 registers there was
                               // slower on config 5: the bound stays
#endif
#define FQ_EPS_DEP 1e-18      // squared sine below which a new normal counts as dependent on the active set
#define FQ_ZZ_FLOOR 1e-30
#define FQ_MAX_ITERS 400

struct FqKernelArgs
{
  // plan (device copies of FqPlanHost tables)
  int N, force_final, ne, nz, nw, NY, ld;
  const double* TZ;      // NY x nz
  const double* T0;      // NY x (3+ne)
  const double* FT;      // ne x 3
  // problems
  int n_prob;
  const double* x0;      // n_prob x 9
  const double* xf;      // n_prob x 9
  const double* lim;     // n_prob x 3
  const int* poly_ofs;   // n_prob+1  -> index into face_ofs
  const int* face_ofs;   // n_poly_total+1 -> row of Ab
  const double* Ab;      // rows [Ax Ay Az b]
  int max_faces;         // max total faces of one problem (sizes the shared staging area)
  int item_cap;          // corridor rows per candidate the item list must hold: N * max_faces
  // candidates
  const int* cand_ofs;   // n_prob+1
  const double* dt;
  const uint8_t* sigma;  // n_cand x N
  // outputs
  uint8_t* feasible;
  double* cost;
  double* coeffs;        // n_cand x N x 12 or nullptr
  int32_t* iters;        // or nullptr
  double row_tol;        // absolute row tolerance (default FQ_ROW_TOL; option "row_tol_1e9")
  // "first feasible dt wins" early exit (option "sweep_early_exit"; specialised kernel only): per problem the smallest dt
  // (bit pattern) of a candidate found feasible so far, or nullptr.  Candidates with a larger dt are not evaluated.
  unsigned long long* first_feasible;
  int sorted_dt;         // candidates of every problem are in ascending dt order (the chained replan's grids)
  int ee_width;          // candidates per time allocation (0: unknown); sizes the grid of an early-exit sweep
  // single-problem sweeps (fq_gen_new_traj*): the warp that finishes the LAST candidate runs genNewTraj's selection itself
  // and writes the winner record straight into mapped host memory -- no selection launch, no device-to-host copy.
  // sweep_done = counter of finished candidates (zeroed with the claim counters), or nullptr.
  int* sweep_done;
  int sweep_n_sigma;     // candidates per time allocation (the list is dt-major)
  int* sweep_idx;        // out (host-mapped): [0] dt index (-1 none), [1] sigma index
  double* sweep_win;     // out (host-mapped): [0] cost, [1 .. 12N] coefficients of the winner (a.coeffs must be set)
  // size-generic kernel only (fq_solve_batch_cert): per infeasible candidate, [n, violation, (row id, multiplier) x n]
  double* cert;
  int cert_stride;
};

struct FqSelectArgs
{
  int n_dt, n_sigma, N;
  const uint8_t* feasible;
  const double* cost;
  const double* coeffs;  // n_dt*n_sigma x N x 12
  int* out_idx;          // [0] dt index (-1 none), [1] sigma index
  double* out_cost;      // [0]
  double* out_coeffs;    // N x 12
};

// device-side fillX (solverGurobi.cpp:122-168) of the winner selected by fq_select_kernel
struct FqFillArgs
{
  int N, n_dt, max_samples;
  double DC;
  const double* dts;        // n_dt, device
  const int* win_idx;       // [0] winning dt index (-1: nothing to sample)
  const double* coeffs;     // N x 12 of the winner
  double* out;              // max_samples x 12
  int* n_samples;           // [0] number of samples written
};
cudaError_t fq_launch_fill(const FqFillArgs& a, cudaStream_t stream);

size_t fq_solve_smem_bytes(const FqKernelArgs& a);
// picks the size-specialised kernel when one exists (4 <= N <= 16, faces <= 2047), else the generic one;
// force_generic selects the generic kernel regardless (differential testing)
// `counters`: a.n_prob ints of device memory owned by the caller's context (per-problem claim counters of the
// persistent kernel; zeroed by the launch on `stream`)
cudaError_t fq_launch_solve(const FqKernelArgs& a, int max_cand_per_prob, cudaStream_t stream, int* counters, int sm_count,
                            bool force_generic = false, bool* used_specialised = nullptr);
bool fq_has_specialised(int N, int force_final, int max_faces);
cudaError_t fq_launch_select(const FqSelectArgs& a, cudaStream_t stream);

// ---- branch-and-bound over assignments (fq_bnb.cuh)
struct FqBnbLevel
{
  FqKernelArgs k;                  // plan + ONE problem
  int n_dt, P;
  const double* dts;               // device
  int depth, n_parents;
  const unsigned char* parents;
  const int* roots;
  unsigned char* children;
  int* n_children;
  int cap;
  unsigned long long* incumbent;
  void* leaves;                    // fqb::LeafRec[leaf_cap]: {int dt_idx, pad; double cost; uchar sigma[16]}
  int* n_leaves;
  int leaf_cap;
  int* flags;
};
size_t fq_bnb_node_bytes(int N, int force_final);     // 0 if unsupported
cudaError_t fq_launch_bnb_level(const FqBnbLevel& l, cudaStream_t stream);

// ---- chained replan (fq_pair.cuh): the small kernels between the whole and the safe sweep
struct FqSelectMultiArgs
{
  int n_prob, N, n_sig;                 // n_sig > 0: candidates are a (factor x assignment) grid, dt index = local / n_sig
  const int* cand_ofs;
  const double* dt;
  const uint8_t* sigma;
  const uint8_t* feasible;
  const double* cost;
  int* win_idx;                         // n_prob: candidate index relative to the problem's first candidate, -1 none
  double* win_cost;                     // n_prob (+inf none)
  double* win_dt;                       // n_prob (NaN none): also the dt list of the winners' re-solve
  uint8_t* win_sigma;                   // n_prob x N
  int* win_ofs;                         // n_prob + 1: 0,1,2,... (cand_ofs of the re-solve)
};

struct FqPairMidArgs
{
  int n_prob, N;
  double DC, r_fraction;
  const double* coeffs;                 // n_prob x N x 12: the whole winners
  const double* win_dt;                 // n_prob (NaN: no winner)
  const int* win_idx;
  double* x0_safe;                      // n_prob x 9 (NaN when there is no whole trajectory to branch from)
  int* n_samples;                       // n_prob
  int* k_safe;                          // n_prob
};

struct FqPairFinalArgs
{
  int n_prob, n_sig_w, n_sig_s;
  const int *win_idx_w, *win_idx_s, *n_samples, *k_safe;
  const double *win_cost_w, *win_cost_s, *win_dt_w, *win_dt_s, *dt_base_w, *dt_base_s, *x0_safe;
  fq_pair_result* out;
};

cudaError_t fq_launch_dtbase(int n_prob, int N, double DC, const double* x0, const double* xf, const double* lim,
                             double* dt_base, cudaStream_t stream);
cudaError_t fq_launch_expand_grid(int n_prob, int N, int n_fac, int n_sig, const double* factors, const uint8_t* sig_list,
                                  const double* dt_base, double* dt, uint8_t* sigma, int* cand_ofs, cudaStream_t stream);
cudaError_t fq_launch_select_multi(const FqSelectMultiArgs& a, cudaStream_t stream);
cudaError_t fq_launch_pair_mid(const FqPairMidArgs& a, cudaStream_t stream);
cudaError_t fq_launch_pair_final(const FqPairFinalArgs& a, cudaStream_t stream);
