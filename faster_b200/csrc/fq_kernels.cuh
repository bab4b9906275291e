// Device-side interface of the batched corridor-QP solver (sm_90a).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "../../include/faster_b200.h"
#include "fq_map.h"

#define FQ_WARPS_PER_CTA 4
#ifndef FQ_MIN_CTAS_PER_SM
#define FQ_MIN_CTAS_PER_SM 4
#endif
#ifndef FQ_MIN_CTAS_WHOLE
#define FQ_MIN_CTAS_WHOLE 4   // whole-mode kernels for N <= 10 (128 registers, no spills); 5 needs <= 96 registers, spills, and
                              // measured slower on config 4 (DESIGN section 9)
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

// ---- branch-and-bound over assignments (fq_bnb.cuh): corridor c of a level is problem c of k, with slices of its own
struct FqBnbLevel
{
  FqKernelArgs k;                  // plan + the corridors (k.n_prob)
  int n_dt;                        // row length of dts / roots / incumbent
  const double* dts;               // device, n_prob x n_dt
  int depth, cpc;                  // cpc: CTAs per corridor
  const int* n_parents;            // device, n_prob
  const unsigned char* parents;
  const int* roots;
  unsigned char* children;
  int* n_children;                 // device, n_prob
  int cap;                         // nodes per corridor
  unsigned long long* incumbent;
  void* leaves;                    // fqb::LeafRec[n_prob x leaf_cap]: {int dt_idx, corridor; double cost; uchar sigma[16]}
  int* n_leaves;
  int leaf_cap;
  int* flags;                      // n_prob x 2
  long long* nodes;                // n_prob, or nullptr
  int keep_ties;
  unsigned long long* lbound;      // keep_ties: n_prob x n_dt each (fq_bnb.cuh), or nullptr
  unsigned char* closed;
};
size_t fq_bnb_node_bytes(int N, int force_final);     // 0 if unsupported
// shared memory of a level launch for max_faces staged rows and item_cap rows per warp (0 if N is unsupported)
size_t fq_bnb_level_smem(int N, int force_final, int max_faces, int item_cap);
cudaError_t fq_launch_bnb_level(const FqBnbLevel& l, cudaStream_t stream);

// the chained replan's exact stage (fq_replan_pairs_exact*): roots before the levels, resolve after them
struct FqBnbChainArgs
{
  int n_prob, N, force_final, stride;   // stride: row length of dts / roots / incumbent (largest factor count)
  int max_faces;                        // rows the level kernel stages (corridors with more get status 2)
  int tree_ok;                          // 0: the level kernel has no instance for N (every tree corridor gets status 2)
  long long all_limit;
  const int *poly_ofs, *face_ofs;
  const double *Ab, *x0, *xf;
  double row_tol;
  const int* cand_ofs;                  // the sweep's candidates: factor-major, |L_c| per factor
  const double* cand_dt;
  int n_fac;                            // factors per corridor, or per corridor n_fac_j[c]
  const int* n_fac_j;
  int* win_idx;                         // the list winners (fq_select_multi_kernel); resolve overwrites them
  double *win_cost, *win_dt;
  uint8_t* win_sig;
  // tree state (ctx->d_bnb)
  double* dts;
  unsigned long long *incumbent, *lbound;
  uint8_t* closed;
  int* roots;
  int* n_par;                           // 2 x n_prob: parent counts of even / odd levels
  int* n_leaves;
  int* flags;
  long long* nodes;
  const void* leaves;
  int leaf_cap;
  uint8_t* status;
  uint8_t* changed;                     // out: the winner is the tree's
  // the list winners, saved by the resolve before it overwrites win_* (restored where the tree's winner does not re-solve)
  int* keep_idx;
  double *keep_cost, *keep_dt;
  uint8_t* keep_sig;
  int* exact_out;                       // out, or nullptr
  long long* nodes_out;                 // out, or nullptr
};
cudaError_t fq_launch_bnb_roots(const FqBnbChainArgs& a, cudaStream_t stream);
cudaError_t fq_launch_bnb_certify(const FqBnbChainArgs& a, cudaStream_t stream);
cudaError_t fq_launch_bnb_resolve(const FqBnbChainArgs& a, cudaStream_t stream);
// after the winners' coefficient solve (feasible = its flags): a tree winner the solve did not confirm is replaced by the
// list winner, whose dt goes to redo_dt (NaN elsewhere) for a second coefficient solve into redo_coeffs; adopt copies
// those coefficients (n_prob x N x 12) where redo_dt is set
cudaError_t fq_launch_bnb_fallback(const FqBnbChainArgs& a, const uint8_t* feasible, double* redo_dt, cudaStream_t stream);
cudaError_t fq_launch_bnb_adopt(int n_prob, int N, const double* redo_dt, const double* redo_coeffs, double* coeffs, cudaStream_t stream);

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
  // fq_replan_pairs_hr*: R's index per corridor from fq_pair_hr_kernel in place of the r_fraction rule; < 0: no safe path
  // is needed (no R, k_safe = n - 1).  NULL: the r_fraction rule.
  const int* r_index = nullptr;
};

// indexH / needToComputeSafePath / indexR of every corridor (fq_pair_hr_kernel, faster.cpp:173-251), after the whole
// sweep's coefficients
struct FqPairHrArgs
{
  int n_prob, N;
  double DC, drone_radius, delta_a, delta_H;
  const double* coeffs;                 // n_prob x N x 12: the whole winners
  const double* win_dt;                 // n_prob (NaN: no winner)
  const int* win_idx;
  const double* lim;                    // n_prob x 3: a_max = lim[3 j + 1]
  const int* unk_ofs;                   // n_prob + 1: corridor j's unknown cloud is rows unk_ofs[j] .. unk_ofs[j+1]-1 of unk
  const double* unk;
  int* r_index;                         // out n_prob: k_safe when a safe path is needed, else -1 (FqPairMidArgs::r_index)
  uint8_t* need;                        // out n_prob: needToComputeSafePath (0 without a whole winner)
  uint8_t* need_out;                    // out n_prob, or NULL: a copy for the caller
  int* index_H;                         // out n_prob, or NULL: indexH (-1 without a whole winner)
  // fq_replan_pairs_map*: corridor j's unknown cloud is the U of maps[map_index[j]] (map_index NULL: maps[0]) in place of
  // unk_ofs / unk, and only its cells near the sample are read
  const FqMapDev* const* maps = nullptr;
  const int* map_index = nullptr;
};

struct FqPairFinalArgs
{
  int n_prob, n_sig_w, n_sig_s;
  const int *win_idx_w, *win_idx_s, *n_samples, *k_safe;
  const double *win_cost_w, *win_cost_s, *win_dt_w, *win_dt_s, *dt_base_w, *dt_base_s, *x0_safe;
  fq_pair_result* out;
  // per-corridor assignment lists (fq_replan_pairs_assign*): the sweeps' candidate offsets, whose ranges are n_fac x the
  // corridor's list, replace n_sig_*; the winners' assignments (N x n_prob each) are copied to sigma_out_* if set.
  // All NULL / 0: one shared list of n_sig_* assignments.
  const int* cand_ofs_w = nullptr;
  const int* cand_ofs_s = nullptr;
  int n_fac_w = 0, n_fac_s = 0, N_w = 0, N_s = 0;
  const uint8_t* win_sig_w = nullptr;
  const uint8_t* win_sig_s = nullptr;
  uint8_t* sigma_out_w = nullptr;
  uint8_t* sigma_out_s = nullptr;
  // per-corridor windows (fq_replan_pairs_window*): corridor j's factor count, which then replaces n_fac_* in the split
  const int* n_fac_j_w = nullptr;
  const int* n_fac_j_s = nullptr;
  // exact stage (fq_replan_pairs_exact*): corridors whose winner came from the tree get *_sigma_index = the rank of the
  // winning assignment in L_j, or -1 when it is not in L_j
  const uint8_t* changed_w = nullptr;
  const uint8_t* changed_s = nullptr;
  const int* poly_ofs_w = nullptr;
  const int* poly_ofs_s = nullptr;
  long long all_limit = 0;
};

// factor_*, trials_* and the next windows of fq_replan_pairs_window* (fq_window.h), from the result records
struct FqPairWindowArgs
{
  int n_prob, max_fac_w, max_fac_s;
  const fq_pair_result* rec;            // n_prob records of the chain
  const int *cand_ofs_w, *cand_ofs_s;   // n_prob + 1 each (all 0: the sweep was emptied)
  const int *n_fac_w, *n_fac_s;         // n_prob: |F_j| (-1 refused)
  const double *fac_w, *fac_s;          // n_prob x max_fac_*: F_j
  const double *init_w, *final_w, *init_s, *final_s;
  double gamma_w, gammap_w, gamma_s, gammap_s;
  double *factor_w, *factor_s;          // out, or NULL
  int *trials_w, *trials_s;             // out, or NULL
  double *next_init_w, *next_final_w, *next_init_s, *next_final_s;   // out, or NULL; may alias init_* / final_*
  // fq_replan_pairs_hr*: need_safe[j] = 0 means the replan needed no safe sweep and still succeeded when the whole sweep
  // won; the safe window then follows last_factor_safe[j] (in/out: the safe winner's factor when the safe sweep wins).
  // NULL: every replan runs both sweeps.
  const uint8_t* need_safe = nullptr;
  double* last_factor_safe = nullptr;
  // fq_replan_pairs_queue*: n_prob FQ_QUEUE_* statuses of the appends; a corridor whose append is not FQ_QUEUE_OK keeps its
  // input windows (replan() returns before the update, faster.cpp:548-551).  NULL: no append gates the update.
  const int* gate = nullptr;
};

// the plan piece of every corridor (fq_replan_pairs_plan*, fq_pair.cuh): whole samples 0 .. k_safe, then every safe sample,
// each as fq_fill_x writes it with the winner's full sample count
struct FqPairPlanArgs
{
  int n_prob, N_w, N_s;
  double DC;
  const int *win_idx_w, *win_idx_s;     // n_prob: the sweeps' winners (-1: none)
  const double *win_dt_w, *win_dt_s;    // n_prob
  const int *n_samples, *k_safe;        // n_prob: fq_pair_mid_kernel's
  const uint8_t* need;                  // n_prob: needToComputeSafePath (fq_pair_hr_kernel), or NULL: a safe path is always needed
  const double *coeffs_w, *coeffs_s;    // n_prob x N x 12: the winners' coefficients
  long long cap;                        // rows of states
  double* states;                       // out: cap x 12
  long long* plan_ofs;                  // out: n_prob + 1, the exclusive scan of every succeeding corridor's rows
  int* status;                          // out n_prob (FQ_PLAN_*), or NULL
};
cudaError_t fq_launch_pair_plan(const FqPairPlanArgs& a, cudaStream_t stream);

// the committed plans of fq_queue_* and fq_replan_pairs_queue* (fq_queue.h, fq_pair.cuh): n_rows rings of cap states;
// corridor j works on row rows[j] (NULL: row j)
struct FqQueueArgs
{
  int n, n_rows, cap, delta_t;
  const int* rows;
  double* states;                       // n_rows x cap x 12
  int *head, *size;                     // n_rows
  const double* pos;                    // reset: n x 3
  double* x0;                           // select: out n x 9
  int* k_end;                           // select: out n; append: in/out
  const int* ticks;                     // pop: n
  int max_ticks;
  double* goals;                        // pop: out n x max_ticks x 12
  const double* G_term;                 // append: n x 3, or NULL
  double goal_radius;
  int* status;                          // append: out n (FQ_QUEUE_*)
  uint8_t* goal_seen;                   // append: out n, or NULL
};
cudaError_t fq_launch_queue_reset(const FqQueueArgs& q, cudaStream_t stream);
cudaError_t fq_launch_queue_select(const FqQueueArgs& q, cudaStream_t stream);
cudaError_t fq_launch_queue_pop(const FqQueueArgs& q, cudaStream_t stream);
// appendToPlan of every corridor's piece (the FqPairPlanArgs of the chain, whose cap, states, plan_ofs and status are not read)
cudaError_t fq_launch_pair_queue(const FqPairPlanArgs& a, const FqQueueArgs& q, cudaStream_t stream);

// the device decomposition of one sweep's corridors (fq_decomp.cuh): fq_decomp_kernel stages every polytope's rows in a slot
// of cap_pf rows (slot j * max_poly + s), fq_decomp_csr_kernel packs them into the sweep's CSR and sets the final states
struct FqDecompArgs
{
  int n_prob, max_poly;
  const int* poly_ofs;                  // n_prob + 1: P_j
  const double* path;                   // corridor j: rows poly_ofs[j] + j .. poly_ofs[j+1] + j
  const double* first;                  // NULL, or n_prob x 9: vertex 0 of corridor j is first[9 j .. 9 j + 2] (R; NaN: not run)
  const int* obs_ofs;                   // n_prob + 1
  const double* obs;
  int max_obs;                          // clouds above it are refused; sizes the spill slices
  double bbox[3], inflate, z_ground;
  int cap_pf;                           // staged rows per polytope: the max_poly_faces cap
  int max_faces;                        // the corridor cap
  double* stage;                        // n_prob x max_poly x cap_pf x 4
  int* stage_n;                         // n_prob x max_poly: rows, or -FQ_DECOMP_* status
  double* spill;                        // n_prob x max_poly x spill_n x 4 (x, y, z, dist of survivors kFitPts and beyond)
  uint8_t* spill_flag;                  // n_prob x max_poly x spill_n
  int spill_n;                          // max(max_obs - kFitPts, 0)
  // fq_decomp_csr_kernel
  const double* goal;                   // n_prob x 3, or NULL
  int face_cap;                         // face_ofs has face_cap + 1 entries (n_prob x max_poly)
  int* face_ofs;                        // out: absolute CSR over poly_ofs
  double* Ab;                           // out: n_prob x max_faces rows of 4
  double* xf;                           // out: n_prob x 9 final states (NaN rows for failed corridors)
  double* pos_out;                      // out n_prob x 3, or NULL
  int* status;                          // out n_prob, or NULL
  // fq_replan_pairs_map*: an indexed map in place of obs_ofs / obs.  Corridor j reads maps[map_index[j]] (map_index NULL:
  // maps[0]; outside 0 .. n_maps-1: FQ_DECOMP_CLOUD): its occupied cloud O (map_unk 0), or its unknown cloud U followed by
  // O (map_unk 1, O's indices after U's), in the cells the segment's AABB overlaps.  max_obs then caps the survivors of one
  // segment, and spill_idx (spill_n per slot) holds the spilled survivors' indices in the cloud.
  const FqMapDev* const* maps = nullptr;
  const int* map_index = nullptr;
  int n_maps = 0, map_unk = 0;
  int* spill_idx = nullptr;
};
size_t fq_decomp_spill_n(int max_obs);
cudaError_t fq_launch_decomp(const FqDecompArgs& a, cudaStream_t stream);

cudaError_t fq_launch_dtbase(int n_prob, int N, double DC, const double* x0, const double* xf, const double* lim,
                             double* dt_base, cudaStream_t stream);
cudaError_t fq_launch_expand_grid(int n_prob, int N, int n_fac, int n_sig, const double* factors, const uint8_t* sig_list,
                                  const double* dt_base, double* dt, uint8_t* sigma, int* cand_ofs, cudaStream_t stream);
// per-corridor assignment lists (fq_pair.cuh, fq_assign.h): offsets of n_fac x |L_j| (emptied when a corridor has more than
// max_poly polytopes or the total is not n_cand), then the factor x list grid with unranked assignments
cudaError_t fq_launch_assign_offsets(int n_prob, int N, int n_fac, long long all_limit, int max_poly, long long n_cand,
                                     const int* poly_ofs, int* cand_ofs, cudaStream_t stream);
cudaError_t fq_launch_expand_assign(int n_prob, int N, int n_fac, long long all_limit, const double* factors, const double* dt_base,
                                    const int* poly_ofs, const int* cand_ofs, double* dt, uint8_t* sigma, cudaStream_t stream);
// per-corridor windows (fq_window.h): F_j into rows of max_fac factors and |F_j| (-1 refused); the offsets and the
// expansion with those rows and counts (n_fac = max_fac; the total must be at most n_cand); the records' window outputs
cudaError_t fq_launch_window_factors(int n_prob, int max_fac, const double* init, const double* final_, double inc, double* fac,
                                     int* n_fac_j, cudaStream_t stream);
cudaError_t fq_launch_window_offsets(int n_prob, int N, int max_fac, long long all_limit, int max_poly, long long cap,
                                     const int* poly_ofs, const int* n_fac_j, int* cand_ofs, cudaStream_t stream);
cudaError_t fq_launch_expand_window(int n_prob, int N, int max_fac, long long all_limit, const double* fac, const int* n_fac_j,
                                    const double* dt_base, const int* poly_ofs, const int* cand_ofs, double* dt, uint8_t* sigma,
                                    cudaStream_t stream);
cudaError_t fq_launch_pair_window(const FqPairWindowArgs& a, cudaStream_t stream);
cudaError_t fq_launch_select_multi(const FqSelectMultiArgs& a, cudaStream_t stream);
cudaError_t fq_launch_pair_mid(const FqPairMidArgs& a, cudaStream_t stream);
cudaError_t fq_launch_pair_hr(const FqPairHrArgs& a, cudaStream_t stream);
// the map table of one submission: table[at + i] = m[i] for i < n, the device addresses of the maps' descriptors (they
// pass through kernel parameters, so that the table needs no host copy and a CUDA graph can capture it; the descriptors
// never move, so a replay reads each map's last update)
struct FqMapTableChunk
{
  static constexpr int kCap = 64;
  const FqMapDev* m[kCap];
  int n, at;
  const FqMapDev** table;
};
cudaError_t fq_launch_map_table(const FqMapTableChunk& c, cudaStream_t stream);
cudaError_t fq_launch_pair_final(const FqPairFinalArgs& a, cudaStream_t stream);
