/* faster_b200 -- C ABI of the H100-native trajectory-optimisation core.
 *
 * This is the drop-in boundary: everything FASTER's SolverGurobi asks of Gurobi (reference
 * faster/src/solverGurobi.cpp, calls m.addVar/addConstr/addGenConstrIndicator/setObjective/optimize/get at
 * :80,:119,:226,:246,:283-286,:349-354,:371-377,:397-404,:513-521,:559-581) is replaced by the entry points below.
 * Plain pointers and sizes only; no C++/torch types; never throws.  All floating point is IEEE double.
 *
 * Model solved per candidate (dt, sigma)  [reference lines in brackets]:
 *   N cubic segments x 3 axes, coefficients x[t][0..11] = ax ay az bx by bz cx cy cz dx dy dz     [:70-84]
 *   minimise sum_t sum_axis (6 a)^2                                                                 [:113-119]
 *   s.t. initial state [:359-380], final state (position only if force_final) [:332-357],
 *        C2 continuity [:499-524], |v|,|a|,|j| boxes at segment starts [:390-407],
 *        the 4 Bezier control points of segment t inside polytope sigma[t] [:180-291,:833-862].
 * A candidate is feasible iff that QP has a solution (row tolerance FQ_ROW_TOL); cost is Gurobi's ObjVal.
 *
 * Return codes: 0 ok; <0 error (FQ_E_*), message via fq_last_error().  Per-candidate status is written to
 * `feasible` (1 optimal, 0 infeasible or numerically abandoned -- the reference maps every non-OPTIMAL Gurobi
 * status to "not solved", solverGurobi.cpp:580-648).
 */
#ifndef FASTER_B200_H
#define FASTER_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FQ_ABI_VERSION 2
#define FQ_MAX_N 16               /* segments per trajectory                                  */
#define FQ_MAX_POLY 32            /* polytopes per corridor problem                           */
/* Faces per problem are bounded by shared memory, and the bound depends on N and mode: a problem's rows and per-warp
 * solver state live in one block's shared memory (227 KB on an H100).  The size-specialised kernel takes up to 2047 faces
 * and less as N grows (N = 10 whole: 951 faces in one polytope, 1279 in three equal ones; N = 16 safe: 463 / 695).  A
 * larger problem runs on the size-generic kernel instead, with the same results to rounding (N = 10 whole: up to 5600
 * faces; N = 16 safe: 2244).  Beyond that every solve entry point refuses the problem with FQ_E_ARG ("problem too large for
 * shared memory").  DESIGN.md section 3.4 has the table. */
#define FQ_ROW_TOL 1e-8           /* DEFAULT absolute row violation tolerance (m, m/s, m/s^2, m/s^3); run-time
                                     option "row_tol_1e9" of fq_set_option                                   */

#define FQ_E_ARG (-1)
#define FQ_E_CUDA (-2)
#define FQ_E_NOMEM (-3)
#define FQ_E_NOGPU (-4)

typedef struct fq_ctx fq_ctx;     /* opaque: device, stream, plan tables, scratch             */

int fq_abi_version(void);
/* 1 if this build has the named feature: "sweep_early_exit", "replan_pairs", "multi_gpu", "row_tol", "certificates",
 * "replan_pairs_assign", "replan_pairs_window", "replan_pairs_exact", "replan_pairs_decomp", "replan_pairs_hr",
 * "replan_pairs_map", "replan_pairs_plan", "map_paths", "replan_pairs_queue", "jps_batch". */
int fq_has_feature(const char* name);

/* Threading: a context is used from one thread at a time, like a SolverGurobi instance in the reference (one replan
 * callback, SURVEY.md 8b); different contexts are independent.  With fq_solve_multi_dev at most 64 launches of one
 * context may be in flight on DIFFERENT streams at once (launches on one stream are ordered and unlimited).
 *
 * Creates a solver context on CUDA device `device`.  Fails with FQ_E_NOGPU when no usable GPU exists:
 * there is no CPU fallback.  Replaces `new GRBEnv()` / GRBModel construction (solverGurobi.hpp:154-155). */
int fq_create(fq_ctx** out, int device);
void fq_destroy(fq_ctx* ctx);
const char* fq_last_error(const fq_ctx* ctx);   /* ctx may be NULL: last creation error */

/* Tuning / testing knobs.  "force_generic_kernel" (0/1): use the size-generic kernel even where a size-specialised one
 * exists (the two are independent implementations of the same solve; tests run both).  "throughput_slices" (1..64, 0 =
 * default: 4, or 2 for fq_solve_multi_async): how many launches a large host batch is cut into (upload / solve / download of consecutive slices
 * overlap on two streams).  "max_faces_per_polytope": see fq_solve_multi_dev.  "row_tol_1e9" (1..1000000): the absolute row
 * tolerance of every later solve of the context in units of 1e-9 -- 10 is the default FQ_ROW_TOL = 1e-8, 1000 is Gurobi's
 * default FeasibilityTol 1e-6 (the reference sets no tolerance parameter, solverGurobi.cpp:479-487).  0 is refused
 * (FQ_E_ARG): at zero tolerance rounding alone keeps a row that was just made active violated, and the active set cycles
 * until the iteration cap gives up on solvable candidates.  1 (1e-9) is also the lowest FeasibilityTol Gurobi accepts.  "cert_memo" (any
 * value) is accepted and ignored: the GPU kernels have no infeasibility-certificate memo.
 * "sweep_early_exit" (0/1, default 0): genNewTraj keeps the FIRST feasible factor (solverGurobi.cpp:445-446), so once a
 * problem has a feasible candidate, candidates with a larger dt cannot win; with this option they are not evaluated
 * (reported feasible = 0, cost = +inf, iters = -3) and claims run in ascending dt.  The winners (fq_replan_pairs results,
 * fq_gen_new_traj*, fq_solve_multi_sharded's winners) are unchanged; the per-candidate arrays are no longer complete.
 * fq_gen_new_traj* pick the first dt INDEX with a feasible assignment, so they apply the option only to an ascending dt
 * list; a list in any other order is evaluated in full.
 * Returns 0 or FQ_E_ARG. */
int fq_set_option(fq_ctx* ctx, const char* key, int value);

/* One corridor problem, n_cand candidates (dt[i], sigma[i*N .. i*N+N-1]); HOST pointers.
 * Replaces the per-trial model rebuild + m.optimize() of genNewTraj (solverGurobi.cpp:449-458) for a whole
 * batch of trials at once.
 *   x0, xf     9 doubles each: pos(3) vel(3) accel(3)            (setX0/setXf, :298-330)
 *   lim        v_max, a_max, j_max                               (setBounds, :409-416)
 *   P          number of polytopes (0 => no corridor rows, sigma ignored, :217)
 *   face_ofs   P+1 ints; polytope p owns rows face_ofs[p] .. face_ofs[p+1]-1 of Ab
 *   Ab         rows [Ax Ay Az b], A x <= b                       (setPolytopes, :175-178; polyhedron.h:114-185)
 *   feasible   n_cand bytes out;  cost n_cand doubles out (+inf when infeasible)
 *   coeffs     n_cand*N*12 doubles out in the x[t][i] order of solverGurobi.cpp:72, or NULL
 *   iters      n_cand int32 out (active-set iterations), or NULL                                         */
int fq_solve_batch(fq_ctx* ctx, int N, int force_final, const double* x0, const double* xf, const double* lim,
                   int P, const int* face_ofs, const double* Ab, int n_cand, const double* dt,
                   const uint8_t* sigma, uint8_t* feasible, double* cost, double* coeffs, int32_t* iters);

/* fq_solve_batch, plus a PROOF for every candidate reported infeasible: the Farkas certificate the solver stopped on, so
 * that a caller (tests/test_certificates_gpu.py) can verify the flag on the literal rows of the reference's model without
 * trusting the solver.  cert[i*cert_stride ..]: [0] n = number of rows, [1] violation of the entering row at the last
 * iterate, then n pairs (row id, multiplier >= 0); the pairs' rows are inconsistent: sum mult_k row_k = 0 in the free
 * directions and sum mult_k rhs_k < 0.  Row ids: box rows (solverGurobi.cpp:390-407) 10000000 + type*10000 + axis*1000 +
 * t*10 + s with type 0/1/2 = v/a/j at the start of segment t, s = 1 for "<= +max", 0 for ">= -max"; corridor rows
 * (:249-287) t*100000 + f*10 + k: face f (row of Ab) on control point k of segment t.  n = 0: feasible, or abandoned.
 * cert_stride >= 4 + 6 FQ_MAX_N.  Runs the size-generic kernel (which tracks row identities); HOST pointers. */
int fq_solve_batch_cert(fq_ctx* ctx, int N, int force_final, const double* x0, const double* xf, const double* lim,
                        int P, const int* face_ofs, const double* Ab, int n_cand, const double* dt,
                        const uint8_t* sigma, uint8_t* feasible, double* cost, double* cert, int cert_stride);

/* n_prob corridor problems in one launch; HOST pointers.  Problem j owns candidates
 * cand_ofs[j] .. cand_ofs[j+1]-1 and polytopes poly_ofs[j] .. poly_ofs[j+1]-1 (indices into face_ofs, which has
 * poly_ofs[n_prob]+1 entries).  x0/xf are n_prob*9, lim n_prob*3.  Outputs as fq_solve_batch. */
int fq_solve_multi(fq_ctx* ctx, int N, int force_final, int n_prob, const double* x0, const double* xf,
                   const double* lim, const int* poly_ofs, const int* face_ofs, const double* Ab,
                   const int* cand_ofs, const double* dt, const uint8_t* sigma, uint8_t* feasible, double* cost,
                   double* coeffs, int32_t* iters);

/* fq_solve_multi without the final wait: returns once the copies and launches are enqueued (large batches; small ones
 * are simply complete on return).  Outputs are valid after fq_wait(ctx) -- or after the next call on the same context,
 * which settles a deferred call before it reuses the context's device buffers.  Input and output arrays must stay
 * alive and untouched until then; pinned (page-locked) arrays make the copies truly asynchronous.  Two contexts (the
 * reference keeps two solver objects, sg_whole_ and sg_safe_: faster.hpp:74-75) can thus have their batches in flight
 * together, the second batch's CTAs filling the SMs that the first one's last launch leaves idle. */
int fq_solve_multi_async(fq_ctx* ctx, int N, int force_final, int n_prob, const double* x0, const double* xf,
                         const double* lim, const int* poly_ofs, const int* face_ofs, const double* Ab,
                         const int* cand_ofs, const double* dt, const uint8_t* sigma, uint8_t* feasible, double* cost,
                         double* coeffs, int32_t* iters);
/* Blocks until everything enqueued on the context's own streams has finished (deferred host batches and
 * fq_solve_multi_dev launches made with stream == NULL). */
int fq_wait(fq_ctx* ctx);

/* Same as fq_solve_multi with every array already resident in DEVICE memory of the context's GPU.  The library
 * cannot read device arrays on the host, so the caller also passes `max_cand_per_prob` (largest
 * cand_ofs[j+1]-cand_ofs[j]) and `max_faces_per_prob` (largest number of Ab rows owned by one problem).  Ab must
 * be 16-byte aligned.  Launches on `stream` (a cudaStream_t; NULL = the context's stream) and returns without
 * synchronising. */
int fq_solve_multi_dev(fq_ctx* ctx, int N, int force_final, int n_prob, const double* d_x0, const double* d_xf,
                       const double* d_lim, const int* d_poly_ofs, const int* d_face_ofs, const double* d_Ab,
                       const int* d_cand_ofs, int max_cand_per_prob, int max_faces_per_prob, const double* d_dt,
                       const uint8_t* d_sigma, uint8_t* d_feasible, double* d_cost, double* d_coeffs,
                       int32_t* d_iters, void* stream);

/* The dt sweep of genNewTraj (solverGurobi.cpp:445-472) as one launch: candidates are the grid
 * dts[0..n_dt) x sigmas[0..n_sigma); the winner is the FIRST dt (ascending index) that has any feasible sigma,
 * and within it the minimum-cost sigma (= the MIQP optimum over the supplied assignments).  HOST pointers.
 * Returns 1 solved / 0 no feasible candidate / <0 error.  Outputs (may be NULL): winning dt index, sigma
 * index, cost, coefficients N*12. */
int fq_gen_new_traj(fq_ctx* ctx, int N, int force_final, const double* x0, const double* xf, const double* lim,
                    int P, const int* face_ofs, const double* Ab, int n_dt, const double* dts, int n_sigma,
                    const uint8_t* sigmas, int* dt_index, int* sigma_index, double* cost, double* coeffs);

/* fq_gen_new_traj followed by fillX ON THE DEVICE (solverGurobi.cpp:122-168, resetX :382-388), chained on the same
 * stream: solve launch -> selection -> sampling kernel -> one D2H.  `samples` receives min(n, max_samples) rows of 12
 * doubles (pos vel accel jerk at t = (i+1) DC, last row's vel/accel/jerk zeroed), n = max(2, (int)(N dt/DC)) for the
 * winning dt; *n_samples is the count.  Same return convention as fq_gen_new_traj.  Provided for completeness and
 * measured in DESIGN.md: sampling on the host from the 96 N bytes of coefficients (fq_fill_x) is the faster route. */
int fq_gen_new_traj_sampled(fq_ctx* ctx, int N, int force_final, const double* x0, const double* xf, const double* lim,
                            int P, const int* face_ofs, const double* Ab, int n_dt, const double* dts, int n_sigma,
                            const uint8_t* sigmas, double DC, int max_samples, int* dt_index, int* sigma_index,
                            double* cost, double* coeffs, double* samples, int* n_samples);

/* genNewTraj with the EXACT MIQP optimum: the minimum over all P^N interval->polytope assignments for every time
 * allocation, which is what Gurobi's branch-and-bound over the binaries b[t][p] returns (solverGurobi.cpp:217-246,
 * :445-472).  Branch-and-bound on the GPU over the segments (dual warm starts from the parent node, bound pruning with the
 * best non-decreasing assignment as incumbent).  Outputs: winning dt index (-1 none), its assignment sigma_out[N], cost,
 * coefficients; *nodes_out = nodes evaluated; *exact_out = 0 if the tree had to be cut (more than 65536 open nodes on one
 * level, a node's solve gave up, N < 4, more than 2047 faces, or the tree's shared-memory footprint is too large) and the
 * result is the best non-decreasing assignment instead.  FQ_E_ARG if that assignment list is too long for the pre-sweep:
 * C(N+P-1, N) > 2^20 or C(N+P-1, N) x n_dt > 2^24.  Returns 1 / 0 / <0. */
int fq_gen_new_traj_exact(fq_ctx* ctx, int N, int force_final, const double* x0, const double* xf, const double* lim,
                          int P, const int* face_ofs, const double* Ab, int n_dt, const double* dts, int* dt_index,
                          uint8_t* sigma_out, double* cost, double* coeffs, long* nodes_out, int* exact_out);

/* ---- chained replan: whole sweep -> R -> safe sweep, many corridors in one submission ----------------------------
 *
 * One Faster::replan() asks its two solver objects (sg_whole_, sg_safe_; faster.hpp:74-75) for two DEPENDENT sweeps:
 *   sg_whole_.setX0(A); setXf(E); setPolytopes(whole corridor); genNewTraj(); fillX()          faster.cpp:406-430
 *   R = sg_whole_.X_temp_[k_safe]                                                             faster.cpp:474-475
 *   sg_safe_.setX0(R); setXf(M); setPolytopes(safe corridor); setForceFinalConstraint(false); genNewTraj(); fillX()
 *                                                                                              faster.cpp:521-537
 * fq_replan_pairs does that for n_prob corridors at once without a host round trip between the sweeps: the selection
 * (first feasible factor, then minimum cost: solverGurobi.cpp:445-472), the sample R of fillX (:122-168), the safe
 * sweep's getDTInitial(R, M) (:659-759) and its time allocations factor * max(dt_initial, 2 DC) (:494-497) are all
 * computed on the device.  k_safe = min(n - 1, (int)(r_fraction * n)), n = resetX's sample count (:382-388), stands in
 * for findIndexR (faster.cpp:173-216), which needs the planner's map.  A corridor whose whole sweep finds nothing gets
 * no safe sweep: all its safe candidates are "not solved".
 *
 * Candidates of corridor j: whole (factors_whole[f], sigmas_whole[s]), index f * n_sig_whole + s; safe likewise. */
typedef struct fq_pair_result
{
  int whole_dt_index, whole_sigma_index;   /* winner of the whole sweep (-1, -1: none)                              */
  int safe_dt_index, safe_sigma_index;     /* winner of the safe sweep                                               */
  double whole_cost, safe_cost;            /* +inf: none                                                             */
  double whole_dt, safe_dt;                /* winning time allocations (NaN: none)                                   */
  double whole_dt_base, safe_dt_base;      /* max(getDTInitial, 2 DC) of the two sweeps, as computed on the device   */
  int n_samples_whole, k_safe;             /* resetX count of the whole winner; index of R among its samples         */
  double R[9];                             /* pos vel accel of R = start state of the safe sweep (NaN: none)         */
} fq_pair_result;

typedef struct fq_pair_args
{
  int n_prob;                              /* corridors = replans                                                    */
  int N_whole, N_safe;                     /* segments (faster.yaml N_whole, N_safe)                                 */
  double DC;                               /* setDC: sampling period of fillX, floor 2 DC of findDT                  */
  double r_fraction;                       /* where R sits on the whole trajectory, in [0, 1]                        */
  const double* x0;                        /* n_prob x 9: A (pos vel accel)            setX0, faster.cpp:406         */
  const double* xf_whole;                  /* n_prob x 9: E                            setXf, faster.cpp:407         */
  const double* xf_safe;                   /* n_prob x 9: M                            setXf, faster.cpp:522         */
  const double* lim;                       /* n_prob x 3: v_max a_max j_max            setBounds                     */
  const int* poly_ofs_whole;               /* corridors in the CSR layout of fq_solve_multi    faster.cpp:408        */
  const int* face_ofs_whole;
  const double* Ab_whole;
  const int* poly_ofs_safe;                /*                                                  faster.cpp:523        */
  const int* face_ofs_safe;
  const double* Ab_safe;
  int n_fac_whole;  const double* factors_whole;   /* ascending factors of the whole sweep (solverGurobi.cpp:445-446) */
  int n_sig_whole;  const uint8_t* sigmas_whole;   /* n_sig_whole x N_whole assignments                               */
  int n_fac_safe;   const double* factors_safe;
  int n_sig_safe;   const uint8_t* sigmas_safe;    /* n_sig_safe x N_safe                                             */
  uint8_t* feasible_whole;  double* cost_whole;    /* out, n_prob x n_fac_whole x n_sig_whole each; may be NULL       */
  uint8_t* feasible_safe;   double* cost_safe;     /* out, n_prob x n_fac_safe x n_sig_safe each; may be NULL         */
  double* coeffs_whole;                    /* out, n_prob x N_whole x 12 (winners, x[t][i] order); may be NULL       */
  double* coeffs_safe;                     /* out, n_prob x N_safe x 12; may be NULL                                 */
  fq_pair_result* results;                 /* out, n_prob                                                            */
  /* fq_replan_pairs_dev only (the library cannot read device arrays): largest number of Ab rows of one corridor and
   * of one polytope, whole and safe */
  int max_faces_whole, max_poly_faces_whole, max_faces_safe, max_poly_faces_safe;
} fq_pair_args;

/* HOST pointers everywhere; blocks until the results are in the caller's arrays.  Returns 0 or FQ_E_*. */
int fq_replan_pairs(fq_ctx* ctx, const fq_pair_args* args);
/* The same, returning once everything is enqueued; results are valid after fq_wait(ctx).  Arrays must stay alive. */
int fq_replan_pairs_async(fq_ctx* ctx, const fq_pair_args* args);
/* DEVICE pointers everywhere (the struct itself lives on the host); enqueues on `stream` (NULL: the context's) and
 * returns without synchronising.  One chain per context may be in flight on a given stream order: calls on the same
 * stream are ordered and may follow each other freely; use one context per concurrently used stream (the chain keeps
 * its intermediate arrays in the context).  With a communicator attached (fq_comm_init / fq_create_multi) and
 * `results_all` != NULL the chain ends with the path's one collective: an all-gather of the n_prob result records of
 * every rank into results_all[world x n_prob] (device). */
int fq_replan_pairs_dev(fq_ctx* ctx, const fq_pair_args* args, fq_pair_result* results_all, void* stream);

/* ---- chained replan with a per-corridor assignment list -------------------------------------------------------------
 *
 * Corridors of one batch need not have the same polytope count: Faster::replan trims the JPS paths to at most max_poly + 1
 * vertices (deleteVertexes, faster.cpp:393,:495) and every segment becomes one polytope, so near the goal or at the first
 * unknown cell a corridor has fewer.  The entry points below give every corridor j of a sweep with N segments its OWN list
 * L(N, P_j, all_limit), P_j = its polytope count, generated on the device (nothing is enumerated on the host):
 *   P_j = 0                   the single all-zero assignment
 *   P_j^N <= all_limit        all P_j^N assignments, lexicographic with segment 0 most significant (base-P_j digits)
 *   otherwise                 the non-decreasing assignments in the order of fq_monotone_sigmas, C(N + P_j - 1, N)
 * all_limit = 0: always non-decreasing.  all_limit = 4096 with N = 6, P <= 3 (729 assignments) enumerates every assignment
 * and so returns the exact MIQP optimum over the factors, as SolverGurobi's AUTO mode does.
 *
 * Corridor j's candidates are n_fac x |L_j|, factor-major (index f * |L_j| + s), at cand_ofs[j] .. cand_ofs[j+1]-1 of the
 * per-candidate outputs (feasible_* / cost_*).  The selection is fq_replan_pairs's; the result records' *_sigma_index is
 * the index in the corridor's own list.  fq_pair_args is used as for fq_replan_pairs except that sigmas_* must be NULL and
 * n_sig_* 0 (FQ_E_ARG otherwise: a caller must not believe that a shared list was used).  FQ_E_ARG also for all_limit < 0,
 * a corridor list longer than 2^20 and more than 2^30 candidates in a sweep. */
typedef struct fq_pair_assign
{
  long all_limit;                          /* rule above                                                             */
  int max_poly_whole, max_poly_safe;       /* _dev only: largest polytope count of one corridor (hint)               */
  long n_cand_whole, n_cand_safe;          /* _dev only: total candidates of each sweep (hint, checked)              */
  int* cand_ofs_whole;                     /* out, n_prob + 1: candidate offsets of the whole sweep, or NULL         */
  int* cand_ofs_safe;                      /* out, n_prob + 1, or NULL                                               */
  uint8_t* sigma_whole;                    /* out, n_prob x N_whole: the whole winners' assignments (0s: none), or NULL */
  uint8_t* sigma_safe;                     /* out, n_prob x N_safe, or NULL                                          */
} fq_pair_assign;

/* |L(N, P, all_limit)|: candidates per factor of a corridor with P polytopes.  < 0 (FQ_E_ARG) if N is not in 1..FQ_MAX_N,
 * P not in 0..FQ_MAX_POLY, all_limit < 0 or the list is longer than 2^20.  Pure host code. */
long fq_pair_assign_count(int N, int P, long all_limit);
/* HOST pointers everywhere; blocks until every output is in the caller's arrays.  On a multi-GPU context the corridors
 * are sharded by candidate count, whole + safe (fq_shard_range over the summed per-corridor offsets, which the host knows
 * from poly_ofs): the shards balance the work, not the corridor count.  DESIGN.md section 6. */
int fq_replan_pairs_assign(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign);
/* The same, returning once everything is enqueued; outputs are valid after fq_wait(ctx).  Arrays must stay alive. */
int fq_replan_pairs_assign_async(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign);
/* DEVICE pointers everywhere (both structs live on the host), as fq_replan_pairs_dev.  The library cannot read poly_ofs, so
 * the caller passes max_poly_* (largest polytope count of one corridor) and n_cand_* (the sweeps' total candidates:
 * n_fac_* x the sum of |L_j|; the per-candidate outputs hold that many).  The device computes the offsets and checks them:
 * if a corridor has more polytopes than max_poly_* or the total is not n_cand_*, that sweep gets NO candidates -- every
 * cand_ofs entry of it is 0, nothing is written to its per-candidate outputs, and every corridor's winner of that sweep is
 * "none" (indices -1; a corridor without a whole winner has no safe winner either).  The call itself still returns 0: it
 * does not synchronise.  Refused up front (FQ_E_ARG): max_poly_* outside 0..FQ_MAX_POLY, n_cand_* outside 0..2^30. */
int fq_replan_pairs_assign_dev(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, fq_pair_result* results_all,
                               void* stream);

/* ---- chained replan with a per-corridor time-allocation window ------------------------------------------------------
 *
 * The one piece of solver state Faster::replan() carries from one replan to the next is each solver object's window of
 * time-allocation factors: [1, 10] with step increment_* at start-up (setFactorInitialAndFinalAndIncrement, faster.cpp:57,
 * :68), then, after every replan in which BOTH sweeps succeed, [max(f* - gamma, 1.0), f* + gammap] around the factor that
 * worked (faster.cpp:582-588).  genNewTraj visits the factors `for (double i = fi; i <= ff; i = i + inc)`
 * (solverGurobi.cpp:445-446).  The entry points below give corridor j its OWN window and list:
 *   F_j = the factors that loop visits for (init_*[j], final_*[j], inc_*), accumulated as it does (never fi + k inc);
 *         final < init gives no factor (no candidate, no winner).  Refused: a bound or inc not finite, init <= 0,
 *         inc <= 0, more than 4096 factors (the drop-in class's cap), or an accumulation that stalls (i + inc == i).
 *   candidates of corridor j: |F_j| x |L_j| (L_j: the per-corridor assignment list of fq_pair_assign), factor-major,
 *         dt = F_j[f] * max(getDTInitial, 2 DC); *_dt_index of the result records indexes F_j.
 *   factor_*[j]  factor_that_worked_ (NaN: no winner)
 *   trials_*[j]  the winner's index in F_j + 1; |F_j| without a winner; 0 for a sweep that did not run (the safe sweep
 *                after a whole sweep without winner; an emptied sweep of the _dev variant)
 *   next_*[j]    the window of the next replan: if both sweeps won, max(f*_w - gamma_whole, 1.0) and f*_w + gammap_whole
 *                (and likewise for safe); otherwise the input window unchanged, since replan() returns before its update
 *                (faster.cpp:420-424, :529-533).  appendToPlan's early return (:548) depends on the planner's plan_ deque
 *                and is not modelled; the states appendToPlan pushes are (fq_replan_pairs_plan below), and with the deque
 *                on the device the early return is too (fq_replan_pairs_queue below).
 * fq_pair_args is used as for fq_replan_pairs_assign except that factors_* must be NULL and n_fac_* 0 (FQ_E_ARG otherwise);
 * `assign` is required.  Feature "replan_pairs_window". */
typedef struct fq_pair_window
{
  const double *init_whole, *final_whole, *init_safe, *final_safe;  /* n_prob each: setFactorInitialAndFinalAndIncrement */
  double inc_whole, inc_safe;                                       /* par_.increment_*                                  */
  double gamma_whole, gammap_whole, gamma_safe, gammap_safe;        /* par_.gamma*_, for the next window                */
  int max_fac_whole, max_fac_safe;                                  /* _dev only: largest |F_j| (hint, checked)          */
  double *factor_whole, *factor_safe;                               /* out n_prob, or NULL                               */
  int *trials_whole, *trials_safe;                                  /* out n_prob, or NULL                               */
  double *next_init_whole, *next_final_whole, *next_init_safe, *next_final_safe;  /* out n_prob, or NULL; MAY alias the inputs */
} fq_pair_window;

/* |F(fi, ff, inc)|, writing its first min(|F|, cap) factors to out (may be NULL); FQ_E_ARG when the window is refused.
 * Pure host code, the same source as the device's. */
long fq_pair_window_factors(double fi, double ff, double inc, double* out, long cap);
/* HOST pointers everywhere (window arrays included); every window is validated here (FQ_E_ARG).  Blocks until every output
 * is in the caller's arrays.  On a multi-GPU context the corridors are sharded by candidate count |F_j| x |L_j|, whole +
 * safe, as fq_replan_pairs_assign does. */
int fq_replan_pairs_window(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window);
/* The same, returning once everything is enqueued; outputs are valid after fq_wait(ctx).  Arrays must stay alive. */
int fq_replan_pairs_window_async(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window);
/* DEVICE pointers everywhere (the three structs live on the host), as fq_replan_pairs_assign_dev, so that consecutive
 * replans of a batch can pass each call's next_* arrays (or the same arrays: they may alias init_* / final_*) to the next
 * call without a host round trip.  The library cannot read the windows, so for this call assign->n_cand_* is a CAPACITY
 * (the per-candidate outputs hold that many; the sweep's total must not exceed it) and window->max_fac_* bounds |F_j|
 * (the rows of factors kept on the device; for gamma = gammap = 20 and inc = 1 every window after the first has at most
 * 41 factors).  cand_ofs_* report the layout used.  If a window of a sweep is refused, a corridor has more than max_fac_*
 * factors or more than max_poly_* polytopes, or the total exceeds the capacity, that sweep gets NO candidates: every winner
 * of it is "none", nothing is written to its per-candidate outputs, and every window is returned unchanged, so a closed
 * loop's state is never corrupted.  The call still returns 0.  Refused up front (FQ_E_ARG): inc_* not finite or <= 0,
 * max_fac_* outside 0..4096, and the hints fq_replan_pairs_assign_dev refuses. */
int fq_replan_pairs_window_dev(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                               fq_pair_result* results_all, void* stream);

/* ---- chained replan with the exact MIQP optimum of every corridor ------------------------------------------------------
 *
 * SolverGurobi solves an MIQP over every binary b[t][p] (solverGurobi.cpp:217-246): at the first factor where ANY of the
 * P^N assignments of segments to polytopes is feasible, the cheapest one.  The entry points below return that answer for
 * every corridor of a batch, by branch-and-bound over all assignments on the device (fq_bnb.cuh), with no host round trip.
 * `assign` is required and used as in fq_replan_pairs_assign; window == NULL takes the shared ascending factor lists of
 * fq_pair_args (as _assign), a window the per-corridor windows of fq_replan_pairs_window (factor_*, trials_*, next_*
 * included).  Feature "replan_pairs_exact".
 *
 * For corridor j and each sweep, with F_j its factors, L_j its list (all_limit still chooses it: the list is the pre-sweep
 * whose winner seeds the tree) and f* the first factor at which L_j has a feasible candidate:
 *   - the winner is at the first factor f <= f* at which ANY assignment is feasible (every factor of F_j without f*);
 *   - at that factor it is the minimum-cost assignment.  The list winner is kept unless some assignment is cheaper by more
 *     than a relative 1e-9, and then the records are byte for byte those of _assign / _window.  Otherwise the winner is
 *     the lexicographically smallest assignment (base-P_j digits, segment 0 most significant) within a relative 1e-9 of the
 *     minimum, so that exact ties of overlapping polytopes never depend on the order in which warps finish (whether a
 *     slice near its capacity overflows can: DESIGN.md 3.2); its cost is the tree's evaluation of that assignment;
 *   - corridors whose list already holds every assignment (P_j <= 1 or P_j^N <= all_limit) run no tree: exact 1, nodes 0;
 *   - *_sigma_index is the winner's index in L_j, or -1 when it is not in L_j (then *_dt_index >= 0 tells it from "no
 *     winner"); assign->sigma_* always holds the winning assignment;
 *   - feasible_* / cost_* stay the list pre-sweep's per-candidate outputs;
 *   - R, the safe sweep, the window update and the records follow the exact whole winner;
 *   - exact_*[j] = 0: the corridor's tree was cut (its node or leaf slice filled up, or a node gave up at the iteration
 *     cap), its faces exceed what the level kernel stages (2047, or less where shared memory runs out; DESIGN.md 3.4), or
 *     the sweep's N has no tree kernel (N < 4), or the winners' coefficient solve rejected the tree's winner (a cold
 *     solve can hit the iteration cap where the warm-started tree did not).  The corridor then gets its list winner,
 *     byte-identical to _assign; the other corridors of the batch are unaffected.
 * Each corridor owns max(64, 65536 / n_prob) nodes of each of two level pools and 4096 leaves in the context's device
 * memory, which the context keeps until it is destroyed (at N = 10 and up to 1024 corridors about 1.3 GB with the
 * arena's headroom; DESIGN.md 3.2). */
typedef struct fq_pair_exact
{
  int *exact_whole, *exact_safe;        /* out n_prob, or NULL: 1 = the minimum over all P_j^N assignments, 0 = list winner kept (above) */
  long long *nodes_whole, *nodes_safe;  /* out n_prob, or NULL: tree nodes the levels considered for the corridor   */
} fq_pair_exact;

/* HOST pointers everywhere; blocks until every output is in the caller's arrays.  FQ_E_ARG: exact or assign NULL, the
 * refusals of _assign / _window, and multi-GPU contexts (gathering exact_* / nodes_* would need a second exchange). */
int fq_replan_pairs_exact(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                          const fq_pair_exact* exact);
/* The same, returning once everything is enqueued; outputs are valid after fq_wait(ctx).  Arrays must stay alive. */
int fq_replan_pairs_exact_async(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                                const fq_pair_exact* exact);
/* DEVICE pointers everywhere (the structs live on the host), with the hint and capacity rules of _assign_dev /
 * _window_dev: a broken hint empties that sweep (exact 1, nodes 0, every winner "none"), nothing is written past the
 * caller's arrays.  Never synchronises: the N level launches of a sweep read their parent counts on the device.  On a
 * rank context the records are all-gathered into results_all as fq_replan_pairs_dev does. */
int fq_replan_pairs_exact_dev(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                              const fq_pair_exact* exact, fq_pair_result* results_all, void* stream);

/* ---- chained replan that decomposes its own corridors on the device ----------------------------------------------------
 *
 * Faster::replan cuts the safe corridor around R (faster.cpp:474-475 R, :485 JPS_safe[0] = R.pos, :495-496 deleteVertexes
 * and M, :499 cvxEllipsoidDecomp over unknown and occupied space, :503-504 M = G when the last safe polytope contains G;
 * the whole corridor likewise at :393-403).  R only exists on the device, so the entry points below take the paths and
 * obstacle clouds instead of polytopes and run fq_ellipsoid_decomp's decomposition on the device: the whole corridors
 * before the whole sweep, the safe corridors around the device's R between the sweeps.  Feature "replan_pairs_decomp".
 *
 * `assign` is required (per-corridor lists, as _assign); window == NULL takes the shared factor lists of fq_pair_args (as
 * _assign), a window the per-corridor windows (as _window); exact == NULL returns the list winners, an fq_pair_exact the
 * exact optimum (as _exact).  In fq_pair_args, poly_ofs_* give the polytope counts P_j (one per path segment),
 * face_ofs_*, Ab_* and xf_* must be NULL (FQ_E_ARG otherwise: the chain makes them), and max_faces_* / max_poly_faces_* are
 * CAPS on a corridor's and a polytope's faces (they also size the solve kernels, as always).
 *
 * Per corridor and sweep the decomposition gives, bit for bit up to the atan2/hypot/sin/cos of the device (a few ulp;
 * DESIGN.md 3.2), the rows fq_ellipsoid_decomp gives for the same path and cloud, and the final state E (whole) / M (safe):
 * the goal when goal != NULL and the last polytope's rows all satisfy a.x - b <= 0 (LinearConstraint::inside), the path's
 * last vertex otherwise; velocity and acceleration 0.  A corridor whose decomposition fails (status != 0) gets no winner for
 * that sweep, and after a failed whole sweep no safe sweep; every other corridor of the batch is unaffected. */
#define FQ_DECOMP_OK 0
#define FQ_DECOMP_POLY_FACES 1      /* a polytope has more than max_poly_faces_* faces                               */
#define FQ_DECOMP_CORRIDOR_FACES 2  /* the corridor has more than max_faces_* faces                                  */
#define FQ_DECOMP_CLOUD 3           /* the corridor's cloud has more than max_obs_* points (_dev)                    */
#define FQ_DECOMP_ZERO_SEGMENT 4    /* two consecutive path vertices coincide (for safe: also R.pos and vertex 1)    */
#define FQ_DECOMP_NOT_RUN 5         /* safe: no whole winner, so no R; either: more than max_poly_* polytopes (_dev)  */

typedef struct fq_pair_decomp
{
  /* inputs, per corridor: corridor j's path has P_j + 1 vertices (x, y, z) at rows poly_ofs_*[j] + j .. poly_ofs_*[j+1] + j,
   * already trimmed by deleteVertexes; vertex 0 of the safe path is replaced by R.pos.  Clouds are CSR: corridor j's
   * points are rows obs_ofs_*[j] .. obs_ofs_*[j+1] of obs_* (occupied space for whole, unknown and occupied for safe; the
   * two may be the same arrays). */
  const double *path_whole, *path_safe;
  const int *obs_ofs_whole, *obs_ofs_safe;
  const double *obs_whole, *obs_safe;
  /* inputs, shared */
  const double* goal;                   /* n_prob x 3, or NULL (then E / M are the last vertices)                    */
  double bbox[3];                       /* local bounding box half sizes (jps_manager.cpp:100: 2, 2, 1)                 */
  double inflate;                       /* obstacle inflation, the drone radius                                          */
  double z_ground;                      /* ground face -z <= -z_ground                                                  */
  int max_obs_whole, max_obs_safe;      /* _dev only: the largest cloud of one corridor (checked: FQ_DECOMP_CLOUD)     */
  /* outputs, each optional (NULL): the corridors the sweeps used (the reference's poly_*_out), as an ordinary gap-free
   * CSR -- face_ofs_* (poly_ofs_*[n_prob] + 1, absolute) and Ab_* (16-byte aligned, room for n_prob x max_faces_* rows);
   * a failed corridor's polytopes are empty -- the E / M positions (n_prob x 3, NaN for a failed corridor), and the status
   * of every corridor's decomposition (n_prob, FQ_DECOMP_*). */
  int *face_ofs_whole, *face_ofs_safe;
  double *Ab_whole, *Ab_safe;
  double *E, *M;
  int *status_whole, *status_safe;
} fq_pair_decomp;

/* HOST pointers everywhere; blocks until every output is in the caller's arrays.  FQ_E_ARG: decomp or assign NULL, the
 * fq_pair_args rules above, the refusals of _assign / _window / _exact, a path, cloud or goal value that is not finite,
 * bbox <= 0, inflate < 0, and multi-GPU contexts. */
int fq_replan_pairs_decomp(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                           const fq_pair_exact* exact, const fq_pair_decomp* decomp);
/* The same, returning once everything is enqueued; outputs are valid after fq_wait(ctx).  Arrays must stay alive. */
int fq_replan_pairs_decomp_async(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                                 const fq_pair_exact* exact, const fq_pair_decomp* decomp);
/* DEVICE pointers everywhere (the structs live on the host), with the hint rules of _assign_dev / _window_dev / _exact_dev
 * and decomp->max_obs_*.  Never synchronises (a CUDA graph can capture it).  On a rank context the records are all-gathered
 * into results_all as fq_replan_pairs_dev does. */
int fq_replan_pairs_decomp_dev(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                               const fq_pair_exact* exact, const fq_pair_decomp* decomp, fq_pair_result* results_all, void* stream);

/* ---- chained replan that chooses H and R from each corridor's unknown space ------------------------------------------
 *
 * Faster::replan places R on the whole trajectory from the map (faster.cpp:452-538): findIndexH (:218-251) and findIndexR
 * (:173-216).  The entry points below do that on the device, between the whole sweep and the safe corridor's decomposition,
 * instead of the r_fraction rule (r_fraction is still validated but not used).  They are fq_replan_pairs_decomp* otherwise:
 * `assign`, `decomp` and `hr` are required, `window` and `exact` optional.  Feature "replan_pairs_hr".
 *
 * Per corridor j whose whole winner has n = resetX samples X_temp_ (fillX's accumulated clock, the last sample at rest):
 *   H   for i = 0, 10, 20, ... < n: q = sample i's position rounded to float (pcl::PointXYZ), d^2 = the minimum over the
 *       corridor's unknown points p (rounded to float) of ((0 + dx^2) + dy^2) + dz^2 in float (FLANN's L2 order).  At the
 *       first i with sqrtf(d^2) < drone_radius (compared in double): need_safe = 1, indexH = (int)(delta_H i).  Without
 *       such a sample, or with an empty cloud: need_safe = 0, indexH = n - 1.  (FLANN's kd-tree may differ from this exact
 *       float minimum only through the rounding of its pruning bounds; DESIGN.md 3.2.)
 *   R   (need_safe = 1) k_safe = the first i in 0 .. indexH whose braking distance (sign(v (H - p)) v^2) / ((2 delta_a) a_max)
 *       exceeds |H - p| in x or in y (double; sign(0) = 0; H = X_temp_[indexH], a_max = lim[3 j + 1]), else indexH.  R is
 *       X_temp_[k_safe], bit-equal to fq_fill_x's sample.
 *   need_safe = 0 (whole won): k_safe = n - 1, R NaN, no safe decomposition (status FQ_DECOMP_NOT_RUN), no safe sweep and
 *       no safe winner; trials_safe 0.  The replan still succeeds: the next whole window follows the whole winner, the next
 *       safe window is [max(last_factor_safe - gamma_safe, 1), last_factor_safe + gammap_safe] (faster.cpp:465-469,
 *       :586-588).
 *   no whole winner: index_H = -1, k_safe = -1, R NaN, as in fq_replan_pairs_decomp.
 * last_factor_safe[j] becomes the safe winner's factor when the safe sweep wins and is unchanged otherwise; every window is
 * read before anything is written, so the outputs may alias the inputs. */
typedef struct fq_pair_hr
{
  const int* unk_ofs;        /* n_prob + 1: corridor j's unknown cloud is rows unk_ofs[j] .. unk_ofs[j+1]-1 of unk       */
  const double* unk;         /* rows x 3; rounded to float on the device, as pcl::PointXYZ holds them. May point into obs_safe */
  double drone_radius;       /* par_.drone_radius (findIndexH)                                                         */
  double delta_a, delta_H;   /* par_.delta_a (findIndexR), par_.delta_H (findIndexH)                                   */
  double* last_factor_safe;  /* in/out n_prob: the safe solver's factor_that_worked_ (0 at start-up).  Required with a window */
  int* index_H;              /* out n_prob, or NULL: indexH (-1: no whole winner)                                      */
  uint8_t* need_safe;        /* out n_prob, or NULL: needToComputeSafePath                                             */
} fq_pair_hr;

/* HOST pointers everywhere; blocks until every output is in the caller's arrays.  FQ_E_ARG: the refusals of
 * fq_replan_pairs_decomp, hr NULL, drone_radius not finite or < 0, delta_a not finite or <= 0, delta_H outside [0, 1],
 * unk_ofs or unk NULL, unk_ofs not starting at 0 or decreasing, a non-finite unknown value, a window without
 * last_factor_safe, and multi-GPU contexts. */
int fq_replan_pairs_hr(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                       const fq_pair_exact* exact, const fq_pair_decomp* decomp, const fq_pair_hr* hr);
/* The same, returning once everything is enqueued; outputs are valid after fq_wait(ctx).  Arrays must stay alive. */
int fq_replan_pairs_hr_async(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                             const fq_pair_exact* exact, const fq_pair_decomp* decomp, const fq_pair_hr* hr);
/* DEVICE pointers everywhere (the structs live on the host), as fq_replan_pairs_decomp_dev; never synchronises.  Every
 * thread of the H/R kernel walks the sample clock itself, so n has no cap.  On a rank context the records are all-gathered
 * into results_all as fq_replan_pairs_dev does. */
int fq_replan_pairs_hr_dev(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                           const fq_pair_exact* exact, const fq_pair_decomp* decomp, const fq_pair_hr* hr, fq_pair_result* results_all,
                           void* stream);

/* ---- an indexed map on the device, shared by every corridor and every later replan ---------------------------------
 *
 * Faster::updateMap (faster.cpp:99-137) keeps, per mapper message, the occupied cloud O (vec_o_), the unknown cloud U and
 * U ++ O (vec_uo_: U with O appended, in that order), which every replan then queries.  An fq_map holds the same three
 * clouds on one GPU, uploaded and indexed once: each of U and O is bucketed into a uniform grid of cells of edge
 * FQ_MAP_CELL_EDGE (doubled until the grid has at most min(max(65536, 4 (|U| + |O|)), 2^26) cells), its points sorted by (cell, index)
 * with a stable device radix sort.  The cell edge changes no answer, only how many points a query reads.  Feature
 * "replan_pairs_map".
 *
 * An empty U is allowed: H/R then finds no unknown point and the safe cloud is O.  (The reference keeps its previous
 * vec_uo_ when the unknown cloud is empty, faster.cpp:121-125; that is not modelled.)  A map must not be updated or
 * destroyed while a submission that reads it is in flight.
 *
 * A submission reads a map through a descriptor that stays at one device address for the map's life and that every
 * update rewrites in full on the update's stream: its grid, its counts and the addresses of its arrays.  So a
 * fq_replan_pairs_map_dev call captured once in a CUDA graph and replayed after later updates -- with or without a grown
 * capacity -- reads each map's last update, as a fresh call would.
 *
 * An update that fails (FQ_E_CUDA: an allocation or a launch) leaves the map empty, with a descriptor that reads no
 * points, and fq_replan_pairs_map* refuse the map until an update succeeds. */
#define FQ_MAP_CELL_EDGE 0.5
typedef struct fq_map fq_map;
/* Errors of fq_map_* are read with fq_last_error(NULL). */
int fq_map_create(fq_map** out, int device);
void fq_map_destroy(fq_map* map);
/* HOST pointers (n x 3 doubles each; NULL with a count of 0); blocks until the map holds the new clouds.  FQ_E_ARG for a
 * negative count, more than 2^30 points in all, a NULL cloud with a positive count or a non-finite coordinate. */
int fq_map_update(fq_map* map, const double* occ, int n_occ, const double* unk, int n_unk);
/* DEVICE pointers, stream-ordered on `stream` (NULL: the legacy default stream): copies the clouds and builds the index
 * without synchronising, as long as the map's capacity holds n_occ + n_unk points.  A larger update first grows the
 * capacity (cudaFree / cudaMalloc, which wait for the whole device); the capacity never shrinks.  The counts are checked
 * as by fq_map_update; the coordinates cannot be checked without synchronising: a non-finite point is left out of the
 * index, so no query ever sees it.  The input arrays may be reused once the stream has passed this call. */
int fq_map_update_dev(fq_map* map, const double* d_occ, int n_occ, const double* d_unk, int n_unk, void* stream);
/* the counts of the last update (either may be NULL) */
int fq_map_size(const fq_map* map, int* n_occ, int* n_unk);

/* ---- chained replan against indexed maps ------------------------------------------------------------------------
 *
 * fq_replan_pairs_hr* (or, with hr == NULL, fq_replan_pairs_decomp*, the r_fraction rule) with each corridor's clouds taken
 * from a map: for corridor j, whose map holds O and U, the outputs are byte for byte those of fq_replan_pairs_hr called with
 * obs_whole_j = O, obs_safe_j = U ++ O and unk_j = U -- records, per-candidate flags and costs, coefficients, corridors,
 * E / M, statuses, index_H / need_safe, windows and exact / nodes -- as long as no segment has more than max_local points
 * in its local box (below).  This holds at any coordinate magnitude: the cells H/R reads are widened by a bound on the
 * float rounding of points, samples and distances.  decomp->obs_* and hr->unk* must be NULL, and decomp->max_obs_* are
 * not used.  The decomposition reads only the cells the segment's local box overlaps, H/R only the cells near each
 * sample.
 *
 * max_local caps the points of one segment's cloud that pass the local-box test; a segment above it gets FQ_DECOMP_CLOUD,
 * and the rest of the batch is unaffected.  It sizes the decomposition's scratch, n_prob x max_poly x (max_local - 1024) x
 * 37 bytes, whatever the maps' sizes. */
typedef struct fq_pair_map
{
  const fq_map* const* maps;  /* n_maps maps, all on the context's device                                          */
  int n_maps;
  const int* map_index;       /* n_prob: corridor j uses maps[map_index[j]], or NULL: every corridor uses maps[0]  */
  int max_local;              /* >= 0                                                                              */
} fq_pair_map;

/* HOST pointers everywhere (map_index included); blocks until every output is in the caller's arrays.  FQ_E_ARG: the
 * refusals of fq_replan_pairs_hr (fq_replan_pairs_decomp when hr == NULL) other than those of the clouds, obs_* / unk*
 * not NULL, map NULL, no maps or a NULL map, a map on another device, a map whose last update failed, a map_index
 * entry outside 0 .. n_maps-1, max_local < 0 or above 2^30, and multi-GPU contexts. */
int fq_replan_pairs_map(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                        const fq_pair_exact* exact, const fq_pair_decomp* decomp, const fq_pair_hr* hr, const fq_pair_map* map);
/* The same, returning once everything is enqueued; outputs are valid after fq_wait(ctx).  Arrays must stay alive. */
int fq_replan_pairs_map_async(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                              const fq_pair_exact* exact, const fq_pair_decomp* decomp, const fq_pair_hr* hr, const fq_pair_map* map);
/* DEVICE pointers everywhere (the structs and the maps array live on the host; map_index is a device array), as
 * fq_replan_pairs_hr_dev; never synchronises.  map_index is not read on the host: a corridor whose entry is out of range
 * gets FQ_DECOMP_CLOUD for both sweeps.  On a rank context the records are all-gathered into results_all as
 * fq_replan_pairs_dev does. */
int fq_replan_pairs_map_dev(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                            const fq_pair_exact* exact, const fq_pair_decomp* decomp, const fq_pair_hr* hr, const fq_pair_map* map,
                            fq_pair_result* results_all, void* stream);

/* ---- whole and safe paths from JPS_in against an indexed map ----------------------------------------------------------
 *
 * Faster::replan decomposes two paths (faster.cpp:373-393, :449-496): JPS_whole = deleteVertexes(JPS_in, max_poly_whole)
 * and JPS_safe, which is JPS_in cropped where it first nears unknown space -- getFirstCollisionJPS(JPS_in, UNKNOWN_MAP,
 * RETURN_INTERSECTION) (:767-921) -- then trimmed by deleteVertexes(., max_poly_safe).  (The reference then replaces vertex
 * 0 of JPS_safe by R, :485; the decomposing chains do that on the device.)  fq_map_paths computes both from each corridor's
 * JPS_in and the U of its map, and writes them in the layout fq_pair_args.poly_ofs_* / fq_pair_decomp.path_* take, so its
 * outputs feed fq_replan_pairs_map* as they are.  Feature "map_paths".
 *
 * The crop, per corridor, in the reference's own mix of float and double (faster_b200/csrc/fq_paths.h):
 *   the head starts at vertex 0; each step takes q = the head rounded to float (eigenPoint2pclPoint), d^2 = the exact float
 *   minimum of FLANN's L2 ((0 + dx^2) + dy^2) + dz^2 over U (as fq_pair_hr's findIndexH; DESIGN.md 3.2) and r = sqrtf(d^2);
 *   r < drone_radius: a collision -- at the first step the path becomes [v0, v0 + (0.01, 0, 0)] (:833-841), later the vertices
 *     passed so far plus the head, shortened by drone_radius (reduceJPSbyDistance, utils.cpp:690-710); crossed = 1;
 *   otherwise the head moves to where the path leaves the sphere (head, r) (getFirstIntersectionWithSphere and
 *     getIntersectionWithSphere, utils.cpp:713-866, with their float temporaries and the fallback of a discriminant <= 0);
 *   no vertex outside the sphere, or an empty U: the path is JPS_in unchanged, crossed = 0.
 * A step reads only the map cells within max(drone_radius, the farthest vertex left) of the head, widened for the float
 * rounding as fq_replan_pairs_map's H/R does: a nearest point beyond that range changes nothing.  A crop that takes
 * FQ_PATHS_MAX_STEPS steps stops with FQ_PATHS_STALL.
 *
 * Outputs: corridor j's whole path has P_w + 1 vertices (P_w = min(n_in - 1, max_poly_whole)) at rows poly_ofs_whole[j] + j
 * .. poly_ofs_whole[j+1] + j of path_whole, the safe path likewise with P_s = min(|cropped| - 1, max_poly_safe).  So
 * neither array ever needs more than n_prob x (max_poly_* + 1) rows.  A corridor whose status is not FQ_PATHS_OK gets one
 * vertex of NaN (P = 0) in both, which the chained replan gives no winner.
 *
 * A map must not be updated or destroyed while a call that reads it is in flight.  The call reads each map through the
 * descriptor of fq_replan_pairs_map*, so a CUDA graph of fq_map_paths_dev replayed after later updates reads the last one. */
#define FQ_PATHS_OK 0
#define FQ_PATHS_SHORT 1      /* JPS_in has fewer than 2 vertices (_dev)                                                */
#define FQ_PATHS_STALL 2      /* the crop took FQ_PATHS_MAX_STEPS steps                                                 */
#define FQ_PATHS_MAP 3        /* map_index out of range (_dev)                                                          */
#define FQ_PATHS_INPUT 4      /* JPS_in has more than max_in vertices, a negative offset or a non-finite vertex (_dev)  */
#define FQ_PATHS_MAX_STEPS 4096
#define FQ_PATHS_MAX_IN 4096  /* vertices of one JPS_in                                                                 */
typedef struct fq_map_paths_args
{
  int n_prob;
  const int* in_ofs;                     /* n_prob + 1: JPS_in of corridor j (faster.cpp:373-384) is rows in_ofs[j] ..     */
  const double* in;                      /*   in_ofs[j+1]-1 of in (x, y, z), >= 2 vertices; fq_jps_in makes it             */
  const fq_map* const* maps;             /* n_maps maps, all on one device: corridor j reads the U of maps[map_index[j]]   */
  int n_maps;
  const int* map_index;                  /* n_prob, or NULL: every corridor reads maps[0]                                  */
  double drone_radius;                   /* par_.drone_radius, > 0                                                          */
  int max_poly_whole, max_poly_safe;     /* par_.max_poly_whole / _safe, 1 .. FQ_MAX_POLY                                   */
  int max_in;                            /* _dev only: the longest JPS_in, 2 .. FQ_PATHS_MAX_IN (longer: FQ_PATHS_INPUT)   */
  int *poly_ofs_whole, *poly_ofs_safe;   /* out n_prob + 1: fq_pair_args.poly_ofs_*                                         */
  double *path_whole, *path_safe;        /* out, room for n_prob x (max_poly_* + 1) rows: fq_pair_decomp.path_*            */
  int* status;                           /* out n_prob, or NULL: FQ_PATHS_*                                                 */
  uint8_t* crossed;                      /* out n_prob, or NULL: getFirstCollisionJPS's thereIsIntersection                 */
} fq_map_paths_args;

/* HOST pointers everywhere (maps and map_index included); blocks until every output is in the caller's arrays.  Runs on
 * the maps' device.  FQ_E_ARG (text in fq_last_error(NULL)): p NULL, n_prob <= 0, a NULL input or output array, in_ofs not
 * starting at 0 or decreasing, a corridor with fewer than 2 or more than FQ_PATHS_MAX_IN vertices, a non-finite vertex,
 * drone_radius not finite or <= 0 (the reference can then loop forever on a point of the path), max_poly_* outside
 * 1 .. FQ_MAX_POLY, no maps, a NULL map, maps on different devices, a map whose last update failed, and a map_index entry
 * outside 0 .. n_maps-1.  max_in is not read. */
int fq_map_paths(const fq_map_paths_args* p);
/* DEVICE pointers (the struct and the maps array live on the host; map_index is a device array); stream-ordered on
 * `stream`, which must belong to the maps' device (NULL: the legacy default stream), and never synchronises, so a CUDA
 * graph can capture it.  Its scratch (n_prob x 40 bytes and the map table) is stream-ordered memory (cudaMallocAsync).
 * Refused as fq_map_paths, except that what only the arrays tell -- offsets, vertex counts and values, map_index -- is
 * reported per corridor in status instead: FQ_PATHS_SHORT, FQ_PATHS_INPUT, FQ_PATHS_MAP. */
int fq_map_paths_dev(const fq_map_paths_args* p, void* stream);
/* The same crop on the host over per-corridor clouds instead of maps: corridor j's U is rows unk_ofs[j] .. unk_ofs[j+1]-1
 * of unk (n_prob + 1 offsets from 0, non-decreasing; unk may be NULL when every cloud is empty), and the nearest point is
 * found by brute force.  For the same JPS_in and clouds it writes what fq_map_paths writes, byte for byte.  maps,
 * n_maps, map_index and max_in are not read; the other refusals are fq_map_paths's, plus a non-finite unknown point.  Pure
 * host code. */
int fq_paths_cloud(const fq_map_paths_args* p, const int* unk_ofs, const double* unk);
/* JPS_in from a path of fq_jps3d_plan_world (faster.cpp:361-384): vertex 0 := start and the last vertex := goal, both with
 * z raised to 0 if below, as solveJPS3D forces them (jps_manager.cpp:143-144, :172-186: a one-vertex path becomes [start,
 * goal]); the path up to where it first leaves the sphere of radius ra around vertex 0 (getFirstIntersectionWithSphere,
 * :373-382; the caller passes ra = min(dist_to_goal - 0.001, Ra)); then createMoreVertexes(dist_max) (:80-97).  Writes
 * the first min(count, cap) vertices to out and returns the count (out may be NULL with cap 0).  FQ_E_ARG: jps, start or
 * goal NULL, n < 1, cap < 0, out NULL with cap > 0, a non-finite vertex, start, goal or ra, dist_max not finite or <= 0,
 * and a count above 2^30.  Pure host code. */
int fq_jps_in(const double* jps, int n, const double* start, const double* goal, double ra, double dist_max, double* out,
              int cap);

/* ---- every planner's JPS search and JPS_in on the device ----------------------------------------------------------------
 *
 * jps_manager_.solveJPS3D(A, G) followed by fq_jps_in (faster.cpp:361-384) for a batch of planners, with fq_jps3d_plan_world's
 * search and post-processing run on the GPU (one warp per planner), so that a replan cycle -- fq_queue_select_dev, this,
 * fq_map_paths_dev, fq_replan_pairs_queue_dev, fq_queue_pop_dev -- needs no host step and can be captured as one CUDA
 * graph.  For planner j: A = x0[j][0..2] and G = goal[j], both with z raised to 0 for the search (jps_manager.cpp:143-144);
 * ra = min(|G - P| - 0.001, Ra) with P = pos[j] (the drone's state, faster.cpp:327), or A when pos is NULL, the norm in
 * Eigen's order sqrt((dx^2 + dy^2) + dz^2).  The search runs on grid grid_index[j] (fq_jps3d_plan's map) from cell
 * to_int(A) to cell to_int(G); the grid is the caller's (no readMap voxelisation, no setFreeVoxelAndSurroundings).
 * JPS_in is written in fq_map_paths_args' layout (in_ofs from 0, compact rows), so fq_map_paths_dev can read it as it is.
 * Every output equals, byte for byte, fq_jps3d_plan_world + fq_jps_in on the host, with these statuses:
 *   FQ_JPS_OK       path found: its JPS_in;                                                           k_end unchanged
 *   FQ_JPS_NO_PATH  start or goal cell outside the grid or not free, or the search exhausted: fq_jps_in([A], A, G, ra,
 *                   dist_max), Faster::replan's early return (no append, window kept);                k_end[j] := -1
 *   FQ_JPS_NODES    the search needed more than max_nodes nodes: one NaN vertex;                      k_end[j] := -1
 *   FQ_JPS_LONG     JPS_in longer than max_in vertices: one NaN vertex;                               k_end[j] := -1
 *   FQ_JPS_INPUT    (_dev only) grid_index out of range, a grid with a dimension <= 0, more than 2^31 cells, a res not
 *                   finite or <= 0 or a non-finite origin, or a non-finite A, G or pos: one NaN vertex; k_end[j] := -1
 * A single NaN vertex makes fq_map_paths_dev report FQ_PATHS_SHORT, so the chain gives that corridor no winner.
 * Device scratch per planner: at most 116 max_nodes + 24 max_in + 112 bytes (node pool, heap, a hash of 2 max_nodes cells, two
 * path buffers, the JPS_in slot), stream-ordered.  Feature "jps_batch". */
#define FQ_JPS_OK 0
#define FQ_JPS_NO_PATH 1
#define FQ_JPS_NODES 2
#define FQ_JPS_LONG 3
#define FQ_JPS_INPUT 4
typedef struct fq_jps_grids {       /* caller-owned, DEVICE arrays for _dev, HOST for fq_jps_batch                           */
  const int8_t* cells;              /* every grid's cells, x fastest; 0 free, > 0 occupied, < 0 unknown (fq_jps3d_plan's map) */
  const long long* cell_ofs;        /* n_grids: first cell of grid g                                                        */
  const int* dims;                  /* n_grids x 3: xd, yd, zd                                                              */
  const double* origin;             /* n_grids x 3                                                                          */
  const double* res;                /* n_grids                                                                              */
  int n_grids;
} fq_jps_grids;
typedef struct fq_jps_batch_args {
  int n_prob;
  fq_jps_grids grids;
  const int* grid_index;            /* n_prob, or NULL: every planner plans on grid 0                                       */
  const double* x0;                 /* n_prob x 9, as fq_queue_select writes it: A = x0[j][0..2]                            */
  const double* goal;               /* n_prob x 3: G                                                                        */
  const double* pos;                /* n_prob x 3 or NULL (= A): the state dist_to_goal is measured from                    */
  double Ra, dist_max;              /* par_.Ra, par_.dist_max_vertexes                                                      */
  int use_jps;                      /* != 0 JPS (the reference's call), 0 plain A*                                          */
  int max_nodes, max_in;            /* per-planner caps: 1 .. 2^26 nodes; max_in 2 .. FQ_PATHS_MAX_IN                       */
  int* in_ofs;                      /* out n_prob + 1: fq_map_paths_args.in_ofs                                             */
  double* in;                       /* out: fq_map_paths_args.in, room for n_prob x max_in rows                             */
  int* status;                      /* out n_prob: FQ_JPS_*                                                                 */
  int* k_end;                       /* in/out n_prob or NULL: set to -1 where status != FQ_JPS_OK                           */
} fq_jps_batch_args;
/* HOST pointers; runs on the current device and blocks.  FQ_E_ARG (text in fq_last_error(NULL)): a NULL, n_prob outside
 * 1..2^24, a NULL required array, n_grids < 1, a dimension <= 0, more than 2^31 cells in a grid, a negative cell_ofs, res
 * not finite or <= 0, a non-finite origin, Ra not finite, dist_max not finite or <= 0, max_nodes outside 1..2^26, max_in
 * outside 2..FQ_PATHS_MAX_IN; and, since it can read them, grid_index out of range and a non-finite A, G or pos. */
int fq_jps_batch(const fq_jps_batch_args* a);
/* DEVICE pointers; stream-ordered, never synchronises (a CUDA graph can capture it).  The refusals of fq_jps_batch that
 * read no array; the grids and the per-planner inputs are checked per planner instead (FQ_JPS_INPUT). */
int fq_jps_batch_dev(const fq_jps_batch_args* a, void* stream);

/* ---- chained replan that returns each corridor's committed plan --------------------------------------------------------
 *
 * What a replan commits is not its coefficients but the states appendToPlan pushes onto the plan (faster.cpp:548,
 * :606-648): the whole winner's fillX samples X_temp_[0 .. k_safe] followed by every sample of the safe winner.  The entry
 * points below run one of the chains above and also return that piece for every corridor, sampled on the device.  Feature
 * "replan_pairs_plan".
 *
 * The chain is chosen by the structs given, with the rules of its own family: assign == NULL is fq_replan_pairs (window,
 * exact, decomp, hr and map must then be NULL); otherwise map != NULL is _map, hr != NULL _hr, decomp != NULL _decomp,
 * exact != NULL _exact, window != NULL _window, else _assign.  Every output other than the plan is byte for byte that
 * family's, and every refusal of that family is refused alike (FQ_E_ARG, same fq_last_error text).
 *
 * Per corridor j, with n_w = n_samples_whole and n_s = max(2, (int)(N_safe safe_dt / DC)) (resetX's count):
 *   the replan succeeds when it has a whole winner and, unless no safe path is needed (need_safe = 0, only with hr), a
 *   safe winner; otherwise status FQ_PLAN_NONE and no rows (faster.cpp:420-424, :529-533);
 *   piece = whole samples 0 .. k_safe, then safe samples 0 .. n_s - 1 (none when no safe path is needed, where k_safe =
 *   n_w - 1): k_safe + 1 + n_s rows of 12 doubles, pos vel accel jerk, the layout of fq_fill_x;
 *   every row is bit-equal to fq_fill_x(N, coeffs_*[j], dt, DC, n, .) called with the FULL count n (n_w or n_s) on the
 *   coefficients the call returns in coeffs_* (for _exact after its fallback).  So whole row k_safe keeps its velocity
 *   unless k_safe = n_w - 1, its first 9 doubles are the record's R bit for bit, and the last safe row is at rest.
 * coeffs_* may be NULL: the chain keeps the winners' coefficients in its own scratch.
 *
 * Capacity: n_s depends on R, so the caller cannot size the plan in advance.  plan_ofs[0 .. n_prob] is the exclusive scan
 * of every succeeding corridor's rows (64 bits), and plan_ofs[n_prob] is the capacity the whole batch needs.  A corridor
 * whose rows would end past cap_states gets FQ_PLAN_CAPACITY and none of its rows are written; those corridors are the
 * succeeding corridors of a suffix of the batch.  Nothing is written past cap_states rows, and the call still returns 0.
 * Refused (FQ_E_ARG) besides the family's refusals: plan NULL, states or plan_ofs NULL, cap_states < 0, and multi-GPU
 * contexts (group or rank): gathering variable-length plans would need a second exchange besides the records'. */
#define FQ_PLAN_OK 0
#define FQ_PLAN_NONE 1      /* the replan appends nothing (above)                                                   */
#define FQ_PLAN_CAPACITY 2  /* the piece does not fit in cap_states rows                                            */
typedef struct fq_pair_plan
{
  long long cap_states;     /* rows of `states`                                                                     */
  double* states;           /* out: cap_states x 12                                                                 */
  long long* plan_ofs;      /* out: n_prob + 1; corridor j is rows plan_ofs[j] .. plan_ofs[j+1]-1                   */
  int* status;              /* out: n_prob (FQ_PLAN_*), or NULL                                                     */
} fq_pair_plan;

/* HOST pointers everywhere; blocks until every output is in the caller's arrays.  Of `states` only the rows of the
 * corridors that fit are copied back (at most min(plan_ofs[n_prob], cap_states)); the rest of the array is untouched. */
int fq_replan_pairs_plan(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                         const fq_pair_exact* exact, const fq_pair_decomp* decomp, const fq_pair_hr* hr, const fq_pair_map* map,
                         const fq_pair_plan* plan);
/* The same, returning once everything is enqueued; outputs are valid after fq_wait(ctx).  Arrays must stay alive.  The
 * plan_ofs total is not known when the copies are enqueued, so all cap_states rows of `states` are copied back; rows past
 * plan_ofs[n_prob] hold whatever the library's staging buffer held. */
int fq_replan_pairs_plan_async(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                               const fq_pair_exact* exact, const fq_pair_decomp* decomp, const fq_pair_hr* hr, const fq_pair_map* map,
                               const fq_pair_plan* plan);
/* DEVICE pointers everywhere (the structs live on the host; plan's arrays are device arrays), with the hint rules of the
 * selected family's _dev entry.  Never synchronises: the offsets and the rows are computed on the device after the
 * records, so a CUDA graph can capture the call. */
int fq_replan_pairs_plan_dev(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                             const fq_pair_exact* exact, const fq_pair_decomp* decomp, const fq_pair_hr* hr, const fq_pair_map* map,
                             const fq_pair_plan* plan, fq_pair_result* results_all, void* stream);

/* ---- each planner's committed plan, kept on the device ----------------------------------------------------------------
 *
 * Faster keeps its committed plan in a deque (plan_, faster.hpp:70) from one replan to the next: replan() takes A from it,
 * appendToPlan replaces its tail with the new piece, and getNextGoal publishes its front on its own timer.  The entries
 * below keep that deque for every planner in caller-owned ring arrays, so a batch planner's loop needs only A back on the
 * host (for JPS).  Feature "replan_pairs_queue".
 *
 * Ring: n_rows rows of cap states (12 doubles each, fq_fill_x's layout: pos vel accel jerk).  Row r holds size[r] states,
 * and its i-th state (0 = front) is states[(r * cap + (head[r] + i) % cap) * 12 ..].  A row is valid when 0 <= head < cap
 * and 0 <= size <= cap.  Corridor (planner) j of a call works on row rows[j], or row j when rows is NULL, so a caller can
 * submit only its active planners.  GOAL_REACHED / YAWING gating, yaw and the G projection stay with the caller.
 *
 * The host entries take HOST pointers and refuse (FQ_E_ARG, text in fq_last_error(NULL)): q or a required array NULL,
 * n < 0, n_rows < 1, cap < 1, delta_t < 1, a row outside 0 .. n_rows-1 or named twice, and an invalid row named.  They are
 * pure host code.  The _dev entries take DEVICE arrays (the struct lives on the host), are stream-ordered on `stream` of
 * the current device (NULL: the legacy default stream) and never synchronise.  They refuse what the struct alone shows;
 * a corridor whose row is out of range, named twice or invalid is skipped: select gives it k_end = -1 and a NaN x0, pop
 * gives it NaN goals, reset leaves the row as it was.  Except: select only reads the rings, so fq_queue_select and
 * fq_queue_select_dev accept a row named by several corridors and give each of them the row's A and k_end (an invalid or
 * out-of-range row is still refused on the host and skipped on the device); reset does not read head and size, so it
 * accepts an invalid row and makes it a ring. */
typedef struct fq_queue
{
  double* states;   /* n_rows x cap x 12                                                                              */
  int* head;        /* n_rows: slot of the front state                                                                */
  int* size;        /* n_rows: states held                                                                            */
  int n_rows;
  int cap;          /* states per row, >= 1                                                                           */
  int delta_t;      /* deltaT_ (faster.hpp:131: 10), >= 1                                                             */
} fq_queue;

/* updateState's first push (faster.cpp:253-266): row rows[j] := [the state with pos = pos[j] (n x 3), the rest 0]. */
int fq_queue_reset(const fq_queue* q, int n, const int* rows, const double* pos);
int fq_queue_reset_dev(const fq_queue* q, int n, const int* rows, const double* pos, void* stream);
/* Choosing A (faster.cpp:350-352): k_end[j] = max(size - delta_t, 0) and x0[j] (n x 9) = pos, vel, accel of the row's
 * state size - 1 - k_end[j].  An empty row gives k_end = -1 and a NaN x0, so that corridor's sweeps have no winner.  x0
 * is fq_pair_args.x0 of the next replan, and the one array a caller reads back (for host JPS from A.pos). */
int fq_queue_select(const fq_queue* q, int n, const int* rows, double* x0, int* k_end);
int fq_queue_select_dev(const fq_queue* q, int n, const int* rows, double* x0, int* k_end, void* stream);
/* getNextGoal (faster.cpp:699-723) called ticks[j] times (clamped to 0 .. max_ticks): goal t of corridor j, goals[(j *
 * max_ticks + t) * 12 ..], is the row's front, which is then popped while the row holds more than one state.  Slots past
 * ticks[j] are not written.  Yaw is not computed. */
int fq_queue_pop(const fq_queue* q, int n, const int* rows, const int* ticks, int max_ticks, double* goals);
int fq_queue_pop_dev(const fq_queue* q, int n, const int* rows, const int* ticks, int max_ticks, double* goals, void* stream);

/* The chained replan that appends each corridor's piece to its row, as appendToPlan does (faster.cpp:548-551, :606-648).
 * The chain is chosen by the structs given, with the rules of fq_replan_pairs_plan, and every output it returns is byte
 * for byte what fq_replan_pairs_plan returns for the same arguments (args->x0 is fq_queue_select's x0).  Then, per
 * corridor j on row r = rows[j], with the piece of fq_replan_pairs_plan (k_safe + 1 + n_s states, or none):
 *   status FQ_QUEUE_NONE: the replan appends nothing (FQ_PLAN_NONE), or k_end[j] < 0 (no select since the last append);
 *   FQ_QUEUE_PUBLISHED: size[r] - 1 - k_end[j] < 0, with size[r] read when the chain appends, so pops enqueued between the
 *     select and this call count (delta_t or more of them): "Already published the point A";
 *   FQ_QUEUE_CAPACITY: size[r] - k_end[j] - 1 + the piece's states > cap, decided for this row alone;
 *   FQ_QUEUE_ROWS (_dev only): the row is out of range, named by another corridor, or invalid;
 *   FQ_QUEUE_OK: the last k_end[j] + 1 states are erased and the piece pushed; size[r] changes, head[r] does not.
 * Only an OK corridor's row changes.  k_end[j] becomes -1 for every corridor (consumed), so a second call without a new
 * select appends nothing.  goal_seen[j] (if given, with G_term) = 1 when OK and |G_term[j] - the row's last pos| <
 * goal_radius (faster.cpp:563-572), else 0.
 * With a window, factor_*, trials_* and last_factor_safe are written as fq_replan_pairs_plan writes them (they are set
 * inside genNewTraj, before the append), but next_* only for OK corridors: replan() returns before its window update when
 * the append fails (faster.cpp:548-551), so every other corridor keeps its input window, also when next_* aliases it.
 * Refused (FQ_E_ARG) besides the family's refusals: q NULL, a NULL ring array, k_end or status NULL, n_rows < 1, cap < 1,
 * delta_t < 1, multi-GPU contexts, and on the host entries the row checks above. */
#define FQ_QUEUE_OK 0
#define FQ_QUEUE_NONE 1        /* nothing appended: no plan piece, or no select                                       */
#define FQ_QUEUE_PUBLISHED 2   /* the state A was already published                                                    */
#define FQ_QUEUE_CAPACITY 3    /* the row would exceed cap                                                             */
#define FQ_QUEUE_ROWS 4        /* the row is out of range, shared with another corridor or invalid (_dev)              */
typedef struct fq_pair_queue
{
  fq_queue ring;            /* in/out                                                                               */
  const int* rows;          /* n_prob, or NULL: corridor j is row j                                                 */
  int* k_end;               /* in/out n_prob: fq_queue_select's                                                     */
  const double* G_term;     /* n_prob x 3, or NULL: no goal_seen                                                    */
  double goal_radius;       /* par_.goal_radius                                                                     */
  int* status;              /* out n_prob: FQ_QUEUE_*                                                               */
  uint8_t* goal_seen;       /* out n_prob, or NULL                                                                  */
} fq_pair_queue;

/* HOST pointers everywhere; blocks until every output is in the caller's arrays (the whole ring is copied back). */
int fq_replan_pairs_queue(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                          const fq_pair_exact* exact, const fq_pair_decomp* decomp, const fq_pair_hr* hr, const fq_pair_map* map,
                          const fq_pair_queue* q);
/* The same, returning once everything is enqueued; outputs are valid after fq_wait(ctx).  Arrays must stay alive. */
int fq_replan_pairs_queue_async(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                                const fq_pair_exact* exact, const fq_pair_decomp* decomp, const fq_pair_hr* hr, const fq_pair_map* map,
                                const fq_pair_queue* q);
/* DEVICE pointers everywhere (the structs live on the host), with the hint rules of the selected family's _dev entry.
 * Never synchronises, so a CUDA graph can capture select, this call and pop together. */
int fq_replan_pairs_queue_dev(fq_ctx* ctx, const fq_pair_args* args, const fq_pair_assign* assign, const fq_pair_window* window,
                              const fq_pair_exact* exact, const fq_pair_decomp* decomp, const fq_pair_hr* hr, const fq_pair_map* map,
                              const fq_pair_queue* q, fq_pair_result* results_all, void* stream);

/* ---- several GPUs behind the boundary (SURVEY.md 8b/8e) ---------------------------------------------------------
 *
 * Candidates of different corridors are independent, so a batch is sharded BY CORRIDOR: contiguous blocks of problems
 * per GPU (fq_shard_range), no data-path communication while solving.  The path's one exchange is an all-gather of the
 * per-corridor winners of the genNewTraj selection (solverGurobi.cpp:445-472) -- a few hundred bytes per corridor, not the
 * per-candidate costs -- with NCCL, the communicator living inside the context.  Nothing like this exists in the
 * reference (one process, one CPU solver per trajectory kind: faster.hpp:74-75); the entry points below are what a
 * planner that evaluates many corridors per cycle would bind.  NCCL is loaded at run time (libnccl.so.2; the
 * environment variable FQ_NCCL_LIB overrides); single-GPU use never touches it.
 *
 * One process, n_gpus devices (devices == NULL: 0..n_gpus-1).  The returned context is the context of devices[0] for
 * every single-GPU entry point, and a GROUP for fq_replan_pairs, fq_replan_pairs_assign and fq_replan_pairs_window (sync
 * and async) and fq_solve_multi_sharded, which spread the corridors over all its devices.
 *
 * Those chained-replan entries check the whole description on a multi-GPU context (group or rank) exactly as on a plain
 * context: what a plain context refuses, they refuse with the same code and fq_last_error text.  They then check every
 * shard as a one-GPU call of its own.  Both checks run before any output is written (cand_ofs_* included) or any work is
 * enqueued, and every rank checks every shard, not only its own, so the ranks of a communicator accept or refuse a
 * description together.  One description passes the first check and not the second: a shared list (sigmas_*) whose
 * entry names a polytope that a corridor lacks.  A plain context lets that entry through when some corridor of the batch
 * has no polytope, but a shard without such a corridor refuses it ("sigmas_* entry >= number of polytopes"). */
int fq_create_multi(fq_ctx** out, int n_gpus, const int* devices);
/* One process per GPU: rank 0 obtains an id (128 bytes), the launcher distributes it (torch.distributed, MPI, a file),
 * every rank attaches its own context.  Afterwards fq_replan_pairs / fq_solve_multi_sharded on that context solve the
 * rank's shard of the (identical) description every rank passes, and fq_replan_pairs_dev / fq_allgather_dev exchange
 * device-resident results. */
int fq_comm_unique_id(void* id128);
int fq_comm_init(fq_ctx* ctx, const void* id128, int rank, int world);
int fq_comm_info(const fq_ctx* ctx, int* rank, int* world, int* nccl_version);
/* All-gather of `bytes` bytes per rank between device buffers on `stream` (NULL: the context's), rank order.  A context
 * without communicator copies (world of one). */
int fq_allgather_dev(fq_ctx* ctx, const void* d_send, void* d_recv, long bytes, void* stream);
/* The partition rule: problems [*lo, *hi) belong to `rank`; balanced by candidate count (cand_ofs[n_prob+1], or NULL for
 * equal problem counts).  Pure host code. */
int fq_shard_range(int n_prob, const int* cand_ofs, int rank, int world, int* lo, int* hi);
/* fq_solve_multi on a multi-GPU context (group: all problems solved by this process, spread over its GPUs; rank context:
 * this rank's shard only, `feasible`/`cost` of other shards stay untouched) plus, for EVERY problem on EVERY rank, the
 * winner of the genNewTraj selection: win_idx[j] = candidate index relative to cand_ofs[j] (-1: none feasible) of the
 * feasible candidate with the smallest dt, then the smallest cost; win_cost[j] its cost (+inf: none).  HOST pointers. */
int fq_solve_multi_sharded(fq_ctx* ctx, int N, int force_final, int n_prob, const double* x0, const double* xf,
                           const double* lim, const int* poly_ofs, const int* face_ofs, const double* Ab,
                           const int* cand_ofs, const double* dt, const uint8_t* sigma, uint8_t* feasible, double* cost,
                           int* win_idx, double* win_cost);

/* ---- host-side helpers (no GPU needed) ------------------------------------------------------------- */

/* getDTInitial (solverGurobi.cpp:659-759), including its float temporaries and MinPositiveElement
 * (solverGurobi_utils.hpp:19-32). */
double fq_dt_initial(const double* x0, const double* xf, const double* lim, int N);

/* resetX (solverGurobi.cpp:382-388): number of samples max(2, (int)(N*dt/DC)). */
int fq_num_samples(int N, double dt, double DC);

/* fillX (solverGurobi.cpp:122-168): out[i*12 .. i*12+11] = pos vel accel jerk at t=(i+1)*DC; the last
 * sample's vel/accel/jerk are zeroed. */
void fq_fill_x(int N, const double* coeffs, double dt, double DC, int n_samples, double* out);

/* Number of non-decreasing assignments C(N+P-1, P-1); if out != NULL writes min(count, cap) rows of N bytes in
 * lexicographic order. */
long fq_monotone_sigmas(int N, int P, uint8_t* out, long cap);

/* Convex decomposition of a polyline path against an obstacle point cloud -- the host-side input generator that feeds
 * setPolytopes in the reference: JPS_Manager::cvxEllipsoidDecomp (faster/src/jps_manager.cpp:80-127) over DecompUtil's
 * EllipsoidDecomp3D (line_segment.h:156-252 ellipsoid, decomp_base.h:83-115 polyhedron, line_segment.h:57-98 local
 * bbox), sign normalisation w.r.t. the segment midpoint (polyhedron.h:131-152) and the ground face appended last.
 *   path (n_seg+1) x 3, obs n_obs x 3, bbox[3] = local bounding box (reference: 2,2,1), inflate = drone radius.
 * Writes face_ofs[n_seg+1] and rows [Ax Ay Az b] into Ab (capacity cap_rows rows).  Returns the number of rows, or
 * FQ_E_NOMEM if cap_rows is too small, FQ_E_ARG on bad input.  Pure host code. */
int fq_ellipsoid_decomp(const double* path, int n_seg, const double* obs, int n_obs, const double* bbox,
                        double inflate, double z_ground, int* face_ofs, double* Ab, int cap_rows);

/* Path search on a voxel grid -- the host-side input generator in front of the decomposition
 * (jps_manager_.solveJPS3D, faster.cpp:361 -> thirdparty/jps3d GraphSearch, graph_search.cpp:123-219,:272-470).
 * map: xd*yd*zd cells, x fastest; 0 free, > 0 occupied, < 0 unknown.  26-connected, Euclidean costs and heuristic;
 * use_jps != 0: jump point search, else plain A*.  path_out receives up to cap (x,y,z) cell triples from start to goal
 * (jump points only with JPS).  Returns the number of path points (0: no path / start or goal not free), <0 on error;
 * *cost = path length in cells, *n_expanded = nodes expanded.  Pure host code. */
int fq_jps3d_plan(const int8_t* map, int xd, int yd, int zd, const int* start, const int* goal, int use_jps,
                  int max_expand, int* path_out, int cap, double* cost, int* n_expanded);

/* The same in world coordinates with the reference's post-processing (JPSPlanner<3>::plan, jps_planner.cpp:196-295:
 * cell = round((p - origin)/res - 0.5), centre = (cell + 0.5) res + origin (map_util.h:334-347), then removeLinePts and
 * removeCornerPts forwards and backwards with ray-traced line of sight (jps_planner.cpp:36-105, map_util.h:349-383)).
 * path_out: up to cap (x,y,z) points.  Returns the number of points, 0 if no path, <0 on error (FQ_E_NOMEM: cap). */
int fq_jps3d_plan_world(const int8_t* map, int xd, int yd, int zd, const double* origin, double res, const double* start,
                        const double* goal, int use_jps, double* path_out, int cap, double* raw_cost);

/* Introspection (tests): the number of nodes fq_jps3d_plan's search creates for this query (0 when start or goal is not
 * free), which is what fq_jps_batch's max_nodes bounds; < 0 on error.  Pure host code. */
long long fq_jps3d_nodes(const int8_t* map, int xd, int yd, int zd, const int* start, const int* goal, int use_jps);

/* Introspection (tests): the pruning rules in the layout of the reference's JPS3DNeib (graph_search.h:104-136):
 * ns[27][3][26], f1[27][3][12], f2[27][3][12], counts[27][2] = (natural, forced) entries per direction id. */
void fq_jps3d_rules(int* ns, int* f1, int* f2, int* counts);

/* Introspection (tests): copies the per-(N, force_final) plan tables documented in faster_b200/csrc/fq_plan.h.
 * Returns NY = 6N+1, or 0 if (N, force_final) is unsupported.  TZ: NY*(N-ne), T0: NY*(3+ne), FT: ne*3,
 * ne = force_final ? 3 : 2.  Any pointer may be NULL. */
int fq_plan_tables(int N, int force_final, double* TZ, double* T0, double* FT);

#ifdef __cplusplus
}
#endif
#endif
