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
#define FQ_ROW_TOL 1e-8           /* DEFAULT absolute row violation tolerance (m, m/s, m/s^2, m/s^3); run-time
                                     option "row_tol_1e9" of fq_set_option                                   */

#define FQ_E_ARG (-1)
#define FQ_E_CUDA (-2)
#define FQ_E_NOMEM (-3)
#define FQ_E_NOGPU (-4)

typedef struct fq_ctx fq_ctx;     /* opaque: device, stream, plan tables, scratch             */

int fq_abi_version(void);
/* 1 if this build has the named feature: "cert_memo" (compile-time switch FQ_CERT_MEMO, off by default: see
 * faster_b200/csrc/fq_kernels.cuh), "sweep_early_exit", "replan_pairs", "multi_gpu", "row_tol", "certificates". */
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
 * until the iteration cap gives up on solvable candidates.  1 (1e-9) is also the lowest FeasibilityTol Gurobi accepts.  "cert_memo" (0/1; only in builds with
 * fq_has_feature("cert_memo")): candidates of one problem share their infeasibility proofs (a candidate whose dt and polytopes on the proof's segments
 * match a recorded Farkas certificate is answered without a solve; same flags, iters = 0 marks them).
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
 * coefficients; *nodes_out = nodes evaluated; *exact_out = 0 if the tree had to be cut (node pool overflow, N < 4 or
 * more than 2047 faces) and the result is the best non-decreasing assignment instead.  Returns 1 / 0 / <0. */
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
 * every single-GPU entry point, and a GROUP for fq_replan_pairs / fq_replan_pairs_async / fq_solve_multi_sharded, which
 * spread the corridors over all its devices. */
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
