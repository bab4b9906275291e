// Chained replan (include/faster_b200.h: fq_replan_pairs*): whole sweep -> selection -> R -> safe sweep -> selection for
// many corridors in one submission.  Reference data flow: faster/src/faster.cpp:406-430 (whole), :474-475 (R), :521-537
// (safe).  Kernels: the batch solve (fq_kernels_t.cuh) and the small kernels of fq_pair.cuh.
#include "fq_assign.h"
#include "fq_ctx.h"
#include "fq_queue.h"
#include "fq_window.h"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace
{
// One sweep of the chain: the _whole or the _safe half of fq_pair_args, fq_pair_assign, fq_pair_window, fq_pair_exact
// and fq_pair_decomp.  Only each_field knows the two halves' names; the rest of this file works on a sweep.
struct Sweep
{
  int N = 0, force_final = 0;
  // fq_pair_args
  const double* xf = nullptr;
  const int *poly_ofs = nullptr, *face_ofs = nullptr;
  const double* Ab = nullptr;
  int max_faces = 0, max_poly_faces = 0;
  int n_fac = 0, n_sig = 0;
  const double* factors = nullptr;
  const uint8_t* sigmas = nullptr;
  uint8_t* feasible = nullptr;
  double *cost = nullptr, *coeffs = nullptr;
  // fq_pair_assign
  int max_poly = 0;
  long n_cand = 0;
  int* cand_ofs_out = nullptr;
  uint8_t* sigma_out = nullptr;
  // fq_pair_window
  const double *init = nullptr, *final_ = nullptr;
  double inc = 0, gamma = 0, gammap = 0;
  int max_fac = 0;
  double* factor = nullptr;
  int* trials = nullptr;
  double *next_init = nullptr, *next_final = nullptr;
  // fq_pair_exact
  int* exact = nullptr;
  long long* nodes = nullptr;
  // fq_pair_decomp
  const double* path = nullptr;
  const int* obs_ofs = nullptr;
  const double* obs = nullptr;
  int max_obs = 0;
  int* face_ofs_out = nullptr;
  double *Ab_out = nullptr, *pos_out = nullptr;   // pos_out: E (whole) or M (safe)
  int* status = nullptr;
  // set by the device entry: the largest candidate count of one corridor (sizes the solve launch) and the candidates per
  // time allocation (sizes an early-exit grid)
  int max_cand = 0, ee_width = 0;
};

// f(the sweep's field, the _whole field, the _safe field) for every field of the structs given (the others may be NULL).
// The one list of the two halves' names: sweep_of reads a side through it, put_sweep writes one.
template <class S, class A, class As, class W, class E, class D, class F>
void each_field(S& s, A* a, As* as, W* win, E* ex, D* dc, F&& f)
{
  f(s.N, a->N_whole, a->N_safe);  f(s.xf, a->xf_whole, a->xf_safe);
  f(s.poly_ofs, a->poly_ofs_whole, a->poly_ofs_safe);  f(s.face_ofs, a->face_ofs_whole, a->face_ofs_safe);  f(s.Ab, a->Ab_whole, a->Ab_safe);
  f(s.max_faces, a->max_faces_whole, a->max_faces_safe);  f(s.max_poly_faces, a->max_poly_faces_whole, a->max_poly_faces_safe);
  f(s.n_fac, a->n_fac_whole, a->n_fac_safe);  f(s.factors, a->factors_whole, a->factors_safe);
  f(s.n_sig, a->n_sig_whole, a->n_sig_safe);  f(s.sigmas, a->sigmas_whole, a->sigmas_safe);
  f(s.feasible, a->feasible_whole, a->feasible_safe);  f(s.cost, a->cost_whole, a->cost_safe);  f(s.coeffs, a->coeffs_whole, a->coeffs_safe);
  if (as)
  {
    f(s.max_poly, as->max_poly_whole, as->max_poly_safe);  f(s.n_cand, as->n_cand_whole, as->n_cand_safe);
    f(s.cand_ofs_out, as->cand_ofs_whole, as->cand_ofs_safe);  f(s.sigma_out, as->sigma_whole, as->sigma_safe);
  }
  if (win)
  {
    f(s.init, win->init_whole, win->init_safe);  f(s.final_, win->final_whole, win->final_safe);  f(s.inc, win->inc_whole, win->inc_safe);
    f(s.gamma, win->gamma_whole, win->gamma_safe);  f(s.gammap, win->gammap_whole, win->gammap_safe);
    f(s.max_fac, win->max_fac_whole, win->max_fac_safe);  f(s.factor, win->factor_whole, win->factor_safe);
    f(s.trials, win->trials_whole, win->trials_safe);
    f(s.next_init, win->next_init_whole, win->next_init_safe);  f(s.next_final, win->next_final_whole, win->next_final_safe);
  }
  if (ex) { f(s.exact, ex->exact_whole, ex->exact_safe);  f(s.nodes, ex->nodes_whole, ex->nodes_safe); }
  if (dc)
  {
    f(s.path, dc->path_whole, dc->path_safe);  f(s.obs_ofs, dc->obs_ofs_whole, dc->obs_ofs_safe);  f(s.obs, dc->obs_whole, dc->obs_safe);
    f(s.max_obs, dc->max_obs_whole, dc->max_obs_safe);  f(s.face_ofs_out, dc->face_ofs_whole, dc->face_ofs_safe);
    f(s.Ab_out, dc->Ab_whole, dc->Ab_safe);  f(s.pos_out, dc->E, dc->M);  f(s.status, dc->status_whole, dc->status_safe);
  }
}

// sweep `side` (0: whole, 1: safe) of the structs given
Sweep sweep_of(int side, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win, const fq_pair_exact* ex,
               const fq_pair_decomp* dc)
{
  Sweep s;
  each_field(s, a, as, win, ex, dc, [&](auto& mine, auto& whole, auto& safe) { mine = side ? safe : whole; });
  s.force_final = side == 0;
  return s;
}

// the inverse: sweep `side` written into the structs
void put_sweep(const Sweep& s, int side, fq_pair_args* a, fq_pair_assign* as, fq_pair_window* win, fq_pair_exact* ex,
               fq_pair_decomp* dc)
{
  each_field(s, a, as, win, ex, dc, [&](auto& mine, auto& whole, auto& safe) { (side ? safe : whole) = mine; });
}

// the checks of one sweep that need no device memory.  as == NULL: one shared assignment list (sigmas); otherwise a list
// per corridor, whose candidate counts the callers check.  win: per-corridor windows instead of the factor list.  dc: the
// chain decomposes the corridors, so the sweep has no faces and no final states.
const char* check_sweep(const Sweep& w, int n_prob, const fq_pair_assign* as, const fq_pair_window* win, const fq_pair_decomp* dc,
                        const fq_pair_map* mp)
{
  if (w.N < (w.force_final ? 3 : 2) || w.N > FQ_MAX_N) return "N out of range";
  if (!as)
  {
    if (w.n_fac <= 0 || w.n_sig <= 0) return "empty factor / assignment grid";
    if ((long long)n_prob * w.n_fac * w.n_sig > (1LL << 30)) return "too many candidates";
  }
  else
  {
    if (win && (w.factors || w.n_fac != 0)) return "per-corridor windows: factors_* must be NULL and n_fac_* 0";
    if (!win && w.n_fac <= 0) return "empty factor grid";
    if (w.sigmas || w.n_sig != 0) return "per-corridor assignment lists: sigmas_* must be NULL and n_sig_* 0";
  }
  if (dc && (w.face_ofs || w.Ab || w.xf))
    return "decomposing chain: face_ofs_*, Ab_* and xf_* must be NULL (the chain makes them)";
  if (dc && (w.max_faces <= 0 || w.max_poly_faces <= 0))
    return "decomposing chain: max_faces_* and max_poly_faces_* are caps and must be > 0";
  if (!w.poly_ofs || (!dc && (!w.xf || !w.face_ofs)) || (!win && !w.factors)) return "NULL argument";
  if (win)
  {
    if (!w.init || !w.final_) return "window arrays must not be NULL";
    if (!fqw::finite(w.inc) || !(w.inc > 0)) return "inc_* must be finite and > 0";
    if (!fqw::finite(w.gamma) || !fqw::finite(w.gammap)) return "gamma* must be finite";
  }
  if (dc)
  {
    if (!w.path || (!mp && (!w.obs_ofs || !w.obs))) return "decomp: path_* / obs_ofs_* / obs_* must not be NULL";
    if (mp && (w.obs_ofs || w.obs)) return "map: obs_ofs_* and obs_* must be NULL (the maps hold the clouds)";
    if ((uintptr_t)w.Ab_out & 15) return "decomp: Ab_* must be 16-byte aligned";
  }
  return nullptr;
}

// the checks every entry makes, and the two sweeps of the call (see check_sweep)
int check_chain(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win, const fq_pair_exact* ex,
                const fq_pair_decomp* dc, Sweep* sw, const fq_pair_map* mp = nullptr)
{
  if (!a) return fq_fail(ctx, FQ_E_ARG, "args is NULL");
  if ((win || ex || dc) && !as) return fq_fail(ctx, FQ_E_ARG, "assign is NULL");
  if (a->n_prob <= 0) return fq_fail(ctx, FQ_E_ARG, "n_prob <= 0");
  if (!(a->DC > 0) || !(a->r_fraction >= 0 && a->r_fraction <= 1)) return fq_fail(ctx, FQ_E_ARG, "DC must be > 0 and r_fraction in [0, 1]");
  if (!a->x0 || !a->lim || !a->results) return fq_fail(ctx, FQ_E_ARG, "NULL argument");
  if (dc)
  {
    for (int k = 0; k < 3; k++)
      if (!std::isfinite(dc->bbox[k]) || !(dc->bbox[k] > 0)) return fq_fail(ctx, FQ_E_ARG, "decomp: bbox must be finite and > 0");
    if (!std::isfinite(dc->inflate) || dc->inflate < 0 || !std::isfinite(dc->z_ground))
      return fq_fail(ctx, FQ_E_ARG, "decomp: inflate must be finite and >= 0, z_ground finite");
  }
  for (int i = 0; i < 2; i++)
  {
    sw[i] = sweep_of(i, a, as, win, ex, dc);
    if (const char* why = check_sweep(sw[i], a->n_prob, as, win, dc, mp)) return fq_fail(ctx, FQ_E_ARG, why);
  }
  return 0;
}

// the checks of fq_pair_hr that need no device memory (the chain with H and R needs the decomposing chain's arguments).
// map: the unknown clouds come from maps, so unk_ofs / unk must be NULL.
int check_hr(fq_ctx* ctx, const fq_pair_window* win, const fq_pair_decomp* dc, const fq_pair_hr* hr, bool map = false)
{
  if (!hr) return fq_fail(ctx, FQ_E_ARG, "hr is NULL");
  if (!dc) return fq_fail(ctx, FQ_E_ARG, "decomp is NULL");
  if (!std::isfinite(hr->drone_radius) || hr->drone_radius < 0) return fq_fail(ctx, FQ_E_ARG, "hr: drone_radius must be finite and >= 0");
  if (!std::isfinite(hr->delta_a) || !(hr->delta_a > 0)) return fq_fail(ctx, FQ_E_ARG, "hr: delta_a must be finite and > 0");
  if (!(hr->delta_H >= 0 && hr->delta_H <= 1)) return fq_fail(ctx, FQ_E_ARG, "hr: delta_H must be in [0, 1]");
  if (map && (hr->unk_ofs || hr->unk)) return fq_fail(ctx, FQ_E_ARG, "map: hr->unk_ofs and hr->unk must be NULL (the maps hold the clouds)");
  if (!map && (!hr->unk_ofs || !hr->unk)) return fq_fail(ctx, FQ_E_ARG, "hr: unk_ofs / unk must not be NULL");
  if (win && !hr->last_factor_safe) return fq_fail(ctx, FQ_E_ARG, "hr: last_factor_safe is required with a window");
  return 0;
}

// the checks of fq_pair_map that need no device memory (map_index is checked by the host entries)
int check_map(fq_ctx* ctx, const fq_pair_decomp* dc, const fq_pair_hr* hr, const fq_pair_window* win, const fq_pair_map* mp)
{
  if (!mp) return fq_fail(ctx, FQ_E_ARG, "map is NULL");
  if (!dc) return fq_fail(ctx, FQ_E_ARG, "decomp is NULL");
  if (hr)
    if (int rc = check_hr(ctx, win, dc, hr, true)) return rc;
  if (!mp->maps || mp->n_maps <= 0) return fq_fail(ctx, FQ_E_ARG, "map: no maps");
  for (int i = 0; i < mp->n_maps; i++)
  {
    if (!mp->maps[i]) return fq_fail(ctx, FQ_E_ARG, "map: a NULL map");
    if (fq_map_device(mp->maps[i]) != ctx->device) return fq_fail(ctx, FQ_E_ARG, "map: a map on another device");
    if (!fq_map_valid(mp->maps[i])) return fq_fail(ctx, FQ_E_ARG, "map: a map whose last update failed");
  }
  if (mp->max_local < 0 || mp->max_local > (1 << 30)) return fq_fail(ctx, FQ_E_ARG, "map: max_local out of range (0..2^30)");
  return 0;
}

// the chain's intermediate arrays, placed in ctx->d_pair: those of both sweeps, and a SweepScratch per sweep
struct Shared
{
  double *x0_safe, *re_cost;            // R, the safe sweep's start states; the winners' re-solves (costs and flags)
  uint8_t* re_feas;
  int *win_ofs, *n_samples, *k_safe;
  int* hr_r;                            // H and R from the unknown clouds: R's index (-1: no safe path) and needToComputeSafePath
  uint8_t* hr_need;
  // decomposing chain: staging and spill, used by one sweep after the other
  double *dc_stage, *dc_spill;
  int* dc_stage_n;
  uint8_t* dc_spill_flag;
  // against maps: the spilled survivors' cloud indices, and the submission's map table
  int* dc_spill_idx;
  const FqMapDev** map_table;
};
struct SweepScratch
{
  double *dt, *cost, *dt_base, *win_cost, *win_dt, *coeffs;
  uint8_t *sig, *feas, *win_sig;
  int *cand_ofs, *win_idx;
  double* fac;                          // per-corridor windows: n_prob x max_fac factor rows
  int* nf;                              // and |F_j| (-1: refused)
  double *dc_Ab, *dc_xf;                // decomposing chain: the corridors (unless the caller takes them), the final states
  int* dc_face;
};

// Exact stage (fq_replan_pairs_exact*): node pools, leaves and per-corridor tree state, placed in ctx->d_bnb.  Corridor c
// owns a slice of kTreeCap(n_prob) nodes in each of the two level pools (parents / children) and of kLeafCap leaves, so a
// cut tree never takes room from another corridor.
const int kLeafCap = 4096;
inline int tree_cap(int n_prob) { return std::max(64, 65536 / std::max(n_prob, 1)); }
struct Tree
{
  double* dts;
  unsigned long long *incumbent, *lbound;
  int *roots, *n_par, *n_leaves, *flags;
  long long* nodes;
  uint8_t *status, *changed_w, *changed_s, *closed;
  int* keep_idx;                       // the list winners of the sweep in progress (fq_bnb_resolve_kernel)
  double *keep_cost, *keep_dt, *redo_dt, *redo_coeffs;
  uint8_t* keep_sig;
  void* leaves;
  unsigned char *pool0, *pool1;
};

void tree_layout(FqPack& p, int n_prob, int stride, int max_N, size_t nb, Tree* t)
{
  const size_t np = (size_t)n_prob, cells = np * (size_t)std::max(stride, 1);
  t->dts = p.scratch<double>(cells);  t->incumbent = p.scratch<unsigned long long>(cells);  t->roots = p.scratch<int>(cells);
  t->lbound = p.scratch<unsigned long long>(cells);  t->closed = p.scratch<uint8_t>(cells);
  t->keep_idx = p.scratch<int>(np);  t->keep_cost = p.scratch<double>(np);  t->keep_dt = p.scratch<double>(np);
  t->keep_sig = p.scratch<uint8_t>(np * max_N);  t->redo_dt = p.scratch<double>(np);  t->redo_coeffs = p.scratch<double>(np * 12 * max_N);
  t->n_par = p.scratch<int>(2 * np);  t->n_leaves = p.scratch<int>(np);  t->flags = p.scratch<int>(2 * np);
  t->nodes = p.scratch<long long>(np);
  t->status = p.scratch<uint8_t>(np); t->changed_w = p.scratch<uint8_t>(np);  t->changed_s = p.scratch<uint8_t>(np);
  t->leaves = p.scratch<char>(np * kLeafCap * 32);
  t->pool0 = p.scratch<unsigned char>(np * tree_cap(n_prob) * nb);
  t->pool1 = p.scratch<unsigned char>(np * tree_cap(n_prob) * nb);
}

// One sweep's exact stage, enqueued on `st` after its selection: roots, N level launches (parent counts stay on the
// device) and the resolve.  `k` holds the sweep's corridors, `c` its candidates and list winners.
int exact_stage(fq_ctx* ctx, const Tree& t, FqKernelArgs k, FqBnbChainArgs& c, int max_poly_faces, uint8_t* changed,
                cudaStream_t st)
{
  const int N = k.N, ff = k.force_final, n = k.n_prob;
  c.n_prob = n; c.N = N; c.force_final = ff; c.poly_ofs = k.poly_ofs; c.face_ofs = k.face_ofs; c.Ab = k.Ab; c.x0 = k.x0;
  c.xf = k.xf; c.row_tol = ctx->row_tol;
  c.dts = t.dts; c.incumbent = t.incumbent; c.lbound = t.lbound; c.closed = t.closed;
  c.keep_idx = t.keep_idx; c.keep_cost = t.keep_cost; c.keep_dt = t.keep_dt; c.keep_sig = t.keep_sig; c.roots = t.roots; c.n_par = t.n_par; c.n_leaves = t.n_leaves; c.flags = t.flags;
  c.nodes = t.nodes; c.leaves = t.leaves; c.leaf_cap = kLeafCap; c.status = t.status; c.changed = changed;
  // rows the level kernel stages: at most 2047 (the item encoding), shrunk until one CTA-wide copy fits in shared memory
  int F = std::min(std::max(k.max_faces, 1), 2047);
  auto items = [&](int f) { return N * std::min(max_poly_faces > 0 ? max_poly_faces : f, f); };
  while (F > 1 && fq_bnb_level_smem(N, ff, F, items(F)) > 227 * 1024) F = F * 15 / 16;
  c.tree_ok = fq_bnb_node_bytes(N, ff) != 0 && fq_bnb_level_smem(N, ff, F, items(F)) <= 227 * 1024;
  c.max_faces = F;
  FQ_CUDA(fq_launch_bnb_roots(c, st));
  if (c.tree_ok)
  {
    FqPlanDev* pd = nullptr;
    if (int rc = fq_get_plan(ctx, N, ff, &pd)) return rc;
    FqBnbLevel L{};
    L.k = k;
    fq_fill_plan_args(*pd, &L.k);
    L.k.max_faces = F; L.k.item_cap = items(F); L.k.row_tol = ctx->row_tol;
    L.n_dt = c.stride; L.dts = t.dts; L.roots = t.roots; L.cap = tree_cap(n); L.incumbent = t.incumbent; L.leaves = t.leaves;
    L.n_leaves = t.n_leaves; L.leaf_cap = kLeafCap; L.flags = t.flags; L.nodes = t.nodes; L.keep_ties = 1;
    L.lbound = t.lbound; L.closed = t.closed;
    L.cpc = std::max(1, (16 * std::max(ctx->sm_count, 1) + n - 1) / n);
    unsigned char* pools[2] = { t.pool0, t.pool1 };
    for (int depth = 0; depth < N; depth++)
    {
      L.depth = depth;
      L.n_parents = t.n_par + (size_t)n * (depth & 1); L.n_children = t.n_par + (size_t)n * ((depth + 1) & 1);
      L.parents = pools[depth & 1]; L.children = pools[(depth + 1) & 1];
      FQ_CUDA(cudaMemsetAsync(L.n_children, 0, sizeof(int) * (size_t)n, st));
      FQ_CUDA(fq_launch_bnb_level(L, st));
      if (depth == 0) FQ_CUDA(fq_launch_bnb_certify(c, st));
    }
  }
  FQ_CUDA(fq_launch_bnb_resolve(c, st));
  return 0;
}

// largest |L(N, P, all_limit)| over P = 0 .. max_poly, or -1 when the list of max_poly polytopes is refused
long long longest_list(int N, int max_poly, long long all_limit)
{
  long long m = 0;
  for (int p = 0; p <= max_poly; p++) m = std::max(m, fqa::list_len(N, p, all_limit));
  return fqa::list_len(N, max_poly, all_limit) < 0 ? -1 : m;
}

// the chain itself, every pointer a device pointer and every argument checked.  as == NULL: the shared lists of `a`;
// sw: the two sweeps, their candidate counts set by the entry
int run_chain(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win, const fq_pair_exact* ex,
              const fq_pair_decomp* dc, const fq_pair_hr* hr, const fq_pair_map* mp, const fq_pair_plan* pl, const fq_pair_queue* qu, const Sweep* sw,
              fq_pair_result* results_all, cudaStream_t st)
{
  const int P = a->n_prob;
  // decomposing chain: staging slots of both sweeps (the larger), rows per slot, spilled survivors per slot
  size_t dslots = 0, dcap = 0, dspill = 0;
  if (dc)
  {
    dslots = (size_t)P * std::max(sw[0].max_poly, sw[1].max_poly);
    dcap = (size_t)std::max(sw[0].max_poly_faces, sw[1].max_poly_faces);
    dspill = fq_decomp_spill_n(std::max(sw[0].max_obs, sw[1].max_obs));
  }
  Shared sh;
  SweepScratch ss[2];
  auto layout = [&](FqPack& p) {
    sh.x0_safe = p.scratch<double>((size_t)9 * P);  sh.re_cost = p.scratch<double>(P);  sh.re_feas = p.scratch<uint8_t>(P);
    sh.win_ofs = p.scratch<int>(P + 1);  sh.n_samples = p.scratch<int>(P);  sh.k_safe = p.scratch<int>(P);
    sh.hr_r = p.scratch<int>(hr ? P : 0);  sh.hr_need = p.scratch<uint8_t>(hr ? P : 0);
    sh.dc_stage = p.scratch<double>(dslots * dcap * 4);    sh.dc_stage_n = p.scratch<int>(dslots);
    sh.dc_spill = p.scratch<double>(dslots * dspill * 4);  sh.dc_spill_flag = p.scratch<uint8_t>(dslots * dspill);
    sh.dc_spill_idx = p.scratch<int>(mp ? dslots * dspill : 0);  sh.map_table = p.scratch<const FqMapDev*>(mp ? mp->n_maps : 0);
    for (int i = 0; i < 2; i++)
    {
      const Sweep& w = sw[i];
      SweepScratch& s = ss[i];
      const size_t nc = (size_t)w.n_cand;
      s.dt = p.scratch<double>(nc);  s.cost = p.scratch<double>(nc);  s.feas = p.scratch<uint8_t>(nc);  s.sig = p.scratch<uint8_t>(nc * w.N);
      s.dt_base = p.scratch<double>(P);  s.win_cost = p.scratch<double>(P);  s.win_dt = p.scratch<double>(P);
      s.coeffs = p.scratch<double>((size_t)12 * w.N * P);
      s.cand_ofs = p.scratch<int>(P + 1);  s.win_idx = p.scratch<int>(P);  s.win_sig = p.scratch<uint8_t>((size_t)P * w.N);
      s.fac = p.scratch<double>(win ? (size_t)P * w.max_fac : 0);  s.nf = p.scratch<int>(win ? P : 0);
      s.dc_Ab = p.scratch<double>(dc && !w.Ab_out ? (size_t)P * w.max_faces * 4 : 0);
      s.dc_face = p.scratch<int>(dc && !w.face_ofs_out ? (size_t)P * w.max_poly + 1 : 0);
      s.dc_xf = p.scratch<double>(dc ? (size_t)9 * P : 0);
    }
  };
  FqPack pk;
  layout(pk);
  FQ_CUDA(ctx->d_pair.reserve(pk.at));   // grows only on the first call / a larger batch (synchronous cudaMalloc)
  pk = pk.place(ctx->d_pair.p);
  layout(pk);
  if (int rc = pk.done(ctx)) return rc;
  if (mp)
    for (int at = 0; at < mp->n_maps; at += FqMapTableChunk::kCap)
    {
      FqMapTableChunk c{};
      c.n = std::min(FqMapTableChunk::kCap, mp->n_maps - at); c.at = at; c.table = sh.map_table;
      for (int i = 0; i < c.n; i++) c.m[i] = fq_map_descriptor(mp->maps[at + i]);
      FQ_CUDA(fq_launch_map_table(c, st));
    }
  Tree tree{};
  const int stride = std::max(win ? std::max(sw[0].max_fac, sw[1].max_fac) : std::max(sw[0].n_fac, sw[1].n_fac), 1);
  if (ex)
  { // the whole tree is done before the safe one starts: one pool serves both
    const int max_N = std::max(sw[0].N, sw[1].N);
    const size_t nb = std::max(fq_bnb_node_bytes(sw[0].N, sw[0].force_final), fq_bnb_node_bytes(sw[1].N, sw[1].force_final));
    FqPack tp;
    tree_layout(tp, P, stride, max_N, nb, &tree);
    FQ_CUDA(ctx->d_bnb.reserve(tp.at));
    tp = tp.place(ctx->d_bnb.p);
    tree_layout(tp, P, stride, max_N, nb, &tree);
    if (int rc = tp.done(ctx)) return rc;
  }

  // One sweep from the start states x0: a decomposing chain's corridors (`first`: their vertex 0, NULL: the path's own),
  // getDTInitial, the candidates, the batch solve, the selection, the exact stage (its tree flags to `changed`), and the
  // winners' coefficients into `coeffs` (NULL: not wanted).
  auto run_sweep = [&](const Sweep& w, SweepScratch& s, const double* x0, const double* first, double* coeffs,
                       uint8_t* changed, int side) -> int {
    FqKernelArgs corr{};                // the sweep's corridors; each launch adds its candidates and outputs
    corr.N = w.N; corr.force_final = w.force_final; corr.n_prob = P; corr.x0 = x0; corr.xf = w.xf; corr.lim = a->lim;
    corr.poly_ofs = w.poly_ofs; corr.face_ofs = w.face_ofs; corr.Ab = w.Ab; corr.max_faces = w.max_faces;
    if (dc)
    { // faster.cpp:393-403 whole, :485-504 safe: the corridors from the paths and clouds, into the caller's outputs or the
      // scratch, and the final states (E / M, which getDTInitial reads) into the scratch
      FqDecompArgs x{};
      x.n_prob = P; x.max_poly = w.max_poly; x.poly_ofs = w.poly_ofs; x.path = w.path; x.first = first;
      x.obs_ofs = w.obs_ofs; x.obs = w.obs; x.max_obs = w.max_obs;
      for (int k = 0; k < 3; k++) x.bbox[k] = dc->bbox[k];
      x.inflate = dc->inflate; x.z_ground = dc->z_ground; x.cap_pf = w.max_poly_faces; x.max_faces = w.max_faces;
      x.stage = sh.dc_stage; x.stage_n = sh.dc_stage_n; x.spill = sh.dc_spill; x.spill_flag = sh.dc_spill_flag; x.spill_n = (int)dspill;
      x.goal = dc->goal; x.face_cap = P * x.max_poly;
      x.face_ofs = w.face_ofs_out ? w.face_ofs_out : s.dc_face; x.Ab = w.Ab_out ? w.Ab_out : s.dc_Ab; x.xf = s.dc_xf;
      x.pos_out = w.pos_out; x.status = w.status;
      if (mp)
      { // the whole sweep reads O, the safe sweep U ++ O (faster.cpp:130-132)
        x.maps = sh.map_table; x.map_index = mp->map_index; x.n_maps = mp->n_maps; x.map_unk = side; x.spill_idx = sh.dc_spill_idx;
      }
      FQ_CUDA(fq_launch_decomp(x, st));
      corr.face_ofs = x.face_ofs; corr.Ab = x.Ab; corr.xf = x.xf;
    }
    FQ_CUDA(fq_launch_dtbase(P, w.N, a->DC, x0, corr.xf, a->lim, s.dt_base, st));
    if (!as)
      FQ_CUDA(fq_launch_expand_grid(P, w.N, w.n_fac, w.n_sig, w.factors, w.sigmas, s.dt_base, s.dt, s.sig, s.cand_ofs, st));
    else if (win)
    {
      FQ_CUDA(fq_launch_window_offsets(P, w.N, w.max_fac, as->all_limit, w.max_poly, (long long)w.n_cand, w.poly_ofs, s.nf,
                                       s.cand_ofs, st));
      FQ_CUDA(fq_launch_expand_window(P, w.N, w.max_fac, as->all_limit, s.fac, s.nf, s.dt_base, w.poly_ofs, s.cand_ofs, s.dt,
                                      s.sig, st));
    }
    else
    {
      FQ_CUDA(fq_launch_assign_offsets(P, w.N, w.n_fac, as->all_limit, w.max_poly, (long long)w.n_cand, w.poly_ofs, s.cand_ofs, st));
      FQ_CUDA(fq_launch_expand_assign(P, w.N, w.n_fac, as->all_limit, w.factors, s.dt_base, w.poly_ofs, s.cand_ofs, s.dt, s.sig, st));
    }
    uint8_t* feas = w.feasible ? w.feasible : s.feas;
    double* cost = w.cost ? w.cost : s.cost;
    FqKernelArgs k = corr;
    k.cand_ofs = s.cand_ofs; k.dt = s.dt; k.sigma = s.sig; k.feasible = feas; k.cost = cost;
    k.sorted_dt = 1; k.ee_width = w.ee_width;             // factor-major grid, ascending factors
    if (int rc = fq_launch_solve_ctx(ctx, k, w.max_cand, w.max_poly_faces, st)) return rc;
    FqSelectMultiArgs m{};
    m.n_prob = P; m.N = w.N; m.n_sig = w.n_sig; m.cand_ofs = s.cand_ofs; m.dt = s.dt; m.sigma = s.sig; m.feasible = feas; m.cost = cost;
    m.win_idx = s.win_idx; m.win_cost = s.win_cost; m.win_dt = s.win_dt; m.win_sigma = s.win_sig; m.win_ofs = sh.win_ofs;
    FQ_CUDA(fq_launch_select_multi(m, st));
    FqBnbChainArgs cx{};                                   // the exact stage's view of the sweep
    if (ex)
    {
      cx.stride = stride; cx.all_limit = as->all_limit; cx.cand_ofs = s.cand_ofs; cx.cand_dt = s.dt;
      cx.n_fac = w.n_fac; cx.n_fac_j = win ? s.nf : nullptr;
      cx.win_idx = s.win_idx; cx.win_cost = s.win_cost; cx.win_dt = s.win_dt; cx.win_sig = s.win_sig;
      cx.exact_out = w.exact; cx.nodes_out = w.nodes;
      if (int rc = exact_stage(ctx, tree, corr, cx, w.max_poly_faces, changed, st)) return rc;
    }
    if (!coeffs) return 0;
    // coefficients of the winners: one candidate per corridor through the same kernel (losers' dt is NaN -> "not solved")
    FqKernelArgs r = corr;
    r.cand_ofs = sh.win_ofs; r.dt = s.win_dt; r.sigma = s.win_sig; r.feasible = sh.re_feas; r.cost = sh.re_cost; r.coeffs = coeffs;
    if (int rc = fq_launch_solve_ctx(ctx, r, 1, w.max_poly_faces, st)) return rc;
    if (ex)
    { // tree winners the solve did not confirm go back to their list winners, whose coefficients a second solve of those
      // corridors provides
      FQ_CUDA(fq_launch_bnb_fallback(cx, sh.re_feas, tree.redo_dt, st));
      r.dt = tree.redo_dt; r.coeffs = tree.redo_coeffs;
      if (int rc = fq_launch_solve_ctx(ctx, r, 1, w.max_poly_faces, st)) return rc;
      FQ_CUDA(fq_launch_bnb_adopt(P, w.N, tree.redo_dt, tree.redo_coeffs, coeffs, st));
    }
    return 0;
  };

  // ---- per-corridor windows: every window is read here, before anything is written (the outputs may alias them)
  if (win)
    for (int i = 0; i < 2; i++)
      FQ_CUDA(fq_launch_window_factors(P, sw[i].max_fac, sw[i].init, sw[i].final_, sw[i].inc, ss[i].fac, ss[i].nf, st));
  // ---- whole sweep (faster.cpp:406-430); R needs its winners' coefficients
  double* coeffs_w = sw[0].coeffs ? sw[0].coeffs : ss[0].coeffs;
  if (int rc = run_sweep(sw[0], ss[0], a->x0, nullptr, coeffs_w, tree.changed_w, 0)) return rc;
  // ---- R (faster.cpp:474-475) and the safe sweep from it (faster.cpp:521-537), in corridors around R when the chain
  //      decomposes them; the exact stage re-solves its winners to confirm them, wanted or not.  With hr, H and R come
  //      from the unknown clouds (faster.cpp:452-475), and a corridor that needs no safe path gets a NaN R, so that the
  //      safe decomposition and sweep skip it as they skip a corridor without a whole winner.
  FqPairMidArgs m;
  m.n_prob = P; m.N = sw[0].N; m.DC = a->DC; m.r_fraction = a->r_fraction; m.coeffs = coeffs_w; m.win_dt = ss[0].win_dt;
  m.win_idx = ss[0].win_idx; m.x0_safe = sh.x0_safe; m.n_samples = sh.n_samples; m.k_safe = sh.k_safe;
  if (hr)
  {
    FqPairHrArgs h;
    h.n_prob = P; h.N = sw[0].N; h.DC = a->DC; h.drone_radius = hr->drone_radius; h.delta_a = hr->delta_a; h.delta_H = hr->delta_H;
    h.coeffs = coeffs_w; h.win_dt = ss[0].win_dt; h.win_idx = ss[0].win_idx; h.lim = a->lim; h.unk_ofs = hr->unk_ofs; h.unk = hr->unk;
    h.r_index = sh.hr_r; h.need = sh.hr_need; h.need_out = hr->need_safe; h.index_H = hr->index_H;
    if (mp) { h.maps = sh.map_table; h.map_index = mp->map_index; }
    FQ_CUDA(fq_launch_pair_hr(h, st));
    m.r_index = sh.hr_r;
  }
  FQ_CUDA(fq_launch_pair_mid(m, st));
  // the safe winners' coefficients: wanted, or needed by the exact stage's confirmation or by the plan
  double* coeffs_s = sw[1].coeffs ? sw[1].coeffs : ex || pl || qu ? ss[1].coeffs : nullptr;
  if (int rc = run_sweep(sw[1], ss[1], sh.x0_safe, sh.x0_safe, coeffs_s, tree.changed_s, 1)) return rc;

  FqPairFinalArgs f;
  f.n_prob = P; f.n_sig_w = sw[0].n_sig; f.n_sig_s = sw[1].n_sig; f.win_idx_w = ss[0].win_idx; f.win_idx_s = ss[1].win_idx;
  f.n_samples = sh.n_samples; f.k_safe = sh.k_safe; f.win_cost_w = ss[0].win_cost; f.win_cost_s = ss[1].win_cost;
  f.win_dt_w = ss[0].win_dt; f.win_dt_s = ss[1].win_dt; f.dt_base_w = ss[0].dt_base; f.dt_base_s = ss[1].dt_base; f.x0_safe = sh.x0_safe;
  f.out = a->results;
  if (as)
  {
    f.cand_ofs_w = ss[0].cand_ofs; f.cand_ofs_s = ss[1].cand_ofs; f.n_fac_w = sw[0].n_fac; f.n_fac_s = sw[1].n_fac;
    f.N_w = sw[0].N; f.N_s = sw[1].N; f.win_sig_w = ss[0].win_sig; f.win_sig_s = ss[1].win_sig;
    f.sigma_out_w = sw[0].sigma_out; f.sigma_out_s = sw[1].sigma_out;
    if (win) { f.n_fac_j_w = ss[0].nf; f.n_fac_j_s = ss[1].nf; }
    if (ex)
    {
      f.changed_w = tree.changed_w; f.changed_s = tree.changed_s; f.poly_ofs_w = sw[0].poly_ofs; f.poly_ofs_s = sw[1].poly_ofs;
      f.all_limit = as->all_limit;
    }
    for (int i = 0; i < 2; i++)
      if (sw[i].cand_ofs_out)
        FQ_CUDA(cudaMemcpyAsync(sw[i].cand_ofs_out, ss[i].cand_ofs, sizeof(int) * (size_t)(P + 1), cudaMemcpyDeviceToDevice, st));
  }
  FQ_CUDA(fq_launch_pair_final(f, st));
  // the plan pieces (appendToPlan, faster.cpp:606-648) from the winners and k_safe
  FqPairPlanArgs q;
  q.n_prob = P; q.N_w = sw[0].N; q.N_s = sw[1].N; q.DC = a->DC;
  q.win_idx_w = ss[0].win_idx; q.win_idx_s = ss[1].win_idx; q.win_dt_w = ss[0].win_dt; q.win_dt_s = ss[1].win_dt;
  q.n_samples = sh.n_samples; q.k_safe = sh.k_safe; q.need = hr ? sh.hr_need : nullptr;
  q.coeffs_w = coeffs_w; q.coeffs_s = coeffs_s;
  if (qu)
  { // ---- the pieces appended to the planners' plans; before the windows, whose update the appends gate
    FqQueueArgs u{};
    u.n = P; u.n_rows = qu->ring.n_rows; u.cap = qu->ring.cap; u.delta_t = qu->ring.delta_t; u.rows = qu->rows;
    u.states = qu->ring.states; u.head = qu->ring.head; u.size = qu->ring.size; u.k_end = qu->k_end;
    u.G_term = qu->G_term; u.goal_radius = qu->goal_radius; u.status = qu->status; u.goal_seen = qu->goal_seen;
    FQ_CUDA(fq_launch_pair_queue(q, u, st));
  }
  if (win)
  {
    FqPairWindowArgs wa;
    wa.n_prob = P; wa.max_fac_w = sw[0].max_fac; wa.max_fac_s = sw[1].max_fac; wa.rec = a->results;
    wa.cand_ofs_w = ss[0].cand_ofs; wa.cand_ofs_s = ss[1].cand_ofs; wa.n_fac_w = ss[0].nf; wa.n_fac_s = ss[1].nf;
    wa.fac_w = ss[0].fac; wa.fac_s = ss[1].fac;
    wa.init_w = sw[0].init; wa.final_w = sw[0].final_; wa.init_s = sw[1].init; wa.final_s = sw[1].final_;
    wa.gamma_w = sw[0].gamma; wa.gammap_w = sw[0].gammap; wa.gamma_s = sw[1].gamma; wa.gammap_s = sw[1].gammap;
    wa.factor_w = sw[0].factor; wa.factor_s = sw[1].factor; wa.trials_w = sw[0].trials; wa.trials_s = sw[1].trials;
    wa.next_init_w = sw[0].next_init; wa.next_final_w = sw[0].next_final;
    wa.next_init_s = sw[1].next_init; wa.next_final_s = sw[1].next_final;
    if (hr) { wa.need_safe = sh.hr_need; wa.last_factor_safe = hr->last_factor_safe; }
    if (qu) wa.gate = qu->status;
    FQ_CUDA(fq_launch_pair_window(wa, st));
  }
  if (pl)
  { // ---- the plan pieces as rows of the caller's array
    q.cap = pl->cap_states; q.states = pl->states; q.plan_ofs = pl->plan_ofs; q.status = pl->status;
    FQ_CUDA(fq_launch_pair_plan(q, st));
  }
  // ---- the path's one exchange: every rank's result records to every rank (north_star: one all-gather, only when the
  //      batch is spread over several GPUs)
  if (results_all && ctx->comm)
    return fq_comm_allgather(ctx, a->results, results_all, sizeof(fq_pair_result) * (size_t)P, st);
  if (results_all)
    FQ_CUDA(cudaMemcpyAsync(results_all, a->results, sizeof(fq_pair_result) * (size_t)P, cudaMemcpyDeviceToDevice, st));
  return 0;
}

// the chains with per-corridor lists (fq_replan_pairs_assign_dev, _window_dev, _exact_dev, _decomp_dev): every pointer
// of the structs is a device pointer; the sweeps' sizes come from the hints of `as` (capacities) and `win` (factor rows)
int chain_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win, const fq_pair_exact* ex,
              const fq_pair_decomp* dc, fq_pair_result* results_all, void* stream_v, const fq_pair_hr* hr = nullptr,
              const fq_pair_map* mp = nullptr, const fq_pair_plan* pl = nullptr, const fq_pair_queue* qu = nullptr)
{
  if (!ctx) return FQ_E_ARG;
  if (!as) return fq_fail(ctx, FQ_E_ARG, "assign is NULL");
  Sweep sw[2];
  if (int rc = check_chain(ctx, a, as, win, ex, dc, sw, mp)) return rc;
  if (as->all_limit < 0) return fq_fail(ctx, FQ_E_ARG, "all_limit < 0");
  for (Sweep& w : sw)
  {
    if (win && (w.max_fac < 0 || w.max_fac > fqw::kMaxFactors)) return fq_fail(ctx, FQ_E_ARG, "max_fac_* out of range (0..4096)");
    if (w.max_poly < 0 || w.max_poly > FQ_MAX_POLY) return fq_fail(ctx, FQ_E_ARG, "max_poly_* out of range (0..FQ_MAX_POLY)");
    if (w.n_cand < 0 || w.n_cand > (1L << 30)) return fq_fail(ctx, FQ_E_ARG, "too many candidates (n_cand_* out of 0..2^30)");
    if (mp) w.max_obs = mp->max_local;                   // the survivors of one segment, not a cloud
    if (dc && w.max_obs < 0) return fq_fail(ctx, FQ_E_ARG, "decomp: max_obs_* < 0");
    if ((uintptr_t)w.Ab & 15) return fq_fail(ctx, FQ_E_ARG, "Ab must be 16-byte aligned");
    // the longest list is the candidates per time allocation; with the factors, the most candidates of one corridor
    const long long longest = longest_list(w.N, w.max_poly, as->all_limit);
    if (longest < 0) return fq_fail(ctx, FQ_E_ARG, "assignment list longer than 2^20");
    const long long most = longest * (win ? w.max_fac : w.n_fac);
    if (most > (1LL << 30)) return fq_fail(ctx, FQ_E_ARG, "too many candidates");
    w.max_cand = (int)(win ? std::max(1LL, most) : most);
    w.ee_width = (int)longest;
  }
  FQ_CUDA(cudaSetDevice(ctx->device));
  return run_chain(ctx, a, as, win, ex, dc, hr, mp, pl, qu, sw, results_all, stream_v ? (cudaStream_t)stream_v : ctx->stream);
}

// the chain with the shared lists of `a` (fq_replan_pairs_dev): every pointer of `a` is a device pointer
int shared_dev(fq_ctx* ctx, const fq_pair_args* a, fq_pair_result* results_all, void* stream_v, const fq_pair_plan* pl = nullptr,
               const fq_pair_queue* qu = nullptr)
{
  if (!ctx) return FQ_E_ARG;
  Sweep sw[2];
  if (int rc = check_chain(ctx, a, nullptr, nullptr, nullptr, nullptr, sw)) return rc;
  for (Sweep& w : sw)
  {
    if ((uintptr_t)w.Ab & 15) return fq_fail(ctx, FQ_E_ARG, "Ab must be 16-byte aligned");
    w.n_cand = (long)a->n_prob * w.n_fac * w.n_sig;
    w.max_cand = w.n_fac * w.n_sig;
    w.ee_width = w.n_sig;
  }
  FQ_CUDA(cudaSetDevice(ctx->device));
  return run_chain(ctx, a, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, pl, qu, sw, results_all,
                   stream_v ? (cudaStream_t)stream_v : ctx->stream);
}

// the plan's own refusals (fq_replan_pairs_plan*)
int check_plan(fq_ctx* ctx, const fq_pair_plan* pl)
{
  if (!pl) return fq_fail(ctx, FQ_E_ARG, "plan is NULL");
  if (!pl->states || !pl->plan_ofs) return fq_fail(ctx, FQ_E_ARG, "plan: states and plan_ofs must not be NULL");
  if (pl->cap_states < 0) return fq_fail(ctx, FQ_E_ARG, "plan: cap_states < 0");
  if (ctx->is_group || ctx->comm)
    return fq_fail(ctx, FQ_E_ARG, "fq_replan_pairs_plan: multi-GPU contexts are not supported (plans are variable-length per corridor)");
  return 0;
}

// what a ring's struct alone shows wrong (fq_queue_*, fq_replan_pairs_queue*), or nullptr
const char* queue_struct(const fq_queue* q)
{
  if (!q) return "queue is NULL";
  if (!q->states || !q->head || !q->size) return "queue: states, head and size must not be NULL";
  if (q->n_rows < 1) return "queue: n_rows < 1";
  if (q->cap < 1) return "queue: cap < 1";
  if (q->delta_t < 1) return "queue: delta_t < 1";
  return nullptr;
}

// the host entries' row checks: every row named in range, named once (`unique`), and a ring (`ring`)
const char* queue_rows(const fq_queue* q, int n, const int* rows, bool unique, bool ring)
{
  std::vector<char> named((size_t)q->n_rows, 0);
  for (int j = 0; j < n; j++)
  {
    const int r = rows ? rows[j] : j;
    if (r < 0 || r >= q->n_rows) return "queue: a row outside 0 .. n_rows-1";
    if (unique && named[(size_t)r]) return "queue: a row named twice";
    named[(size_t)r] = 1;
    if (ring && !fqq::ring_ok(q->head[r], q->size[r], q->cap)) return "queue: an invalid row (head outside 0 .. cap-1 or size outside 0 .. cap)";
  }
  return nullptr;
}

// the queue's own refusals (fq_replan_pairs_queue*)
int check_queue(fq_ctx* ctx, const fq_pair_queue* qu)
{
  if (!qu) return fq_fail(ctx, FQ_E_ARG, "queue is NULL");
  if (const char* why = queue_struct(&qu->ring)) return fq_fail(ctx, FQ_E_ARG, why);
  if (!qu->k_end || !qu->status) return fq_fail(ctx, FQ_E_ARG, "queue: k_end and status must not be NULL");
  if (ctx->is_group || ctx->comm)
    return fq_fail(ctx, FQ_E_ARG, "fq_replan_pairs_queue: multi-GPU contexts are not supported");
  return 0;
}

// The device chain the non-NULL structs select (fq_replan_pairs_plan*; the same dispatch as the host entries): the shared
// lists without assign, else _map, _hr, _decomp, _exact, _window or _assign, each with its own family's checks.
int family_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win, const fq_pair_exact* ex,
               const fq_pair_decomp* dc, const fq_pair_hr* hr, const fq_pair_map* mp, const fq_pair_plan* pl,
               fq_pair_result* results_all, void* stream_v, const fq_pair_queue* qu = nullptr)
{
  if (!as)
  {
    if (win || ex || dc || hr || mp) return fq_fail(ctx, FQ_E_ARG, "assign is NULL");
    return shared_dev(ctx, a, results_all, stream_v, pl, qu);
  }
  if (mp)
  {
    if (int rc = check_map(ctx, dc, hr, win, mp)) return rc;
  }
  else if (hr)
  {
    if (int rc = check_hr(ctx, win, dc, hr)) return rc;
  }
  return chain_dev(ctx, a, as, win, ex, dc, results_all, stream_v, hr, mp, pl, qu);
}
}  // namespace

extern "C" int fq_replan_pairs_dev(fq_ctx* ctx, const fq_pair_args* a, fq_pair_result* results_all, void* stream_v)
{
  return shared_dev(ctx, a, results_all, stream_v);
}

extern "C" int fq_replan_pairs_plan_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                        const fq_pair_exact* ex, const fq_pair_decomp* dc, const fq_pair_hr* hr, const fq_pair_map* mp,
                                        const fq_pair_plan* pl, fq_pair_result* results_all, void* stream_v)
{
  if (!ctx) return FQ_E_ARG;
  if (int rc = check_plan(ctx, pl)) return rc;
  return family_dev(ctx, a, as, win, ex, dc, hr, mp, pl, results_all, stream_v);
}

extern "C" int fq_replan_pairs_queue_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                         const fq_pair_exact* ex, const fq_pair_decomp* dc, const fq_pair_hr* hr, const fq_pair_map* mp,
                                         const fq_pair_queue* qu, fq_pair_result* results_all, void* stream_v)
{
  if (!ctx) return FQ_E_ARG;
  if (int rc = check_queue(ctx, qu)) return rc;
  return family_dev(ctx, a, as, win, ex, dc, hr, mp, nullptr, results_all, stream_v, qu);
}

namespace
{
// the FqQueueArgs of a small ring kernel
FqQueueArgs queue_args(const fq_queue* q, int n, const int* rows)
{
  FqQueueArgs u{};
  u.n = n; u.n_rows = q->n_rows; u.cap = q->cap; u.delta_t = q->delta_t; u.rows = rows;
  u.states = q->states; u.head = q->head; u.size = q->size;
  return u;
}

int queue_launched(cudaError_t e) { return e == cudaSuccess ? 0 : fq_cuda_fail(nullptr, e, "fq_queue_*_dev launch"); }
}  // namespace

extern "C" int fq_queue_reset(const fq_queue* q, int n, const int* rows, const double* pos)
{
  if (const char* why = queue_struct(q)) return fq_fail(nullptr, FQ_E_ARG, why);
  if (n < 0 || (n > 0 && !pos)) return fq_fail(nullptr, FQ_E_ARG, "queue: n < 0, or pos NULL");
  if (const char* why = queue_rows(q, n, rows, true, false)) return fq_fail(nullptr, FQ_E_ARG, why);
  for (int j = 0; j < n; j++)
  {
    const int r = rows ? rows[j] : j;
    fqq::reset(q->states + (size_t)r * q->cap * fqq::kState, q->head + r, q->size + r, pos + 3 * (size_t)j);
  }
  return 0;
}

extern "C" int fq_queue_select(const fq_queue* q, int n, const int* rows, double* x0, int* k_end)
{
  if (const char* why = queue_struct(q)) return fq_fail(nullptr, FQ_E_ARG, why);
  if (n < 0 || (n > 0 && (!x0 || !k_end))) return fq_fail(nullptr, FQ_E_ARG, "queue: n < 0, or x0 or k_end NULL");
  if (const char* why = queue_rows(q, n, rows, false, true)) return fq_fail(nullptr, FQ_E_ARG, why);
  for (int j = 0; j < n; j++)
  {
    const int r = rows ? rows[j] : j;
    k_end[j] = fqq::select(q->states + (size_t)r * q->cap * fqq::kState, q->head[r], q->size[r], q->cap, q->delta_t, x0 + 9 * (size_t)j);
  }
  return 0;
}

extern "C" int fq_queue_pop(const fq_queue* q, int n, const int* rows, const int* ticks, int max_ticks, double* goals)
{
  if (const char* why = queue_struct(q)) return fq_fail(nullptr, FQ_E_ARG, why);
  if (n < 0 || max_ticks < 0 || (n > 0 && (!ticks || (max_ticks > 0 && !goals))))
    return fq_fail(nullptr, FQ_E_ARG, "queue: n < 0, max_ticks < 0, or ticks or goals NULL");
  if (const char* why = queue_rows(q, n, rows, true, true)) return fq_fail(nullptr, FQ_E_ARG, why);
  for (int j = 0; j < n; j++)
  {
    const int r = rows ? rows[j] : j;
    const int t = ticks[j] < 0 ? 0 : std::min(ticks[j], max_ticks);
    fqq::pop(q->states + (size_t)r * q->cap * fqq::kState, q->head + r, q->size + r, q->cap, t,
             goals + (size_t)j * max_ticks * fqq::kState);
  }
  return 0;
}

extern "C" int fq_queue_reset_dev(const fq_queue* q, int n, const int* rows, const double* pos, void* stream)
{
  if (const char* why = queue_struct(q)) return fq_fail(nullptr, FQ_E_ARG, why);
  if (n < 0 || (n > 0 && !pos)) return fq_fail(nullptr, FQ_E_ARG, "queue: n < 0, or pos NULL");
  FqQueueArgs u = queue_args(q, n, rows);
  u.pos = pos;
  return queue_launched(fq_launch_queue_reset(u, (cudaStream_t)stream));
}

extern "C" int fq_queue_select_dev(const fq_queue* q, int n, const int* rows, double* x0, int* k_end, void* stream)
{
  if (const char* why = queue_struct(q)) return fq_fail(nullptr, FQ_E_ARG, why);
  if (n < 0 || (n > 0 && (!x0 || !k_end))) return fq_fail(nullptr, FQ_E_ARG, "queue: n < 0, or x0 or k_end NULL");
  FqQueueArgs u = queue_args(q, n, rows);
  u.x0 = x0; u.k_end = k_end;
  return queue_launched(fq_launch_queue_select(u, (cudaStream_t)stream));
}

extern "C" int fq_queue_pop_dev(const fq_queue* q, int n, const int* rows, const int* ticks, int max_ticks, double* goals, void* stream)
{
  if (const char* why = queue_struct(q)) return fq_fail(nullptr, FQ_E_ARG, why);
  if (n < 0 || max_ticks < 0 || (n > 0 && (!ticks || (max_ticks > 0 && !goals))))
    return fq_fail(nullptr, FQ_E_ARG, "queue: n < 0, max_ticks < 0, or ticks or goals NULL");
  FqQueueArgs u = queue_args(q, n, rows);
  u.ticks = ticks; u.max_ticks = max_ticks; u.goals = goals;
  return queue_launched(fq_launch_queue_pop(u, (cudaStream_t)stream));
}

extern "C" int fq_replan_pairs_assign_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, fq_pair_result* results_all,
                                          void* stream_v)
{
  return chain_dev(ctx, a, as, nullptr, nullptr, nullptr, results_all, stream_v);
}

extern "C" int fq_replan_pairs_window_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                          fq_pair_result* results_all, void* stream_v)
{
  if (!ctx) return FQ_E_ARG;
  if (!win) return fq_fail(ctx, FQ_E_ARG, "window is NULL");
  return chain_dev(ctx, a, as, win, nullptr, nullptr, results_all, stream_v);
}

extern "C" int fq_replan_pairs_exact_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                         const fq_pair_exact* ex, fq_pair_result* results_all, void* stream_v)
{
  if (!ctx) return FQ_E_ARG;
  if (!ex) return fq_fail(ctx, FQ_E_ARG, "exact is NULL");
  return chain_dev(ctx, a, as, win, ex, nullptr, results_all, stream_v);
}

extern "C" int fq_replan_pairs_decomp_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                          const fq_pair_exact* ex, const fq_pair_decomp* dc, fq_pair_result* results_all, void* stream_v)
{
  if (!ctx) return FQ_E_ARG;
  if (!dc) return fq_fail(ctx, FQ_E_ARG, "decomp is NULL");
  return chain_dev(ctx, a, as, win, ex, dc, results_all, stream_v);
}

extern "C" int fq_replan_pairs_hr_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                      const fq_pair_exact* ex, const fq_pair_decomp* dc, const fq_pair_hr* hr, fq_pair_result* results_all,
                                      void* stream_v)
{
  if (!ctx) return FQ_E_ARG;
  if (int rc = check_hr(ctx, win, dc, hr)) return rc;
  return chain_dev(ctx, a, as, win, ex, dc, results_all, stream_v, hr);
}

extern "C" int fq_replan_pairs_map_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                       const fq_pair_exact* ex, const fq_pair_decomp* dc, const fq_pair_hr* hr, const fq_pair_map* mp,
                                       fq_pair_result* results_all, void* stream_v)
{
  if (!ctx) return FQ_E_ARG;
  if (int rc = check_map(ctx, dc, hr, win, mp)) return rc;
  return chain_dev(ctx, a, as, win, ex, dc, results_all, stream_v, hr, mp);
}

namespace
{
// Candidate offsets of one sweep with per-corridor assignment lists, the only code that counts them: corridor j (P_j
// polytopes) has |L(N, P_j, all_limit)| candidates per factor and n_fac factors, or the |F_j| of its window (init[j],
// final_[j], inc) when init is not NULL.  Fills ofs[0 .. n_prob], *max_fac (largest |F_j|, 0 without windows) and
// *max_poly (largest P_j), and returns why the sweep is refused, or nullptr.
const char* fq_list_offsets(int n_prob, const int* poly_ofs, int N, long all_limit, int n_fac, const double* init,
                            const double* final_, double inc, std::vector<long long>* ofs, int* max_fac, int* max_poly)
{
  if (all_limit < 0) return "all_limit < 0";
  ofs->assign(n_prob + 1, 0);
  *max_fac = *max_poly = 0;
  for (int j = 0; j < n_prob; j++)
  {
    const int p = poly_ofs[j + 1] - poly_ofs[j];
    if (p > FQ_MAX_POLY) return "more than FQ_MAX_POLY polytopes in a corridor";
    const long long len = fqa::list_len(N, p, all_limit);
    if (len < 0) return "assignment list of a corridor longer than 2^20";
    const int nf = init ? fqw::factors(init[j], final_[j], inc, nullptr, 0) : n_fac;
    if (nf < 0) return "time-allocation window refused (not finite, init <= 0, more than 4096 factors or a stalled accumulation)";
    (*ofs)[j + 1] = (*ofs)[j] + len * nf;
    if ((*ofs)[j + 1] > (1LL << 30)) return "too many candidates";
    if (init) *max_fac = std::max(*max_fac, nf);
    *max_poly = std::max(*max_poly, p);
  }
  return nullptr;
}

bool scan_offsets(const int* o, int n, int max_step, int* total, int* largest)
{ // o[0] = 0 and steps of 0 .. max_step
  if (o[0] != 0) return false;
  for (int j = 0; j < n; j++)
  {
    const int d = o[j + 1] - o[j];
    if (d < 0 || d > max_step) return false;
    *largest = std::max(*largest, d);
  }
  *total = o[n];
  return true;
}

// The host-side checks of one sweep's arrays (host pointers), which also set the sizes the _dev entries take as hints:
// max_faces / max_poly_faces (a decomposing chain keeps the caller's caps), max_obs, and with per-corridor lists n_cand,
// max_fac and max_poly.  *c receives the corridors' sizes (a decomposing chain: n_poly only), *n_obs the clouds' points,
// *ofs the candidate offsets of per-corridor lists (left empty with a shared list).
const char* scan_sweep(Sweep& w, int P, const fq_pair_assign* as, const fq_pair_decomp* dc, FqCorridorSizes* c, int* n_obs,
                       std::vector<long long>* ofs)
{
  if (!dc)
  {
    if (w.poly_ofs[0] != 0 || w.face_ofs[0] != 0) return "offset arrays must start at 0";
    if (const char* why = fq_scan_corridors(P, w.poly_ofs, w.face_ofs, c)) return why;
    if (c->n_face > 0 && !w.Ab) return "polytopes given but Ab is NULL";
    if (c->n_face > 0 && !fq_scan_all_finite(w.Ab, 4 * (size_t)c->n_face)) return "non-finite value in Ab";
    if (!fq_scan_all_finite(w.xf, 9 * (size_t)P)) return "non-finite value in x0/xf";
    w.max_faces = std::max(c->max_faces, 1);
    w.max_poly_faces = c->max_poly_faces;
  }
  else
  { // polytope counts, paths and clouds
    int mp = 0;
    w.max_obs = 0;
    if (!scan_offsets(w.poly_ofs, P, FQ_MAX_POLY, &c->n_poly, &mp)) return "poly_ofs_* must start at 0 and step by 0..FQ_MAX_POLY";
    if (w.obs_ofs && !scan_offsets(w.obs_ofs, P, 1 << 30, n_obs, &w.max_obs))   // (against maps there are no clouds here)
      return "decomp: obs_ofs_* must start at 0 and be non-decreasing";
    if (!fq_scan_all_finite(w.path, 3 * (size_t)(c->n_poly + P)) || (w.obs && !fq_scan_all_finite(w.obs, 3 * (size_t)*n_obs)))
      return "decomp: non-finite value in a path, a cloud or the goal";
  }
  if (!fq_scan_all_positive_finite(w.factors, (size_t)w.n_fac)) return "limits and factors must be finite and > 0";
  for (int i = 1; i < w.n_fac; i++)
    if (w.factors[i] < w.factors[i - 1]) return "factors_* must be ascending";
  // a NULL cost/flag output still needs a device array of its own kind: the chain allocates it in its scratch
  if ((w.feasible == nullptr) != (w.cost == nullptr)) return "feasible_* and cost_* must be given (or omitted) together";
  if (as)
  {
    if (const char* why = fq_list_offsets(P, w.poly_ofs, w.N, as->all_limit, w.n_fac, w.init, w.final_, w.inc, ofs, &w.max_fac,
                                          &w.max_poly))
      return why;
    w.n_cand = (long)(*ofs)[P];
    return nullptr;
  }
  if (c->n_poly > 0 && !w.sigmas) return "sigmas_* is NULL";
  // assignments must name existing polytopes of EVERY corridor they are applied to
  int min_p = FQ_MAX_POLY;
  for (int j = 0; j < P; j++) min_p = std::min(min_p, w.poly_ofs[j + 1] - w.poly_ofs[j]);
  if (min_p > 0 && fq_scan_max_u8(w.sigmas, (size_t)w.n_sig * w.N) >= min_p) return "sigmas_* entry >= number of polytopes";
  w.n_cand = (long)P * w.n_fac * w.n_sig;
  return nullptr;
}

// A submission checked against the caller's host arrays: its two sweeps, sized by scan_sweep, their corridors' sizes and
// clouds' points, the unknown clouds' points, and with per-corridor lists each sweep's candidate offsets
struct Checked
{
  Sweep sw[2];
  FqCorridorSizes cs[2];
  int n_obs[2] = { 0, 0 };
  int n_unk = 0;
  std::vector<long long> cand_ofs[2];
};

// Every check of a host-pointer submission: everything that reads the caller's host memory and can refuse.  It writes
// nothing but *k, so a refused submission leaves every output as it was.
int check_host(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win, const fq_pair_exact* ex,
               const fq_pair_decomp* dc, const fq_pair_hr* hr, const fq_pair_map* mp, Checked* k)
{
  if (int rc = check_chain(ctx, a, as, win, ex, dc, k->sw, mp)) return rc;
  const int P = a->n_prob;
  if (!fq_scan_all_finite(a->x0, 9 * (size_t)P)) return fq_fail(ctx, FQ_E_ARG, "non-finite value in x0/xf");
  if (!fq_scan_all_positive_finite(a->lim, 3 * (size_t)P)) return fq_fail(ctx, FQ_E_ARG, "limits and factors must be finite and > 0");
  if (dc && dc->goal && !fq_scan_all_finite(dc->goal, 3 * (size_t)P))
    return fq_fail(ctx, FQ_E_ARG, "decomp: non-finite value in a path, a cloud or the goal");
  if (mp)
  {
    if (int rc = check_map(ctx, dc, hr, win, mp)) return rc;
    for (int j = 0; mp->map_index && j < P; j++)
      if (mp->map_index[j] < 0 || mp->map_index[j] >= mp->n_maps) return fq_fail(ctx, FQ_E_ARG, "map: map_index out of range");
  }
  else if (hr)
  {
    int largest_unk = 0;
    if (int rc = check_hr(ctx, win, dc, hr)) return rc;
    if (!scan_offsets(hr->unk_ofs, P, 1 << 30, &k->n_unk, &largest_unk)) return fq_fail(ctx, FQ_E_ARG, "hr: unk_ofs must start at 0 and be non-decreasing");
    if (!fq_scan_all_finite(hr->unk, 3 * (size_t)k->n_unk)) return fq_fail(ctx, FQ_E_ARG, "hr: non-finite value in an unknown cloud");
  }
  for (int i = 0; i < 2; i++)
    if (const char* why = scan_sweep(k->sw[i], P, as, dc, &k->cs[i], &k->n_obs[i], &k->cand_ofs[i])) return fq_fail(ctx, FQ_E_ARG, why);
  return 0;
}

// A checked submission onto the device and back: one packed upload, the chain (through the _dev entry of its kind), the
// outputs straight into the caller's arrays.  d_results (may be NULL) receives the device address of the result records;
// copy_results = false leaves the caller's `results` untouched (the sharded chain reads the all-gathered table instead).
int submit_host(fq_ctx* ctx, const Checked& k, const fq_pair_args* a, bool deferred, fq_pair_result** d_results, bool copy_results,
                const fq_pair_assign* as, const fq_pair_window* win, const fq_pair_exact* ex, const fq_pair_decomp* dc,
                const fq_pair_hr* hr, const fq_pair_map* mp, const fq_pair_plan* pl = nullptr, const fq_pair_queue* qu = nullptr)
{
  const int P = a->n_prob, n_unk = k.n_unk;
  const Sweep* sw = k.sw;
  const FqCorridorSizes* cs = k.cs;
  const int* n_obs = k.n_obs;
  FQ_CUDA(cudaSetDevice(ctx->device));
  // ---- one packed upload of the inputs (pi) and, after it in d_pair_io, one block for the outputs (po).  stage() runs
  //      twice: to size them, then to copy the inputs into the pinned staging buffer and point the device copies of the
  //      structs at both
  fq_pair_args d = *a;
  fq_pair_assign da{};
  fq_pair_window dw{};
  fq_pair_exact dx{};
  fq_pair_decomp dd = dc ? *dc : fq_pair_decomp{};
  fq_pair_hr dh = hr ? *hr : fq_pair_hr{};
  fq_pair_map dm = mp ? *mp : fq_pair_map{};
  fq_pair_plan dp = pl ? *pl : fq_pair_plan{};
  fq_pair_queue du = qu ? *qu : fq_pair_queue{};
  const size_t ring_n = qu ? (size_t)qu->ring.n_rows * qu->ring.cap * fqq::kState : 0;
  if (as) da.all_limit = as->all_limit;
  Sweep dv[2];
  FqPack pi, po;
  // f(the caller's array, its device copy, elements) for every output of sweep i
  auto each_output = [&](int i, auto&& f) {
    const Sweep& w = sw[i];
    Sweep& v = dv[i];
    const size_t nc = (size_t)w.n_cand, NP = (size_t)w.N * P;
    f(w.coeffs, v.coeffs, 12 * NP);  f(w.cost, v.cost, nc);  f(w.feasible, v.feasible, nc);
    f(w.cand_ofs_out, v.cand_ofs_out, P + 1);  f(w.sigma_out, v.sigma_out, NP);
    f(w.factor, v.factor, P);  f(w.trials, v.trials, P);  f(w.next_init, v.next_init, P);  f(w.next_final, v.next_final, P);
    f(w.exact, v.exact, P);  f(w.nodes, v.nodes, P);
    f(w.face_ofs_out, v.face_ofs_out, cs[i].n_poly + 1);  f(w.Ab_out, v.Ab_out, 4 * (size_t)P * w.max_faces);
    f(w.pos_out, v.pos_out, 3 * P);  f(w.status, v.status, P);
  };
  auto stage = [&] {
    d.x0 = pi.in(a->x0, 9 * (size_t)P);
    d.lim = pi.in(a->lim, 3 * (size_t)P);
    d.results = po.out(a->results, P);
    if (dc) dd.goal = pi.in(dc->goal, 3 * (size_t)P);
    if (mp) dm.map_index = pi.in(mp->map_index, P);
    if (hr)
    { // last_factor_safe is updated in its uploaded copy, which goes back to the caller's array
      dh.unk_ofs = pi.in(hr->unk_ofs, P + 1);  dh.unk = pi.in(hr->unk, 3 * (size_t)n_unk);
      dh.last_factor_safe = pi.in(hr->last_factor_safe, P);
      dh.index_H = po.out(hr->index_H, P);  dh.need_safe = po.out(hr->need_safe, P);
    }
    if (pl)
    {
      dp.states = po.out(pl->states, 12 * (size_t)pl->cap_states);
      dp.plan_ofs = po.out(pl->plan_ofs, P + 1);  dp.status = po.out(pl->status, P);
    }
    if (qu)
    { // the rings and k_end are updated in their uploaded copies, which go back to the caller's arrays
      du.ring.states = pi.in(qu->ring.states, ring_n);
      du.ring.head = pi.in(qu->ring.head, qu->ring.n_rows);  du.ring.size = pi.in(qu->ring.size, qu->ring.n_rows);
      du.rows = pi.in(qu->rows, P);  du.k_end = pi.in(qu->k_end, P);  du.G_term = pi.in(qu->G_term, 3 * (size_t)P);
      du.status = po.out(qu->status, P);  du.goal_seen = po.out(qu->goal_seen, P);
    }
    for (int i = 0; i < 2; i++)
    {
      const Sweep& w = sw[i];
      Sweep& v = dv[i];
      v = w;
      v.xf = pi.in(w.xf, 9 * (size_t)P);  v.poly_ofs = pi.in(w.poly_ofs, P + 1);  v.face_ofs = pi.in(w.face_ofs, cs[i].n_poly + 1);
      v.Ab = pi.in(w.Ab, 4 * (size_t)cs[i].n_face);  v.factors = pi.in(w.factors, w.n_fac);  v.sigmas = pi.in(w.sigmas, (size_t)w.n_sig * w.N);
      v.init = pi.in(w.init, P);  v.final_ = pi.in(w.final_, P);
      v.path = pi.in(w.path, 3 * (size_t)(cs[i].n_poly + P));  v.obs_ofs = pi.in(w.obs_ofs, P + 1);  v.obs = pi.in(w.obs, 3 * (size_t)n_obs[i]);
      each_output(i, [&](auto* host, auto*& dev, size_t n) { dev = po.out(host, n); });
    }
  };
  stage();
  FQ_CUDA(ctx->h_in.reserve(pi.at));
  FQ_CUDA(ctx->d_pair_io.reserve(pi.at + po.at));
  pi = pi.place(ctx->d_pair_io.p, ctx->h_in.p);
  po = po.place((char*)ctx->d_pair_io.p + pi.sized);
  stage();
  if (int rc = pi.done(ctx)) return rc;
  if (int rc = po.done(ctx)) return rc;
  cudaStream_t st = ctx->stream;
  FQ_CUDA(cudaMemcpyAsync(pi.base, pi.host, pi.at, cudaMemcpyHostToDevice, st));
  for (int i = 0; i < 2; i++) put_sweep(dv[i], i, &d, &da, &dw, &dx, &dd);
  int rc = family_dev(ctx, &d, as ? &da : nullptr, win ? &dw : nullptr, ex ? &dx : nullptr, dc ? &dd : nullptr, hr ? &dh : nullptr,
                      mp ? &dm : nullptr, pl ? &dp : nullptr, nullptr, st, qu ? &du : nullptr);
  if (rc) return rc;
  // ---- results straight into the caller's arrays (asynchronous when they are pinned).  The caller's window arrays were
  //      copied into the upload above, so the next_* outputs may alias them.
  if (d_results) *d_results = d.results;
  if (copy_results) FQ_CUDA(cudaMemcpyAsync(a->results, d.results, sizeof(fq_pair_result) * (size_t)P, cudaMemcpyDeviceToHost, st));
  cudaError_t e = cudaSuccess;
  for (int i = 0; i < 2; i++)
    each_output(i, [&](auto* host, auto*& dev, size_t n) {
      if (host && e == cudaSuccess) e = cudaMemcpyAsync(host, dev, sizeof(*host) * n, cudaMemcpyDeviceToHost, st);
    });
  FQ_CUDA(e);
  if (hr)
  {
    if (hr->last_factor_safe) FQ_CUDA(cudaMemcpyAsync(hr->last_factor_safe, dh.last_factor_safe, sizeof(double) * P, cudaMemcpyDeviceToHost, st));
    if (hr->index_H) FQ_CUDA(cudaMemcpyAsync(hr->index_H, dh.index_H, sizeof(int) * P, cudaMemcpyDeviceToHost, st));
    if (hr->need_safe) FQ_CUDA(cudaMemcpyAsync(hr->need_safe, dh.need_safe, P, cudaMemcpyDeviceToHost, st));
  }
  if (pl)
  {
    FQ_CUDA(cudaMemcpyAsync(pl->plan_ofs, dp.plan_ofs, sizeof(long long) * (size_t)(P + 1), cudaMemcpyDeviceToHost, st));
    if (pl->status) FQ_CUDA(cudaMemcpyAsync(pl->status, dp.status, sizeof(int) * (size_t)P, cudaMemcpyDeviceToHost, st));
    if (deferred && pl->cap_states > 0)      // the rows' total is not known yet: all cap_states rows
      FQ_CUDA(cudaMemcpyAsync(pl->states, dp.states, sizeof(double) * 12 * (size_t)pl->cap_states, cudaMemcpyDeviceToHost, st));
  }
  if (qu)
  {
    FQ_CUDA(cudaMemcpyAsync(qu->ring.states, du.ring.states, sizeof(double) * ring_n, cudaMemcpyDeviceToHost, st));
    FQ_CUDA(cudaMemcpyAsync(qu->ring.size, du.ring.size, sizeof(int) * (size_t)qu->ring.n_rows, cudaMemcpyDeviceToHost, st));
    FQ_CUDA(cudaMemcpyAsync(qu->k_end, du.k_end, sizeof(int) * (size_t)P, cudaMemcpyDeviceToHost, st));
    FQ_CUDA(cudaMemcpyAsync(qu->status, du.status, sizeof(int) * (size_t)P, cudaMemcpyDeviceToHost, st));
    if (qu->goal_seen) FQ_CUDA(cudaMemcpyAsync(qu->goal_seen, du.goal_seen, (size_t)P, cudaMemcpyDeviceToHost, st));
  }
  if (deferred) { ctx->pending = true; return 0; }
  FQ_CUDA(cudaStreamSynchronize(st));
  if (pl)
  { // only the rows of the corridors that fit: those before the first FQ_PLAN_CAPACITY corridor
    long long rows = 0;
    for (int j = 0; j <= P; j++)
      if (pl->plan_ofs[j] <= pl->cap_states) rows = pl->plan_ofs[j];
    if (rows > 0)
    {
      FQ_CUDA(cudaMemcpyAsync(pl->states, dp.states, sizeof(double) * 12 * (size_t)rows, cudaMemcpyDeviceToHost, st));
      FQ_CUDA(cudaStreamSynchronize(st));
    }
  }
  return 0;
}

// a host-pointer chain on one GPU.  The context settles before the check: a deferred call may still be copying into
// arrays this one reads (a window's next_* passed on as the next init_* / final_*).
int host_chain(fq_ctx* ctx, const fq_pair_args* a, bool deferred, fq_pair_result** d_results, bool copy_results,
               const fq_pair_assign* as = nullptr, const fq_pair_window* win = nullptr, const fq_pair_exact* ex = nullptr,
               const fq_pair_decomp* dc = nullptr, const fq_pair_hr* hr = nullptr, const fq_pair_map* mp = nullptr,
               const fq_pair_plan* pl = nullptr, const fq_pair_queue* qu = nullptr)
{
  if (!ctx) return FQ_E_ARG;
  if (int rc = fq_settle(ctx)) return rc;
  Checked k;
  if (int rc = check_host(ctx, a, as, win, ex, dc, hr, mp, &k)) return rc;
  if (qu)
    if (const char* why = queue_rows(&qu->ring, a->n_prob, qu->rows, true, true)) return fq_fail(ctx, FQ_E_ARG, why);
  return submit_host(ctx, k, a, deferred, d_results, copy_results, as, win, ex, dc, hr, mp, pl, qu);
}

// checked sweep w cut to the corridors [lo, hi) (ofs: its candidate offsets, empty with a shared list): corridor offsets
// rebased into *sub, per-corridor arrays from corridor lo, per-candidate outputs from the shard's first candidate.  The
// candidate offsets are not the shard's to write.  The exact and decomposing fields are not cut: those chains are refused
// on multi-GPU contexts (lists_host), so they are NULL here.
Sweep cut_sweep(Sweep w, const std::vector<long long>& ofs, int lo, int hi, FqSubCorridors* sub)
{
  sub->build(w.poly_ofs, w.face_ofs, w.Ab, lo, hi);
  w.poly_ofs = sub->poly_ofs.data();  w.face_ofs = sub->face_ofs.data();  w.Ab = sub->Ab;
  const size_t j = (size_t)lo, NP = (size_t)w.N * lo, c0 = ofs.empty() ? (size_t)w.n_fac * w.n_sig * lo : (size_t)ofs[lo];
  auto at = [](auto* p, size_t o) { return p ? p + o : p; };
  w.xf = at(w.xf, 9 * j);  w.coeffs = at(w.coeffs, 12 * NP);  w.sigma_out = at(w.sigma_out, NP);
  w.feasible = at(w.feasible, c0);  w.cost = at(w.cost, c0);
  w.init = at(w.init, j);  w.final_ = at(w.final_, j);  w.factor = at(w.factor, j);  w.trials = at(w.trials, j);
  w.next_init = at(w.next_init, j);  w.next_final = at(w.next_final, j);
  w.cand_ofs_out = nullptr;
  return w;
}

// one shard of a sharded call: its structs (pointing into the caller's arrays and the rebased offsets) and its check
struct Shard
{
  fq_pair_args a{};
  fq_pair_assign as{};
  fq_pair_window win{};
  FqSubCorridors sub[2];
  Checked k;
};

// The chain on a multi-GPU context (fq_replan_pairs*, _assign*, _window*).  Group (one process): corridors [lo_i, hi_i) go
// to member i, every member runs its chain, the result records are all-gathered (padded to the largest shard) and read
// back once from member 0; the per-candidate arrays travel straight from each member into the caller's arrays.  Rank
// context (one process per GPU): every rank passes the SAME full description and solves its own shard; after the
// all-gather every rank holds every corridor's result record, while per-candidate outputs are filled for the rank's own
// corridors only.
// Nothing is written or enqueued before two checks pass, on every rank alike.  The whole description is checked as a
// plain context checks it, so what a plain context refuses is refused with the same message.  Then every shard of the
// world is cut and checked, which also sizes it as the same batch on one GPU.  A shard's check is not always implied by
// the whole one: a shared list may name a polytope a corridor lacks when some corridor of the batch has none (the bound
// is then skipped), so corridors with P = {0, 1} and the entry 1 pass as a whole but not as the shard [1, 2).  Checking
// every shard on every rank keeps the ranks' decisions equal even then.
// Shared lists: equal corridor counts per shard.  Per-corridor lists: the shards are balanced by candidates (fq_shard_range
// over the summed whole + safe offsets), and each shard's per-candidate outputs start at its first offset.
int sharded_chain(fq_ctx* g, const fq_pair_args* a, bool deferred, const fq_pair_assign* as, const fq_pair_window* win)
{
  fq_ctx* ctx = g;
  if (int rc = fq_settle(g)) return rc;            // every member (see host_chain)
  Checked k;
  if (int rc = check_host(g, a, as, win, nullptr, nullptr, nullptr, nullptr, &k)) return rc;
  const int P = a->n_prob, world = g->world;
  const bool group = g->is_group;
  const int n_local = group ? world : 1;
  std::vector<int> weight;
  if (as)
  {
    weight.assign(P + 1, 0);
    for (int j = 1; j <= P; j++) weight[j] = (int)std::min<long long>(k.cand_ofs[0][j] + k.cand_ofs[1][j], 0x7fffffffLL);
  }
  int pad = 0;
  std::vector<int> lo(world), hi(world);
  std::vector<Shard> shard(world);
  for (int r = 0; r < world; r++)
  {
    fq_shard_range(P, as ? weight.data() : nullptr, r, world, &lo[r], &hi[r]);
    pad = std::max(pad, hi[r] - lo[r]);
    if (hi[r] <= lo[r]) continue;
    Shard& s = shard[r];
    s.a = *a;
    s.a.n_prob = hi[r] - lo[r];  s.a.x0 = a->x0 + 9 * (size_t)lo[r];  s.a.lim = a->lim + 3 * (size_t)lo[r];
    s.a.results = a->results + lo[r];           // not copied back (copy_results = false): the gathered table is
    if (as) s.as = *as;
    if (win) s.win = *win;
    for (int h = 0; h < 2; h++)
      put_sweep(cut_sweep(k.sw[h], k.cand_ofs[h], lo[r], hi[r], &s.sub[h]), h, &s.a, as ? &s.as : nullptr, win ? &s.win : nullptr,
                nullptr, nullptr);
    if (int rc = check_host(g, &s.a, as ? &s.as : nullptr, win ? &s.win : nullptr, nullptr, nullptr, nullptr, nullptr, &s.k)) return rc;
  }
  for (int i = 0; as && i < 2; i++)
    for (int j = 0; k.sw[i].cand_ofs_out && j <= P; j++) k.sw[i].cand_ofs_out[j] = (int)k.cand_ofs[i][j];
  std::vector<void*> d_res(n_local, nullptr), d_all(n_local, nullptr);
  for (int i = 0; i < n_local; i++)
  {
    fq_ctx* c = group ? fq_member(g, i) : g;
    const int r = group ? i : g->rank;
    cudaSetDevice(c->device);
    // gather buffers: [pad records to send | world x pad records received]
    cudaError_t e = c->d_out.reserve(sizeof(fq_pair_result) * (size_t)pad * (world + 1));
    if (e != cudaSuccess) return fq_cuda_fail(g, e, "gather buffer");
    fq_pair_result* res = (fq_pair_result*)c->d_out.p;
    d_res[i] = res;
    d_all[i] = res + pad;
    e = cudaMemsetAsync(res, 0xff, sizeof(fq_pair_result) * (size_t)pad, c->stream);
    if (e != cudaSuccess) return fq_cuda_fail(g, e, "gather buffer");
    if (hi[r] <= lo[r]) continue;
    Shard& s = shard[r];
    fq_pair_result* dr = nullptr;
    int rc = submit_host(c, s.k, &s.a, true, &dr, false, as ? &s.as : nullptr, win ? &s.win : nullptr, nullptr, nullptr, nullptr, nullptr);
    if (rc) { if (c != g) g->err = c->err; return rc; }
    e = cudaMemcpyAsync(res, dr, sizeof(fq_pair_result) * (size_t)s.a.n_prob, cudaMemcpyDeviceToDevice, c->stream);
    if (e != cudaSuccess) return fq_cuda_fail(g, e, "gather staging");
  }
  if (int rc = fq_exchange(g, d_res, d_all, sizeof(fq_pair_result) * (size_t)pad)) return rc;
  // ---- the gathered table, shard by shard, into the caller's results (from member 0 / this rank)
  FQ_CUDA(cudaSetDevice(g->device));
  const fq_pair_result* all = (const fq_pair_result*)d_all[0];
  for (int r = 0; r < world; r++)
    if (hi[r] > lo[r])
      FQ_CUDA(cudaMemcpyAsync(a->results + lo[r], all + (size_t)r * pad, sizeof(fq_pair_result) * (size_t)(hi[r] - lo[r]),
                              cudaMemcpyDeviceToHost, g->stream));
  g->pending = true;
  if (deferred) return 0;
  return fq_settle(g);
}
}  // namespace

extern "C" int fq_replan_pairs(fq_ctx* ctx, const fq_pair_args* a)
{
  if (ctx && (ctx->is_group || ctx->comm)) return sharded_chain(ctx, a, false, nullptr, nullptr);
  return host_chain(ctx, a, false, nullptr, true);
}
extern "C" int fq_replan_pairs_async(fq_ctx* ctx, const fq_pair_args* a)
{
  if (ctx && (ctx->is_group || ctx->comm)) return sharded_chain(ctx, a, true, nullptr, nullptr);
  return host_chain(ctx, a, true, nullptr, true);
}

namespace
{
// the host entries with per-corridor lists.  A multi-GPU context shards _assign and _window; the exact and decomposing
// chains run on one GPU only, since gathering their per-corridor exact / nodes / corridor arrays would need a second
// exchange besides the records'.
int lists_host(fq_ctx* ctx, const fq_pair_args* a, bool deferred, const fq_pair_assign* as, const fq_pair_window* win,
               const fq_pair_exact* ex = nullptr, const fq_pair_decomp* dc = nullptr, const fq_pair_hr* hr = nullptr,
               const fq_pair_map* mp = nullptr, const fq_pair_plan* pl = nullptr, const fq_pair_queue* qu = nullptr)
{
  if (!as) return fq_fail(ctx, FQ_E_ARG, "assign is NULL");
  if ((ex || dc) && (ctx->is_group || ctx->comm))
    return fq_fail(ctx, FQ_E_ARG, "fq_replan_pairs_exact / _decomp / _hr / _map: multi-GPU contexts are not supported (use the _dev entry)");
  if (ctx->is_group || ctx->comm) return sharded_chain(ctx, a, deferred, as, win);
  return host_chain(ctx, a, deferred, nullptr, true, as, win, ex, dc, hr, mp, pl, qu);
}

// fq_replan_pairs_plan / _async: the plan's refusals (multi-GPU contexts among them, so nothing here is sharded), then the
// host entry of the family the structs select, with its own checks in its own order
// (fq_replan_pairs_queue / _async: the same with the queue's refusals instead of the plan's)
int plan_host(fq_ctx* ctx, const fq_pair_args* a, bool deferred, const fq_pair_assign* as, const fq_pair_window* win,
              const fq_pair_exact* ex, const fq_pair_decomp* dc, const fq_pair_hr* hr, const fq_pair_map* mp, const fq_pair_plan* pl,
              const fq_pair_queue* qu = nullptr)
{
  if (!ctx) return FQ_E_ARG;
  if (int rc = qu ? check_queue(ctx, qu) : check_plan(ctx, pl)) return rc;
  if (!as)
  {
    if (win || ex || dc || hr || mp) return fq_fail(ctx, FQ_E_ARG, "assign is NULL");
    return host_chain(ctx, a, deferred, nullptr, true, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, pl, qu);
  }
  if (hr && !mp)
    if (int rc = check_hr(ctx, win, dc, hr)) return rc;
  return lists_host(ctx, a, deferred, as, win, ex, dc, hr, mp, pl, qu);
}
}  // namespace

extern "C" int fq_replan_pairs_plan(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                    const fq_pair_exact* ex, const fq_pair_decomp* dc, const fq_pair_hr* hr, const fq_pair_map* mp,
                                    const fq_pair_plan* pl)
{
  return plan_host(ctx, a, false, as, win, ex, dc, hr, mp, pl);
}
extern "C" int fq_replan_pairs_plan_async(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                          const fq_pair_exact* ex, const fq_pair_decomp* dc, const fq_pair_hr* hr,
                                          const fq_pair_map* mp, const fq_pair_plan* pl)
{
  return plan_host(ctx, a, true, as, win, ex, dc, hr, mp, pl);
}

extern "C" int fq_replan_pairs_queue(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                     const fq_pair_exact* ex, const fq_pair_decomp* dc, const fq_pair_hr* hr, const fq_pair_map* mp,
                                     const fq_pair_queue* qu)
{
  if (!ctx) return FQ_E_ARG;
  if (int rc = check_queue(ctx, qu)) return rc;
  return plan_host(ctx, a, false, as, win, ex, dc, hr, mp, nullptr, qu);
}
extern "C" int fq_replan_pairs_queue_async(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                           const fq_pair_exact* ex, const fq_pair_decomp* dc, const fq_pair_hr* hr,
                                           const fq_pair_map* mp, const fq_pair_queue* qu)
{
  if (!ctx) return FQ_E_ARG;
  if (int rc = check_queue(ctx, qu)) return rc;
  return plan_host(ctx, a, true, as, win, ex, dc, hr, mp, nullptr, qu);
}

extern "C" int fq_replan_pairs_assign(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as)
{
  return ctx ? lists_host(ctx, a, false, as, nullptr) : FQ_E_ARG;
}
extern "C" int fq_replan_pairs_assign_async(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as)
{
  return ctx ? lists_host(ctx, a, true, as, nullptr) : FQ_E_ARG;
}

extern "C" int fq_replan_pairs_window(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win)
{
  if (!ctx) return FQ_E_ARG;
  return win ? lists_host(ctx, a, false, as, win) : fq_fail(ctx, FQ_E_ARG, "window is NULL");
}
extern "C" int fq_replan_pairs_window_async(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win)
{
  if (!ctx) return FQ_E_ARG;
  return win ? lists_host(ctx, a, true, as, win) : fq_fail(ctx, FQ_E_ARG, "window is NULL");
}

extern "C" int fq_replan_pairs_exact(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                     const fq_pair_exact* ex)
{
  if (!ctx) return FQ_E_ARG;
  return ex ? lists_host(ctx, a, false, as, win, ex) : fq_fail(ctx, FQ_E_ARG, "exact is NULL");
}
extern "C" int fq_replan_pairs_exact_async(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                           const fq_pair_exact* ex)
{
  if (!ctx) return FQ_E_ARG;
  return ex ? lists_host(ctx, a, true, as, win, ex) : fq_fail(ctx, FQ_E_ARG, "exact is NULL");
}

extern "C" int fq_replan_pairs_decomp(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                      const fq_pair_exact* ex, const fq_pair_decomp* dc)
{
  if (!ctx) return FQ_E_ARG;
  return dc ? lists_host(ctx, a, false, as, win, ex, dc) : fq_fail(ctx, FQ_E_ARG, "decomp is NULL");
}
extern "C" int fq_replan_pairs_decomp_async(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                            const fq_pair_exact* ex, const fq_pair_decomp* dc)
{
  if (!ctx) return FQ_E_ARG;
  return dc ? lists_host(ctx, a, true, as, win, ex, dc) : fq_fail(ctx, FQ_E_ARG, "decomp is NULL");
}

extern "C" int fq_replan_pairs_hr(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                  const fq_pair_exact* ex, const fq_pair_decomp* dc, const fq_pair_hr* hr)
{
  if (!ctx) return FQ_E_ARG;
  if (int rc = check_hr(ctx, win, dc, hr)) return rc;
  return lists_host(ctx, a, false, as, win, ex, dc, hr);
}
extern "C" int fq_replan_pairs_hr_async(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                        const fq_pair_exact* ex, const fq_pair_decomp* dc, const fq_pair_hr* hr)
{
  if (!ctx) return FQ_E_ARG;
  if (int rc = check_hr(ctx, win, dc, hr)) return rc;
  return lists_host(ctx, a, true, as, win, ex, dc, hr);
}

extern "C" int fq_replan_pairs_map(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                   const fq_pair_exact* ex, const fq_pair_decomp* dc, const fq_pair_hr* hr, const fq_pair_map* mp)
{
  if (!ctx) return FQ_E_ARG;
  if (!mp) return fq_fail(ctx, FQ_E_ARG, "map is NULL");
  return lists_host(ctx, a, false, as, win, ex, dc, hr, mp);
}
extern "C" int fq_replan_pairs_map_async(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                         const fq_pair_exact* ex, const fq_pair_decomp* dc, const fq_pair_hr* hr, const fq_pair_map* mp)
{
  if (!ctx) return FQ_E_ARG;
  if (!mp) return fq_fail(ctx, FQ_E_ARG, "map is NULL");
  return lists_host(ctx, a, true, as, win, ex, dc, hr, mp);
}
