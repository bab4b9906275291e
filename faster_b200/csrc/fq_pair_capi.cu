// Chained replan (include/faster_b200.h: fq_replan_pairs*): whole sweep -> selection -> R -> safe sweep -> selection for
// many corridors in one submission.  Reference data flow: faster/src/faster.cpp:406-430 (whole), :474-475 (R), :521-537
// (safe).  Kernels: the batch solve (fq_kernels_t.cuh) and the small kernels of fq_pair.cuh.
#include "fq_assign.h"
#include "fq_ctx.h"
#include "fq_window.h"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace
{
struct Scratch
{ // intermediate arrays of one chain, carved from ctx->d_pair
  double *dt_w, *dt_s, *dt_base_w, *dt_base_s, *win_cost_w, *win_cost_s, *win_dt_w, *win_dt_s, *x0_safe, *coeffs_w, *coeffs_s,
      *cost_w, *cost_s, *re_cost;
  uint8_t *sig_w, *sig_s, *win_sig_w, *win_sig_s, *feas_w, *feas_s, *re_feas;
  int *cand_ofs_w, *cand_ofs_s, *win_idx_w, *win_idx_s, *win_ofs, *n_samples, *k_safe;
  double *fac_w, *fac_s;                // per-corridor windows: n_prob x max_fac factor rows
  int *nf_w, *nf_s;                     // and |F_j| (-1: refused)
  // decomposing chain: both sweeps' staging and spill (used one sweep after the other), the corridors, the final states
  double *dc_stage, *dc_spill, *dc_Ab_w, *dc_Ab_s, *dc_xf_w, *dc_xf_s;
  int *dc_stage_n, *dc_face_w, *dc_face_s;
  uint8_t* dc_spill_flag;
};

template <class T>
T* carve(char*& p, size_t count)
{
  T* r = reinterpret_cast<T*>(p);
  p += fq_align16(sizeof(T) * count);
  return r;
}

// shared = false: per-corridor lists (fq_replan_pairs_assign*), whose candidate counts the callers check themselves;
// windows = true (with shared = false): per-corridor windows (fq_replan_pairs_window*), no factor list in `a`;
// decomp = true: the chain decomposes the corridors (fq_replan_pairs_decomp*), so `a` has no faces and no final states
int check_common(fq_ctx* ctx, const fq_pair_args* a, bool shared = true, bool windows = false, bool decomp = false)
{
  if (!a) return fq_fail(ctx, FQ_E_ARG, "args is NULL");
  if (a->n_prob <= 0) return fq_fail(ctx, FQ_E_ARG, "n_prob <= 0");
  if (a->N_whole < 3 || a->N_whole > FQ_MAX_N || a->N_safe < 2 || a->N_safe > FQ_MAX_N) return fq_fail(ctx, FQ_E_ARG, "N out of range");
  if (!(a->DC > 0) || !(a->r_fraction >= 0 && a->r_fraction <= 1)) return fq_fail(ctx, FQ_E_ARG, "DC must be > 0 and r_fraction in [0, 1]");
  if (!shared)
  {
    if (windows && (a->factors_whole || a->factors_safe || a->n_fac_whole != 0 || a->n_fac_safe != 0))
      return fq_fail(ctx, FQ_E_ARG, "per-corridor windows: factors_* must be NULL and n_fac_* 0");
    if (!windows && (a->n_fac_whole <= 0 || a->n_fac_safe <= 0)) return fq_fail(ctx, FQ_E_ARG, "empty factor grid");
    if (a->sigmas_whole || a->sigmas_safe || a->n_sig_whole != 0 || a->n_sig_safe != 0)
      return fq_fail(ctx, FQ_E_ARG, "per-corridor assignment lists: sigmas_* must be NULL and n_sig_* 0");
  }
  else if (a->n_fac_whole <= 0 || a->n_fac_safe <= 0 || a->n_sig_whole <= 0 || a->n_sig_safe <= 0)
    return fq_fail(ctx, FQ_E_ARG, "empty factor / assignment grid");
  if (shared &&
      ((long long)a->n_prob * a->n_fac_whole * a->n_sig_whole > (1LL << 30) || (long long)a->n_prob * a->n_fac_safe * a->n_sig_safe > (1LL << 30)))
    return fq_fail(ctx, FQ_E_ARG, "too many candidates");
  if (decomp && (a->face_ofs_whole || a->face_ofs_safe || a->Ab_whole || a->Ab_safe || a->xf_whole || a->xf_safe))
    return fq_fail(ctx, FQ_E_ARG, "decomposing chain: face_ofs_*, Ab_* and xf_* must be NULL (the chain makes them)");
  if (decomp && (a->max_faces_whole <= 0 || a->max_faces_safe <= 0 || a->max_poly_faces_whole <= 0 || a->max_poly_faces_safe <= 0))
    return fq_fail(ctx, FQ_E_ARG, "decomposing chain: max_faces_* and max_poly_faces_* are caps and must be > 0");
  if (!a->x0 || (!decomp && (!a->xf_whole || !a->xf_safe || !a->face_ofs_whole || !a->face_ofs_safe)) || !a->lim || !a->poly_ofs_whole ||
      !a->poly_ofs_safe || (!windows && (!a->factors_whole || !a->factors_safe)) || !a->results)
    return fq_fail(ctx, FQ_E_ARG, "NULL argument");
  return 0;
}

// the assignment lists of one chain: one shared list per sweep (fq_replan_pairs*), or a list per corridor generated on the
// device (fq_replan_pairs_assign*)
struct Lists
{
  const fq_pair_assign* as = nullptr;   // per-corridor lists (outputs are device pointers), or nullptr: fq_pair_args' lists
  size_t ncw = 0, ncs = 0;              // candidates of the whole / safe sweep
  int mcw = 0, mcs = 0;                 // largest candidate count of one corridor
  int eew = 0, ees = 0;                 // candidates per time allocation (sizes an early-exit grid): the longest list
  const fq_pair_window* win = nullptr;  // per-corridor windows (device pointers; needs `as`), or nullptr
  int mfw = 0, mfs = 0;                 // with `win`: the factor rows' length (largest |F_j| allowed)
  const fq_pair_exact* ex = nullptr;    // exact stage after each sweep's selection (device pointers; needs `as`), or nullptr
  const fq_pair_decomp* dc = nullptr;   // the chain decomposes the corridors (device pointers; needs `as`), or nullptr
};

// the checks of fq_pair_decomp that need no device memory
const char* check_decomp_scalars(const fq_pair_decomp* d)
{
  if (!d) return "decomp is NULL";
  if (!d->path_whole || !d->path_safe || !d->obs_ofs_whole || !d->obs_ofs_safe || !d->obs_whole || !d->obs_safe)
    return "decomp: path_* / obs_ofs_* / obs_* must not be NULL";
  for (int k = 0; k < 3; k++)
    if (!std::isfinite(d->bbox[k]) || !(d->bbox[k] > 0)) return "decomp: bbox must be finite and > 0";
  if (!std::isfinite(d->inflate) || d->inflate < 0 || !std::isfinite(d->z_ground)) return "decomp: inflate must be finite and >= 0, z_ground finite";
  if (((uintptr_t)d->Ab_whole & 15) || ((uintptr_t)d->Ab_safe & 15)) return "decomp: Ab_* must be 16-byte aligned";
  return nullptr;
}

// Exact stage (fq_replan_pairs_exact*): node pools, leaves and per-corridor tree state, carved from ctx->d_bnb.  Corridor c
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

size_t tree_layout(char* base, int n_prob, int stride, int max_N, size_t nb, Tree* t)
{
  char* p = base;
  const size_t np = (size_t)n_prob, cells = np * (size_t)std::max(stride, 1);
  t->dts = carve<double>(p, cells);  t->incumbent = carve<unsigned long long>(p, cells);  t->roots = carve<int>(p, cells);
  t->lbound = carve<unsigned long long>(p, cells);  t->closed = carve<uint8_t>(p, cells);
  t->keep_idx = carve<int>(p, np);  t->keep_cost = carve<double>(p, np);  t->keep_dt = carve<double>(p, np);
  t->keep_sig = carve<uint8_t>(p, np * max_N);  t->redo_dt = carve<double>(p, np);  t->redo_coeffs = carve<double>(p, np * 12 * max_N);
  t->n_par = carve<int>(p, 2 * np);  t->n_leaves = carve<int>(p, np);  t->flags = carve<int>(p, 2 * np);
  t->nodes = carve<long long>(p, np);
  t->status = carve<uint8_t>(p, np); t->changed_w = carve<uint8_t>(p, np);  t->changed_s = carve<uint8_t>(p, np);
  t->leaves = carve<char>(p, np * kLeafCap * 32);
  t->pool0 = carve<unsigned char>(p, np * tree_cap(n_prob) * nb);
  t->pool1 = carve<unsigned char>(p, np * tree_cap(n_prob) * nb);
  return (size_t)(p - base);
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

// the hints of fq_pair_assign for the _dev entries -> the longest list of each sweep
int check_assign_hints(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, long long* lw, long long* ls)
{
  if (!as) return fq_fail(ctx, FQ_E_ARG, "assign is NULL");
  if (as->all_limit < 0) return fq_fail(ctx, FQ_E_ARG, "all_limit < 0");
  if (as->max_poly_whole < 0 || as->max_poly_whole > FQ_MAX_POLY || as->max_poly_safe < 0 || as->max_poly_safe > FQ_MAX_POLY)
    return fq_fail(ctx, FQ_E_ARG, "max_poly_* out of range (0..FQ_MAX_POLY)");
  if (as->n_cand_whole < 0 || as->n_cand_whole > (1L << 30) || as->n_cand_safe < 0 || as->n_cand_safe > (1L << 30))
    return fq_fail(ctx, FQ_E_ARG, "too many candidates (n_cand_* out of 0..2^30)");
  *lw = longest_list(a->N_whole, as->max_poly_whole, as->all_limit);
  *ls = longest_list(a->N_safe, as->max_poly_safe, as->all_limit);
  if (*lw < 0 || *ls < 0) return fq_fail(ctx, FQ_E_ARG, "assignment list longer than 2^20");
  if (((uintptr_t)a->Ab_whole & 15) || ((uintptr_t)a->Ab_safe & 15)) return fq_fail(ctx, FQ_E_ARG, "Ab must be 16-byte aligned");
  return 0;
}

// the scalar parts of fq_pair_window, checked by every window entry
const char* check_window_scalars(const fq_pair_window* w)
{
  if (!w) return "window is NULL";
  if (!w->init_whole || !w->final_whole || !w->init_safe || !w->final_safe) return "window arrays must not be NULL";
  if (!fqw::finite(w->inc_whole) || !(w->inc_whole > 0) || !fqw::finite(w->inc_safe) || !(w->inc_safe > 0))
    return "inc_* must be finite and > 0";
  if (!fqw::finite(w->gamma_whole) || !fqw::finite(w->gammap_whole) || !fqw::finite(w->gamma_safe) || !fqw::finite(w->gammap_safe))
    return "gamma* must be finite";
  return nullptr;
}

// the chain itself, every pointer a device pointer; `a` and the lists are checked
int run_chain(fq_ctx* ctx, const fq_pair_args* a, const Lists& l, fq_pair_result* results_all, cudaStream_t st)
{
  const int P = a->n_prob, Nw = a->N_whole, Ns = a->N_safe;
  const size_t ncw = l.ncw, ncs = l.ncs;
  // ---- scratch
  size_t need = 0;
  // decomposing chain: staging slots of both sweeps (the larger), rows per slot, spilled survivors per slot
  size_t dslots = 0, dcap = 0, dspill = 0;
  if (l.dc)
  {
    dslots = (size_t)P * std::max(l.as->max_poly_whole, l.as->max_poly_safe);
    dcap = (size_t)std::max(a->max_poly_faces_whole, a->max_poly_faces_safe);
    dspill = fq_decomp_spill_n(std::max(l.dc->max_obs_whole, l.dc->max_obs_safe));
  }
  {
    char* p = nullptr;
    Scratch s;
    auto layout = [&](char* base) {
      p = base;
      s.dt_w = carve<double>(p, ncw);          s.dt_s = carve<double>(p, ncs);
      s.cost_w = carve<double>(p, ncw);        s.cost_s = carve<double>(p, ncs);
      s.dt_base_w = carve<double>(p, P);       s.dt_base_s = carve<double>(p, P);
      s.win_cost_w = carve<double>(p, P);      s.win_cost_s = carve<double>(p, P);
      s.win_dt_w = carve<double>(p, P);        s.win_dt_s = carve<double>(p, P);
      s.x0_safe = carve<double>(p, (size_t)9 * P);
      s.coeffs_w = carve<double>(p, (size_t)12 * Nw * P);
      s.coeffs_s = carve<double>(p, (size_t)12 * Ns * P);
      s.re_cost = carve<double>(p, P);
      s.cand_ofs_w = carve<int>(p, P + 1);     s.cand_ofs_s = carve<int>(p, P + 1);
      s.win_idx_w = carve<int>(p, P);          s.win_idx_s = carve<int>(p, P);
      s.win_ofs = carve<int>(p, P + 1);        s.n_samples = carve<int>(p, P);      s.k_safe = carve<int>(p, P);
      s.sig_w = carve<uint8_t>(p, ncw * Nw);   s.sig_s = carve<uint8_t>(p, ncs * Ns);
      s.win_sig_w = carve<uint8_t>(p, (size_t)P * Nw);  s.win_sig_s = carve<uint8_t>(p, (size_t)P * Ns);
      s.feas_w = carve<uint8_t>(p, ncw);       s.feas_s = carve<uint8_t>(p, ncs);   s.re_feas = carve<uint8_t>(p, P);
      s.fac_w = carve<double>(p, l.win ? (size_t)P * l.mfw : 0);  s.fac_s = carve<double>(p, l.win ? (size_t)P * l.mfs : 0);
      s.nf_w = carve<int>(p, l.win ? P : 0);   s.nf_s = carve<int>(p, l.win ? P : 0);
      s.dc_stage = carve<double>(p, dslots * dcap * 4);     s.dc_stage_n = carve<int>(p, dslots);
      s.dc_spill = carve<double>(p, dslots * dspill * 4);   s.dc_spill_flag = carve<uint8_t>(p, dslots * dspill);
      s.dc_Ab_w = carve<double>(p, l.dc && !l.dc->Ab_whole ? (size_t)P * a->max_faces_whole * 4 : 0);
      s.dc_Ab_s = carve<double>(p, l.dc && !l.dc->Ab_safe ? (size_t)P * a->max_faces_safe * 4 : 0);
      s.dc_face_w = carve<int>(p, l.dc && !l.dc->face_ofs_whole ? (size_t)P * l.as->max_poly_whole + 1 : 0);
      s.dc_face_s = carve<int>(p, l.dc && !l.dc->face_ofs_safe ? (size_t)P * l.as->max_poly_safe + 1 : 0);
      s.dc_xf_w = carve<double>(p, l.dc ? (size_t)9 * P : 0);  s.dc_xf_s = carve<double>(p, l.dc ? (size_t)9 * P : 0);
      return (size_t)(p - base);
    };
    need = layout(nullptr);
    FQ_CUDA(ctx->d_pair.reserve(need));       // grows only on the first call / a larger batch (synchronous cudaMalloc)
    layout((char*)ctx->d_pair.p);
    Tree tree{};
    const int stride = std::max(l.win ? std::max(l.mfw, l.mfs) : std::max(a->n_fac_whole, a->n_fac_safe), 1);
    if (l.ex)
    { // the whole tree is done before the safe one starts: one pool serves both
      const size_t nb = std::max(fq_bnb_node_bytes(Nw, 1), fq_bnb_node_bytes(Ns, 0));
      FQ_CUDA(ctx->d_bnb.reserve(tree_layout(nullptr, P, stride, std::max(Nw, Ns), nb, &tree)));
      tree_layout((char*)ctx->d_bnb.p, P, stride, std::max(Nw, Ns), nb, &tree);
    }

    uint8_t* feas_w = a->feasible_whole ? a->feasible_whole : s.feas_w;
    uint8_t* feas_s = a->feasible_safe ? a->feasible_safe : s.feas_s;
    double* cost_w = a->cost_whole ? a->cost_whole : s.cost_w;
    double* cost_s = a->cost_safe ? a->cost_safe : s.cost_s;
    double* coeffs_w = a->coeffs_whole ? a->coeffs_whole : s.coeffs_w;
    double* coeffs_s = a->coeffs_safe ? a->coeffs_safe : s.coeffs_s;
    const int mcw = l.mcw, mcs = l.mcs;
    // the corridors of the two sweeps; each launch adds its candidates and outputs
    FqKernelArgs whole{}, safe{};
    whole.N = Nw; whole.force_final = 1; whole.n_prob = P; whole.x0 = a->x0; whole.xf = a->xf_whole; whole.lim = a->lim;
    whole.poly_ofs = a->poly_ofs_whole; whole.face_ofs = a->face_ofs_whole; whole.Ab = a->Ab_whole; whole.max_faces = a->max_faces_whole;
    safe.N = Ns; safe.force_final = 0; safe.n_prob = P; safe.x0 = s.x0_safe; safe.xf = a->xf_safe; safe.lim = a->lim;
    safe.poly_ofs = a->poly_ofs_safe; safe.face_ofs = a->face_ofs_safe; safe.Ab = a->Ab_safe; safe.max_faces = a->max_faces_safe;
    // decomposing chain (faster.cpp:393-403 whole, :485-504 safe): one sweep's corridors from its paths and clouds, into
    // the caller's outputs or the scratch; the final states go to the scratch
    auto decompose = [&](bool is_whole, FqKernelArgs* sweep) -> cudaError_t {
      const fq_pair_decomp* d = l.dc;
      FqDecompArgs x{};
      x.n_prob = P; x.max_poly = is_whole ? l.as->max_poly_whole : l.as->max_poly_safe;
      x.poly_ofs = is_whole ? a->poly_ofs_whole : a->poly_ofs_safe;
      x.path = is_whole ? d->path_whole : d->path_safe;
      x.first = is_whole ? nullptr : s.x0_safe;
      x.obs_ofs = is_whole ? d->obs_ofs_whole : d->obs_ofs_safe; x.obs = is_whole ? d->obs_whole : d->obs_safe;
      x.max_obs = is_whole ? d->max_obs_whole : d->max_obs_safe;
      for (int k = 0; k < 3; k++) x.bbox[k] = d->bbox[k];
      x.inflate = d->inflate; x.z_ground = d->z_ground;
      x.cap_pf = is_whole ? a->max_poly_faces_whole : a->max_poly_faces_safe;
      x.max_faces = is_whole ? a->max_faces_whole : a->max_faces_safe;
      x.stage = s.dc_stage; x.stage_n = s.dc_stage_n; x.spill = s.dc_spill; x.spill_flag = s.dc_spill_flag; x.spill_n = (int)dspill;
      x.goal = d->goal; x.face_cap = P * x.max_poly;
      x.face_ofs = is_whole ? (d->face_ofs_whole ? d->face_ofs_whole : s.dc_face_w) : (d->face_ofs_safe ? d->face_ofs_safe : s.dc_face_s);
      x.Ab = is_whole ? (d->Ab_whole ? d->Ab_whole : s.dc_Ab_w) : (d->Ab_safe ? d->Ab_safe : s.dc_Ab_s);
      x.xf = is_whole ? s.dc_xf_w : s.dc_xf_s;
      x.pos_out = is_whole ? d->E : d->M;
      x.status = is_whole ? d->status_whole : d->status_safe;
      sweep->face_ofs = x.face_ofs; sweep->Ab = x.Ab; sweep->xf = x.xf;
      return fq_launch_decomp(x, st);
    };

    // ---- per-corridor windows: every window is read here, before anything is written (the outputs may alias them)
    const fq_pair_window* win = l.win;
    if (win)
    {
      FQ_CUDA(fq_launch_window_factors(P, l.mfw, win->init_whole, win->final_whole, win->inc_whole, s.fac_w, s.nf_w, st));
      FQ_CUDA(fq_launch_window_factors(P, l.mfs, win->init_safe, win->final_safe, win->inc_safe, s.fac_s, s.nf_s, st));
    }
    // ---- whole sweep (faster.cpp:406-418); a decomposing chain first makes its corridors and E (which getDTInitial reads)
    if (l.dc) FQ_CUDA(decompose(true, &whole));
    FQ_CUDA(fq_launch_dtbase(P, Nw, a->DC, a->x0, whole.xf, a->lim, s.dt_base_w, st));
    if (!l.as)
      FQ_CUDA(fq_launch_expand_grid(P, Nw, a->n_fac_whole, a->n_sig_whole, a->factors_whole, a->sigmas_whole, s.dt_base_w, s.dt_w,
                                    s.sig_w, s.cand_ofs_w, st));
    else if (win)
    {
      FQ_CUDA(fq_launch_window_offsets(P, Nw, l.mfw, l.as->all_limit, l.as->max_poly_whole, (long long)ncw, a->poly_ofs_whole, s.nf_w,
                                       s.cand_ofs_w, st));
      FQ_CUDA(fq_launch_expand_window(P, Nw, l.mfw, l.as->all_limit, s.fac_w, s.nf_w, s.dt_base_w, a->poly_ofs_whole, s.cand_ofs_w,
                                      s.dt_w, s.sig_w, st));
    }
    else
    {
      FQ_CUDA(fq_launch_assign_offsets(P, Nw, a->n_fac_whole, l.as->all_limit, l.as->max_poly_whole, (long long)ncw, a->poly_ofs_whole,
                                       s.cand_ofs_w, st));
      FQ_CUDA(fq_launch_expand_assign(P, Nw, a->n_fac_whole, l.as->all_limit, a->factors_whole, s.dt_base_w, a->poly_ofs_whole,
                                      s.cand_ofs_w, s.dt_w, s.sig_w, st));
    }
    FqKernelArgs k = whole;
    k.cand_ofs = s.cand_ofs_w; k.dt = s.dt_w; k.sigma = s.sig_w; k.feasible = feas_w; k.cost = cost_w;
    k.sorted_dt = 1; k.ee_width = l.eew;                  // factor-major grid, ascending factors
    int rc = fq_launch_solve_ctx(ctx, k, mcw, a->max_poly_faces_whole, st);
    if (rc) return rc;
    FqSelectMultiArgs sw;
    sw.n_prob = P; sw.N = Nw; sw.n_sig = a->n_sig_whole; sw.cand_ofs = s.cand_ofs_w; sw.dt = s.dt_w; sw.sigma = s.sig_w;
    sw.feasible = feas_w; sw.cost = cost_w; sw.win_idx = s.win_idx_w; sw.win_cost = s.win_cost_w; sw.win_dt = s.win_dt_w;
    sw.win_sigma = s.win_sig_w; sw.win_ofs = s.win_ofs;
    FQ_CUDA(fq_launch_select_multi(sw, st));
    FqBnbChainArgs cx{};                                   // the exact stage's view of a sweep
    // after a sweep's coefficient solve: tree winners it did not confirm go back to their list winners, whose
    // coefficients a second solve of those corridors provides
    auto confirm = [&](const FqKernelArgs& sweep, double* coeffs, int mpf) -> int {
      FQ_CUDA(fq_launch_bnb_fallback(cx, s.re_feas, tree.redo_dt, st));
      FqKernelArgs r = sweep;
      r.cand_ofs = s.win_ofs; r.dt = tree.redo_dt; r.sigma = cx.win_sig; r.feasible = s.re_feas; r.cost = s.re_cost; r.coeffs = tree.redo_coeffs;
      if (int e = fq_launch_solve_ctx(ctx, r, 1, mpf, st)) return e;
      FQ_CUDA(fq_launch_bnb_adopt(P, sweep.N, tree.redo_dt, tree.redo_coeffs, coeffs, st));
      return 0;
    };
    if (l.ex)
    {
      cx.stride = stride; cx.all_limit = l.as->all_limit; cx.cand_ofs = s.cand_ofs_w; cx.cand_dt = s.dt_w;
      cx.n_fac = a->n_fac_whole; cx.n_fac_j = win ? s.nf_w : nullptr;
      cx.win_idx = s.win_idx_w; cx.win_cost = s.win_cost_w; cx.win_dt = s.win_dt_w; cx.win_sig = s.win_sig_w;
      cx.exact_out = l.ex->exact_whole; cx.nodes_out = l.ex->nodes_whole;
      rc = exact_stage(ctx, tree, whole, cx, a->max_poly_faces_whole, tree.changed_w, st);
      if (rc) return rc;
    }
    // coefficients of the winners: one candidate per corridor through the same kernel (losers' dt is NaN -> "not solved")
    k = whole;
    k.cand_ofs = s.win_ofs; k.dt = s.win_dt_w; k.sigma = s.win_sig_w; k.feasible = s.re_feas; k.cost = s.re_cost; k.coeffs = coeffs_w;
    rc = fq_launch_solve_ctx(ctx, k, 1, a->max_poly_faces_whole, st);
    if (rc) return rc;
    if (l.ex && (rc = confirm(whole, coeffs_w, a->max_poly_faces_whole))) return rc;
    // ---- R (faster.cpp:474-475) and the safe sweep from it (faster.cpp:521-527)
    FqPairMidArgs m;
    m.n_prob = P; m.N = Nw; m.DC = a->DC; m.r_fraction = a->r_fraction; m.coeffs = coeffs_w; m.win_dt = s.win_dt_w;
    m.win_idx = s.win_idx_w; m.x0_safe = s.x0_safe; m.n_samples = s.n_samples; m.k_safe = s.k_safe;
    FQ_CUDA(fq_launch_pair_mid(m, st));
    if (l.dc) FQ_CUDA(decompose(false, &safe));            // the safe corridors around R, and M
    FQ_CUDA(fq_launch_dtbase(P, Ns, a->DC, s.x0_safe, safe.xf, a->lim, s.dt_base_s, st));
    if (!l.as)
      FQ_CUDA(fq_launch_expand_grid(P, Ns, a->n_fac_safe, a->n_sig_safe, a->factors_safe, a->sigmas_safe, s.dt_base_s, s.dt_s,
                                    s.sig_s, s.cand_ofs_s, st));
    else if (win)
    {
      FQ_CUDA(fq_launch_window_offsets(P, Ns, l.mfs, l.as->all_limit, l.as->max_poly_safe, (long long)ncs, a->poly_ofs_safe, s.nf_s,
                                       s.cand_ofs_s, st));
      FQ_CUDA(fq_launch_expand_window(P, Ns, l.mfs, l.as->all_limit, s.fac_s, s.nf_s, s.dt_base_s, a->poly_ofs_safe, s.cand_ofs_s,
                                      s.dt_s, s.sig_s, st));
    }
    else
    {
      FQ_CUDA(fq_launch_assign_offsets(P, Ns, a->n_fac_safe, l.as->all_limit, l.as->max_poly_safe, (long long)ncs, a->poly_ofs_safe,
                                       s.cand_ofs_s, st));
      FQ_CUDA(fq_launch_expand_assign(P, Ns, a->n_fac_safe, l.as->all_limit, a->factors_safe, s.dt_base_s, a->poly_ofs_safe,
                                      s.cand_ofs_s, s.dt_s, s.sig_s, st));
    }
    k = safe;
    k.cand_ofs = s.cand_ofs_s; k.dt = s.dt_s; k.sigma = s.sig_s; k.feasible = feas_s; k.cost = cost_s;
    k.sorted_dt = 1; k.ee_width = l.ees;
    rc = fq_launch_solve_ctx(ctx, k, mcs, a->max_poly_faces_safe, st);
    if (rc) return rc;
    FqSelectMultiArgs ss = sw;
    ss.N = Ns; ss.n_sig = a->n_sig_safe; ss.cand_ofs = s.cand_ofs_s; ss.dt = s.dt_s; ss.sigma = s.sig_s; ss.feasible = feas_s;
    ss.cost = cost_s; ss.win_idx = s.win_idx_s; ss.win_cost = s.win_cost_s; ss.win_dt = s.win_dt_s; ss.win_sigma = s.win_sig_s;
    FQ_CUDA(fq_launch_select_multi(ss, st));
    if (l.ex)
    {
      cx.cand_ofs = s.cand_ofs_s; cx.cand_dt = s.dt_s; cx.n_fac = a->n_fac_safe; cx.n_fac_j = win ? s.nf_s : nullptr;
      cx.win_idx = s.win_idx_s; cx.win_cost = s.win_cost_s; cx.win_dt = s.win_dt_s; cx.win_sig = s.win_sig_s;
      cx.exact_out = l.ex->exact_safe; cx.nodes_out = l.ex->nodes_safe;
      rc = exact_stage(ctx, tree, safe, cx, a->max_poly_faces_safe, tree.changed_s, st);
      if (rc) return rc;
    }
    if (a->coeffs_safe || l.ex)           // the exact stage re-solves its winners to confirm them, wanted or not
    {
      k = safe;
      k.cand_ofs = s.win_ofs; k.dt = s.win_dt_s; k.sigma = s.win_sig_s; k.feasible = s.re_feas; k.cost = s.re_cost; k.coeffs = coeffs_s;
      rc = fq_launch_solve_ctx(ctx, k, 1, a->max_poly_faces_safe, st);
      if (rc) return rc;
      if (l.ex && (rc = confirm(safe, coeffs_s, a->max_poly_faces_safe))) return rc;
    }
    FqPairFinalArgs f;
    f.n_prob = P; f.n_sig_w = a->n_sig_whole; f.n_sig_s = a->n_sig_safe; f.win_idx_w = s.win_idx_w; f.win_idx_s = s.win_idx_s;
    f.n_samples = s.n_samples; f.k_safe = s.k_safe; f.win_cost_w = s.win_cost_w; f.win_cost_s = s.win_cost_s;
    f.win_dt_w = s.win_dt_w; f.win_dt_s = s.win_dt_s; f.dt_base_w = s.dt_base_w; f.dt_base_s = s.dt_base_s; f.x0_safe = s.x0_safe;
    f.out = a->results;
    if (l.as)
    {
      f.cand_ofs_w = s.cand_ofs_w; f.cand_ofs_s = s.cand_ofs_s; f.n_fac_w = a->n_fac_whole; f.n_fac_s = a->n_fac_safe;
      f.N_w = Nw; f.N_s = Ns; f.win_sig_w = s.win_sig_w; f.win_sig_s = s.win_sig_s;
      f.sigma_out_w = l.as->sigma_whole; f.sigma_out_s = l.as->sigma_safe;
      if (win) { f.n_fac_j_w = s.nf_w; f.n_fac_j_s = s.nf_s; }
      if (l.ex)
      {
        f.changed_w = tree.changed_w; f.changed_s = tree.changed_s; f.poly_ofs_w = a->poly_ofs_whole; f.poly_ofs_s = a->poly_ofs_safe;
        f.all_limit = l.as->all_limit;
      }
      if (l.as->cand_ofs_whole)
        FQ_CUDA(cudaMemcpyAsync(l.as->cand_ofs_whole, s.cand_ofs_w, sizeof(int) * (size_t)(P + 1), cudaMemcpyDeviceToDevice, st));
      if (l.as->cand_ofs_safe)
        FQ_CUDA(cudaMemcpyAsync(l.as->cand_ofs_safe, s.cand_ofs_s, sizeof(int) * (size_t)(P + 1), cudaMemcpyDeviceToDevice, st));
    }
    FQ_CUDA(fq_launch_pair_final(f, st));
    if (win)
    {
      FqPairWindowArgs wa;
      wa.n_prob = P; wa.max_fac_w = l.mfw; wa.max_fac_s = l.mfs; wa.rec = a->results;
      wa.cand_ofs_w = s.cand_ofs_w; wa.cand_ofs_s = s.cand_ofs_s; wa.n_fac_w = s.nf_w; wa.n_fac_s = s.nf_s; wa.fac_w = s.fac_w; wa.fac_s = s.fac_s;
      wa.init_w = win->init_whole; wa.final_w = win->final_whole; wa.init_s = win->init_safe; wa.final_s = win->final_safe;
      wa.gamma_w = win->gamma_whole; wa.gammap_w = win->gammap_whole; wa.gamma_s = win->gamma_safe; wa.gammap_s = win->gammap_safe;
      wa.factor_w = win->factor_whole; wa.factor_s = win->factor_safe; wa.trials_w = win->trials_whole; wa.trials_s = win->trials_safe;
      wa.next_init_w = win->next_init_whole; wa.next_final_w = win->next_final_whole;
      wa.next_init_s = win->next_init_safe; wa.next_final_s = win->next_final_safe;
      FQ_CUDA(fq_launch_pair_window(wa, st));
    }
    // ---- the path's one exchange: every rank's result records to every rank (north_star: one all-gather, only when the
    //      batch is spread over several GPUs)
    if (results_all && ctx->comm)
    {
      rc = fq_comm_allgather(ctx, a->results, results_all, sizeof(fq_pair_result) * (size_t)P, st);
      if (rc) return rc;
    }
    else if (results_all)
      FQ_CUDA(cudaMemcpyAsync(results_all, a->results, sizeof(fq_pair_result) * (size_t)P, cudaMemcpyDeviceToDevice, st));
  }
  return 0;
}
}  // namespace

// every pointer of `a` is a device pointer
extern "C" int fq_replan_pairs_dev(fq_ctx* ctx, const fq_pair_args* a, fq_pair_result* results_all, void* stream_v)
{
  if (!ctx) return FQ_E_ARG;
  if (int rc = check_common(ctx, a)) return rc;
  if (((uintptr_t)a->Ab_whole & 15) || ((uintptr_t)a->Ab_safe & 15)) return fq_fail(ctx, FQ_E_ARG, "Ab must be 16-byte aligned");
  FQ_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = stream_v ? (cudaStream_t)stream_v : ctx->stream;
  Lists l;
  l.ncw = (size_t)a->n_prob * a->n_fac_whole * a->n_sig_whole; l.ncs = (size_t)a->n_prob * a->n_fac_safe * a->n_sig_safe;
  l.mcw = a->n_fac_whole * a->n_sig_whole; l.mcs = a->n_fac_safe * a->n_sig_safe;
  l.eew = a->n_sig_whole; l.ees = a->n_sig_safe;
  return run_chain(ctx, a, l, results_all, st);
}

namespace
{
// every pointer of `a` and of `as` (and `ex`) is a device pointer; the sweeps' sizes come from the hints of `as`
int assign_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_exact* ex, fq_pair_result* results_all,
               void* stream_v, const fq_pair_decomp* dc = nullptr)
{
  if (!ctx) return FQ_E_ARG;
  if (int rc = check_common(ctx, a, false, false, dc != nullptr)) return rc;
  long long lw = 0, ls = 0;
  if (int rc = check_assign_hints(ctx, a, as, &lw, &ls)) return rc;
  if (lw * a->n_fac_whole > (1LL << 30) || ls * a->n_fac_safe > (1LL << 30)) return fq_fail(ctx, FQ_E_ARG, "too many candidates");
  FQ_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = stream_v ? (cudaStream_t)stream_v : ctx->stream;
  Lists l;
  l.as = as;
  l.ncw = (size_t)as->n_cand_whole; l.ncs = (size_t)as->n_cand_safe;
  l.mcw = (int)(lw * a->n_fac_whole); l.mcs = (int)(ls * a->n_fac_safe);
  l.eew = (int)lw; l.ees = (int)ls;
  l.ex = ex; l.dc = dc;
  return run_chain(ctx, a, l, results_all, st);
}

// every pointer of `a`, `as` and `win` (and `ex`) is a device pointer; the sweeps' sizes come from the hints of `as`
// (capacities) and `win` (factor rows)
int window_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win, const fq_pair_exact* ex,
               fq_pair_result* results_all, void* stream_v, const fq_pair_decomp* dc = nullptr)
{
  if (!ctx) return FQ_E_ARG;
  if (int rc = check_common(ctx, a, false, true, dc != nullptr)) return rc;
  if (const char* why = check_window_scalars(win)) return fq_fail(ctx, FQ_E_ARG, why);
  if (win->max_fac_whole < 0 || win->max_fac_whole > fqw::kMaxFactors || win->max_fac_safe < 0 || win->max_fac_safe > fqw::kMaxFactors)
    return fq_fail(ctx, FQ_E_ARG, "max_fac_* out of range (0..4096)");
  long long lw = 0, ls = 0;
  if (int rc = check_assign_hints(ctx, a, as, &lw, &ls)) return rc;
  if (lw * win->max_fac_whole > (1LL << 30) || ls * win->max_fac_safe > (1LL << 30)) return fq_fail(ctx, FQ_E_ARG, "too many candidates");
  FQ_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = stream_v ? (cudaStream_t)stream_v : ctx->stream;
  Lists l;
  l.as = as; l.win = win;
  l.ncw = (size_t)as->n_cand_whole; l.ncs = (size_t)as->n_cand_safe;
  l.mfw = win->max_fac_whole; l.mfs = win->max_fac_safe;
  l.mcw = (int)std::max(1LL, lw * l.mfw); l.mcs = (int)std::max(1LL, ls * l.mfs);
  l.eew = (int)lw; l.ees = (int)ls;
  l.ex = ex; l.dc = dc;
  return run_chain(ctx, a, l, results_all, st);
}
}  // namespace

extern "C" int fq_replan_pairs_assign_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, fq_pair_result* results_all,
                                          void* stream_v)
{
  return assign_dev(ctx, a, as, nullptr, results_all, stream_v);
}

extern "C" int fq_replan_pairs_window_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                          fq_pair_result* results_all, void* stream_v)
{
  return window_dev(ctx, a, as, win, nullptr, results_all, stream_v);
}

extern "C" int fq_replan_pairs_exact_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                         const fq_pair_exact* ex, fq_pair_result* results_all, void* stream_v)
{
  if (!ctx) return FQ_E_ARG;
  if (!ex) return fq_fail(ctx, FQ_E_ARG, "exact is NULL");
  if (!as) return fq_fail(ctx, FQ_E_ARG, "assign is NULL");
  return win ? window_dev(ctx, a, as, win, ex, results_all, stream_v) : assign_dev(ctx, a, as, ex, results_all, stream_v);
}

extern "C" int fq_replan_pairs_decomp_dev(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                          const fq_pair_exact* ex, const fq_pair_decomp* dc, fq_pair_result* results_all, void* stream_v)
{
  if (!ctx) return FQ_E_ARG;
  if (!as) return fq_fail(ctx, FQ_E_ARG, "assign is NULL");
  if (const char* why = check_decomp_scalars(dc)) return fq_fail(ctx, FQ_E_ARG, why);
  if (dc->max_obs_whole < 0 || dc->max_obs_safe < 0) return fq_fail(ctx, FQ_E_ARG, "decomp: max_obs_* < 0");
  return win ? window_dev(ctx, a, as, win, ex, results_all, stream_v, dc) : assign_dev(ctx, a, as, ex, results_all, stream_v, dc);
}

int fq_replan_pairs_host_ex(fq_ctx* ctx, const fq_pair_args* a, bool deferred, fq_pair_result** d_results, bool copy_results,
                            const fq_pair_assign* as, const fq_pair_window* win, const fq_pair_exact* ex, const fq_pair_decomp* dc)
{
  if (!ctx) return FQ_E_ARG;
  if (int rc = fq_settle(ctx)) return rc;
  if ((win || dc) && !as) return fq_fail(ctx, FQ_E_ARG, "assign is NULL");
  if (int rc = check_common(ctx, a, as == nullptr, win != nullptr, dc != nullptr)) return rc;
  if (dc)
    if (const char* why = check_decomp_scalars(dc)) return fq_fail(ctx, FQ_E_ARG, why);
  if (win)
    if (const char* why = check_window_scalars(win)) return fq_fail(ctx, FQ_E_ARG, why);
  const int P = a->n_prob, Nw = a->N_whole, Ns = a->N_safe;
  // ---- validate the two corridor descriptions
  auto check = [&](const int* po, const int* fo, const double* Ab, FqCorridorSizes* sizes) -> const char* {
    if (po[0] != 0 || fo[0] != 0) return "offset arrays must start at 0";
    if (const char* why = fq_scan_corridors(P, po, fo, sizes)) return why;
    if (sizes->n_face > 0 && !Ab) return "polytopes given but Ab is NULL";
    if (sizes->n_face > 0 && !fq_scan_all_finite(Ab, 4 * (size_t)sizes->n_face)) return "non-finite value in Ab";
    return nullptr;
  };
  FqCorridorSizes cw, cs;
  int n_obs_w = 0, n_obs_s = 0, max_obs_w = 0, max_obs_s = 0;   // decomposing chain: the clouds
  if (!dc)
  {
    if (const char* why = check(a->poly_ofs_whole, a->face_ofs_whole, a->Ab_whole, &cw)) return fq_fail(ctx, FQ_E_ARG, why);
    if (const char* why = check(a->poly_ofs_safe, a->face_ofs_safe, a->Ab_safe, &cs)) return fq_fail(ctx, FQ_E_ARG, why);
  }
  else
  { // polytope counts, paths, clouds and the goal
    auto ofs = [&](const int* o, int max_step, int* total, int* largest) -> bool {
      if (o[0] != 0) return false;
      for (int j = 0; j < P; j++)
      {
        const int d = o[j + 1] - o[j];
        if (d < 0 || d > max_step) return false;
        *largest = std::max(*largest, d);
      }
      *total = o[P];
      return true;
    };
    int mp = 0;
    if (!ofs(a->poly_ofs_whole, FQ_MAX_POLY, &cw.n_poly, &mp) || !ofs(a->poly_ofs_safe, FQ_MAX_POLY, &cs.n_poly, &mp))
      return fq_fail(ctx, FQ_E_ARG, "poly_ofs_* must start at 0 and step by 0..FQ_MAX_POLY");
    if (!ofs(dc->obs_ofs_whole, 1 << 30, &n_obs_w, &max_obs_w) || !ofs(dc->obs_ofs_safe, 1 << 30, &n_obs_s, &max_obs_s))
      return fq_fail(ctx, FQ_E_ARG, "decomp: obs_ofs_* must start at 0 and be non-decreasing");
    if (!fq_scan_all_finite(dc->path_whole, 3 * (size_t)(cw.n_poly + P)) || !fq_scan_all_finite(dc->path_safe, 3 * (size_t)(cs.n_poly + P)) ||
        !fq_scan_all_finite(dc->obs_whole, 3 * (size_t)n_obs_w) || !fq_scan_all_finite(dc->obs_safe, 3 * (size_t)n_obs_s) ||
        (dc->goal && !fq_scan_all_finite(dc->goal, 3 * (size_t)P)))
      return fq_fail(ctx, FQ_E_ARG, "decomp: non-finite value in a path, a cloud or the goal");
  }
  if (!fq_scan_all_finite(a->x0, 9 * (size_t)P) ||
      (!dc && (!fq_scan_all_finite(a->xf_whole, 9 * (size_t)P) || !fq_scan_all_finite(a->xf_safe, 9 * (size_t)P))))
    return fq_fail(ctx, FQ_E_ARG, "non-finite value in x0/xf");
  if (!fq_scan_all_positive_finite(a->lim, 3 * (size_t)P) || !fq_scan_all_positive_finite(a->factors_whole, (size_t)a->n_fac_whole) ||
      !fq_scan_all_positive_finite(a->factors_safe, (size_t)a->n_fac_safe))
    return fq_fail(ctx, FQ_E_ARG, "limits and factors must be finite and > 0");
  for (int i = 1; i < a->n_fac_whole; i++)
    if (a->factors_whole[i] < a->factors_whole[i - 1]) return fq_fail(ctx, FQ_E_ARG, "factors_whole must be ascending");
  for (int i = 1; i < a->n_fac_safe; i++)
    if (a->factors_safe[i] < a->factors_safe[i - 1]) return fq_fail(ctx, FQ_E_ARG, "factors_safe must be ascending");
  size_t ncw = (size_t)P * a->n_fac_whole * a->n_sig_whole, ncs = (size_t)P * a->n_fac_safe * a->n_sig_safe;
  fq_pair_assign da{};                 // per-corridor lists: the device-side outputs and exact sizes
  fq_pair_window dw{};                 // per-corridor windows: device copies and the longest factor lists
  if (as)
  {
    if (as->all_limit < 0) return fq_fail(ctx, FQ_E_ARG, "all_limit < 0");
    long long tw = 0, ts = 0;
    int mpw = 0, mps = 0;
    for (int j = 0; j < P; j++)
    {
      const int pw = a->poly_ofs_whole[j + 1] - a->poly_ofs_whole[j], ps = a->poly_ofs_safe[j + 1] - a->poly_ofs_safe[j];
      const long long lw = fqa::list_len(Nw, pw, as->all_limit), ls = fqa::list_len(Ns, ps, as->all_limit);
      if (lw < 0 || ls < 0) return fq_fail(ctx, FQ_E_ARG, "assignment list of a corridor longer than 2^20");
      int nfw = a->n_fac_whole, nfs = a->n_fac_safe;
      if (win)
      {
        nfw = fqw::factors(win->init_whole[j], win->final_whole[j], win->inc_whole, nullptr, 0);
        nfs = fqw::factors(win->init_safe[j], win->final_safe[j], win->inc_safe, nullptr, 0);
        if (nfw < 0 || nfs < 0) return fq_fail(ctx, FQ_E_ARG, "time-allocation window refused (not finite, init <= 0, more than 4096 factors or a stalled accumulation)");
        dw.max_fac_whole = std::max(dw.max_fac_whole, nfw); dw.max_fac_safe = std::max(dw.max_fac_safe, nfs);
      }
      tw += lw * nfw; ts += ls * nfs;
      mpw = std::max(mpw, pw); mps = std::max(mps, ps);
    }
    if (tw > (1LL << 30) || ts > (1LL << 30)) return fq_fail(ctx, FQ_E_ARG, "too many candidates");
    ncw = (size_t)tw; ncs = (size_t)ts;
    da.all_limit = as->all_limit; da.max_poly_whole = mpw; da.max_poly_safe = mps; da.n_cand_whole = (long)tw; da.n_cand_safe = (long)ts;
  }
  if (!as && cw.n_poly > 0 && !a->sigmas_whole) return fq_fail(ctx, FQ_E_ARG, "sigmas_whole is NULL");
  if (!as && cs.n_poly > 0 && !a->sigmas_safe) return fq_fail(ctx, FQ_E_ARG, "sigmas_safe is NULL");
  // assignments must name existing polytopes of EVERY corridor they are applied to
  if (!as)
  {
    int min_pw = FQ_MAX_POLY, min_ps = FQ_MAX_POLY;
    for (int j = 0; j < P; j++)
    {
      min_pw = std::min(min_pw, a->poly_ofs_whole[j + 1] - a->poly_ofs_whole[j]);
      min_ps = std::min(min_ps, a->poly_ofs_safe[j + 1] - a->poly_ofs_safe[j]);
    }
    if (min_pw > 0 && fq_scan_max_u8(a->sigmas_whole, (size_t)a->n_sig_whole * Nw) >= min_pw) return fq_fail(ctx, FQ_E_ARG, "sigmas_whole entry >= number of polytopes");
    if (min_ps > 0 && fq_scan_max_u8(a->sigmas_safe, (size_t)a->n_sig_safe * Ns) >= min_ps) return fq_fail(ctx, FQ_E_ARG, "sigmas_safe entry >= number of polytopes");
  }
  FQ_CUDA(cudaSetDevice(ctx->device));
  // ---- one packed upload
  size_t o = 0;
  auto put = [&](size_t bytes) { const size_t at = o; o = fq_align16(o + bytes); return at; };
  const size_t oAbw = put(32 * (size_t)std::max(cw.n_face, 1)), oAbs = put(32 * (size_t)std::max(cs.n_face, 1));
  const size_t ox0 = put(72 * (size_t)P), oxfw = put(72 * (size_t)P), oxfs = put(72 * (size_t)P), olim = put(24 * (size_t)P);
  const size_t ofw = put(8 * (size_t)a->n_fac_whole), ofs = put(8 * (size_t)a->n_fac_safe);
  const size_t opow = put(4 * (size_t)(P + 1)), ofow = put(4 * (size_t)(cw.n_poly + 1));
  const size_t opos = put(4 * (size_t)(P + 1)), ofos = put(4 * (size_t)(cs.n_poly + 1));
  const size_t osw = put((size_t)a->n_sig_whole * Nw), oss = put((size_t)a->n_sig_safe * Ns);
  const size_t owin = win ? put(8 * 4 * (size_t)P) : 0;   // init_whole, final_whole, init_safe, final_safe
  size_t opaw = 0, opas = 0, ooow = 0, ooos = 0, oobw = 0, oobs = 0, ogoal = 0;   // decomposing chain: paths, clouds, goal
  if (dc)
  {
    opaw = put(24 * (size_t)(cw.n_poly + P)); opas = put(24 * (size_t)(cs.n_poly + P));
    ooow = put(4 * (size_t)(P + 1)); ooos = put(4 * (size_t)(P + 1));
    oobw = put(24 * (size_t)n_obs_w); oobs = put(24 * (size_t)n_obs_s); ogoal = put(24 * (size_t)P);
  }
  const size_t in_bytes = o;
  o = 0;
  const size_t ores = put(sizeof(fq_pair_result) * (size_t)P);
  const size_t ocow = put(96 * (size_t)Nw * P), ocos = put(96 * (size_t)Ns * P);
  const size_t ocw = put(8 * ncw), ocs = put(8 * ncs), ofew = put(ncw), ofes = put(ncs);
  size_t ocaw = 0, ocas = 0, osgw = 0, osgs = 0;        // per-corridor lists: offsets and winners' assignments
  if (as) { ocaw = put(4 * (size_t)(P + 1)); ocas = put(4 * (size_t)(P + 1)); osgw = put((size_t)P * Nw); osgs = put((size_t)P * Ns); }
  size_t ofac = 0, otri = 0, onext = 0;                 // windows: factor_* (2 P), trials_* (2 P), next_* (4 P)
  if (win) { ofac = put(8 * 2 * (size_t)P); otri = put(4 * 2 * (size_t)P); onext = put(8 * 4 * (size_t)P); }
  size_t oex = 0, ond = 0;                              // exact stage: exact_* (2 P ints), nodes_* (2 P)
  if (ex) { oex = put(4 * 2 * (size_t)P); ond = put(8 * 2 * (size_t)P); }
  size_t odfw = 0, odfs = 0, odaw = 0, odas = 0, oE = 0, oM = 0, ostw = 0, osts = 0;   // decomposing chain: its outputs
  if (dc)
  {
    odfw = put(4 * (size_t)(cw.n_poly + 1)); odfs = put(4 * (size_t)(cs.n_poly + 1));
    odaw = put(32 * (size_t)P * a->max_faces_whole); odas = put(32 * (size_t)P * a->max_faces_safe);
    oE = put(24 * (size_t)P); oM = put(24 * (size_t)P); ostw = put(4 * (size_t)P); osts = put(4 * (size_t)P);
  }
  const size_t out_bytes = o;
  FQ_CUDA(ctx->h_in.reserve(in_bytes));
  FQ_CUDA(ctx->d_pair_io.reserve(in_bytes + out_bytes));
  char* hi = (char*)ctx->h_in.p;
  char* din = (char*)ctx->d_pair_io.p;
  char* dout = din + in_bytes;
  if (cw.n_face) std::memcpy(hi + oAbw, a->Ab_whole, 32 * (size_t)cw.n_face);
  if (cs.n_face) std::memcpy(hi + oAbs, a->Ab_safe, 32 * (size_t)cs.n_face);
  std::memcpy(hi + ox0, a->x0, 72 * (size_t)P);      std::memcpy(hi + olim, a->lim, 24 * (size_t)P);
  if (!dc) { std::memcpy(hi + oxfw, a->xf_whole, 72 * (size_t)P); std::memcpy(hi + oxfs, a->xf_safe, 72 * (size_t)P); }
  else
  {
    std::memcpy(hi + opaw, dc->path_whole, 24 * (size_t)(cw.n_poly + P)); std::memcpy(hi + opas, dc->path_safe, 24 * (size_t)(cs.n_poly + P));
    std::memcpy(hi + ooow, dc->obs_ofs_whole, 4 * (size_t)(P + 1));       std::memcpy(hi + ooos, dc->obs_ofs_safe, 4 * (size_t)(P + 1));
    if (n_obs_w) std::memcpy(hi + oobw, dc->obs_whole, 24 * (size_t)n_obs_w);
    if (n_obs_s) std::memcpy(hi + oobs, dc->obs_safe, 24 * (size_t)n_obs_s);
    if (dc->goal) std::memcpy(hi + ogoal, dc->goal, 24 * (size_t)P);
  }
  if (a->n_fac_whole) std::memcpy(hi + ofw, a->factors_whole, 8 * (size_t)a->n_fac_whole);
  if (a->n_fac_safe) std::memcpy(hi + ofs, a->factors_safe, 8 * (size_t)a->n_fac_safe);
  if (win)
  {
    const double* w4[4] = { win->init_whole, win->final_whole, win->init_safe, win->final_safe };
    for (int i = 0; i < 4; i++) std::memcpy(hi + owin + 8 * (size_t)P * i, w4[i], 8 * (size_t)P);
  }
  std::memcpy(hi + opow, a->poly_ofs_whole, 4 * (size_t)(P + 1)); std::memcpy(hi + opos, a->poly_ofs_safe, 4 * (size_t)(P + 1));
  if (!dc)
  {
    std::memcpy(hi + ofow, a->face_ofs_whole, 4 * (size_t)(cw.n_poly + 1)); std::memcpy(hi + ofos, a->face_ofs_safe, 4 * (size_t)(cs.n_poly + 1));
  }
  if (a->sigmas_whole) std::memcpy(hi + osw, a->sigmas_whole, (size_t)a->n_sig_whole * Nw);
  if (a->sigmas_safe) std::memcpy(hi + oss, a->sigmas_safe, (size_t)a->n_sig_safe * Ns);
  cudaStream_t st = ctx->stream;
  FQ_CUDA(cudaMemcpyAsync(din, hi, in_bytes, cudaMemcpyHostToDevice, st));
  fq_pair_args d = *a;
  d.x0 = (const double*)(din + ox0); d.xf_whole = (const double*)(din + oxfw); d.xf_safe = (const double*)(din + oxfs);
  d.lim = (const double*)(din + olim);
  d.poly_ofs_whole = (const int*)(din + opow); d.face_ofs_whole = (const int*)(din + ofow); d.Ab_whole = (const double*)(din + oAbw);
  d.poly_ofs_safe = (const int*)(din + opos); d.face_ofs_safe = (const int*)(din + ofos); d.Ab_safe = (const double*)(din + oAbs);
  d.factors_whole = a->factors_whole ? (const double*)(din + ofw) : nullptr;
  d.factors_safe = a->factors_safe ? (const double*)(din + ofs) : nullptr;
  d.sigmas_whole = a->sigmas_whole ? (const uint8_t*)(din + osw) : nullptr;
  d.sigmas_safe = a->sigmas_safe ? (const uint8_t*)(din + oss) : nullptr;
  d.feasible_whole = a->feasible_whole ? (uint8_t*)(dout + ofew) : nullptr; d.cost_whole = a->cost_whole ? (double*)(dout + ocw) : nullptr;
  d.feasible_safe = a->feasible_safe ? (uint8_t*)(dout + ofes) : nullptr;   d.cost_safe = a->cost_safe ? (double*)(dout + ocs) : nullptr;
  d.coeffs_whole = a->coeffs_whole ? (double*)(dout + ocow) : nullptr;       d.coeffs_safe = a->coeffs_safe ? (double*)(dout + ocos) : nullptr;
  d.results = (fq_pair_result*)(dout + ores);
  if (!dc)
  {
    d.max_faces_whole = std::max(cw.max_faces, 1); d.max_poly_faces_whole = cw.max_poly_faces; d.max_faces_safe = std::max(cs.max_faces, 1); d.max_poly_faces_safe = cs.max_poly_faces;
  }
  else
  { // the chain makes the corridors and final states; max_*faces_* stay the caller's caps
    d.xf_whole = d.xf_safe = nullptr; d.face_ofs_whole = d.face_ofs_safe = nullptr; d.Ab_whole = d.Ab_safe = nullptr;
  }
  // a NULL cost/flag output still needs a device array of its own kind: the chain allocates it in its scratch
  if ((d.feasible_whole == nullptr) != (d.cost_whole == nullptr) || (d.feasible_safe == nullptr) != (d.cost_safe == nullptr))
    return fq_fail(ctx, FQ_E_ARG, "feasible_* and cost_* must be given (or omitted) together");
  if (as)
  {
    da.cand_ofs_whole = as->cand_ofs_whole ? (int*)(dout + ocaw) : nullptr; da.cand_ofs_safe = as->cand_ofs_safe ? (int*)(dout + ocas) : nullptr;
    da.sigma_whole = as->sigma_whole ? (uint8_t*)(dout + osgw) : nullptr;  da.sigma_safe = as->sigma_safe ? (uint8_t*)(dout + osgs) : nullptr;
  }
  if (win)
  {
    const double* wi = (const double*)(din + owin);
    double* fo = (double*)(dout + ofac);
    int* to = (int*)(dout + otri);
    double* no = (double*)(dout + onext);
    dw.init_whole = wi; dw.final_whole = wi + P; dw.init_safe = wi + 2 * (size_t)P; dw.final_safe = wi + 3 * (size_t)P;
    dw.inc_whole = win->inc_whole; dw.inc_safe = win->inc_safe;
    dw.gamma_whole = win->gamma_whole; dw.gammap_whole = win->gammap_whole; dw.gamma_safe = win->gamma_safe; dw.gammap_safe = win->gammap_safe;
    dw.factor_whole = win->factor_whole ? fo : nullptr;               dw.factor_safe = win->factor_safe ? fo + P : nullptr;
    dw.trials_whole = win->trials_whole ? to : nullptr;               dw.trials_safe = win->trials_safe ? to + P : nullptr;
    dw.next_init_whole = win->next_init_whole ? no : nullptr;         dw.next_final_whole = win->next_final_whole ? no + P : nullptr;
    dw.next_init_safe = win->next_init_safe ? no + 2 * (size_t)P : nullptr; dw.next_final_safe = win->next_final_safe ? no + 3 * (size_t)P : nullptr;
  }
  fq_pair_exact dx{};
  if (ex)
  {
    int* eo = (int*)(dout + oex);
    long long* no = (long long*)(dout + ond);
    dx.exact_whole = ex->exact_whole ? eo : nullptr;  dx.exact_safe = ex->exact_safe ? eo + P : nullptr;
    dx.nodes_whole = ex->nodes_whole ? no : nullptr;  dx.nodes_safe = ex->nodes_safe ? no + P : nullptr;
  }
  fq_pair_decomp dd{};
  if (dc)
  {
    dd = *dc;
    dd.path_whole = (const double*)(din + opaw); dd.path_safe = (const double*)(din + opas);
    dd.obs_ofs_whole = (const int*)(din + ooow); dd.obs_ofs_safe = (const int*)(din + ooos);
    dd.obs_whole = (const double*)(din + oobw); dd.obs_safe = (const double*)(din + oobs);
    dd.goal = dc->goal ? (const double*)(din + ogoal) : nullptr;
    dd.max_obs_whole = max_obs_w; dd.max_obs_safe = max_obs_s;
    dd.face_ofs_whole = (int*)(dout + odfw); dd.face_ofs_safe = (int*)(dout + odfs);
    dd.Ab_whole = (double*)(dout + odaw); dd.Ab_safe = (double*)(dout + odas);
    dd.E = (double*)(dout + oE); dd.M = (double*)(dout + oM); dd.status_whole = (int*)(dout + ostw); dd.status_safe = (int*)(dout + osts);
  }
  int rc = dc ? fq_replan_pairs_decomp_dev(ctx, &d, &da, win ? &dw : nullptr, ex ? &dx : nullptr, &dd, nullptr, st)
         : ex ? fq_replan_pairs_exact_dev(ctx, &d, &da, win ? &dw : nullptr, &dx, nullptr, st)
         : win ? fq_replan_pairs_window_dev(ctx, &d, &da, &dw, nullptr, st)
         : as ? fq_replan_pairs_assign_dev(ctx, &d, &da, nullptr, st) : fq_replan_pairs_dev(ctx, &d, nullptr, st);
  if (rc) return rc;
  // ---- results straight into the caller's arrays (asynchronous when they are pinned)
  if (d_results) *d_results = (fq_pair_result*)(dout + ores);
  if (copy_results) FQ_CUDA(cudaMemcpyAsync(a->results, dout + ores, sizeof(fq_pair_result) * (size_t)P, cudaMemcpyDeviceToHost, st));
  if (a->coeffs_whole) FQ_CUDA(cudaMemcpyAsync(a->coeffs_whole, dout + ocow, 96 * (size_t)Nw * P, cudaMemcpyDeviceToHost, st));
  if (a->coeffs_safe) FQ_CUDA(cudaMemcpyAsync(a->coeffs_safe, dout + ocos, 96 * (size_t)Ns * P, cudaMemcpyDeviceToHost, st));
  if (a->cost_whole)
  {
    FQ_CUDA(cudaMemcpyAsync(a->cost_whole, dout + ocw, 8 * ncw, cudaMemcpyDeviceToHost, st));
    FQ_CUDA(cudaMemcpyAsync(a->feasible_whole, dout + ofew, ncw, cudaMemcpyDeviceToHost, st));
  }
  if (a->cost_safe)
  {
    FQ_CUDA(cudaMemcpyAsync(a->cost_safe, dout + ocs, 8 * ncs, cudaMemcpyDeviceToHost, st));
    FQ_CUDA(cudaMemcpyAsync(a->feasible_safe, dout + ofes, ncs, cudaMemcpyDeviceToHost, st));
  }
  if (as)
  {
    if (as->cand_ofs_whole) FQ_CUDA(cudaMemcpyAsync(as->cand_ofs_whole, dout + ocaw, 4 * (size_t)(P + 1), cudaMemcpyDeviceToHost, st));
    if (as->cand_ofs_safe) FQ_CUDA(cudaMemcpyAsync(as->cand_ofs_safe, dout + ocas, 4 * (size_t)(P + 1), cudaMemcpyDeviceToHost, st));
    if (as->sigma_whole) FQ_CUDA(cudaMemcpyAsync(as->sigma_whole, dout + osgw, (size_t)P * Nw, cudaMemcpyDeviceToHost, st));
    if (as->sigma_safe) FQ_CUDA(cudaMemcpyAsync(as->sigma_safe, dout + osgs, (size_t)P * Ns, cudaMemcpyDeviceToHost, st));
  }
  if (win)
  { // the caller's window arrays were copied into the upload above, so the next_* outputs may alias them
    auto back = [&](void* host, const void* dev, size_t elem) {
      return host ? cudaMemcpyAsync(host, dev, elem * (size_t)P, cudaMemcpyDeviceToHost, st) : cudaSuccess;
    };
    FQ_CUDA(back(win->factor_whole, dw.factor_whole, 8));   FQ_CUDA(back(win->factor_safe, dw.factor_safe, 8));
    FQ_CUDA(back(win->trials_whole, dw.trials_whole, 4));   FQ_CUDA(back(win->trials_safe, dw.trials_safe, 4));
    FQ_CUDA(back(win->next_init_whole, dw.next_init_whole, 8)); FQ_CUDA(back(win->next_final_whole, dw.next_final_whole, 8));
    FQ_CUDA(back(win->next_init_safe, dw.next_init_safe, 8));   FQ_CUDA(back(win->next_final_safe, dw.next_final_safe, 8));
  }
  if (ex)
  {
    if (ex->exact_whole) FQ_CUDA(cudaMemcpyAsync(ex->exact_whole, dx.exact_whole, 4 * (size_t)P, cudaMemcpyDeviceToHost, st));
    if (ex->exact_safe) FQ_CUDA(cudaMemcpyAsync(ex->exact_safe, dx.exact_safe, 4 * (size_t)P, cudaMemcpyDeviceToHost, st));
    if (ex->nodes_whole) FQ_CUDA(cudaMemcpyAsync(ex->nodes_whole, dx.nodes_whole, 8 * (size_t)P, cudaMemcpyDeviceToHost, st));
    if (ex->nodes_safe) FQ_CUDA(cudaMemcpyAsync(ex->nodes_safe, dx.nodes_safe, 8 * (size_t)P, cudaMemcpyDeviceToHost, st));
  }
  if (dc)
  {
    auto back = [&](void* host, const void* dev, size_t bytes) { return host ? cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, st) : cudaSuccess; };
    FQ_CUDA(back(dc->face_ofs_whole, dd.face_ofs_whole, 4 * (size_t)(cw.n_poly + 1)));
    FQ_CUDA(back(dc->face_ofs_safe, dd.face_ofs_safe, 4 * (size_t)(cs.n_poly + 1)));
    FQ_CUDA(back(dc->Ab_whole, dd.Ab_whole, 32 * (size_t)P * a->max_faces_whole));
    FQ_CUDA(back(dc->Ab_safe, dd.Ab_safe, 32 * (size_t)P * a->max_faces_safe));
    FQ_CUDA(back(dc->E, dd.E, 24 * (size_t)P));                   FQ_CUDA(back(dc->M, dd.M, 24 * (size_t)P));
    FQ_CUDA(back(dc->status_whole, dd.status_whole, 4 * (size_t)P)); FQ_CUDA(back(dc->status_safe, dd.status_safe, 4 * (size_t)P));
  }
  if (deferred) { ctx->pending = true; return 0; }
  FQ_CUDA(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int fq_replan_pairs(fq_ctx* ctx, const fq_pair_args* a)
{
  if (ctx && (ctx->is_group || ctx->comm)) return fq_replan_pairs_sharded(ctx, a, false);
  return fq_replan_pairs_host_ex(ctx, a, false, nullptr, true);
}
extern "C" int fq_replan_pairs_async(fq_ctx* ctx, const fq_pair_args* a)
{
  if (ctx && (ctx->is_group || ctx->comm)) return fq_replan_pairs_sharded(ctx, a, true);
  return fq_replan_pairs_host_ex(ctx, a, true, nullptr, true);
}

extern "C" int fq_replan_pairs_assign(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as)
{
  if (!ctx) return FQ_E_ARG;
  if (!as) return fq_fail(ctx, FQ_E_ARG, "assign is NULL");
  if (ctx->is_group || ctx->comm) return fq_replan_pairs_sharded(ctx, a, false, as);
  return fq_replan_pairs_host_ex(ctx, a, false, nullptr, true, as);
}
extern "C" int fq_replan_pairs_assign_async(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as)
{
  if (!ctx) return FQ_E_ARG;
  if (!as) return fq_fail(ctx, FQ_E_ARG, "assign is NULL");
  if (ctx->is_group || ctx->comm) return fq_replan_pairs_sharded(ctx, a, true, as);
  return fq_replan_pairs_host_ex(ctx, a, true, nullptr, true, as);
}

extern "C" int fq_replan_pairs_window(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win)
{
  if (!ctx) return FQ_E_ARG;
  if (!as) return fq_fail(ctx, FQ_E_ARG, "assign is NULL");
  if (!win) return fq_fail(ctx, FQ_E_ARG, "window is NULL");
  if (ctx->is_group || ctx->comm) return fq_replan_pairs_sharded(ctx, a, false, as, win);
  return fq_replan_pairs_host_ex(ctx, a, false, nullptr, true, as, win);
}
extern "C" int fq_replan_pairs_window_async(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win)
{
  if (!ctx) return FQ_E_ARG;
  if (!as) return fq_fail(ctx, FQ_E_ARG, "assign is NULL");
  if (!win) return fq_fail(ctx, FQ_E_ARG, "window is NULL");
  if (ctx->is_group || ctx->comm) return fq_replan_pairs_sharded(ctx, a, true, as, win);
  return fq_replan_pairs_host_ex(ctx, a, true, nullptr, true, as, win);
}

// host variants of the exact chain: one context on one GPU.  Gathering the per-corridor exact / nodes arrays of a
// multi-GPU context would need a second exchange besides the records', so those contexts are refused.
namespace
{
int exact_host(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win, const fq_pair_exact* ex,
               bool deferred)
{
  if (!ctx) return FQ_E_ARG;
  if (!ex) return fq_fail(ctx, FQ_E_ARG, "exact is NULL");
  if (!as) return fq_fail(ctx, FQ_E_ARG, "assign is NULL");
  if (ctx->is_group || ctx->comm) return fq_fail(ctx, FQ_E_ARG, "fq_replan_pairs_exact: multi-GPU contexts are not supported (use _exact_dev)");
  return fq_replan_pairs_host_ex(ctx, a, deferred, nullptr, true, as, win, ex);
}
}  // namespace

extern "C" int fq_replan_pairs_exact(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                     const fq_pair_exact* ex)
{
  return exact_host(ctx, a, as, win, ex, false);
}
extern "C" int fq_replan_pairs_exact_async(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                           const fq_pair_exact* ex)
{
  return exact_host(ctx, a, as, win, ex, true);
}

// host variants of the decomposing chain: one context on one GPU, as the exact chain's
namespace
{
int decomp_host(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win, const fq_pair_exact* ex,
                const fq_pair_decomp* dc, bool deferred)
{
  if (!ctx) return FQ_E_ARG;
  if (!dc) return fq_fail(ctx, FQ_E_ARG, "decomp is NULL");
  if (!as) return fq_fail(ctx, FQ_E_ARG, "assign is NULL");
  if (ctx->is_group || ctx->comm) return fq_fail(ctx, FQ_E_ARG, "fq_replan_pairs_decomp: multi-GPU contexts are not supported (use _decomp_dev)");
  return fq_replan_pairs_host_ex(ctx, a, deferred, nullptr, true, as, win, ex, dc);
}
}  // namespace

extern "C" int fq_replan_pairs_decomp(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                      const fq_pair_exact* ex, const fq_pair_decomp* dc)
{
  return decomp_host(ctx, a, as, win, ex, dc, false);
}
extern "C" int fq_replan_pairs_decomp_async(fq_ctx* ctx, const fq_pair_args* a, const fq_pair_assign* as, const fq_pair_window* win,
                                            const fq_pair_exact* ex, const fq_pair_decomp* dc)
{
  return decomp_host(ctx, a, as, win, ex, dc, true);
}
