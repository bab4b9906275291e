// Chained replan (include/faster_b200.h: fq_replan_pairs*): whole sweep -> selection -> R -> safe sweep -> selection for
// many corridors in one submission.  Reference data flow: faster/src/faster.cpp:406-430 (whole), :474-475 (R), :521-537
// (safe).  Kernels: the batch solve (fq_kernels_t.cuh) and the small kernels of fq_pair.cuh.
#include "fq_ctx.h"

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
};

template <class T>
T* carve(char*& p, size_t count)
{
  T* r = reinterpret_cast<T*>(p);
  p += fq_align16(sizeof(T) * count);
  return r;
}

int check_common(fq_ctx* ctx, const fq_pair_args* a)
{
  if (!a) return fq_fail(ctx, FQ_E_ARG, "args is NULL");
  if (a->n_prob <= 0) return fq_fail(ctx, FQ_E_ARG, "n_prob <= 0");
  if (a->N_whole < 3 || a->N_whole > FQ_MAX_N || a->N_safe < 2 || a->N_safe > FQ_MAX_N) return fq_fail(ctx, FQ_E_ARG, "N out of range");
  if (!(a->DC > 0) || !(a->r_fraction >= 0 && a->r_fraction <= 1)) return fq_fail(ctx, FQ_E_ARG, "DC must be > 0 and r_fraction in [0, 1]");
  if (a->n_fac_whole <= 0 || a->n_fac_safe <= 0 || a->n_sig_whole <= 0 || a->n_sig_safe <= 0)
    return fq_fail(ctx, FQ_E_ARG, "empty factor / assignment grid");
  if ((long long)a->n_prob * a->n_fac_whole * a->n_sig_whole > (1LL << 30) || (long long)a->n_prob * a->n_fac_safe * a->n_sig_safe > (1LL << 30))
    return fq_fail(ctx, FQ_E_ARG, "too many candidates");
  if (!a->x0 || !a->xf_whole || !a->xf_safe || !a->lim || !a->poly_ofs_whole || !a->face_ofs_whole || !a->poly_ofs_safe ||
      !a->face_ofs_safe || !a->factors_whole || !a->factors_safe || !a->results)
    return fq_fail(ctx, FQ_E_ARG, "NULL argument");
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
  const int P = a->n_prob, Nw = a->N_whole, Ns = a->N_safe;
  const size_t ncw = (size_t)P * a->n_fac_whole * a->n_sig_whole, ncs = (size_t)P * a->n_fac_safe * a->n_sig_safe;
  // ---- scratch
  size_t need = 0;
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
      return (size_t)(p - base);
    };
    need = layout(nullptr);
    FQ_CUDA(ctx->d_pair.reserve(need));       // grows only on the first call / a larger batch (synchronous cudaMalloc)
    layout((char*)ctx->d_pair.p);

    uint8_t* feas_w = a->feasible_whole ? a->feasible_whole : s.feas_w;
    uint8_t* feas_s = a->feasible_safe ? a->feasible_safe : s.feas_s;
    double* cost_w = a->cost_whole ? a->cost_whole : s.cost_w;
    double* cost_s = a->cost_safe ? a->cost_safe : s.cost_s;
    double* coeffs_w = a->coeffs_whole ? a->coeffs_whole : s.coeffs_w;
    double* coeffs_s = a->coeffs_safe ? a->coeffs_safe : s.coeffs_s;
    const int mcw = a->n_fac_whole * a->n_sig_whole, mcs = a->n_fac_safe * a->n_sig_safe;
    // the corridors of the two sweeps; each launch adds its candidates and outputs
    FqKernelArgs whole{}, safe{};
    whole.N = Nw; whole.force_final = 1; whole.n_prob = P; whole.x0 = a->x0; whole.xf = a->xf_whole; whole.lim = a->lim;
    whole.poly_ofs = a->poly_ofs_whole; whole.face_ofs = a->face_ofs_whole; whole.Ab = a->Ab_whole; whole.max_faces = a->max_faces_whole;
    safe.N = Ns; safe.force_final = 0; safe.n_prob = P; safe.x0 = s.x0_safe; safe.xf = a->xf_safe; safe.lim = a->lim;
    safe.poly_ofs = a->poly_ofs_safe; safe.face_ofs = a->face_ofs_safe; safe.Ab = a->Ab_safe; safe.max_faces = a->max_faces_safe;

    // ---- whole sweep (faster.cpp:406-418)
    FQ_CUDA(fq_launch_dtbase(P, Nw, a->DC, a->x0, a->xf_whole, a->lim, s.dt_base_w, st));
    FQ_CUDA(fq_launch_expand_grid(P, Nw, a->n_fac_whole, a->n_sig_whole, a->factors_whole, a->sigmas_whole, s.dt_base_w, s.dt_w,
                                  s.sig_w, s.cand_ofs_w, st));
    FqKernelArgs k = whole;
    k.cand_ofs = s.cand_ofs_w; k.dt = s.dt_w; k.sigma = s.sig_w; k.feasible = feas_w; k.cost = cost_w;
    k.sorted_dt = 1; k.ee_width = a->n_sig_whole;         // factor-major grid, ascending factors
    int rc = fq_launch_solve_ctx(ctx, k, mcw, a->max_poly_faces_whole, st);
    if (rc) return rc;
    FqSelectMultiArgs sw;
    sw.n_prob = P; sw.N = Nw; sw.n_sig = a->n_sig_whole; sw.cand_ofs = s.cand_ofs_w; sw.dt = s.dt_w; sw.sigma = s.sig_w;
    sw.feasible = feas_w; sw.cost = cost_w; sw.win_idx = s.win_idx_w; sw.win_cost = s.win_cost_w; sw.win_dt = s.win_dt_w;
    sw.win_sigma = s.win_sig_w; sw.win_ofs = s.win_ofs;
    FQ_CUDA(fq_launch_select_multi(sw, st));
    // coefficients of the winners: one candidate per corridor through the same kernel (losers' dt is NaN -> "not solved")
    k = whole;
    k.cand_ofs = s.win_ofs; k.dt = s.win_dt_w; k.sigma = s.win_sig_w; k.feasible = s.re_feas; k.cost = s.re_cost; k.coeffs = coeffs_w;
    rc = fq_launch_solve_ctx(ctx, k, 1, a->max_poly_faces_whole, st);
    if (rc) return rc;
    // ---- R (faster.cpp:474-475) and the safe sweep from it (faster.cpp:521-527)
    FqPairMidArgs m;
    m.n_prob = P; m.N = Nw; m.DC = a->DC; m.r_fraction = a->r_fraction; m.coeffs = coeffs_w; m.win_dt = s.win_dt_w;
    m.win_idx = s.win_idx_w; m.x0_safe = s.x0_safe; m.n_samples = s.n_samples; m.k_safe = s.k_safe;
    FQ_CUDA(fq_launch_pair_mid(m, st));
    FQ_CUDA(fq_launch_dtbase(P, Ns, a->DC, s.x0_safe, a->xf_safe, a->lim, s.dt_base_s, st));
    FQ_CUDA(fq_launch_expand_grid(P, Ns, a->n_fac_safe, a->n_sig_safe, a->factors_safe, a->sigmas_safe, s.dt_base_s, s.dt_s,
                                  s.sig_s, s.cand_ofs_s, st));
    k = safe;
    k.cand_ofs = s.cand_ofs_s; k.dt = s.dt_s; k.sigma = s.sig_s; k.feasible = feas_s; k.cost = cost_s;
    k.sorted_dt = 1; k.ee_width = a->n_sig_safe;
    rc = fq_launch_solve_ctx(ctx, k, mcs, a->max_poly_faces_safe, st);
    if (rc) return rc;
    FqSelectMultiArgs ss = sw;
    ss.N = Ns; ss.n_sig = a->n_sig_safe; ss.cand_ofs = s.cand_ofs_s; ss.dt = s.dt_s; ss.sigma = s.sig_s; ss.feasible = feas_s;
    ss.cost = cost_s; ss.win_idx = s.win_idx_s; ss.win_cost = s.win_cost_s; ss.win_dt = s.win_dt_s; ss.win_sigma = s.win_sig_s;
    FQ_CUDA(fq_launch_select_multi(ss, st));
    if (a->coeffs_safe)
    {
      k = safe;
      k.cand_ofs = s.win_ofs; k.dt = s.win_dt_s; k.sigma = s.win_sig_s; k.feasible = s.re_feas; k.cost = s.re_cost; k.coeffs = coeffs_s;
      rc = fq_launch_solve_ctx(ctx, k, 1, a->max_poly_faces_safe, st);
      if (rc) return rc;
    }
    FqPairFinalArgs f;
    f.n_prob = P; f.n_sig_w = a->n_sig_whole; f.n_sig_s = a->n_sig_safe; f.win_idx_w = s.win_idx_w; f.win_idx_s = s.win_idx_s;
    f.n_samples = s.n_samples; f.k_safe = s.k_safe; f.win_cost_w = s.win_cost_w; f.win_cost_s = s.win_cost_s;
    f.win_dt_w = s.win_dt_w; f.win_dt_s = s.win_dt_s; f.dt_base_w = s.dt_base_w; f.dt_base_s = s.dt_base_s; f.x0_safe = s.x0_safe;
    f.out = a->results;
    FQ_CUDA(fq_launch_pair_final(f, st));
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

int fq_replan_pairs_host_ex(fq_ctx* ctx, const fq_pair_args* a, bool deferred, fq_pair_result** d_results, bool copy_results)
{
  if (!ctx) return FQ_E_ARG;
  if (int rc = fq_settle(ctx)) return rc;
  if (int rc = check_common(ctx, a)) return rc;
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
  if (const char* why = check(a->poly_ofs_whole, a->face_ofs_whole, a->Ab_whole, &cw)) return fq_fail(ctx, FQ_E_ARG, why);
  if (const char* why = check(a->poly_ofs_safe, a->face_ofs_safe, a->Ab_safe, &cs)) return fq_fail(ctx, FQ_E_ARG, why);
  if (!fq_scan_all_finite(a->x0, 9 * (size_t)P) || !fq_scan_all_finite(a->xf_whole, 9 * (size_t)P) || !fq_scan_all_finite(a->xf_safe, 9 * (size_t)P))
    return fq_fail(ctx, FQ_E_ARG, "non-finite value in x0/xf");
  if (!fq_scan_all_positive_finite(a->lim, 3 * (size_t)P) || !fq_scan_all_positive_finite(a->factors_whole, (size_t)a->n_fac_whole) ||
      !fq_scan_all_positive_finite(a->factors_safe, (size_t)a->n_fac_safe))
    return fq_fail(ctx, FQ_E_ARG, "limits and factors must be finite and > 0");
  for (int i = 1; i < a->n_fac_whole; i++)
    if (a->factors_whole[i] < a->factors_whole[i - 1]) return fq_fail(ctx, FQ_E_ARG, "factors_whole must be ascending");
  for (int i = 1; i < a->n_fac_safe; i++)
    if (a->factors_safe[i] < a->factors_safe[i - 1]) return fq_fail(ctx, FQ_E_ARG, "factors_safe must be ascending");
  if (cw.n_poly > 0 && !a->sigmas_whole) return fq_fail(ctx, FQ_E_ARG, "sigmas_whole is NULL");
  if (cs.n_poly > 0 && !a->sigmas_safe) return fq_fail(ctx, FQ_E_ARG, "sigmas_safe is NULL");
  // assignments must name existing polytopes of EVERY corridor they are applied to
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
  const size_t ncw = (size_t)P * a->n_fac_whole * a->n_sig_whole, ncs = (size_t)P * a->n_fac_safe * a->n_sig_safe;
  size_t o = 0;
  auto put = [&](size_t bytes) { const size_t at = o; o = fq_align16(o + bytes); return at; };
  const size_t oAbw = put(32 * (size_t)std::max(cw.n_face, 1)), oAbs = put(32 * (size_t)std::max(cs.n_face, 1));
  const size_t ox0 = put(72 * (size_t)P), oxfw = put(72 * (size_t)P), oxfs = put(72 * (size_t)P), olim = put(24 * (size_t)P);
  const size_t ofw = put(8 * (size_t)a->n_fac_whole), ofs = put(8 * (size_t)a->n_fac_safe);
  const size_t opow = put(4 * (size_t)(P + 1)), ofow = put(4 * (size_t)(cw.n_poly + 1));
  const size_t opos = put(4 * (size_t)(P + 1)), ofos = put(4 * (size_t)(cs.n_poly + 1));
  const size_t osw = put((size_t)a->n_sig_whole * Nw), oss = put((size_t)a->n_sig_safe * Ns);
  const size_t in_bytes = o;
  o = 0;
  const size_t ores = put(sizeof(fq_pair_result) * (size_t)P);
  const size_t ocow = put(96 * (size_t)Nw * P), ocos = put(96 * (size_t)Ns * P);
  const size_t ocw = put(8 * ncw), ocs = put(8 * ncs), ofew = put(ncw), ofes = put(ncs);
  const size_t out_bytes = o;
  FQ_CUDA(ctx->h_in.reserve(in_bytes));
  FQ_CUDA(ctx->d_pair_io.reserve(in_bytes + out_bytes));
  char* hi = (char*)ctx->h_in.p;
  char* din = (char*)ctx->d_pair_io.p;
  char* dout = din + in_bytes;
  if (cw.n_face) std::memcpy(hi + oAbw, a->Ab_whole, 32 * (size_t)cw.n_face);
  if (cs.n_face) std::memcpy(hi + oAbs, a->Ab_safe, 32 * (size_t)cs.n_face);
  std::memcpy(hi + ox0, a->x0, 72 * (size_t)P);      std::memcpy(hi + oxfw, a->xf_whole, 72 * (size_t)P);
  std::memcpy(hi + oxfs, a->xf_safe, 72 * (size_t)P); std::memcpy(hi + olim, a->lim, 24 * (size_t)P);
  std::memcpy(hi + ofw, a->factors_whole, 8 * (size_t)a->n_fac_whole);
  std::memcpy(hi + ofs, a->factors_safe, 8 * (size_t)a->n_fac_safe);
  std::memcpy(hi + opow, a->poly_ofs_whole, 4 * (size_t)(P + 1)); std::memcpy(hi + ofow, a->face_ofs_whole, 4 * (size_t)(cw.n_poly + 1));
  std::memcpy(hi + opos, a->poly_ofs_safe, 4 * (size_t)(P + 1));  std::memcpy(hi + ofos, a->face_ofs_safe, 4 * (size_t)(cs.n_poly + 1));
  if (a->sigmas_whole) std::memcpy(hi + osw, a->sigmas_whole, (size_t)a->n_sig_whole * Nw);
  if (a->sigmas_safe) std::memcpy(hi + oss, a->sigmas_safe, (size_t)a->n_sig_safe * Ns);
  cudaStream_t st = ctx->stream;
  FQ_CUDA(cudaMemcpyAsync(din, hi, in_bytes, cudaMemcpyHostToDevice, st));
  fq_pair_args d = *a;
  d.x0 = (const double*)(din + ox0); d.xf_whole = (const double*)(din + oxfw); d.xf_safe = (const double*)(din + oxfs);
  d.lim = (const double*)(din + olim);
  d.poly_ofs_whole = (const int*)(din + opow); d.face_ofs_whole = (const int*)(din + ofow); d.Ab_whole = (const double*)(din + oAbw);
  d.poly_ofs_safe = (const int*)(din + opos); d.face_ofs_safe = (const int*)(din + ofos); d.Ab_safe = (const double*)(din + oAbs);
  d.factors_whole = (const double*)(din + ofw); d.factors_safe = (const double*)(din + ofs);
  d.sigmas_whole = a->sigmas_whole ? (const uint8_t*)(din + osw) : nullptr;
  d.sigmas_safe = a->sigmas_safe ? (const uint8_t*)(din + oss) : nullptr;
  d.feasible_whole = a->feasible_whole ? (uint8_t*)(dout + ofew) : nullptr; d.cost_whole = a->cost_whole ? (double*)(dout + ocw) : nullptr;
  d.feasible_safe = a->feasible_safe ? (uint8_t*)(dout + ofes) : nullptr;   d.cost_safe = a->cost_safe ? (double*)(dout + ocs) : nullptr;
  d.coeffs_whole = a->coeffs_whole ? (double*)(dout + ocow) : nullptr;       d.coeffs_safe = a->coeffs_safe ? (double*)(dout + ocos) : nullptr;
  d.results = (fq_pair_result*)(dout + ores);
  d.max_faces_whole = std::max(cw.max_faces, 1); d.max_poly_faces_whole = cw.max_poly_faces; d.max_faces_safe = std::max(cs.max_faces, 1); d.max_poly_faces_safe = cs.max_poly_faces;
  // a NULL cost/flag output still needs a device array of its own kind: the chain allocates it in its scratch
  if ((d.feasible_whole == nullptr) != (d.cost_whole == nullptr) || (d.feasible_safe == nullptr) != (d.cost_safe == nullptr))
    return fq_fail(ctx, FQ_E_ARG, "feasible_* and cost_* must be given (or omitted) together");
  int rc = fq_replan_pairs_dev(ctx, &d, nullptr, st);
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
