// Device side of the chained replan (Faster::replan(), reference faster/src/faster.cpp:406-430,:475,:521-537): for many
// corridors at once
//     whole sweep  ->  genNewTraj selection  ->  R = sample k_safe of fillX  ->  safe sweep from R  ->  selection
// without a host round trip.  The solves are the ordinary batch kernel (fq_kernels_t.cuh); this file holds the small
// kernels between them.  All of them are latency-trivial (one thread / one CTA per corridor, or a grid-stride copy).
#pragma once
#include "fq_assign.h"
#include "fq_dtinit.h"
#include "fq_paths.h"
#include "fq_queue.h"
#include "fq_window.h"

namespace fqp
{
// dt_base[j] = max(getDTInitial(x0_j, xf_j), 2 DC)  (findDT, solverGurobi.cpp:494-497).  x0 rows with a NaN (a safe
// problem whose whole sweep found nothing) give NaN, which makes every candidate of the problem "not solved".
__global__ void fq_dtbase_kernel(int n_prob, int N, double DC, const double* __restrict__ x0, const double* __restrict__ xf,
                                 const double* __restrict__ lim, double* __restrict__ dt_base)
{ // four lanes per problem: one per axis (the cubic / quadratic root finding is the long part), the fourth idles
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  const int j = tid >> 2, ax = tid & 3;
  const bool live = j < n_prob;
  double a[9], b[9], l[3];
  bool ok = live;
  float worst = 0;
  if (live)
  {
    for (int i = 0; i < 9; i++) { a[i] = x0[j * 9 + i]; b[i] = xf[j * 9 + i]; ok = ok && isfinite(a[i]) && isfinite(b[i]); }
    for (int i = 0; i < 3; i++) { l[i] = lim[j * 3 + i]; ok = ok && l[i] > 0 && isfinite(l[i]); }
    if (ok && ax < 3) worst = fqdt::dt_axis(a, b, l, ax);
  }
  worst = fmaxf(worst, __shfl_xor_sync(0xffffffffu, worst, 1));
  worst = fmaxf(worst, __shfl_xor_sync(0xffffffffu, worst, 2));
  if (!live || ax != 0) return;
  if (!ok) { dt_base[j] = __longlong_as_double(0x7ff8000000000000ll); return; }
  const double dti = fqdt::dt_from_worst(worst, N);
  const double floor2 = FQ_MUL(2.0, DC);
  dt_base[j] = dti > floor2 ? dti : floor2;            // std::max(getDTInitial(), 2 * DC)
}

// candidates of problem j = factors x assignments: dt = factor * dt_base[j] (findDT), sigma from the shared list
__global__ void fq_expand_grid_kernel(int n_prob, int N, int n_fac, int n_sig, const double* __restrict__ factors,
                                      const uint8_t* __restrict__ sig_list, const double* __restrict__ dt_base,
                                      double* __restrict__ dt, uint8_t* __restrict__ sigma, int* __restrict__ cand_ofs)
{
  const long long per = (long long)n_fac * n_sig, total = per * n_prob;
  for (long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x; c < total; c += (long long)gridDim.x * blockDim.x)
  {
    const int j = (int)(c / per);
    const int r = (int)(c - (long long)j * per);
    const int f = r / n_sig, s = r - f * n_sig;
    dt[c] = FQ_MUL(factors[f], dt_base[j]);
    for (int t = 0; t < N; t++) sigma[c * N + t] = sig_list ? sig_list[(size_t)s * N + t] : (uint8_t)0;
  }
  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j <= n_prob; j += (long long)gridDim.x * blockDim.x)
    cand_ofs[j] = (int)(j * per);
}

// ---- per-corridor assignment lists (fq_replan_pairs_assign*; the lists are defined in fq_assign.h)

// per-corridor windows (fq_replan_pairs_window*, fq_window.h): one thread per corridor accumulates F_j = F(init[j],
// final[j], inc) into row j of fac (its first max_fac factors) and writes |F_j|, or -1 when the window is refused.  A count
// above max_fac makes fq_assign_offsets_kernel empty the sweep.
__global__ void fq_window_factors_kernel(int n_prob, int max_fac, const double* __restrict__ init, const double* __restrict__ final_,
                                         double inc, double* __restrict__ fac, int* __restrict__ n_fac_j)
{
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_prob) return;
  n_fac_j[j] = fqw::factors(init[j], final_[j], inc, fac + (size_t)j * max_fac, max_fac);
}

// cand_ofs[0 .. n_prob] = exclusive scan of n_fac x |L(N, P_j, all_limit)|, P_j from poly_ofs.  One CTA (any size up to
// 1024): every thread scans a contiguous run of corridors.  The sweep's buffers were sized for n_cand candidates; when a
// corridor has more than max_poly polytopes, a list is refused (longer than 2^20) or the total is not n_cand, EVERY range
// is left empty (cand_ofs all 0): no candidate is expanded or solved and every corridor's winner of the sweep is "none".
// Per-corridor windows (n_fac_j != NULL): corridor j has n_fac_j[j] factors instead of n_fac, which then bounds them (a
// refused window, -1, or more than n_fac factors also empties the sweep), and n_cand is a capacity: the total must not
// exceed it.
__global__ void __launch_bounds__(1024) fq_assign_offsets_kernel(int n_prob, int N, int n_fac, long long all_limit, int max_poly,
                                                                 long long n_cand, const int* __restrict__ poly_ofs,
                                                                 int* __restrict__ cand_ofs, const int* __restrict__ n_fac_j = nullptr)
{
  __shared__ long long s_run[1024];
  __shared__ long long s_total;
  __shared__ int s_bad;
  const int T = blockDim.x, tid = threadIdx.x;
  const int per = (n_prob + T - 1) / T;
  const int j0 = min(n_prob, tid * per), j1 = min(n_prob, j0 + per);
  if (tid == 0) s_bad = 0;
  __syncthreads();
  long long sum = 0;
  bool bad = false;
  for (int j = j0; j < j1; j++)
  {
    const int P = poly_ofs[j + 1] - poly_ofs[j];
    const long long L = fqa::list_len(N, P, all_limit);
    const int nf = n_fac_j ? n_fac_j[j] : n_fac;
    if (P < 0 || P > max_poly || L < 0 || nf < 0 || nf > n_fac) bad = true;
    else sum += L * nf;
  }
  if (bad) s_bad = 1;
  s_run[tid] = sum;
  __syncthreads();
  if (tid == 0)
  {
    long long run = 0;
    for (int i = 0; i < T; i++) { const long long x = s_run[i]; s_run[i] = run; run += x; }
    s_total = run;
    if (n_fac_j ? run > n_cand : run != n_cand) s_bad = 1;
  }
  __syncthreads();
  const bool empty = s_bad != 0;
  long long run = s_run[tid];
  for (int j = j0; j < j1; j++)
  {
    cand_ofs[j] = empty ? 0 : (int)run;
    if (!empty) run += fqa::list_len(N, poly_ofs[j + 1] - poly_ofs[j], all_limit) * (n_fac_j ? n_fac_j[j] : n_fac);
  }
  if (tid == 0) cand_ofs[n_prob] = empty ? 0 : (int)s_total;
}

// candidates of corridor j = factors x L_j, factor-major: dt = factor * dt_base[j] (as fq_expand_grid_kernel), sigma =
// the assignment's unranked index within L_j.  One CTA per corridor, grid-striding over its own candidates; the binomials
// of the non-decreasing unranking sit in shared memory.  Per-corridor windows (n_fac_j != NULL): `factors` holds one row of
// n_fac factors per corridor, of which corridor j uses the first n_fac_j[j].
__global__ void __launch_bounds__(256) fq_expand_assign_kernel(int n_prob, int N, int n_fac, long long all_limit,
                                                               const double* __restrict__ factors, const double* __restrict__ dt_base,
                                                               const int* __restrict__ poly_ofs, const int* __restrict__ cand_ofs,
                                                               double* __restrict__ dt, uint8_t* __restrict__ sigma,
                                                               const int* __restrict__ n_fac_j = nullptr)
{
  __shared__ long long s_binom[48 * 17];
  for (int i = threadIdx.x; i < 48 * 17; i += blockDim.x) s_binom[i] = fqa::binom(i / 17, i % 17);
  __syncthreads();
  const int j = blockIdx.x;
  if (j >= n_prob) return;
  const int c0 = cand_ofs[j], n = cand_ofs[j + 1] - c0;
  const int P = poly_ofs[j + 1] - poly_ofs[j];
  const long long L = fqa::list_len(N, P, all_limit);
  const int nf = n_fac_j ? n_fac_j[j] : n_fac;
  const double* fac = n_fac_j ? factors + (size_t)j * n_fac : factors;
  if (n <= 0 || L <= 0 || (long long)n != L * nf) return;           // an emptied sweep (fq_assign_offsets_kernel)
  const bool all = fqa::use_all(N, P, all_limit);
  const double base = dt_base[j];
  for (int i = threadIdx.x; i < n; i += blockDim.x)
  {
    const int f = (int)(i / L);
    dt[c0 + i] = FQ_MUL(fac[f], base);
    fqa::unrank(N, P, all, i - (long long)f * L, s_binom, sigma + (size_t)(c0 + i) * N);
  }
}

// genNewTraj's selection (solverGurobi.cpp:445-472) for every problem of a batch: the winner is the feasible candidate
// with the smallest dt (= first feasible factor of the ascending sweep), among those the smallest cost, among those the
// lowest index -- three exact reductions on the ordered bit patterns of the (positive) doubles.  One CTA per problem.
// Also emits the one-candidate-per-problem list that the coefficient re-solve of the winners runs on.

__global__ void __launch_bounds__(128) fq_select_multi_kernel(const FqSelectMultiArgs a)
{
  __shared__ unsigned long long s_dt, s_cost;
  __shared__ int s_idx;
  const int j = blockIdx.x;
  if (j >= a.n_prob) return;
  const int c0 = a.cand_ofs[j], n = a.cand_ofs[j + 1] - c0;
  if (threadIdx.x == 0) { s_dt = ~0ull; s_cost = ~0ull; s_idx = 0x7fffffff; }
  __syncthreads();
  unsigned long long m = ~0ull;
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (a.feasible[c0 + i])
    {
      const unsigned long long b = (unsigned long long)__double_as_longlong(a.dt[c0 + i]);
      m = b < m ? b : m;
    }
  if (m != ~0ull) atomicMin(&s_dt, m);
  __syncthreads();
  const unsigned long long dtb = s_dt;
  if (dtb != ~0ull)
  {
    m = ~0ull;
    for (int i = threadIdx.x; i < n; i += blockDim.x)
      if (a.feasible[c0 + i] && (unsigned long long)__double_as_longlong(a.dt[c0 + i]) == dtb)
      {
        const unsigned long long b = (unsigned long long)__double_as_longlong(a.cost[c0 + i]);
        m = b < m ? b : m;
      }
    if (m != ~0ull) atomicMin(&s_cost, m);
    __syncthreads();
    const unsigned long long cb = s_cost;
    int mi = 0x7fffffff;
    for (int i = threadIdx.x; i < n; i += blockDim.x)
      if (a.feasible[c0 + i] && (unsigned long long)__double_as_longlong(a.dt[c0 + i]) == dtb &&
          (unsigned long long)__double_as_longlong(a.cost[c0 + i]) == cb)
      { mi = i; break; }
    if (mi != 0x7fffffff) atomicMin(&s_idx, mi);
    __syncthreads();
  }
  const int w = dtb != ~0ull ? s_idx : -1;
  if (threadIdx.x == 0)
  {
    a.win_idx[j] = w;
    a.win_cost[j] = w >= 0 ? a.cost[c0 + w] : INFINITY;
    a.win_dt[j] = w >= 0 ? a.dt[c0 + w] : __longlong_as_double(0x7ff8000000000000ll);
    a.win_ofs[j] = j;
    if (j == a.n_prob - 1) a.win_ofs[a.n_prob] = a.n_prob;
  }
  if (a.win_sigma)
    for (int t = threadIdx.x; t < a.N; t += blockDim.x) a.win_sigma[(size_t)j * a.N + t] = w >= 0 && a.sigma ? a.sigma[(size_t)(c0 + w) * a.N + t] : (uint8_t)0;
}

// fillX's sample clock (solverGurobi.cpp:122-168): the reference's accumulated sample time and lagging interval index.  A
// clock only moves forward; sample i is always reached through samples 0 .. i-1, so every sample has the bits of fillX's.
struct SampleClock
{
  double t = 0;
  int interval = 0, next = 0;           // `next`: the first sample not reached yet
};

// sample i (>= the clock's last one) of corridor j's whole winner: pos vel accel jerk into o; the last sample (n - 1) is at rest
FQ_HD void sample_at(SampleClock& c, int i, const double* coeffs_j, int N, double dt, double DC, int n, double* o)
{
  for (; c.next <= i; c.next++)
  {
    c.t = FQ_ADD(c.t, DC);
    if (c.t > FQ_MUL(dt, (double)(c.interval + 1))) c.interval = c.interval + 1 < N - 1 ? c.interval + 1 : N - 1;
  }
  const double tau = FQ_SUB(c.t, FQ_MUL((double)c.interval, dt));
  double x[12];
  for (int q = 0; q < 12; q++) x[q] = coeffs_j[c.interval * 12 + q];
  fqdt::eval_sample(x, tau, o);
  if (i == n - 1)
    for (int q = 3; q < 12; q++) o[q] = 0.0;                       // :165-167: the last sample is at rest
}

// Between the two sweeps: R = X_temp_[k_safe] of the whole winner (faster.cpp:475; fillX, solverGurobi.cpp:122-168).  k_safe
// is r_index[j] from fq_pair_hr_kernel (findIndexR, faster.cpp:173-216; < 0: no safe path is needed, so no R and k_safe =
// indexH = n - 1, :465-469), or without r_index min(n - 1, (int)(r_fraction * n)).  One thread per problem.

__global__ void fq_pair_mid_kernel(const FqPairMidArgs a)
{
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.n_prob) return;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  if (a.win_idx[j] < 0)
  {
    for (int i = 0; i < 9; i++) a.x0_safe[j * 9 + i] = nan;
    a.n_samples[j] = 0; a.k_safe[j] = -1;
    return;
  }
  const double dt = a.win_dt[j], DC = a.DC;
  const int n = fqdt::num_samples(a.N, dt, DC);
  int k;
  if (a.r_index)
  {
    k = a.r_index[j];
    if (k < 0)
    {
      for (int i = 0; i < 9; i++) a.x0_safe[j * 9 + i] = nan;
      a.n_samples[j] = n; a.k_safe[j] = n - 1;
      return;
    }
  }
  else
  {
    k = (int)(a.r_fraction * (double)n);
    k = k < 0 ? 0 : (k > n - 1 ? n - 1 : k);
  }
  SampleClock c;
  double o[12];
  sample_at(c, k, a.coeffs + (size_t)j * a.N * 12, a.N, dt, DC, n, o);
  for (int i = 0; i < 9; i++) a.x0_safe[j * 9 + i] = o[i];
  a.n_samples[j] = n; a.k_safe[j] = k;
}

// findIndexH and findIndexR (faster.cpp:173-251) for every corridor, from its whole winner and its unknown cloud; one CTA per
// corridor, any block size.
//   H: for the samples i = 0, 10, 20, ... < n of X_temp_ in order, the nearest unknown point (kdtree_unk_.nearestKSearch)
//      with pcl::PointXYZ's float coordinates and FLANN's float L2 order ((0 + dx^2) + dy^2) + dz^2; the first sample with
//      sqrtf(d^2) < drone_radius (in double) sets needToComputeSafePath and indexH = (int)(delta_H i); none: indexH = n - 1.
//      Since sqrtf is monotone, "the nearest point is that close" is "some point is that close": the CTA scans the cloud for
//      any such point (__syncthreads_or), which neither thread count nor warp order can change.  With an indexed map
//      (fq_map.h) it scans only the cells within drone_radius of the sample, widened by a bound on the float rounding of
//      the point and of the distance ((|q| + drone_radius) 2^-20, far above it) and by one cell: they hold every point that
//      close, at any coordinate magnitude.
//   R: the first i in 0 .. indexH whose braking distance sign(v (H - p)) v^2 / (2 delta_a a_max) exceeds |H - p| in x or y,
//      else indexH.  Threads take strided samples, each walking its own sample clock; the first index is a block minimum.
// (flann_l2 and the float FQ_F* operations: fq_paths.h)

// findIndexR's test of one sample (faster.cpp:186-196): any of x, y with a braking distance above |H - p|
FQ_HD bool brakes_past(const double* H, const double* o, double delta_a, double a_max)
{
  const double den = FQ_MUL(FQ_MUL(2.0, delta_a), a_max);
  bool hit = false;
  for (int ax = 0; ax < 2; ax++)
  {
    const double d = FQ_SUB(H[ax], o[ax]), v = o[3 + ax], sv = FQ_MUL(v, d);
    const double sgn = sv > 0 ? 1.0 : (sv < 0 ? -1.0 : 0.0);             // Eigen's sign(): 0 for 0
    const double b = FQ_DIV(FQ_MUL(sgn, FQ_MUL(v, v)), den);
    hit = hit || b > fabs(d);
  }
  return hit;
}

__global__ void __launch_bounds__(256) fq_pair_hr_kernel(const FqPairHrArgs a)
{
  __shared__ float s_q[3];
  __shared__ double s_H[2];
  __shared__ int s_k;
  const int j = blockIdx.x, tid = threadIdx.x, T = blockDim.x;
  if (j >= a.n_prob) return;
  auto put = [&](int r, int need, int h) {
    if (tid != 0) return;
    a.r_index[j] = r; a.need[j] = (uint8_t)need;
    if (a.need_out) a.need_out[j] = (uint8_t)need;
    if (a.index_H) a.index_H[j] = h;
  };
  if (a.win_idx[j] < 0) { put(-1, 0, -1); return; }
  const double dt = a.win_dt[j], DC = a.DC;
  const int N = a.N, n = fqdt::num_samples(N, dt, DC);
  const double* co = a.coeffs + (size_t)j * N * 12;
  const FqMapDev* M = a.maps ? a.maps[a.map_index ? a.map_index[j] : 0] : nullptr;
  const int lo = M ? 0 : a.unk_ofs[j], hi = M ? M->unk.n : a.unk_ofs[j + 1];
  SampleClock c0;                                                   // thread 0's clock through the H queries
  int hit_i = -1;
  for (int i = 0; i < n && hi > lo; i += 10)
  {
    if (tid == 0)
    {
      double o[12];
      sample_at(c0, i, co, N, dt, DC, n, o);
      for (int q = 0; q < 3; q++) s_q[q] = FQ_F2(o[q]);            // pcl::PointXYZ searchPoint(tmp(0), tmp(1), tmp(2))
    }
    __syncthreads();
    const float q[3] = { s_q[0], s_q[1], s_q[2] };
    int near = 0;
    if (!M)
      for (int p = lo + tid; p < hi && !near; p += T)
        near = (double)FQ_FSQRT(flann_l2(q, a.unk + 3 * (size_t)p)) < a.drone_radius;
    else
    {
      const FqMapGrid& g = M->grid;
      double qlo[3], qhi[3];
      for (int k = 0; k < 3; k++)
      {
        const double r = a.drone_radius + (fabs((double)q[k]) + a.drone_radius) * 0x1p-20;
        qlo[k] = (double)q[k] - r; qhi[k] = (double)q[k] + r;
      }
      int cl[3], ch[3];
      fq_map_range(g, qlo, qhi, cl, ch);
      for (int k = 0; k < 3; k++) { cl[k] = cl[k] > 0 ? cl[k] - 1 : 0; ch[k] = ch[k] < g.dims[k] - 1 ? ch[k] + 1 : g.dims[k] - 1; }
      const int rows = (ch[1] - cl[1] + 1) * (ch[2] - cl[2] + 1);
      for (int r = 0; r < rows && !near; r++)
      {
        int b, e;
        fq_map_row(g, M->unk, cl, ch, r, &b, &e);
        for (int p = b + tid; p < e && !near; p += T)
          near = (double)FQ_FSQRT(flann_l2(q, M->unk.xyz + 3 * (size_t)p)) < a.drone_radius;
      }
    }
    if (__syncthreads_or(near)) { hit_i = i; break; }               // also the barrier before s_q is written again
  }
  if (hit_i < 0) { put(-1, 0, n - 1); return; }
  const int iH = (int)FQ_MUL(a.delta_H, (double)hit_i);
  if (tid == 0)
  {
    SampleClock c;
    double o[12];
    sample_at(c, iH, co, N, dt, DC, n, o);
    s_H[0] = o[0]; s_H[1] = o[1];
    s_k = 0x7fffffff;
  }
  __syncthreads();
  const double H[2] = { s_H[0], s_H[1] }, a_max = a.lim[3 * j + 1];
  SampleClock c;
  for (int i = tid; i <= iH; i += T)
  {
    double o[12];
    sample_at(c, i, co, N, dt, DC, n, o);
    if (brakes_past(H, o, a.delta_a, a_max)) { atomicMin(&s_k, i); break; }
  }
  __syncthreads();
  put(s_k == 0x7fffffff ? iH : s_k, 1, iH);
}

// result records (fq_pair_result of include/faster_b200.h; 16 doubles each)

__global__ void fq_pair_final_kernel(const FqPairFinalArgs a)
{
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.n_prob) return;
  fq_pair_result r;
  const int ww = a.win_idx_w[j], ws = a.win_idx_s[j];
  // list lengths: shared (n_sig_*), or per corridor (its candidates / n_fac; a corridor without candidates has no winner).
  // With per-corridor windows n_fac is the corridor's own |F_j|, which may be 0 (then so are its candidates).
  const int nfw = a.n_fac_j_w ? a.n_fac_j_w[j] : a.n_fac_w, nfs = a.n_fac_j_s ? a.n_fac_j_s[j] : a.n_fac_s;
  const int lw = a.cand_ofs_w ? (nfw > 0 ? (a.cand_ofs_w[j + 1] - a.cand_ofs_w[j]) / nfw : 0) : a.n_sig_w;
  const int ls = a.cand_ofs_s ? (nfs > 0 ? (a.cand_ofs_s[j + 1] - a.cand_ofs_s[j]) / nfs : 0) : a.n_sig_s;
  r.whole_dt_index = ww >= 0 && lw > 0 ? ww / lw : -1;
  r.whole_sigma_index = ww >= 0 && lw > 0 ? ww % lw : -1;
  r.safe_dt_index = ws >= 0 && ls > 0 ? ws / ls : -1;
  r.safe_sigma_index = ws >= 0 && ls > 0 ? ws % ls : -1;
  if (a.changed_w && a.changed_w[j])
  {
    const int P = a.poly_ofs_w[j + 1] - a.poly_ofs_w[j];
    r.whole_sigma_index = (int)fqa::rank(a.N_w, P, fqa::use_all(a.N_w, P, a.all_limit), a.win_sig_w + (size_t)j * a.N_w);
  }
  if (a.changed_s && a.changed_s[j])
  {
    const int P = a.poly_ofs_s[j + 1] - a.poly_ofs_s[j];
    r.safe_sigma_index = (int)fqa::rank(a.N_s, P, fqa::use_all(a.N_s, P, a.all_limit), a.win_sig_s + (size_t)j * a.N_s);
  }
  if (a.sigma_out_w)
    for (int t = 0; t < a.N_w; t++) a.sigma_out_w[(size_t)j * a.N_w + t] = a.win_sig_w[(size_t)j * a.N_w + t];
  if (a.sigma_out_s)
    for (int t = 0; t < a.N_s; t++) a.sigma_out_s[(size_t)j * a.N_s + t] = a.win_sig_s[(size_t)j * a.N_s + t];
  r.whole_cost = a.win_cost_w[j]; r.safe_cost = a.win_cost_s[j];
  r.whole_dt = a.win_dt_w[j]; r.safe_dt = a.win_dt_s[j];
  r.whole_dt_base = a.dt_base_w[j]; r.safe_dt_base = a.dt_base_s[j];
  r.n_samples_whole = a.n_samples[j]; r.k_safe = a.k_safe[j];
  for (int i = 0; i < 9; i++) r.R[i] = a.x0_safe[j * 9 + i];
  a.out[j] = r;
}

// factor_that_worked_, trials_ and the next windows of every corridor (fq_window.h), after fq_pair_final_kernel (and with
// a gate after fq_pair_queue_kernel, whose failed appends keep the input windows).  trials:
// the winner's index in F_j + 1; |F_j| without a winner; 0 for a sweep that did not run (a safe sweep after a whole sweep
// without winner, or a sweep the offsets kernel emptied).  Each thread reads its corridor's windows before it writes the
// next ones, so those may alias.  With need_safe (fq_replan_pairs_hr*), a replan that needed no safe path ran no safe sweep
// (trials 0) and succeeds when the whole sweep won; its safe window then follows the safe solver's previous
// factor_that_worked_ (faster.cpp:586-588), last_factor_safe, which only a safe winner changes.
__global__ void fq_pair_window_kernel(const FqPairWindowArgs a)
{
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= a.n_prob) return;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  const int dw = a.rec[j].whole_dt_index, ds = a.rec[j].safe_dt_index;
  const bool no_safe = a.need_safe && !a.need_safe[j];
  const bool ran_w = a.cand_ofs_w[a.n_prob] > 0, ran_s = ran_w && dw >= 0 && a.cand_ofs_s[a.n_prob] > 0 && !no_safe;
  const double fw = dw >= 0 ? a.fac_w[(size_t)j * a.max_fac_w + dw] : nan;
  const double fs = ds >= 0 ? a.fac_s[(size_t)j * a.max_fac_s + ds] : nan;
  const double iw = a.init_w[j], ew = a.final_w[j], is = a.init_s[j], es = a.final_s[j];
  const double last_s = a.last_factor_safe ? a.last_factor_safe[j] : nan;
  if (a.factor_w) a.factor_w[j] = fw;
  if (a.factor_s) a.factor_s[j] = fs;
  if (a.trials_w) a.trials_w[j] = !ran_w ? 0 : (dw >= 0 ? dw + 1 : a.n_fac_w[j]);
  if (a.trials_s) a.trials_s[j] = !ran_s ? 0 : (ds >= 0 ? ds + 1 : a.n_fac_s[j]);
  if (a.last_factor_safe && ds >= 0) a.last_factor_safe[j] = fs;
  const bool both = dw >= 0 && (ds >= 0 || no_safe) && (!a.gate || a.gate[j] == FQ_QUEUE_OK);
  double ni, nf;
  fqw::next_window(both, fw, a.gamma_w, a.gammap_w, iw, ew, &ni, &nf);
  if (a.next_init_w) a.next_init_w[j] = ni;
  if (a.next_final_w) a.next_final_w[j] = nf;
  fqw::next_window(both, no_safe ? last_s : fs, a.gamma_s, a.gammap_s, is, es, &ni, &nf);
  if (a.next_init_s) a.next_init_s[j] = ni;
  if (a.next_final_s) a.next_final_s[j] = nf;
}

// ---- the plan piece of every corridor (fq_replan_pairs_plan*): what appendToPlan pushes (faster.cpp:606-648), whole
//      X_temp_[0 .. k_safe] followed by the whole safe X_temp_, each sampled as fillX does with the winner's full count

// corridor j's rows: 0 when the replan returns early (no whole winner, or a needed safe path without a safe winner:
// faster.cpp:420-424, :529-533), else k_safe + 1 + n_s (n_s = 0 when no safe path is needed; then k_safe = n_w - 1).
// *k and *n_s receive k_safe and the safe sample count.
FQ_HD long long plan_rows(const FqPairPlanArgs& a, int j, int* k, int* n_s)
{
  *k = -1; *n_s = 0;
  if (a.win_idx_w[j] < 0) return 0;
  const bool need = !a.need || a.need[j];
  if (need && a.win_idx_s[j] < 0) return 0;
  *k = a.k_safe[j];
  *n_s = need ? fqdt::num_samples(a.N_s, a.win_dt_s[j], a.DC) : 0;
  return (long long)*k + 1 + *n_s;
}

// plan_ofs = the exclusive scan of every corridor's rows (64 bits: nothing bounds the sum), and the statuses: a corridor
// whose rows end past cap is FQ_PLAN_CAPACITY.  One CTA (any size up to 1024): every thread takes a contiguous run of
// corridors, thread 0 scans the runs' sums.
__global__ void __launch_bounds__(1024) fq_pair_plan_offsets_kernel(const FqPairPlanArgs a)
{
  __shared__ long long s_run[1024];
  const int T = blockDim.x, tid = threadIdx.x;
  const int per = (a.n_prob + T - 1) / T;
  const int j0 = min(a.n_prob, tid * per), j1 = min(a.n_prob, j0 + per);
  int k, ns;
  long long sum = 0;
  for (int j = j0; j < j1; j++) sum += plan_rows(a, j, &k, &ns);
  s_run[tid] = sum;
  __syncthreads();
  if (tid == 0)
  {
    long long run = 0;
    for (int i = 0; i < T; i++) { const long long x = s_run[i]; s_run[i] = run; run += x; }
    a.plan_ofs[a.n_prob] = run;
  }
  __syncthreads();
  long long run = s_run[tid];
  for (int j = j0; j < j1; j++)
  {
    const long long r = plan_rows(a, j, &k, &ns);
    a.plan_ofs[j] = run;
    if (a.status) a.status[j] = r == 0 ? FQ_PLAN_NONE : (run + r > a.cap ? FQ_PLAN_CAPACITY : FQ_PLAN_OK);
    run += r;
  }
}

// the rows of every corridor that fits, after fq_pair_plan_offsets_kernel.  One CTA per corridor (any block size): each
// thread takes a contiguous run of the piece's rows, replays the sample clock of its side to the run's first sample and
// walks on from there, so a corridor costs O(threads x rows) clock steps, not O(rows^2).
__global__ void __launch_bounds__(128) fq_pair_plan_sample_kernel(const FqPairPlanArgs a)
{
  const int j = blockIdx.x;
  if (j >= a.n_prob) return;
  const long long base = a.plan_ofs[j], rows = a.plan_ofs[j + 1] - base;
  if (rows <= 0 || base + rows > a.cap) return;          // nothing to append, or past the capacity (FQ_PLAN_CAPACITY)
  int k, ns;
  plan_rows(a, j, &k, &ns);
  const int nw = a.n_samples[j];
  const long long per = (rows + blockDim.x - 1) / blockDim.x, r0 = per * threadIdx.x;
  const long long r1 = r0 + per < rows ? r0 + per : rows;
  const double* cw = a.coeffs_w + (size_t)j * a.N_w * 12;
  const double* cs = a.coeffs_s + (size_t)j * a.N_s * 12;
  SampleClock clock_w, clock_s;
  for (long long r = r0; r < r1; r++)
  {
    double o[12];
    if (r <= k) sample_at(clock_w, (int)r, cw, a.N_w, a.win_dt_w[j], a.DC, nw, o);
    else sample_at(clock_s, (int)(r - k - 1), cs, a.N_s, a.win_dt_s[j], a.DC, ns, o);
    double* out = a.states + 12 * (size_t)(base + r);
    for (int q = 0; q < 12; q++) out[q] = o[q];
  }
}

// ---- each planner's committed plan kept on the device (fq_queue_*, fq_replan_pairs_queue*; the row operations are
//      fq_queue.h's)

// corridor j's row, or -1 when the device may not touch it: out of range, not a ring (unless `any`: reset makes one), or
// (`unique`) named by another corridor as well
FQ_HD int queue_row(const FqQueueArgs& q, int j, bool unique, bool any)
{
  const int r = q.rows ? q.rows[j] : j;
  if (r < 0 || r >= q.n_rows || (!any && !fqq::ring_ok(q.head[r], q.size[r], q.cap))) return -1;
  for (int i = 0; unique && q.rows && i < q.n; i++)
    if (i != j && q.rows[i] == r) return -1;
  return r;
}

FQ_HD double* queue_states(const FqQueueArgs& q, int r) { return q.states + (size_t)r * q.cap * fqq::kState; }

// one thread per corridor
__global__ void fq_queue_reset_kernel(const FqQueueArgs q)
{
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= q.n) return;
  const int r = queue_row(q, j, true, true);
  if (r >= 0) fqq::reset(queue_states(q, r), q.head + r, q.size + r, q.pos + 3 * (size_t)j);
}

__global__ void fq_queue_select_kernel(const FqQueueArgs q)
{
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= q.n) return;
  const int r = queue_row(q, j, false, false);
  q.k_end[j] = r < 0 ? fqq::select(nullptr, 0, 0, q.cap, q.delta_t, q.x0 + 9 * (size_t)j)
                     : fqq::select(queue_states(q, r), q.head[r], q.size[r], q.cap, q.delta_t, q.x0 + 9 * (size_t)j);
}

__global__ void fq_queue_pop_kernel(const FqQueueArgs q)
{
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= q.n) return;
  const int r = queue_row(q, j, true, false);
  const int t = q.ticks[j] < 0 ? 0 : q.ticks[j] > q.max_ticks ? q.max_ticks : q.ticks[j];
  double* g = q.goals + (size_t)j * q.max_ticks * fqq::kState;
  int head = 0, size = 0;
  if (r < 0)
  {
    fqq::pop(nullptr, &head, &size, q.cap, t, g);
    return;
  }
  head = q.head[r]; size = q.size[r];
  fqq::pop(queue_states(q, r), &head, &size, q.cap, t, g);
  q.head[r] = head; q.size[r] = size;
}

// appendToPlan (faster.cpp:606-648) of corridor j's piece onto its row, after the chain's records.  The piece is sampled
// straight into the ring (plan_rows / sample_at, as fq_pair_plan_sample_kernel samples it): its length is known before a
// row is sampled, so each row's decision needs nothing from any other corridor and no staging.  One CTA per corridor (any
// block size): thread 0 decides, every thread samples a contiguous run of the piece, thread 0 then moves the row's size.
__global__ void __launch_bounds__(128) fq_pair_queue_kernel(const FqPairPlanArgs a, const FqQueueArgs q)
{
  __shared__ int s_status;
  __shared__ long long s_keep;
  const int j = blockIdx.x;
  if (j >= a.n_prob) return;
  const int r = q.rows ? q.rows[j] : j;
  int clash = 0;
  for (int i = threadIdx.x; q.rows && i < a.n_prob; i += blockDim.x) clash |= i != j && q.rows[i] == r;
  clash = __syncthreads_or(clash);
  int k, ns;
  const long long rows = plan_rows(a, j, &k, &ns);
  if (threadIdx.x == 0)
  {
    long long keep = 0;
    const bool mine = !clash && r >= 0 && r < q.n_rows && fqq::ring_ok(q.head[r], q.size[r], q.cap);
    s_status = mine ? fqq::append_status(q.size[r], q.cap, q.k_end[j], rows, &keep) : FQ_QUEUE_ROWS;
    s_keep = keep;
  }
  __syncthreads();
  const int st = s_status;
  const long long keep = s_keep;
  if (st == FQ_QUEUE_OK)
  {
    double* row = queue_states(q, r);
    const int head = q.head[r], nw = a.n_samples[j];
    const long long per = (rows + blockDim.x - 1) / blockDim.x, r0 = per * threadIdx.x;
    const long long r1 = r0 + per < rows ? r0 + per : rows;
    const double* cw = a.coeffs_w + (size_t)j * a.N_w * 12;
    const double* cs = a.coeffs_s + (size_t)j * a.N_s * 12;
    SampleClock clock_w, clock_s;
    for (long long i = r0; i < r1; i++)
    {
      double o[12];
      if (i <= k) sample_at(clock_w, (int)i, cw, a.N_w, a.win_dt_w[j], a.DC, nw, o);
      else sample_at(clock_s, (int)(i - k - 1), cs, a.N_s, a.win_dt_s[j], a.DC, ns, o);
      double* out = row + fqq::kState * fqq::slot(head, keep + i, q.cap);
      for (int c = 0; c < 12; c++) out[c] = o[c];
    }
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  bool seen = false;
  if (st == FQ_QUEUE_OK)
  {
    q.size[r] = (int)(keep + rows);
    const double* last = queue_states(q, r) + fqq::kState * fqq::slot(q.head[r], keep + rows - 1, q.cap);
    seen = q.G_term && fqq::goal_seen(last, q.G_term + 3 * (size_t)j, q.goal_radius);
  }
  q.k_end[j] = -1;
  q.status[j] = st;
  if (q.goal_seen) q.goal_seen[j] = seen;
}
}  // namespace fqp
