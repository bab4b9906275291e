// Batched corridor-QP solver for sm_90a (H100): one warp per candidate (dt, sigma).
//
// Each candidate is the strictly convex QP that FASTER's SolverGurobi hands to Gurobi once the binaries are
// fixed (reference faster/src/solverGurobi.cpp:113-119 cost, :332-407,:499-524 rows, :180-291 corridor rows),
// written in the normalised, equality-eliminated variables of fq_plan.h:  min |w|^2  s.t.  rows(w) <= rhs.
// It is solved exactly by a dual active-set method (Goldfarb-Idnani with identity Hessian): start at w = 0,
// repeatedly pick the most violated row, step along the projection of its normal onto the null space of the
// active normals until the row is tight (dropping active rows whose multiplier reaches zero on the way),
// stop when nothing is violated (optimal) or a violated row cannot be reached (infeasible).
//
// Data placement.  Per CTA (shared, staged once with coalesced loads): plan tables TZ/T0 and the problem's
// polytope rows [Ax Ay Az b] (32-byte rows, read as two 16-byte loads).  Per warp (shared): the orthogonal
// factor J (nw x nw, odd leading dimension so both row- and column-walks are conflict-free), the triangular
// factor R, the state rows Y of the current iterate (3 axes x NY), and a handful of nw-vectors.  Reductions
// (row selection, norms, ratio test) are warp shuffles / redux.  HBM traffic per candidate is the ~200 B of
// inputs and 9 B (+ 96 N B coefficients) of outputs; the kernel is FP64-issue / shared-latency bound.
#include "fq_kernels.cuh"
#include "../../include/faster_b200.h"

#include <cmath>

namespace
{
constexpr unsigned FULL = 0xffffffffu;
constexpr int W = FQ_WARPS_PER_CTA;

__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}
__device__ __forceinline__ double warp_min(double v)
{
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmin(v, __shfl_xor_sync(FULL, v, o));
  return v;
}

struct WarpMem
{
  double *J, *R, *Y, *Yeq, *w, *g, *d, *z, *lam, *r, *rdinv, *hdr;
  int *seg_ofs, *sig, *act;     // act[k]: id of the k-th active row (certificate export)
};

__host__ __device__ inline int per_warp_doubles(int nw, int ld, int NY)
{
  const int nwp = nw > 0 ? nw : 1;
  return 2 * nwp * ld + 2 * 3 * NY + 7 * nwp + 24;
}
__host__ __device__ inline int per_warp_ints() { return 2 * (FQ_MAX_N + 2) + 3 * FQ_MAX_N; }

// Y = Yeq + TZ w
__device__ __forceinline__ void recompute_Y(const FqKernelArgs& a, const double* TZ, const WarpMem& m, int lane)
{
  const int NY = a.NY, nz = a.nz;
  for (int idx = lane; idx < 3 * NY; idx += 32)
  {
    const int ax = idx / NY, y = idx - ax * NY;
    double acc = m.Yeq[idx];
    const double* tz = TZ + y * nz;
    const double* wa = m.w + ax * nz;
    for (int k = 0; k < nz; k++) acc = fma(tz[k], wa[k], acc);
    m.Y[idx] = acc;
  }
  __syncwarp();
}

// remove active row at position l (0 <= l < q) from the factorisation
__device__ __forceinline__ void drop_row(const FqKernelArgs& a, const WarpMem& m, int lane, int l, int q)
{
  const int nw = a.nw, ld = a.ld;
  for (int i = lane; i < q; i += 32)
    for (int j = l; j < q - 1; j++) m.R[i * ld + j] = m.R[i * ld + j + 1];
  for (int base = l; base < q - 1; base += 32)
  {
    const int k = base + lane;
    double t = 0;
    int ta = 0;
    if (k < q - 1) { t = m.lam[k + 1]; ta = m.act[k + 1]; }
    __syncwarp();
    if (k < q - 1) { m.lam[k] = t; m.act[k] = ta; }
    __syncwarp();
  }
  __syncwarp();
  for (int j = l; j < q - 1; j++)
  {
    const double p = m.R[j * ld + j], s = m.R[(j + 1) * ld + j];
    const double h = sqrt(p * p + s * s);
    double c = 1.0, sn = 0.0;
    if (h > 0) { const double hi = 1.0 / h; c = p * hi; sn = s * hi; }
    __syncwarp();
    for (int k = j + lane; k < q - 1; k += 32)
    {
      const double u = m.R[j * ld + k], v = m.R[(j + 1) * ld + k];
      m.R[j * ld + k] = c * u + sn * v;
      m.R[(j + 1) * ld + k] = c * v - sn * u;
    }
    for (int i = lane; i < nw; i += 32)
    {
      const double u = m.J[i * ld + j], v = m.J[i * ld + j + 1];
      m.J[i * ld + j] = c * u + sn * v;
      m.J[i * ld + j + 1] = c * v - sn * u;
    }
    __syncwarp();
  }
  for (int k = l + lane; k < q - 1; k += 32) m.rdinv[k] = 1.0 / m.R[k * ld + k];
  __syncwarp();
}

__device__ void solve_candidate(const FqKernelArgs& a, const double* TZ, const double* T0, const double* sAb,
                                const int* sfo, const WarpMem& m, int prob, int cand, int lane, int rows_bad)
{
  const int N = a.N, nz = a.nz, nw = a.nw, NY = a.NY, ld = a.ld, ne = a.ne;
  const double dt = a.dt[cand], dt2 = dt * dt;
  const double inv1 = 1.0 / dt, inv2 = inv1 * inv1, inv3 = inv2 * inv1;
  const double lim0 = a.lim[prob * 3 + 0], lim1 = a.lim[prob * 3 + 1], lim2 = a.lim[prob * 3 + 2];
  const int P = a.poly_ofs[prob + 1] - a.poly_ofs[prob];

  // ---- normalised boundary data: hdr[ax*6 + 0..2] = (P0, V0, A0), hdr[ax*6 + 3..3+ne) = rhs
  if (lane < 3)
  {
    const int ax = lane;
    const double* x0 = a.x0 + prob * 9;
    const double* xf = a.xf + prob * 9;
    const double s0 = x0[ax], s1 = x0[3 + ax] * dt, s2 = x0[6 + ax] * dt2;
    m.hdr[ax * 6 + 0] = s0; m.hdr[ax * 6 + 1] = s1; m.hdr[ax * 6 + 2] = s2;
    double tgt[3];
    int e = 0;
    if (a.force_final) tgt[e++] = xf[ax];
    tgt[e++] = xf[3 + ax] * dt;
    tgt[e++] = xf[6 + ax] * dt2;
    for (int k = 0; k < ne; k++)
      m.hdr[ax * 6 + 3 + k] = tgt[k] - (a.FT[k * 3 + 0] * s0 + a.FT[k * 3 + 1] * s1 + a.FT[k * 3 + 2] * s2);
  }
  // ---- corridor row ranges per segment
  int total_rows = 0;
  if (P > 0)
  {
    int F = 0, p = 0;
    if (lane < N) { p = a.sigma[(size_t)cand * N + lane]; if (p >= P) p = P - 1; F = sfo[p + 1] - sfo[p]; }
    int incl = F;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1)
    {
      const int v = __shfl_up_sync(FULL, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane < N) { m.seg_ofs[lane + 1] = incl; m.sig[lane] = p; }
    if (lane == 0) m.seg_ofs[0] = 0;
    total_rows = __shfl_sync(FULL, incl, N - 1);
  }
  for (int idx = lane; idx < nw * ld; idx += 32) m.J[idx] = 0.0;
  __syncwarp();
  for (int j = lane; j < nw; j += 32) { m.J[j * ld + j] = 1.0; m.w[j] = 0.0; }
  for (int idx = lane; idx < 3 * NY; idx += 32)
  {
    const int ax = idx / NY, y = idx - ax * NY;
    const double* t0 = T0 + y * (3 + ne);
    const double* h = m.hdr + ax * 6;
    double v = 0;
    for (int k = 0; k < 3 + ne; k++) v = fma(t0[k], h[k], v);
    m.Yeq[idx] = v; m.Y[idx] = v;
  }
  __syncwarp();

  int q = 0, status = -1, it = 0;
  { // non-finite / non-positive inputs (unvalidated device-pointer entry): report "not solved", never fault
    bool okc = dt > 0 && dt < 1e100 && lim0 > 0 && lim0 < 1e300 && lim1 > 0 && lim1 < 1e300 && lim2 > 0 && lim2 < 1e300 &&
               rows_bad == 0;
    for (int idx = lane; idx < 3 * NY; idx += 32) okc = okc && fabs(m.Yeq[idx]) < 1e300;
    if (!__all_sync(FULL, okc))
    {
      if (lane == 0)
      {
        a.feasible[cand] = 0;
        a.cost[cand] = INFINITY;
        if (a.iters) a.iters[cand] = rows_bad == 2 ? -2 : -1;
      }
      if (a.coeffs)
        for (int idx = lane; idx < 12 * N; idx += 32) a.coeffs[(size_t)cand * N * 12 + idx] = 0.0;
      return;
    }
  }
  for (;;)
  {
    // ================= most violated row =================
    double bv = a.row_tol, bw0 = 0, bw1 = 0, bw2 = 0, bh = 0;
    int by = 0, bid = 0;   // bid: row identity for the certificate export (fq_solve_batch_cert): box rows
                           // 10000000 + type*10000 + axis*1000 + t*10 + (upper bound ? 1 : 0); corridor rows t*100000 + face*10 + cp
    for (int i = lane; i < 9 * N; i += 32)
    { // |v|,|a|,|j| boxes at segment starts (solverGurobi.cpp:390-407); type 0 v, 1 a, 2 j
      const int type = i / (3 * N), rem = i - type * 3 * N, ax = rem / N, t = rem - ax * N;
      const int y = (type + 1) * N + 1 + t;
      const double val = m.Y[ax * NY + y];
      const double sinv = type == 0 ? inv1 : (type == 1 ? inv2 : inv3);
      const double L = type == 0 ? lim0 : (type == 1 ? lim1 : lim2);
      const double viol = fabs(val) * sinv - L;
      if (viol > bv)
      {
        const double s = val > 0 ? sinv : -sinv;
        bv = viol; by = y; bh = L;
        bid = 10000000 + type * 10000 + ax * 1000 + t * 10 + (val > 0 ? 1 : 0);
        bw0 = ax == 0 ? s : 0.0; bw1 = ax == 1 ? s : 0.0; bw2 = ax == 2 ? s : 0.0;
      }
    }
    for (int i = lane; i < total_rows; i += 32)
    { // control points of segment t inside polytope sigma[t] (solverGurobi.cpp:249-287)
      int t = 0;
      for (int s = 1; s < N; s++) t += (i >= m.seg_ofs[s]);
      const int gf = sfo[m.sig[t]] + (i - m.seg_ofs[t]);
      const double2 a01 = *reinterpret_cast<const double2*>(sAb + 4 * gf);
      const double2 a23 = *reinterpret_cast<const double2*>(sAb + 4 * gf + 2);
      const int ys[4] = { t, 4 * N + 1 + t, 5 * N + 1 + t, t + 1 };
#pragma unroll
      for (int k = 0; k < 4; k++)
      {
        const int y = ys[k];
        const double v = fma(a01.x, m.Y[y], fma(a01.y, m.Y[NY + y], fma(a23.x, m.Y[2 * NY + y], -a23.y)));
        if (v > bv) { bv = v; by = y; bw0 = a01.x; bw1 = a01.y; bw2 = a23.x; bh = a23.y; bid = t * 100000 + gf * 10 + k; }
      }
    }
    const unsigned key = bv > a.row_tol ? __float_as_uint(fmaxf((float)bv, 1e-30f)) : 0u;
    const unsigned mk = __reduce_max_sync(FULL, key);
    if (mk == 0u) { status = 1; break; }
    const int src = __ffs(__ballot_sync(FULL, key == mk)) - 1;
    const int y = __shfl_sync(FULL, by, src);
    const int eid = __shfl_sync(FULL, bid, src);
    const double w0 = __shfl_sync(FULL, bw0, src), w1 = __shfl_sync(FULL, bw1, src),
                 w2 = __shfl_sync(FULL, bw2, src), h = __shfl_sync(FULL, bh, src);

    // ================= normal of the chosen row in w-space =================
    double ggp = 0;
    for (int j = lane; j < nw; j += 32)
    {
      const int ax = j / nz, k = j - ax * nz;
      const double wa = ax == 0 ? w0 : (ax == 1 ? w1 : w2);
      const double gj = wa * TZ[y * nz + k];
      m.g[j] = gj; ggp += gj * gj;
    }
    const double gg = warp_sum(ggp);
    __syncwarp();
    double lam_p = 0;
    bool done = false;
    for (;;)
    {
      if (++it > FQ_MAX_ITERS) { status = -1; done = true; break; }
      const double viol = fma(w0, m.Y[y], fma(w1, m.Y[NY + y], fma(w2, m.Y[2 * NY + y], -h)));
      // d = J' g ;  zz = |d2|^2
      double zzp = 0;
      for (int j = lane; j < nw; j += 32)
      {
        double acc = 0;
        for (int i = 0; i < nw; i++) acc = fma(m.J[i * ld + j], m.g[i], acc);
        m.d[j] = acc;
        if (j >= q) zzp += acc * acc;
      }
      const double zz = warp_sum(zzp);
      __syncwarp();
      // z = -J2 d2
      for (int i = lane; i < nw; i += 32)
      {
        double acc = 0;
        for (int j = q; j < nw; j++) acc = fma(m.J[i * ld + j], m.d[j], acc);
        m.z[i] = -acc;
      }
      // r = R^-1 d1
      for (int k = lane; k < q; k += 32) m.r[k] = m.d[k];
      __syncwarp();
      for (int k = q - 1; k >= 0; k--)
      {
        const double rk = m.r[k] * m.rdinv[k];
        __syncwarp();
        if (lane == 0) m.r[k] = rk;
        for (int j = lane; j < k; j += 32) m.r[j] = fma(-m.R[j * ld + k], rk, m.r[j]);
        __syncwarp();
      }
      const bool dep = zz <= fmax(FQ_EPS_DEP * gg, FQ_ZZ_FLOOR) || q >= nw;   // a full active set: nothing more fits
      // dual ratio test
      double best = INFINITY;
      int bk = -1;
      for (int k = lane; k < q; k += 32)
      {
        const double rk = m.r[k];
        if (rk > 0)
        {
          const double ratio = m.lam[k] / rk;
          if (ratio < best) { best = ratio; bk = k; }
        }
      }
      const double t1 = warp_min(best);
      int l = -1;
      if (t1 < INFINITY)
      {
        const int s2 = __ffs(__ballot_sync(FULL, best == t1)) - 1;
        l = __shfl_sync(FULL, bk, s2);
      }
      const double t2 = dep ? INFINITY : viol / zz;
      if (t1 == INFINITY && t2 == INFINITY)
      {
        status = 0; done = true;
        if (a.cert)
        { // Farkas certificate: entering row with multiplier 1, active rows with -r_k >= 0 (g_e = sum r_k n_k, r <= 0)
          double* c = a.cert + (size_t)cand * a.cert_stride;
          if (lane == 0) { c[0] = (double)(q + 1); c[1] = viol; c[2] = (double)eid; c[3] = 1.0; }
          for (int k = lane; k < q; k += 32)
            if (4 + 2 * k + 1 < a.cert_stride) { c[4 + 2 * k] = (double)m.act[k]; c[4 + 2 * k + 1] = -m.r[k]; }
        }
        break;
      }
      if (t2 <= t1)
      { // full step: the row becomes active (Householder update of J2, new column of R)
        for (int j = lane; j < nw; j += 32) m.w[j] = fma(t2, m.z[j], m.w[j]);
        for (int k = lane; k < q; k += 32) m.lam[k] = fma(-t2, m.r[k], m.lam[k]);
        lam_p += t2;
        const double dq = m.d[q], nrm = sqrt(zz), sgn = dq >= 0 ? 1.0 : -1.0;
        const double beta = 1.0 / (zz + fabs(dq) * nrm), vq = dq + sgn * nrm;
        for (int i = lane; i < nw; i += 32)
        {
          double* Ji = m.J + i * ld;
          const double bu = beta * fma(sgn * nrm, Ji[q], -m.z[i]);
          Ji[q] = fma(-bu, vq, Ji[q]);
          for (int j = q + 1; j < nw; j++) Ji[j] = fma(-bu, m.d[j], Ji[j]);
        }
        for (int k = lane; k < q; k += 32) m.R[k * ld + q] = m.d[k];
        if (lane == 0) { m.R[q * ld + q] = -sgn * nrm; m.rdinv[q] = -sgn / nrm; m.lam[q] = lam_p; m.act[q] = eid; }
        q++;
        __syncwarp();
        recompute_Y(a, TZ, m, lane);
        break;
      }
      // partial step: active row l leaves.  (l < 0 here means t1/t2 are NaN -- non-finite input: give up)
      if (l < 0) { status = -1; done = true; break; }
      if (!dep)
        for (int j = lane; j < nw; j += 32) m.w[j] = fma(t1, m.z[j], m.w[j]);
      for (int k = lane; k < q; k += 32) m.lam[k] = fma(-t1, m.r[k], m.lam[k]);
      lam_p += t1;
      __syncwarp();
      drop_row(a, m, lane, l, q);
      q--;
      if (!dep) recompute_Y(a, TZ, m, lane);
    }
    if (done) break;
  }

  // ================= outputs =================
  double cp = 0;
  if (status == 1)
    for (int i = lane; i < 3 * N; i += 32)
    {
      const int ax = i / N, t = i - ax * N;
      const double u = m.Y[ax * NY + 3 * N + 1 + t];
      cp = fma(u, u, cp);
    }
  const double cost = warp_sum(cp) * (inv3 * inv3);   // sum (u dt^3)^2 / dt^6
  if (lane == 0)
  {
    a.feasible[cand] = status == 1;
    a.cost[cand] = status == 1 ? cost : INFINITY;
    if (a.iters) a.iters[cand] = status == -1 ? -it : it;
  }
  if (a.coeffs)
  {
    double* out = a.coeffs + (size_t)cand * N * 12;
    for (int idx = lane; idx < 12 * N; idx += 32)
    { // x[t][0..11] = ax ay az bx by bz cx cy cz dx dy dz (solverGurobi.cpp:72)
      const int t = idx / 12, c = idx - 12 * t, kind = c / 3, ax = c - 3 * kind;
      const double* Ya = m.Y + ax * NY;
      double v;
      if (kind == 0) v = Ya[3 * N + 1 + t] * inv3 * (1.0 / 6.0);
      else if (kind == 1) v = Ya[2 * N + 1 + t] * inv2 * 0.5;
      else if (kind == 2) v = Ya[N + 1 + t] * inv1;
      else v = Ya[t];
      out[idx] = status == 1 ? v : 0.0;
    }
  }
}

__global__ void __launch_bounds__(W * 32) fq_solve_kernel(const FqKernelArgs a, int chunks_per_prob)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int prob = blockIdx.x / chunks_per_prob, chunk = blockIdx.x - prob * chunks_per_prob;
  const int c_begin = a.cand_ofs[prob], c_end = a.cand_ofs[prob + 1];
  const int first = c_begin + chunk * W;
  if (first >= c_end) return;

  const int nzp = a.nz > 0 ? a.nz : 1;
  double* sm = reinterpret_cast<double*>(smem_raw);
  double* sAb = sm;                         sm += 4 * a.max_faces;          // 16-byte aligned rows first
  double* TZ = sm;                          sm += a.NY * nzp;
  double* T0 = sm;                          sm += a.NY * (3 + a.ne);
  const int pwd = per_warp_doubles(a.nw, a.ld, a.NY);
  double* wbase = sm;                       sm += W * pwd;
  int* ibase = reinterpret_cast<int*>(sm);
  int* sfo = ibase;                         ibase += 36;

  // ---- stage plan tables and this problem's polytopes (coalesced)
  for (int i = threadIdx.x; i < a.NY * a.nz; i += blockDim.x) TZ[i] = a.TZ[i];
  for (int i = threadIdx.x; i < a.NY * (3 + a.ne); i += blockDim.x) T0[i] = a.T0[i];
  const int p0 = a.poly_ofs[prob], P = a.poly_ofs[prob + 1] - p0;
  const int f0 = a.face_ofs[p0];
  const int nf = P > 0 ? a.face_ofs[p0 + P] - f0 : 0;
  int rows_bad = 0;
  {
    const bool fits = nf >= 0 && nf <= a.max_faces;   // a too small max_faces hint must not overrun the staging area
    const double2* src = reinterpret_cast<const double2*>(a.Ab + (size_t)4 * f0);
    double2* dst = reinterpret_cast<double2*>(sAb);
    int bad = 0;
    for (int i = threadIdx.x; fits && i < 2 * nf; i += blockDim.x)
    {
      const double2 v = src[i];
      bad |= !(fabs(v.x) < 1e300) || !(fabs(v.y) < 1e300);
      dst[i] = v;
    }
    for (int i = threadIdx.x; i <= P && i < 36; i += blockDim.x) sfo[i] = a.face_ofs[p0 + i] - f0;
    rows_bad = __syncthreads_or(bad) != 0 ? 1 : 0;
    if (!fits) rows_bad = 2;
  }

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cand = first + warp;
  if (cand >= c_end) return;
  const int nwp = a.nw > 0 ? a.nw : 1;
  WarpMem m;
  double* p = wbase + warp * pwd;
  m.J = p;      p += nwp * a.ld;
  m.R = p;      p += nwp * a.ld;
  m.Y = p;      p += 3 * a.NY;
  m.Yeq = p;    p += 3 * a.NY;
  m.w = p;      p += nwp;
  m.g = p;      p += nwp;
  m.d = p;      p += nwp;
  m.z = p;      p += nwp;
  m.lam = p;    p += nwp;
  m.r = p;      p += nwp;
  m.rdinv = p;  p += nwp;
  m.hdr = p;
  int* ip = ibase + warp * per_warp_ints();
  m.seg_ofs = ip; m.sig = ip + FQ_MAX_N + 2; m.act = ip + 2 * (FQ_MAX_N + 2);
  solve_candidate(a, TZ, T0, sAb, sfo, m, prob, cand, lane, rows_bad);
}

// genNewTraj selection (solverGurobi.cpp:445-472): first dt with a feasible assignment, then min cost.
__global__ void __launch_bounds__(256) fq_select_kernel(const FqSelectArgs a)
{
  __shared__ int s_dt;
  __shared__ unsigned long long s_best;
  if (threadIdx.x == 0) { s_dt = 0x7fffffff; s_best = ~0ull; }
  __syncthreads();
  const int total = a.n_dt * a.n_sigma;
  int mine = 0x7fffffff;
  for (int i = threadIdx.x; i < total; i += blockDim.x)
    if (a.feasible[i]) { const int d = i / a.n_sigma; if (d < mine) mine = d; }
  if (mine != 0x7fffffff) atomicMin(&s_dt, mine);
  __syncthreads();
  const int dtw = s_dt;
  if (dtw == 0x7fffffff)
  {
    if (threadIdx.x == 0) { a.out_idx[0] = -1; a.out_idx[1] = -1; a.out_cost[0] = INFINITY; }
    return;
  }
  // costs are non-negative doubles: their bit patterns order like unsigned integers.  Exact two-step reduction: the
  // minimum cost, then the lowest assignment index that attains it (ties are exact cost ties).
  unsigned long long best = ~0ull;
  for (int s = threadIdx.x; s < a.n_sigma; s += blockDim.x)
  {
    const int i = dtw * a.n_sigma + s;
    if (!a.feasible[i]) continue;
    const unsigned long long bits = (unsigned long long)__double_as_longlong(a.cost[i]);
    if (bits < best) best = bits;
  }
  if (best != ~0ull) atomicMin(&s_best, best);
  __syncthreads();
  const unsigned long long cb = s_best;
  __shared__ int s_sig;
  if (threadIdx.x == 0) s_sig = 0x7fffffff;
  __syncthreads();
  for (int s = threadIdx.x; s < a.n_sigma; s += blockDim.x)
  {
    const int i = dtw * a.n_sigma + s;
    if (a.feasible[i] && (unsigned long long)__double_as_longlong(a.cost[i]) == cb) { atomicMin(&s_sig, s); break; }
  }
  __syncthreads();
  const int sw = s_sig;
  const int win = dtw * a.n_sigma + sw;
  if (threadIdx.x == 0) { a.out_idx[0] = dtw; a.out_idx[1] = sw; a.out_cost[0] = a.cost[win]; }
  if (a.coeffs && a.out_coeffs)
    for (int i = threadIdx.x; i < 12 * a.N; i += blockDim.x) a.out_coeffs[i] = a.coeffs[(size_t)win * 12 * a.N + i];
}

// fillX on the device (reference solverGurobi.cpp:122-168, resetX :382-388).  The reference accumulates the sample time
// (`t = t + DC`) and advances the interval index by at most one per sample; both are reproduced exactly: thread i
// replays the i+1 additions, and -- because findDT keeps dt >= 2 DC (:494-497) so that a sample crosses at most one knot --
// the lagging interval index equals the number of knots m*dt (m >= 1) strictly below t, capped at N-1.  A sample that
// would need more than one advance (dt < DC, impossible through findDT) is detected and handled by a sequential replay.
__global__ void __launch_bounds__(256) fq_fill_kernel(const FqFillArgs a)
{
  const int w = a.win_idx[0];
  if (w < 0) { if (threadIdx.x == 0 && blockIdx.x == 0) a.n_samples[0] = 0; return; }
  const double dt = a.dts[w], DC = a.DC;
  int n = (int)((int)(a.N)*dt / DC);
  n = n < 2 ? 2 : n;
  if (n > a.max_samples) n = a.max_samples;
  if (threadIdx.x == 0 && blockIdx.x == 0) a.n_samples[0] = n;
  const bool lagging_ok = dt >= DC;            // at most one knot per sample
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
  {
    double t = 0;
    int interval = 0;
    if (lagging_ok)
    {
      for (int k = 0; k <= i; k++) t = t + DC;
      while (interval < a.N - 1 && t > dt * (interval + 1)) interval++;
    }
    else
    {
      for (int k = 0; k <= i; k++)
      {
        t = t + DC;
        if (t > dt * (interval + 1)) interval = min(interval + 1, a.N - 1);
      }
    }
    const double tau = t - interval * dt;
    const double* x = a.coeffs + 12 * interval;
    double* o = a.out + (size_t)12 * i;
    const bool last = i == n - 1;              // :165-167: the last sample's vel/accel/jerk are zeroed
#pragma unroll
    for (int ax = 0; ax < 3; ax++)
    {
      o[ax] = x[ax] * tau * tau * tau + x[3 + ax] * tau * tau + x[6 + ax] * tau + x[9 + ax];
      o[3 + ax] = last ? 0.0 : 3 * x[ax] * tau * tau + 2 * x[3 + ax] * tau + x[6 + ax];
      o[6 + ax] = last ? 0.0 : 6 * x[ax] * tau + 2 * x[3 + ax];
      o[9 + ax] = last ? 0.0 : 6 * x[ax];
    }
  }
}
}  // namespace

#include "fq_kernels_t.cuh"
#include "fq_bnb.cuh"
#include "fq_pair.cuh"
#include "fq_decomp.cuh"

size_t fq_solve_smem_bytes(const FqKernelArgs& a)
{
  const int nzp = a.nz > 0 ? a.nz : 1;
  size_t doubles = (size_t)4 * a.max_faces + (size_t)a.NY * nzp + (size_t)a.NY * (3 + a.ne) +
                   (size_t)W * per_warp_doubles(a.nw, a.ld, a.NY);
  return doubles * sizeof(double) + (36 + W * per_warp_ints()) * sizeof(int);
}

bool fq_has_specialised(int N, int force_final, int max_faces)
{
  return N >= 4 && N <= 16 && max_faces <= 2047 && (force_final ? N >= 4 : N >= 3);
}

cudaError_t fq_launch_solve(const FqKernelArgs& a, int max_cand_per_prob, cudaStream_t stream, int* counters, int sm_count,
                            bool force_generic, bool* used_specialised)
{
  if (used_specialised) *used_specialised = false;
  if (a.n_prob <= 0 || max_cand_per_prob <= 0) return cudaSuccess;
  if (!force_generic && fq_has_specialised(a.N, a.force_final, a.max_faces))
  {
    const long long total_hint = (long long)max_cand_per_prob * a.n_prob;
    cudaError_t e = cudaErrorInvalidConfiguration;
#define FQ_CASE(NN)                                                                                        \
  case NN:                                                                                                 \
    e = a.force_final ? fqt::launch_t<NN, true>(a, total_hint, stream, counters, sm_count)                            \
                      : fqt::launch_t<NN, false>(a, total_hint, stream, counters, sm_count);                          \
    break;
    switch (a.N)
    {
      FQ_CASE(4) FQ_CASE(5) FQ_CASE(6) FQ_CASE(7) FQ_CASE(8) FQ_CASE(9) FQ_CASE(10) FQ_CASE(11) FQ_CASE(12)
      FQ_CASE(13) FQ_CASE(14) FQ_CASE(15) FQ_CASE(16)
      default: break;
    }
#undef FQ_CASE
    // cudaErrorInvalidConfiguration: the problem (very many faces per polytope) does not fit the specialised kernel's
    // shared-memory layout -> the size-generic kernel below takes it
    if (e != cudaErrorInvalidConfiguration) { if (used_specialised) *used_specialised = e == cudaSuccess; return e; }
  }
  const size_t smem = fq_solve_smem_bytes(a);
  {  // per-device attribute; cheap enough to set on every launch (contexts on several GPUs share this code)
    cudaError_t e = cudaFuncSetAttribute(fq_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  const int chunks = (max_cand_per_prob + W - 1) / W;
  const long long blocks = (long long)chunks * a.n_prob;
  if (blocks > 0x7fffffffLL) return cudaErrorInvalidValue;
  fq_solve_kernel<<<(unsigned)blocks, W * 32, smem, stream>>>(a, chunks);
  return cudaGetLastError();
}

cudaError_t fq_launch_fill(const FqFillArgs& a, cudaStream_t stream)
{
  int blocks = (a.max_samples + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > 64) blocks = 64;
  fq_fill_kernel<<<blocks, 256, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t fq_launch_select(const FqSelectArgs& a, cudaStream_t stream)
{
  fq_select_kernel<<<1, 256, 0, stream>>>(a);
  return cudaGetLastError();
}

size_t fq_bnb_node_bytes(int N, int force_final)
{
#define FQ_CASE(NN) case NN: return force_final ? fqb::node_bytes<fqt::Dims<NN, true>>() : fqb::node_bytes<fqt::Dims<NN, false>>();
  switch (N)
  {
    FQ_CASE(4) FQ_CASE(5) FQ_CASE(6) FQ_CASE(7) FQ_CASE(8) FQ_CASE(9) FQ_CASE(10) FQ_CASE(11) FQ_CASE(12)
    FQ_CASE(13) FQ_CASE(14) FQ_CASE(15) FQ_CASE(16)
    default: return 0;
  }
#undef FQ_CASE
}

size_t fq_bnb_level_smem(int N, int force_final, int max_faces, int item_cap)
{
#define FQ_CASE(NN) case NN: return force_final ? fqb::level_smem<NN, true>(max_faces, item_cap) : fqb::level_smem<NN, false>(max_faces, item_cap);
  switch (N)
  {
    FQ_CASE(4) FQ_CASE(5) FQ_CASE(6) FQ_CASE(7) FQ_CASE(8) FQ_CASE(9) FQ_CASE(10) FQ_CASE(11) FQ_CASE(12)
    FQ_CASE(13) FQ_CASE(14) FQ_CASE(15) FQ_CASE(16)
    default: return 0;
  }
#undef FQ_CASE
}

cudaError_t fq_launch_bnb_level(const FqBnbLevel& l, cudaStream_t stream)
{
  fqb::BnbArgs b;
  b.k = l.k; b.n_dt = l.n_dt; b.dts = l.dts; b.depth = l.depth; b.cpc = l.cpc; b.n_parents = l.n_parents;
  b.parents = l.parents; b.roots = l.roots; b.children = l.children; b.n_children = l.n_children; b.cap = l.cap;
  b.incumbent = l.incumbent; b.leaves = (fqb::LeafRec*)l.leaves; b.n_leaves = l.n_leaves; b.leaf_cap = l.leaf_cap;
  b.flags = l.flags; b.nodes = l.nodes; b.keep_ties = l.keep_ties; b.lbound = l.lbound; b.closed = l.closed;
#define FQ_CASE(NN) case NN: return l.k.force_final ? fqb::launch_level<NN, true>(b, stream) : fqb::launch_level<NN, false>(b, stream);
  switch (l.k.N)
  {
    FQ_CASE(4) FQ_CASE(5) FQ_CASE(6) FQ_CASE(7) FQ_CASE(8) FQ_CASE(9) FQ_CASE(10) FQ_CASE(11) FQ_CASE(12)
    FQ_CASE(13) FQ_CASE(14) FQ_CASE(15) FQ_CASE(16)
    default: return cudaErrorInvalidConfiguration;
  }
#undef FQ_CASE
}

cudaError_t fq_launch_bnb_roots(const FqBnbChainArgs& a, cudaStream_t stream)
{
  if (a.n_prob <= 0) return cudaSuccess;
  fqb::fq_bnb_roots_kernel<<<(a.n_prob + 63) / 64, 64, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t fq_launch_bnb_certify(const FqBnbChainArgs& a, cudaStream_t stream)
{
  if (a.n_prob <= 0) return cudaSuccess;
  fqb::fq_bnb_certify_kernel<<<(a.n_prob + 63) / 64, 64, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t fq_launch_bnb_resolve(const FqBnbChainArgs& a, cudaStream_t stream)
{
  if (a.n_prob <= 0) return cudaSuccess;
  fqb::fq_bnb_resolve_kernel<<<(a.n_prob + 63) / 64, 64, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t fq_launch_bnb_fallback(const FqBnbChainArgs& a, const uint8_t* feasible, double* redo_dt, cudaStream_t stream)
{
  if (a.n_prob <= 0) return cudaSuccess;
  fqb::fq_bnb_fallback_kernel<<<(a.n_prob + 63) / 64, 64, 0, stream>>>(a, feasible, redo_dt);
  return cudaGetLastError();
}

cudaError_t fq_launch_bnb_adopt(int n_prob, int N, const double* redo_dt, const double* redo_coeffs, double* coeffs, cudaStream_t stream)
{
  if (n_prob <= 0) return cudaSuccess;
  fqb::fq_bnb_adopt_kernel<<<n_prob, 128, 0, stream>>>(n_prob, N, redo_dt, redo_coeffs, coeffs);
  return cudaGetLastError();
}

cudaError_t fq_launch_dtbase(int n_prob, int N, double DC, const double* x0, const double* xf, const double* lim,
                             double* dt_base, cudaStream_t stream)
{
  if (n_prob <= 0) return cudaSuccess;
  fqp::fq_dtbase_kernel<<<(4 * n_prob + 127) / 128, 128, 0, stream>>>(n_prob, N, DC, x0, xf, lim, dt_base);
  return cudaGetLastError();
}

cudaError_t fq_launch_expand_grid(int n_prob, int N, int n_fac, int n_sig, const double* factors, const uint8_t* sig_list,
                                  const double* dt_base, double* dt, uint8_t* sigma, int* cand_ofs, cudaStream_t stream)
{
  if (n_prob <= 0) return cudaSuccess;
  const long long total = (long long)n_prob * n_fac * n_sig;
  long long blocks = (total + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > 132 * 8) blocks = 132 * 8;          // grid-stride loop: 8 blocks per SM of an H100 SXM
  fqp::fq_expand_grid_kernel<<<(unsigned)blocks, 256, 0, stream>>>(n_prob, N, n_fac, n_sig, factors, sig_list, dt_base, dt, sigma,
                                                                  cand_ofs);
  return cudaGetLastError();
}

cudaError_t fq_launch_assign_offsets(int n_prob, int N, int n_fac, long long all_limit, int max_poly, long long n_cand,
                                     const int* poly_ofs, int* cand_ofs, cudaStream_t stream)
{
  if (n_prob <= 0) return cudaSuccess;
  fqp::fq_assign_offsets_kernel<<<1, 1024, 0, stream>>>(n_prob, N, n_fac, all_limit, max_poly, n_cand, poly_ofs, cand_ofs);
  return cudaGetLastError();
}

cudaError_t fq_launch_expand_assign(int n_prob, int N, int n_fac, long long all_limit, const double* factors, const double* dt_base,
                                    const int* poly_ofs, const int* cand_ofs, double* dt, uint8_t* sigma, cudaStream_t stream)
{
  if (n_prob <= 0) return cudaSuccess;
  fqp::fq_expand_assign_kernel<<<n_prob, 256, 0, stream>>>(n_prob, N, n_fac, all_limit, factors, dt_base, poly_ofs, cand_ofs, dt, sigma);
  return cudaGetLastError();
}

cudaError_t fq_launch_window_factors(int n_prob, int max_fac, const double* init, const double* final_, double inc, double* fac,
                                     int* n_fac_j, cudaStream_t stream)
{
  if (n_prob <= 0) return cudaSuccess;
  fqp::fq_window_factors_kernel<<<(n_prob + 63) / 64, 64, 0, stream>>>(n_prob, max_fac, init, final_, inc, fac, n_fac_j);
  return cudaGetLastError();
}

cudaError_t fq_launch_window_offsets(int n_prob, int N, int max_fac, long long all_limit, int max_poly, long long cap,
                                     const int* poly_ofs, const int* n_fac_j, int* cand_ofs, cudaStream_t stream)
{
  if (n_prob <= 0) return cudaSuccess;
  fqp::fq_assign_offsets_kernel<<<1, 1024, 0, stream>>>(n_prob, N, max_fac, all_limit, max_poly, cap, poly_ofs, cand_ofs, n_fac_j);
  return cudaGetLastError();
}

cudaError_t fq_launch_expand_window(int n_prob, int N, int max_fac, long long all_limit, const double* fac, const int* n_fac_j,
                                    const double* dt_base, const int* poly_ofs, const int* cand_ofs, double* dt, uint8_t* sigma,
                                    cudaStream_t stream)
{
  if (n_prob <= 0) return cudaSuccess;
  fqp::fq_expand_assign_kernel<<<n_prob, 256, 0, stream>>>(n_prob, N, max_fac, all_limit, fac, dt_base, poly_ofs, cand_ofs, dt, sigma,
                                                           n_fac_j);
  return cudaGetLastError();
}

cudaError_t fq_launch_pair_window(const FqPairWindowArgs& a, cudaStream_t stream)
{
  if (a.n_prob <= 0) return cudaSuccess;
  fqp::fq_pair_window_kernel<<<(a.n_prob + 127) / 128, 128, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t fq_launch_select_multi(const FqSelectMultiArgs& a, cudaStream_t stream)
{
  if (a.n_prob <= 0) return cudaSuccess;
  fqp::fq_select_multi_kernel<<<a.n_prob, 128, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t fq_launch_pair_mid(const FqPairMidArgs& a, cudaStream_t stream)
{
  if (a.n_prob <= 0) return cudaSuccess;
  fqp::fq_pair_mid_kernel<<<(a.n_prob + 63) / 64, 64, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t fq_launch_pair_hr(const FqPairHrArgs& a, cudaStream_t stream)
{
  if (a.n_prob <= 0) return cudaSuccess;
  fqp::fq_pair_hr_kernel<<<a.n_prob, 256, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t fq_launch_pair_final(const FqPairFinalArgs& a, cudaStream_t stream)
{
  if (a.n_prob <= 0) return cudaSuccess;
  fqp::fq_pair_final_kernel<<<(a.n_prob + 127) / 128, 128, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t fq_launch_pair_plan(const FqPairPlanArgs& a, cudaStream_t stream)
{
  if (a.n_prob <= 0) return cudaSuccess;
  fqp::fq_pair_plan_offsets_kernel<<<1, 1024, 0, stream>>>(a);
  fqp::fq_pair_plan_sample_kernel<<<a.n_prob, 128, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t fq_launch_queue_reset(const FqQueueArgs& q, cudaStream_t stream)
{
  if (q.n <= 0) return cudaSuccess;
  fqp::fq_queue_reset_kernel<<<(q.n + 127) / 128, 128, 0, stream>>>(q);
  return cudaGetLastError();
}

cudaError_t fq_launch_queue_select(const FqQueueArgs& q, cudaStream_t stream)
{
  if (q.n <= 0) return cudaSuccess;
  fqp::fq_queue_select_kernel<<<(q.n + 127) / 128, 128, 0, stream>>>(q);
  return cudaGetLastError();
}

cudaError_t fq_launch_queue_pop(const FqQueueArgs& q, cudaStream_t stream)
{
  if (q.n <= 0) return cudaSuccess;
  fqp::fq_queue_pop_kernel<<<(q.n + 127) / 128, 128, 0, stream>>>(q);
  return cudaGetLastError();
}

cudaError_t fq_launch_pair_queue(const FqPairPlanArgs& a, const FqQueueArgs& q, cudaStream_t stream)
{
  if (a.n_prob <= 0) return cudaSuccess;
  fqp::fq_pair_queue_kernel<<<a.n_prob, 128, 0, stream>>>(a, q);
  return cudaGetLastError();
}

size_t fq_decomp_spill_n(int max_obs) { return max_obs > fqd::kFitPts ? (size_t)(max_obs - fqd::kFitPts) : 0; }

cudaError_t fq_launch_decomp(const FqDecompArgs& a, cudaStream_t stream)
{
  if (a.n_prob <= 0) return cudaSuccess;
  if (a.max_poly > 0) fqd::fq_decomp_kernel<<<a.n_prob * a.max_poly, fqd::kThreads, 0, stream>>>(a);
  fqd::fq_decomp_csr_kernel<<<1, 1024, 0, stream>>>(a);
  return cudaGetLastError();
}

namespace
{
__global__ void fq_map_table_kernel(const FqMapTableChunk c)
{
  const int i = threadIdx.x;
  if (i < c.n) c.table[c.at + i] = c.m[i];
}
}  // namespace

cudaError_t fq_launch_map_table(const FqMapTableChunk& c, cudaStream_t stream)
{
  if (c.n <= 0) return cudaSuccess;
  fq_map_table_kernel<<<1, FqMapTableChunk::kCap, 0, stream>>>(c);
  return cudaGetLastError();
}

#ifdef FQ_PHASE_CLOCKS
// measurement builds (tools/phase_clocks.py): fqt::fq_phase_clk of the current device summed over its replicas into
// out[whole][settled][9] (seven phase totals in clock cycles, the candidate count, then the corridor-scan total); reset != 0
// zeroes it afterwards
extern "C" int fq_phase_clocks(unsigned long long* out, int reset)
{
  static unsigned long long h[32][2][2][9];
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(h, fqt::fq_phase_clk, sizeof(h)) != cudaSuccess) return -1;
  for (int k = 0; k < 36; k++) out[k] = 0;
  for (int i = 0; i < 32; i++)
    for (int k = 0; k < 36; k++) out[k] += (&h[i][0][0][0])[k];
  if (reset)
  {
    static const unsigned long long z[32][2][2][9] = {};
    if (cudaMemcpyToSymbol(fqt::fq_phase_clk, z, sizeof(z)) != cudaSuccess) return -1;
  }
  return 0;
}
#endif
