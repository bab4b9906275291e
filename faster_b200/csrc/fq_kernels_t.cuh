// Size-specialised solver kernel (compile-time N and whole/safe mode) -- the product path.  Same algorithm as the
// generic kernel in fq_kernels.cu (dual active-set on the normalised, equality-eliminated QP of fq_plan.h) and the same
// answers (the two are differential-tested on the GPU); what changes is where things live and how the lanes are used:
//   * sizes are template constants: no integer division, bounded loops unroll, small vectors live in registers;
//   * every lane OWNS fixed rows of Y (row y = lane + 32 r, all three axes): the plan's constant part Yeq stays in
//     registers, Y = Yeq + TZ w costs one broadcast read of w per column, and the |v|,|a|,|j| box rows
//     (solverGurobi.cpp:390-407) are ranked by the owning lane while the value is still in a register;
//   * corridor rows (solverGurobi.cpp:249-287) are scanned through a per-candidate item list (segment, face), each lane
//     taking a run of faces of one segment whose control points it reads once; the control point shared with the
//     previous segment is skipped when both segments use the same polytope;
//   * the entering row is the one farthest beyond its hyperplane in w-space: rank = (violation - tol) / |TZ[y]|, compared
//     through the hi word of that double as a signed int (positive <=> violated), so the warp arg-max is one redux.sync,
//     and a second one on a tie code picks among equal keys.  This "normalised pivoting" halves the iteration count
//     relative to "largest violation";
//   * THIN factorisation: only J1 (NW x q, an orthonormal basis of the active normals, N = J1 R) is kept instead of the
//     full orthogonal J of the generic kernel.  The projection of a row normal g is z = -(g - J1 J1' g) (q columns, not
//     NW - q), a new active row appends one column -z/|z| (Gram-Schmidt, with one re-orthogonalisation pass when
//     |z|^2 < 0.01 |g|^2), nothing has to be initialised per candidate, and leaving rows rotate columns as before;
//   * duals, the triangular solve and the ratio test are register/shuffle based (element k of an NW-vector lives in
//     lane k%32, slot k/32); reciprocals and square roots use the MUFU seed + Newton steps instead of IEEE division;
//   * persistent CTAs, warp-independent: per-problem claim counters in global memory; every warp adopts a problem that
//     still has unclaimed candidates, stages its polytope rows into its own copy ([Ax Ay Az b+tol], checked for
//     non-finite values), and claims candidates one at a time from the end of the problem's list, so nobody idles behind
//     a slow candidate and no block barrier follows the staging of the plan tables; the triangular factor R is stored
//     packed, which is what leaves room for the four row copies at 4 CTAs per SM;
//   * non-finite or non-positive inputs make a candidate "not solved" up front (NaN rank keys would look satisfied).
#pragma once

namespace fqt
{
constexpr unsigned FULL = 0xffffffffu;
constexpr int W = FQ_WARPS_PER_CTA;
constexpr unsigned BOX_FLAG = 0x40000000u;

template <int N_, bool WHOLE_>
struct Dims
{
  static constexpr int N = N_;
  static constexpr int NE = WHOLE_ ? 3 : 2;
  static constexpr int NZ = N_ - NE;
  static constexpr int NW = 3 * NZ;
  static constexpr int NY = 6 * N_ + 1;
  static constexpr int NYP = NY | 1;             // odd row stride of Y per axis
  static constexpr int LD = NW | 1;              // odd leading dimension of J
  static constexpr int TZLD = NZ | 1;            // odd row stride of TZ in shared memory
  static constexpr int SLOTS = (NW + 31) / 32;   // elements of an NW-vector per lane
  static constexpr int RPL = (NY + 31) / 32;     // Y rows per lane
  static constexpr int RSZ = NW * (NW + 1) / 2;  // doubles of the packed triangular factor
  static constexpr int JR = NW * LD + RSZ;       // J then R, contiguous
  static constexpr int PER_WARP_DOUBLES = JR + 3 * NYP + 3 * NW + 2;
  // element (row j, column k), j <= k, of R: column k starts at k(k+1)/2
  __host__ __device__ static constexpr int ri(int j, int k) { return (k * (k + 1)) / 2 + j; }
};
// per-warp bytes: solver state + item list (item_cap 16-bit entries)
template <class D>
__host__ __device__ inline int per_warp_bytes(int item_cap) { return D::PER_WARP_DOUBLES * 8 + ((item_cap * 2 + 15) & ~15); }

// -DFQ_PHASE_CLOCKS (measurement builds only, tools/phase_clocks.py): clock64() stamps at the ends of the phases of one
// candidate's solve, accumulated per (mode, outcome) into fq_phase_clk[replica][whole][settled] = 7 phase totals, a
// count and the corridor-scan total.  Stamp 0 is taken before the claim, stamp k (1..6) ends phase k-1, the return from
// solve_candidate ends phase 6: claim and input loads, setup_rows and the guards, the segment-0 check, build_items, the
// first scan (with w = 0 and update_Y), the iterations, the outputs.  Stamp 8 holds the outcome: settled at w = 0 means
// optimal with no iteration or infeasible at the first entering row.  Slot 9 sums the cycles of every corridor-row scan of
// gi_loop (the first one and those of the iterations, up to the warp's choice of the entering row): a part of phases 4
// and 5, not a phase of its own.  32 replicas (by CTA) keep the atomics from queueing on one address.
#ifdef FQ_PHASE_CLOCKS
#define FQ_STAMP(clk, k) do { if (clk) (clk)[k] = clock64(); } while (0)
static __device__ unsigned long long fq_phase_clk[32][2][2][9];
#else
#define FQ_STAMP(clk, k) do { } while (0)
#endif

__device__ __forceinline__ double fast_rcp(double x)
{
  double r;
#ifdef FQ_EMULATE_ON_HOST          // tests/cpp/kernel_emu.cpp: this source under a host-side warp emulation (no inline PTX there)
  r = (double)(float)(1.0 / x);
#else
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
#endif
  r = fma(fma(-x, r, 1.0), r, r);
  r = fma(fma(-x, r, 1.0), r, r);
  return r;
}
__device__ __forceinline__ double fast_rsqrt(double x)
{
  double r;
#ifdef FQ_EMULATE_ON_HOST
  r = (double)(float)(1.0 / sqrt(x));
#else
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
#endif
  const double hx = 0.5 * x;
  r = fma(fma(-hx * r, r, 0.5), r, r);
  r = fma(fma(-hx * r, r, 0.5), r, r);
  r = fma(fma(-hx * r, r, 0.5), r, r);
  return r;
}
__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}
__device__ __forceinline__ double warp_min(double v)
{
  // order-preserving integer image of a double (no NaN here): for negative values the magnitude bits are inverted, so the
  // signed order of the hi words and the unsigned order of the lo words are the numeric order; two redux.sync give the
  // exact minimum
  const int hi = __double2hiint(v), neg = hi >> 31;
  const int khi = hi ^ (neg & 0x7fffffff);
  const unsigned klo = (unsigned)__double2loint(v) ^ (unsigned)neg;
  const int mh = __reduce_min_sync(FULL, khi);
  const unsigned ml = __reduce_min_sync(FULL, khi == mh ? klo : 0xffffffffu);
  const int mneg = mh >> 31;
  return __hiloint2double(mh ^ (mneg & 0x7fffffff), (int)(ml ^ (unsigned)mneg));
}

// staged polytope rows, 32 bytes each: row gf = (a01 = [Ax Ay], a23 = [Az b+tol])
__device__ __forceinline__ double2 row_a01(const double* __restrict__ sAb, int gf)
{
  return *reinterpret_cast<const double2*>(sAb + 4 * gf);
}
__device__ __forceinline__ double2 row_a23(const double* __restrict__ sAb, int gf)
{
  return *reinterpret_cast<const double2*>(sAb + 4 * gf + 2);
}
// staging: double2 number i of the source rows (even: [Ax Ay] of row i/2, odd: [Az b] of row i/2)
__device__ __forceinline__ void row_store(double* __restrict__ sAb, int i, double2 v)
{
  reinterpret_cast<double2*>(sAb)[i] = v;
}

template <class D>
struct WarpState
{
  double* J;            // NW x LD row-major
  double* R;            // upper triangular, packed column-major: R(j,k) at R[D::ri(j,k)]
  double* Y;            // 3 x NYP
  double* w;            // NW
  double* d;            // NW
  double* zb;           // NW: scratch for the re-orthogonalisation pass
  unsigned short* items;
};

// Ranking key of a row: hi word of (violation - tol) * S[y] as a signed int, S[y] = 1/|TZ[y]| (distance of the
// iterate to the row's hyperplane in w-space, for unit face normals).  Positive iff the row is violated; ordering
// positive doubles by their hi word keeps 20 mantissa bits, plenty for choosing the entering row.
__device__ __forceinline__ int rank_key(double u) { return __double2hiint(u); }

// Y = Yeq + TZ w for the lane's rows, box rows checked on the fly.  Updates the lane's best (key, code).
// bthr[r] = (limit + tol) * dt^k for box rows (huge for other rows), srow[r] = S[y].
template <class D, bool ZERO_W = false>
__device__ __forceinline__ void update_Y(const WarpState<D>& m, const double* __restrict__ TZ,
                                         const double (&Yeq)[D::RPL][3], const double (&bthr)[D::RPL],
                                         const double* __restrict__ SY, int lane, int& bkey, unsigned& bcode)
{
  double acc[D::RPL][3];
#pragma unroll
  for (int r = 0; r < D::RPL; r++)
#pragma unroll
    for (int ax = 0; ax < 3; ax++) acc[r][ax] = Yeq[r][ax];
#pragma unroll
  for (int k = 0; k < (ZERO_W ? 0 : D::NZ); k++)      // ZERO_W: first evaluation of a candidate, w = 0
  {
    const double w0 = m.w[k], w1 = m.w[D::NZ + k], w2 = m.w[2 * D::NZ + k];
#pragma unroll
    for (int r = 0; r < D::RPL; r++)
    {
      const int y = lane + 32 * r;
      if (y < D::NY)
      {
        const double t = TZ[y * D::TZLD + k];
        acc[r][0] = fma(t, w0, acc[r][0]);
        acc[r][1] = fma(t, w1, acc[r][1]);
        acc[r][2] = fma(t, w2, acc[r][2]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < D::RPL; r++)
  {
    const int y = lane + 32 * r;
    if (y < D::NY)
    {
      const double sr = SY[y];
#pragma unroll
      for (int ax = 0; ax < 3; ax++)
      {
        m.Y[ax * D::NYP + y] = acc[r][ax];
        const int key = rank_key((fabs(acc[r][ax]) - bthr[r]) * sr);
        if (key > bkey) { bkey = key; bcode = BOX_FLAG | (unsigned)(ax << 8) | (unsigned)y; }
      }
    }
  }
  __syncwarp();
}

// remove active element l (0 <= l < q); lam / rdinv are per-lane register slots
template <class D>
__device__ __forceinline__ void drop_row(const WarpState<D>& m, int lane, int l, int q, double (&lam)[D::SLOTS],
                                         double (&rdinv)[D::SLOTS])
{
  constexpr int LD = D::LD;
  // The columns right of l move one place left and become upper Hessenberg: the element below the new diagonal of
  // column k is the OLD diagonal of column k+1.  Packed storage has no room for it, so each lane keeps the old
  // diagonal of "its" column in a register; rotation j reads it by shuffle (no earlier rotation touches row j+1).
  double dg[D::SLOTS];
#pragma unroll
  for (int s = 0; s < D::SLOTS; s++)
  {
    const int k = lane + 32 * s;
    dg[s] = k < q ? m.R[D::ri(k, k)] : 0.0;
  }
  __syncwarp();
#pragma unroll
  for (int s = 0; s < D::SLOTS; s++)
  {
    const int j = lane + 32 * s;                 // this lane moves row j of every column that keeps a row j
    if (j < q)
      for (int k = (l > j ? l : j); k < q - 1; k++) m.R[D::ri(j, k)] = m.R[D::ri(j, k + 1)];
  }
  // lam: element k <- element k+1 for k in [l, q-1)
  {
    double nxt[D::SLOTS];
#pragma unroll
    for (int s = 0; s < D::SLOTS; s++)
    {
      const double same = __shfl_sync(FULL, lam[s], (lane + 1) & 31);
      const double wrap = (s + 1 < D::SLOTS) ? __shfl_sync(FULL, lam[(s + 1 < D::SLOTS) ? s + 1 : s], 0) : 0.0;
      nxt[s] = lane == 31 ? wrap : same;
    }
#pragma unroll
    for (int s = 0; s < D::SLOTS; s++)
    {
      const int k = lane + 32 * s;
      if (k >= l && k < q - 1) lam[s] = nxt[s];
    }
  }
  __syncwarp();
  for (int j = l; j < q - 1; j++)
  {
    const double p = m.R[D::ri(j, j)];
    const int js = (j + 1) >> 5;
    const double sb = __shfl_sync(FULL, (D::SLOTS > 1 && js == 1) ? dg[D::SLOTS - 1] : dg[0], (j + 1) & 31);
    const double h2 = fma(p, p, sb * sb);
    double c = 1.0, sn = 0.0, hi = 0.0;
    if (h2 > 0) { hi = fast_rsqrt(h2); c = p * hi; sn = sb * hi; }
    __syncwarp();
#pragma unroll
    for (int s = 0; s < D::SLOTS; s++)
    {
      const int k = lane + 32 * s;
      if (k > j && k < q - 1)
      { // rows j, j+1 of R at column k (both inside the triangle)
        const double u = m.R[D::ri(j, k)], v = m.R[D::ri(j + 1, k)];
        m.R[D::ri(j, k)] = fma(c, u, sn * v);
        m.R[D::ri(j + 1, k)] = fma(c, v, -sn * u);
      }
      if (k == j) { m.R[D::ri(j, j)] = fma(c, p, sn * sb); rdinv[s] = hi; }   // the element below it rotates to zero
      if (k < D::NW)
      { // columns j, j+1 of J at row k
        const double u = m.J[k * LD + j], v = m.J[k * LD + j + 1];
        m.J[k * LD + j] = fma(c, u, sn * v);
        m.J[k * LD + j + 1] = fma(c, v, -sn * u);
      }
    }
    __syncwarp();
  }
}

// Per-lane constants of one (problem, dt): Yeq of the lane's rows and the box thresholds (limit + tol) * dt^k.
template <class D>
__device__ __forceinline__ void setup_rows(const FqKernelArgs& a, int prob, double dt, double lim0, double lim1, double lim2,
                                           int lane, double (&Yeq)[D::RPL][3], double (&bthr)[D::RPL])
{
  constexpr int N = D::N, NY = D::NY, NE = D::NE;
  const double dt2 = dt * dt;
  {
    double hdr[3][3 + NE];
    const double* x0 = a.x0 + prob * 9;
    const double* xf = a.xf + prob * 9;
#pragma unroll
    for (int ax = 0; ax < 3; ax++)
    {
      const double s0 = x0[ax], s1 = x0[3 + ax] * dt, s2 = x0[6 + ax] * dt2;
      hdr[ax][0] = s0; hdr[ax][1] = s1; hdr[ax][2] = s2;
      double tgt[3];
      int e = 0;
      if (NE == 3) tgt[e++] = xf[ax];
      tgt[e++] = xf[3 + ax] * dt;
      tgt[e++] = xf[6 + ax] * dt2;
#pragma unroll
      for (int k = 0; k < NE; k++)
        hdr[ax][3 + k] = tgt[k] - fma(a.FT[k * 3 + 0], s0, fma(a.FT[k * 3 + 1], s1, a.FT[k * 3 + 2] * s2));
    }
#pragma unroll
    for (int r = 0; r < D::RPL; r++)
    {
      const int y = lane + 32 * r;
      // box type of the row: v (rows N+1..2N), a (2N+1..3N), j (3N+1..4N), none otherwise
      bthr[r] = (y >= N + 1 && y <= 2 * N) ? (lim0 + a.row_tol) * dt
                : ((y >= 2 * N + 1 && y <= 3 * N) ? (lim1 + a.row_tol) * dt2
                                                  : ((y >= 3 * N + 1 && y <= 4 * N) ? (lim2 + a.row_tol) * dt2 * dt : 1e300));
#pragma unroll
      for (int ax = 0; ax < 3; ax++) Yeq[r][ax] = 0.0;
      if (y < NY)
      {
        const double* t0 = a.T0 + y * (3 + NE);
#pragma unroll
        for (int k = 0; k < 3 + NE; k++)
        {
          const double t = __ldg(t0 + k);
#pragma unroll
          for (int ax = 0; ax < 3; ax++) Yeq[r][ax] = fma(t, hdr[ax][k], Yeq[r][ax]);
        }
      }
    }
  }
}

// Corridor item list of the first n_seg segments: item = t << 12 | need_cp0 << 11 | face (row of the staged Ab), segment
// by segment, in face order within a segment.  `p` = polytope of segment `lane` (meaningful for lane < n_seg).
// The scan of gi_loop gives every lane one RUN of consecutive items of ONE segment, so that the lane reads the segment's
// control points once per scan and then only the face rows: each segment is shared by 32 / n_seg lanes in equal runs.
// Returns this lane's run, count << 20 | first item (count 0: no run), or -1 when the list does not fit item_cap (the
// same for every lane); the caller's next __syncwarp publishes the items to the warp.
template <class D>
__device__ __forceinline__ int build_items(const WarpState<D>& m, const int* __restrict__ sfo, int lane, int n_seg, int p,
                                           int item_cap)
{
  int F = 0;
  if (lane < n_seg) F = sfo[p + 1] - sfo[p];
  const int pprev = __shfl_up_sync(FULL, p, 1);
  const int need0 = (lane == 0 || pprev != p) ? 1 : 0;
  int incl = F;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1)
  {
    const int v = __shfl_up_sync(FULL, incl, o);
    if (lane >= o) incl += v;
  }
  const int total_rows = __shfl_sync(FULL, incl, n_seg - 1);
  if (total_rows > item_cap) return -1;     // a wrong max_faces_per_polytope hint (device-pointer entry): refuse, never overrun
  // lane t writes segment t's items, in face order from its first item: independent stores, where a search of every item's
  // segment would chain dependent shared-memory loads.  item_cap >= N * (faces of the largest polytope) >= total_rows by
  // construction (host side)
  if (lane < n_seg)
  {
    unsigned short* dst = m.items + (incl - F);
    const int meta = (lane << 12) | (need0 << 11) | sfo[p];
    for (int k = 0; k < F; k++) dst[k] = (unsigned short)(meta + k);
  }
  // ---- runs: G = 32 / n_seg lanes per segment (a constant in the solve kernels); lane l takes run l % G of segment l / G,
  //      ceil(F / G) items long.  Lanes past G * n_seg fall on a segment beyond n_seg (F = 0) and get no items
  const int G = 32 / n_seg;
  const int s = lane / G, k = lane - s * G;
  const int fs = __shfl_sync(FULL, F, s), f0 = __shfl_sync(FULL, incl - F, s);
  const int len = (fs + G - 1) / G;
  const int cnt = max(0, min(len, fs - k * len));
  return (cnt << 20) | (cnt > 0 ? f0 + k * len : 0);
}

// The dual active-set iteration: from the current state (w, J, R in shared; lam, rdinv, q in registers; Y and the lane's
// rank key/code already evaluated for the current w) run until no enabled row is violated (returns 1), a violated row
// cannot be reached (0) or the iteration cap / a NaN is hit (-1).  Enabled rows = box rows + the items of m.items, which
// the lanes scan in the runs build_items gave them (`run`: this lane's).  Used by the fixed-assignment solve below and by
// the branch-and-bound node solve (fq_bnb.cuh), which enters with a parent's factorisation instead of the identity.
// A box row's scale 1/dt^k (inv1..3) and limit (lim0..2) are held in registers through the iteration, except with
// BOX_AT_ENTRY: then they are read through `dtp` (the time allocation dt) and `lim` (the problem's three limits) and
// recomputed, bit for bit, where such a row enters.  That frees twelve registers in the N <= 10 solve kernels, which fill
// the register file at 4 CTAs per SM and spilled without it; the other instances keep the registers.
template <class D, bool BOX_AT_ENTRY = false>
__device__ __forceinline__ int gi_loop(const WarpState<D>& m, const double* __restrict__ TZ, const double* __restrict__ SY,
                                       const double* __restrict__ sAb, const double (&Yeq)[D::RPL][3],
                                       const double (&bthr)[D::RPL], int lane, int run, double inv1, double inv2,
                                       double inv3, double lim0, double lim1, double lim2, double row_tol,
                                       double (&lam)[D::SLOTS], double (&rdinv)[D::SLOTS], int& q, int& it, int bkey,
                                       unsigned bcode, const double* __restrict__ dtp = nullptr,
                                       const double* __restrict__ lim = nullptr, long long* clk = nullptr)
{
  constexpr int N = D::N, NZ = D::NZ, NW = D::NW, NYP = D::NYP, LD = D::LD, SLOTS = D::SLOTS;
  double r[SLOTS], z[SLOTS], dreg[SLOTS];
#pragma unroll
  for (int s = 0; s < SLOTS; s++) { r[s] = 0; z[s] = 0; dreg[s] = 0; }
  int status = -2;
  while (status == -2)
  {
    // ================= most violated corridor row (box rows were checked by update_Y) =================
#ifdef FQ_PHASE_CLOCKS
    const long long scan0 = clock64();
#endif
    // The lane scans its run (build_items): items i0 .. i0 + cnt - 1, faces gf0 .. of ONE segment t, whose control points
    // are read once.  Ties of the rank key are broken as a lane-strided scan (item i on lane i & 31 in pass i >> 5) breaks
    // them, by a tie code per candidate row: box rows of lane L (bkey/bcode, set by update_Y) L << 16, item i
    // (i & 31) << 16 | (i >> 5) + 1.  The entering row is the one of largest key, and of smallest tie code among those: the
    // lowest lane's, its box rows before its items, its earliest item -- the same row, so the same path, bit for bit.
    int btie = lane << 16;
    {
      const int cnt = run >> 20;
      if (cnt > 0)
      {
        const int i0 = run & 0xfffff;
        const unsigned item = m.items[i0];
        const int t = item >> 12, gf0 = item & 0x7ff;
        const bool need0 = (item & 0x800u) != 0;
        const double* Y0 = m.Y; const double* Y1 = m.Y + NYP; const double* Y2 = m.Y + 2 * NYP;
        const int y1 = 4 * N + 1 + t, y2 = 5 * N + 1 + t;
        const double c10 = Y0[y1], c11 = Y1[y1], c12 = Y2[y1], s1 = SY[y1];
        const double c20 = Y0[y2], c21 = Y1[y2], c22 = Y2[y2], s2 = SY[y2];
        const double c30 = Y0[t + 1], c31 = Y1[t + 1], c32 = Y2[t + 1], s3 = SY[t + 1];
        double c00 = 0, c01 = 0, c02 = 0, s0 = 0;
        if (need0) { c00 = Y0[t]; c01 = Y1[t]; c02 = Y2[t]; s0 = SY[t]; }
#pragma unroll 1
        for (int k = 0; k < cnt; k++)
        {
          const int gf = gf0 + k;
          const double2 a01 = row_a01(sAb, gf);
          const double2 a23 = row_a23(sAb, gf);                                       // a23.y = b + tol
          const double u1 = fma(a01.x, c10, fma(a01.y, c11, fma(a23.x, c12, -a23.y))) * s1;
          const double u2 = fma(a01.x, c20, fma(a01.y, c21, fma(a23.x, c22, -a23.y))) * s2;
          const double u3 = fma(a01.x, c30, fma(a01.y, c31, fma(a23.x, c32, -a23.y))) * s3;
          int km = max(max(rank_key(u1), rank_key(u2)), rank_key(u3));
          if (need0) km = max(km, rank_key(fma(a01.x, c00, fma(a01.y, c01, fma(a23.x, c02, -a23.y))) * s0));
          const int i = i0 + k, tie = ((i & 31) << 16) | ((i >> 5) + 1);
          if (km > bkey || (km == bkey && tie < btie)) { bkey = km; btie = tie; }
        }
      }
    }
    const int mk = __reduce_max_sync(FULL, bkey);
#ifdef FQ_PHASE_CLOCKS
    if (clk)
    {
      const long long scan1 = clock64();
      if (clk[5] == 0) clk[5] = scan1;
      clk[9] += scan1 - scan0;
    }
#endif
    if (mk <= 0) { status = 1; break; }
    const int mt = __reduce_min_sync(FULL, bkey == mk ? btie : 0x7fffffff);
    // a box row: lane mt >> 16 holds it in bcode (items never overwrite bcode); an item: its index, from the tie code
    const unsigned boxc = __shfl_sync(FULL, bcode, (mt >> 16) & 31);
    const unsigned code = (mt & 0xffff) == 0 ? boxc : (unsigned)((((mt & 0xffff) - 1) << 5) | (mt >> 16));
    // ---- decode the chosen row: Y row y, weights (w0,w1,w2), right-hand side h
    int y;
    double w0 = 0, w1 = 0, w2 = 0, h;
    if (code & BOX_FLAG)
    {
      y = code & 0xff;
      const int ax = (code >> 8) & 3;
      const double val = m.Y[ax * NYP + y];
      double sinv;
      if (BOX_AT_ENTRY)
      { // inv2 = inv1 * inv1, inv3 = inv2 * inv1, as the callers compute them
        const double i1 = 1.0 / *dtp;
        sinv = y <= 2 * N ? i1 : (y <= 3 * N ? i1 * i1 : i1 * i1 * i1);
        h = lim[y <= 2 * N ? 0 : (y <= 3 * N ? 1 : 2)];
      }
      else
      {
        sinv = y <= 2 * N ? inv1 : (y <= 3 * N ? inv2 : inv3);
        h = y <= 2 * N ? lim0 : (y <= 3 * N ? lim1 : lim2);
      }
      const double s = val > 0 ? sinv : -sinv;
      w0 = ax == 0 ? s : 0.0; w1 = ax == 1 ? s : 0.0; w2 = ax == 2 ? s : 0.0;
    }
    else
    {
      const unsigned item = m.items[code & 0x0fffffffu];
      const int t = item >> 12, gf = item & 0x7ff;
      const double2 r01 = row_a01(sAb, gf), r23 = row_a23(sAb, gf);
      w0 = r01.x; w1 = r01.y; w2 = r23.x;
      const double hb = r23.y;                      // b + tol
      h = hb - row_tol;
      const int ys[4] = { 4 * N + 1 + t, 5 * N + 1 + t, t + 1, t };
      y = ys[0];
      int best = -0x7fffffff;
#pragma unroll
      for (int k = 0; k < 4; k++)
      {
        if (k == 3 && !(item & 0x800u)) break;
        const int kk = rank_key(fma(w0, m.Y[ys[k]], fma(w1, m.Y[NYP + ys[k]], fma(w2, m.Y[2 * NYP + ys[k]], -hb))) * SY[ys[k]]);
        if (kk > best) { best = kk; y = ys[k]; }
      }
    }
    const double sy = SY[y];
    // |g|^2 = |w|^2 |TZ[y]|^2; the fma chain is spelled out so that the rounding of |w|^2 does not depend on which
    // product the compiler chooses to contract
    const double gg = fma(w2, w2, fma(w0, w0, w1 * w1)) * fast_rcp(sy * sy);
    double lam_p = 0;
    for (;;)
    {
      if (++it > FQ_MAX_ITERS) { status = -1; break; }
      const double viol = fma(w0, m.Y[y], fma(w1, m.Y[NYP + y], fma(w2, m.Y[2 * NYP + y], -h)));
      // ---- thin factorisation: J1 = first q columns of J, an orthonormal basis of the active normals (N = J1 R).
      //      d1 = J1' g with g = (w0, w1, w2) (x) TZ[y];  z = -(g - J1 d1) = minus the part of g outside span(J1)
      double gi[SLOTS];
      {
        double s0[SLOTS], s1[SLOTS], s2[SLOTS];
#pragma unroll
        for (int s = 0; s < SLOTS; s++) { s0[s] = 0; s1[s] = 0; s2[s] = 0; }
        if (q > 0)
        {
#pragma unroll
          for (int k = 0; k < NZ; k++)
          {
            const double tk = TZ[y * D::TZLD + k];
#pragma unroll
            for (int s = 0; s < SLOTS; s++)
            {
              const int j = lane + 32 * s;
              if (j < q)
              {
                s0[s] = fma(tk, m.J[k * LD + j], s0[s]);
                s1[s] = fma(tk, m.J[(NZ + k) * LD + j], s1[s]);
                s2[s] = fma(tk, m.J[(2 * NZ + k) * LD + j], s2[s]);
              }
            }
          }
        }
#pragma unroll
        for (int s = 0; s < SLOTS; s++)
        {
          const int j = lane + 32 * s;
          dreg[s] = fma(w0, s0[s], fma(w1, s1[s], w2 * s2[s]));
          if (j < q) m.d[j] = dreg[s];
          // this lane's component of g: variable j = (axis, column) of the plan table
          const int ax = j / NZ, kk = j - ax * NZ;
          gi[s] = j < NW ? (ax == 0 ? w0 : (ax == 1 ? w1 : w2)) * TZ[y * D::TZLD + kk] : 0.0;
        }
      }
      __syncwarp();
      double zzp = 0;
#pragma unroll
      for (int s = 0; s < SLOTS; s++)
      {
        const int i = lane + 32 * s;
        double acc0 = -gi[s], acc1 = 0;
        if (i < NW)
        {
          const double* Ji = m.J + i * LD;
          int k = 0;
          for (; k + 1 < q; k += 2)
          {
            acc0 = fma(Ji[k], m.d[k], acc0);
            acc1 = fma(Ji[k + 1], m.d[k + 1], acc1);
          }
          if (k < q) acc0 = fma(Ji[k], m.d[k], acc0);
        }
        z[s] = acc0 + acc1;
        zzp = fma(z[s], z[s], zzp);
      }
      // re-orthogonalise once when most of g lies in span(J1) (the subtraction above lost digits): "twice is enough"
      double zz = warp_sum(zzp);
      {
        if (q > 0 && zz < 0.01 * gg && zz > fmax(FQ_EPS_DEP * gg, FQ_ZZ_FLOOR))
        {
          __syncwarp();
#pragma unroll
          for (int s = 0; s < SLOTS; s++)
          {
            const int i = lane + 32 * s;
            if (i < NW) m.zb[i] = z[s];
          }
          __syncwarp();
          double c[SLOTS];
#pragma unroll
          for (int s = 0; s < SLOTS; s++)
          {
            const int k = lane + 32 * s;
            c[s] = 0;
            if (k < q)
            {
              for (int i = 0; i < NW; i++) c[s] = fma(m.J[i * LD + k], m.zb[i], c[s]);
              dreg[s] -= c[s];                       // g = J1 (d1 - c) - z': the new R column stays consistent
              m.d[k] = c[s];
            }
          }
          __syncwarp();
          zzp = 0;
#pragma unroll
          for (int s = 0; s < SLOTS; s++)
          {
            const int i = lane + 32 * s;
            if (i < NW)
            {
              const double* Ji = m.J + i * LD;
              double acc = z[s];
              for (int k = 0; k < q; k++) acc = fma(-Ji[k], m.d[k], acc);
              z[s] = acc;
            }
            zzp = fma(z[s], z[s], zzp);
          }
          __syncwarp();
#pragma unroll
          for (int s = 0; s < SLOTS; s++)
          {
            const int k = lane + 32 * s;
            if (k < q) m.d[k] = dreg[s];
          }
          zz = warp_sum(zzp);
        }
      }
      // ---- r = R^-1 d1 (registers + shuffles)
      // every lane pre-divides its own row by the diagonal (R(j,k) / R(j,j) does not depend on r_k), so the chain from
      // one r_k to the next is a shuffle and one FMA
#pragma unroll
      for (int s = 0; s < SLOTS; s++) r[s] = dreg[s] * rdinv[s];
      for (int k = q - 1; k >= 0; k--)
      {
        const int ks = k >> 5;
        const double rk = __shfl_sync(FULL, (SLOTS > 1 && ks == 1) ? r[SLOTS - 1] : r[0], k & 31);
#pragma unroll
        for (int s = 0; s < SLOTS; s++)
        {
          const int j = lane + 32 * s;
          if (j < k) r[s] = fma(-m.R[D::ri(j, k)] * rdinv[s], rk, r[s]);
        }
      }
      // ---- dual ratio test and the step scalars
      double best = INFINITY;
      int bk = -1;
#pragma unroll
      for (int s = 0; s < SLOTS; s++)
      {
        const int k = lane + 32 * s;
        if (k < q && r[s] > 0)
        {
          const double ratio = lam[s] * fast_rcp(r[s]);
          if (ratio < best) { best = ratio; bk = k; }
        }
      }
      const double t1 = warp_min(best);
      const double zzs = fmax(zz, 1e-300);
      const double rn = fast_rsqrt(zzs), rzz = fast_rcp(zzs);
      // q == NW: the active normals already span the space; whatever rounding leaves in z, the row is dependent (and a
      // further column would not fit the factorisation's storage)
      const bool dep = zz <= fmax(FQ_EPS_DEP * gg, FQ_ZZ_FLOOR) || q >= NW;
      int l = -1;
      if (t1 < INFINITY)
      {
        const int s2 = __ffs(__ballot_sync(FULL, best == t1)) - 1;
        l = __shfl_sync(FULL, bk, s2);
      }
      const double t2 = dep ? INFINITY : viol * rzz;
      if (t1 == INFINITY && t2 == INFINITY) { status = 0; break; }
      if (t2 <= t1)
      { // ---- full step: the row becomes active; new basis vector = normalised residual of g
        const double nrm = zz * rn;
#pragma unroll
        for (int s = 0; s < SLOTS; s++)
        {
          const int i = lane + 32 * s;
          if (i < NW)
          {
            m.w[i] = fma(t2, z[s], m.w[i]);
            m.J[i * LD + q] = -z[s] * rn;
          }
          if (i < q) { lam[s] = fma(-t2, r[s], lam[s]); m.R[D::ri(i, q)] = dreg[s]; }
          if (i == q) { lam[s] = lam_p + t2; rdinv[s] = rn; m.R[D::ri(q, q)] = nrm; }
        }
        q++;
        __syncwarp();
        bkey = 0; bcode = 0;
        update_Y<D>(m, TZ, Yeq, bthr, SY, lane, bkey, bcode);
        break;
      }
      // ---- partial step: active element l leaves.  (l < 0 here means t1/t2 are NaN -- non-finite input: give up)
      if (l < 0) { status = -1; break; }
#pragma unroll
      for (int s = 0; s < SLOTS; s++)
      {
        const int i = lane + 32 * s;
        if (!dep && i < NW) m.w[i] = fma(t1, z[s], m.w[i]);
        if (i < q) lam[s] = fma(-t1, r[s], lam[s]);
      }
      lam_p += t1;
      __syncwarp();
      drop_row<D>(m, lane, l, q, lam, rdinv);
      q--;
      if (!dep)
      {
        int dummy_k = 0;
        unsigned dummy_c = 0;
        update_Y<D>(m, TZ, Yeq, bthr, SY, lane, dummy_k, dummy_c);
      }
    }
  }

  return status;
}

template <class D>
__device__ void solve_candidate(const FqKernelArgs& a, const double* __restrict__ TZ,
                                const double* __restrict__ SY, const double* __restrict__ sAb,
                                const int* __restrict__ sfo, const WarpState<D>& m,
                                int prob, int cand, int lane, int rows_bad, long long* clk = nullptr)
{
  constexpr int N = D::N, NW = D::NW, NYP = D::NYP, SLOTS = D::SLOTS;
  // N <= 10: 4 CTAs per SM at 128 registers, the whole register file.  These instances keep nothing through the
  // iteration that can be read or recomputed after it (gi_loop's BOX_AT_ENTRY); the others have registers to spare.
  constexpr bool LEAN = N <= 10;
  const double dt = a.dt[cand];
  const double inv1 = 1.0 / dt, inv2 = inv1 * inv1, inv3 = inv2 * inv1;
  const double lim0 = a.lim[prob * 3 + 0], lim1 = a.lim[prob * 3 + 1], lim2 = a.lim[prob * 3 + 2];
  const int P = a.poly_ofs[prob + 1] - a.poly_ofs[prob];
  FQ_STAMP(clk, 1);

  // ---- per-lane constants of the owned rows: Yeq, box scale and limit
  double Yeq[D::RPL][3], bthr[D::RPL];
  setup_rows<D>(a, prob, dt, lim0, lim1, lim2, lane, Yeq, bthr);
  // ---- non-finite or non-positive inputs (the device-pointer entry cannot be validated on the host): such a
  //      candidate is reported "not solved" right away.  NaN keys would otherwise rank as "satisfied".
  {
    bool okc = dt > 0 && dt < 1e100 && lim0 > 0 && lim0 < 1e300 && lim1 > 0 && lim1 < 1e300 && lim2 > 0 && lim2 < 1e300 &&
               rows_bad == 0;
#pragma unroll
    for (int r = 0; r < D::RPL; r++)
#pragma unroll
      for (int ax = 0; ax < 3; ax++) okc = okc && fabs(Yeq[r][ax]) < 1e300;
    FQ_STAMP(clk, 2);
    if (!__all_sync(FULL, okc))
    {
      if (lane == 0)
      {
        a.feasible[cand] = 0;
        a.cost[cand] = INFINITY;
        if (a.iters) a.iters[cand] = rows_bad == 2 ? -2 : -1;   // -2: the problem's rows exceed the max_faces hint
      }
      if (a.coeffs)
        for (int idx = lane; idx < 12 * N; idx += 32) a.coeffs[(size_t)cand * N * 12 + idx] = 0.0;
      return;
    }
  }
  // ---- corridor item list
  int run = 0;                                   // this lane's run of corridor items (none without polytopes)
  if (P > 0)
  {
    int p = 0;
    if (lane < N)
    {
      p = a.sigma[(size_t)cand * N + lane];
      if (p >= P) p = P - 1;
    }
    // ---- control points 0..2 of segment 0 depend on x0 and dt only (rows 0, 4N+1, 5N+1 of the plan are zero, SY = 1e15):
    //      one outside a face of sigma[0] refutes the candidate.  Same expression and rank key as the scan of gi_loop,
    //      which would pick such a row first (SY outranks everything) and stop on it: flags are unchanged, iters = 1.
    {
      constexpr int YS[3] = { 0, 4 * N + 1, 5 * N + 1 };
      if (SY[YS[0]] == 1e15 && SY[YS[1]] == 1e15 && SY[YS[2]] == 1e15)
      {
        double c[3][3];
#pragma unroll
        for (int k = 0; k < 3; k++)
#pragma unroll
          for (int ax = 0; ax < 3; ax++) c[k][ax] = __shfl_sync(FULL, Yeq[YS[k] >> 5][ax], YS[k] & 31);
        const int p0 = __shfl_sync(FULL, p, 0);
        bool out = false;
        for (int gf = sfo[p0] + lane; gf < sfo[p0 + 1]; gf += 32)
        {
          const double2 a01 = row_a01(sAb, gf), a23 = row_a23(sAb, gf);
#pragma unroll
          for (int k = 0; k < 3; k++)
            out = out || rank_key(fma(a01.x, c[k][0], fma(a01.y, c[k][1], fma(a23.x, c[k][2], -a23.y))) * 1e15) > 0;
        }
        FQ_STAMP(clk, 3);
        if (__any_sync(FULL, out))
        {
#ifdef FQ_PHASE_CLOCKS
          if (clk) clk[8] = 1;
#endif
          if (lane == 0)
          {
            a.feasible[cand] = 0;
            a.cost[cand] = INFINITY;
            if (a.iters) a.iters[cand] = 1;
          }
          if (a.coeffs)
            for (int idx = lane; idx < 12 * N; idx += 32) a.coeffs[(size_t)cand * N * 12 + idx] = 0.0;
          return;
        }
      }
    }
    FQ_STAMP(clk, 3);
    run = build_items<D>(m, sfo, lane, N, p, a.item_cap);
    FQ_STAMP(clk, 4);
    if (run < 0)
    { // the row list does not fit: report "not solved" (iters = -2 marks the cause)
      if (lane == 0)
      {
        a.feasible[cand] = 0;
        a.cost[cand] = INFINITY;
        if (a.iters) a.iters[cand] = -2;
      }
      if (a.coeffs)
        for (int idx = lane; idx < 12 * N; idx += 32) a.coeffs[(size_t)cand * N * 12 + idx] = 0.0;
      return;
    }
  }
  // ---- w = 0 (the thin factor J1 starts empty: nothing to initialise)
#pragma unroll
  for (int s = 0; s < SLOTS; s++)
  {
    const int j = lane + 32 * s;
    if (j < NW) m.w[j] = 0.0;
  }
  __syncwarp();

  double lam[SLOTS], rdinv[SLOTS];
#pragma unroll
  for (int s = 0; s < SLOTS; s++) { lam[s] = 0; rdinv[s] = 0; }
  int q = 0, it = 0;
  int bkey = 0;
  unsigned bcode = 0;
  update_Y<D, true>(m, TZ, Yeq, bthr, SY, lane, bkey, bcode);
  const int status = gi_loop<D, LEAN>(m, TZ, SY, sAb, Yeq, bthr, lane, run, inv1, inv2, inv3, lim0, lim1, lim2,
                                      a.row_tol, lam, rdinv, q, it, bkey, bcode, a.dt + cand, a.lim + prob * 3, clk);
  FQ_STAMP(clk, 6);
#ifdef FQ_PHASE_CLOCKS
  if (clk) clk[8] = (status == 1 && it == 0) || (status == 0 && it == 1);
#endif

  // ================= outputs =================
#ifndef FQ_EMULATE_ON_HOST
  // LEAN: the output addresses are formed here from the 32-bit index; the compiler would otherwise form them once before
  // the solve (every exit path writes them) and hold them through the iteration
  if (LEAN) asm("" : "+r"(cand));
#endif
  // LEAN: the scales are recomputed (bit for bit) rather than held through the iteration
  const double oinv1 = LEAN ? 1.0 / dt : inv1, oinv2 = LEAN ? oinv1 * oinv1 : inv2, oinv3 = LEAN ? oinv2 * oinv1 : inv3;
  double cp = 0;
  if (status == 1)
    for (int i = lane; i < 3 * N; i += 32)
    {
      const int ax = i / N, t = i - ax * N;
      const double u = m.Y[ax * NYP + 3 * N + 1 + t];
      cp = fma(u, u, cp);
    }
  const double cost = status == 1 ? warp_sum(cp) * (oinv3 * oinv3) : INFINITY;   // (status is warp-uniform)
  if (lane == 0)
  {
    a.feasible[cand] = status == 1;
    a.cost[cand] = status == 1 ? cost : INFINITY;
    if (a.iters) a.iters[cand] = status == -1 ? -it : it;
    if (status == 1 && a.first_feasible) atomicMin(a.first_feasible + prob, (unsigned long long)__double_as_longlong(dt));
  }
  if (a.coeffs)
  {
    double* out = a.coeffs + (size_t)cand * N * 12;
    for (int idx = lane; idx < 12 * N; idx += 32)
    {
      const int t = idx / 12, c = idx - 12 * t, kind = c / 3, ax = c - 3 * kind;
      const double* Ya = m.Y + ax * NYP;
      double v;
      if (kind == 0) v = Ya[3 * N + 1 + t] * oinv3 * (1.0 / 6.0);
      else if (kind == 1) v = Ya[2 * N + 1 + t] * oinv2 * 0.5;
      else if (kind == 2) v = Ya[N + 1 + t] * oinv1;
      else v = Ya[t];
      out[idx] = status == 1 ? v : 0.0;
    }
  }
  __syncwarp();
}

// genNewTraj's selection (solverGurobi.cpp:445-472) by ONE warp, for a single-problem sweep whose candidates are dt-major
// with n_sigma assignments per time allocation: first time allocation with a feasible assignment, then the minimum cost,
// then the lowest assignment index (exact).  Writes the winner record to (host-mapped) memory.
template <int N_>
__device__ void sweep_tail_select(const FqKernelArgs& a, int c_begin, int count, int lane)
{
  const int ns = a.sweep_n_sigma;
  int first = 0x7fffffff;
  for (int i = lane; i < count; i += 32)
    if (a.feasible[c_begin + i]) { first = i; break; }
  first = __reduce_min_sync(FULL, first);
  if (first == 0x7fffffff)
  {
    if (lane == 0) { a.sweep_idx[0] = -1; a.sweep_idx[1] = -1; a.sweep_win[0] = INFINITY; }
    __threadfence_system();
    return;
  }
  const int dtw = first / ns;
  unsigned long long best = ~0ull;
  for (int s = lane; s < ns; s += 32)
  {
    const int i = c_begin + dtw * ns + s;
    if (a.feasible[i]) { const unsigned long long b = (unsigned long long)__double_as_longlong(a.cost[i]); best = b < best ? b : best; }
  }
  unsigned hi = __reduce_min_sync(FULL, (unsigned)(best >> 32));
  unsigned lo = __reduce_min_sync(FULL, (unsigned)(best >> 32) == hi ? (unsigned)best : 0xffffffffu);
  const unsigned long long cb = (unsigned long long)hi << 32 | lo;
  int sw = 0x7fffffff;
  for (int s = lane; s < ns; s += 32)
  {
    const int i = c_begin + dtw * ns + s;
    if (a.feasible[i] && (unsigned long long)__double_as_longlong(a.cost[i]) == cb) { sw = s; break; }
  }
  sw = __reduce_min_sync(FULL, sw);
  const int win = c_begin + dtw * ns + sw;
  if (lane == 0) { a.sweep_idx[0] = dtw; a.sweep_idx[1] = sw; a.sweep_win[0] = a.cost[win]; }
  for (int i = lane; i < 12 * N_; i += 32) a.sweep_win[1 + i] = a.coeffs[(size_t)win * 12 * N_ + i];
  __threadfence_system();
}

// Persistent CTAs.  counters[j] = next unclaimed candidate of problem j (zeroed before the launch).  Every warp on its own
// adopts a problem that still has unclaimed candidates (scanning from its own start so the adopters spread over the
// problems), stages the problem's polytope rows into its own copy, and claims candidates one by one with a global atomic
// until the problem is drained; several adopters may drain the same problem.  No barrier follows the staging of the plan
// tables: a warp never waits for its CTA-mates' last solves.
template <int N_, bool WHOLE_>
__global__ void __launch_bounds__(W * 32, (N_ <= 10 ? (WHOLE_ ? FQ_MIN_CTAS_WHOLE : FQ_MIN_CTAS_PER_SM) : (N_ <= FQ_MAX_N_3CTAS ? 3 : 2)))
    fq_solve_kernel_t(const FqKernelArgs a, int* __restrict__ counters)
{
  using D = Dims<N_, WHOLE_>;
  extern __shared__ __align__(16) unsigned char smem_raw[];

  double* sm = reinterpret_cast<double*>(smem_raw);
  double* sAb0 = sm;           sm += W * 4 * a.max_faces;
  double* TZ = sm;             sm += D::NY * D::TZLD;
  double* SY = sm;             sm += D::NY;
  unsigned char* wraw = reinterpret_cast<unsigned char*>(sm);
  const int pwb = per_warp_bytes<D>(a.item_cap);
  int* sfo0 = reinterpret_cast<int*>(wraw + (size_t)W * pwb);

  // ---- plan tables: once per CTA
  for (int i = threadIdx.x; i < D::NY * D::NZ; i += blockDim.x)
  {
    const int y = i / D::NZ, k = i - y * D::NZ;
    TZ[y * D::TZLD + k] = a.TZ[i];
  }
  for (int y = threadIdx.x; y < D::NY; y += blockDim.x)
  {
    double s = 0;
    for (int k = 0; k < D::NZ; k++) { const double t = a.TZ[y * D::NZ + k]; s = fma(t, t, s); }
    SY[y] = s > 1e-30 ? rsqrt(s) : 1e15;       // constant rows: any violation outranks everything (=> infeasible)
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  WarpState<D> m;
  {
    double* p = reinterpret_cast<double*>(wraw + (size_t)warp * pwb);
    m.J = p;   p += D::NW * D::LD;
    m.R = p;   p += D::RSZ;
    m.Y = p;   p += 3 * D::NYP;
    m.w = p;   p += D::NW;
    m.d = p;   p += D::NW + 2;
    m.zb = p;  p += D::NW;
    m.items = reinterpret_cast<unsigned short*>(p);
  }
  // smem_bytes_t (and the branch-and-bound's level_smem) still count 32 ints per warp after the sfo tables, which nothing
  // uses any more: left in, so that the shared-memory size limits of both kernels stay where they are
  __syncthreads();
  const int n_prob = a.n_prob;
  double* sAb = sAb0 + (size_t)warp * 4 * a.max_faces;
  int* sfo = sfo0 + 40 * warp;
  const long long me = (long long)blockIdx.x * W + warp, adopters = (long long)gridDim.x * W;
  const int cursor = (int)((me * n_prob) / adopters);            // warp-specific starting problem
  int visited = 0;
  for (;;)
  {
    // ---- adopt the next problem (cyclically from `cursor`) that still has unclaimed candidates
    int found = -1;
    while (visited < n_prob && found < 0)
    {
      const int j = visited + lane;
      int pj = cursor + j;
      if (pj >= n_prob) pj -= n_prob;
      bool open = false;
      if (j < n_prob)
        open = *reinterpret_cast<volatile int*>(counters + pj) < a.cand_ofs[pj + 1] - a.cand_ofs[pj];
      const unsigned bal = __ballot_sync(FULL, open);
      if (bal) { const int first = __ffs(bal) - 1; found = cursor + visited + first; visited += first + 1; }
      else visited += 32;
    }
    if (found < 0) break;
    const int prob = found >= n_prob ? found - n_prob : found;
    const int c_begin = a.cand_ofs[prob], count = a.cand_ofs[prob + 1] - c_begin;
    const int p0 = a.poly_ofs[prob], P = a.poly_ofs[prob + 1] - p0;
    const int f0 = a.face_ofs[p0];
    const int nf = P > 0 ? a.face_ofs[p0 + P] - f0 : 0;
    int rows_bad = 0;
    if (nf > a.max_faces || nf < 0) rows_bad = 2;  // a too small max_faces_per_prob hint (device-pointer entry): never
    else                                           // overrun the staging area, report the problem "not solved"
    {
      const double2* src = reinterpret_cast<const double2*>(a.Ab + (size_t)4 * f0);
      int bad = 0;
      for (int i = lane; i < 2 * nf; i += 32)
      {
        double2 v = src[i];
        bad |= !(fabs(v.x) < 1e300) || !(fabs(v.y) < 1e300);
        if (i & 1) v.y += a.row_tol;               // rows are staged as [Ax Ay Az b+tol]
        row_store(sAb, i, v);
      }
      for (int i = lane; i <= P && i < 36; i += 32) sfo[i] = a.face_ofs[p0 + i] - f0;
      rows_bad = __any_sync(FULL, bad) != 0 ? 1 : 0;
      __syncwarp();                                // publishes the staged rows to the warp
    }
    // claim candidates one ahead: the global atomic for the NEXT candidate is issued before the current one is solved,
    // so its round trip hides behind the solve instead of idling the warp between candidates
    int c = 0;
    if (lane == 0) c = atomicAdd(counters + prob, 1);
    c = __shfl_sync(FULL, c, 0);
    const bool ee = a.first_feasible != nullptr;   // early exit: genNewTraj's "first feasible factor wins" (solverGurobi.cpp:445-446)
    while (c < count)
    {
#ifdef FQ_PHASE_CLOCKS
      long long clk[10] = {};
      clk[0] = clock64();
#else
      long long* clk = nullptr;
#endif
      int cn = 0;
      if (lane == 0) cn = atomicAdd(counters + prob, 1);
      // claims run from the end of the list (long solves first); with the early exit from its start (smallest dt first)
      const int cand = c_begin + (ee ? c : count - 1 - c);
      int n_done = 1;                                // candidates this iteration finishes (more when it drains the list)
      bool skip = false;
      if (ee)
      {
        const unsigned long long best = *reinterpret_cast<volatile unsigned long long*>(a.first_feasible + prob);
        skip = (unsigned long long)__double_as_longlong(a.dt[cand]) > best;   // a smaller dt already has a feasible candidate
      }
      if (!skip)
      {
        solve_candidate<D>(a, TZ, SY, sAb, sfo, m, prob, cand, lane, rows_bad, clk);
#ifdef FQ_PHASE_CLOCKS
        const long long end = clock64();
        if (lane == 0)
        { // a phase an early exit skipped ends where the previous one did
          unsigned long long* acc = fq_phase_clk[blockIdx.x & 31][WHOLE_ ? 1 : 0][clk[8] ? 1 : 0];
          for (int k = 1; k <= 6; k++)
            if (clk[k] == 0) clk[k] = clk[k - 1];
          for (int k = 0; k < 6; k++) atomicAdd(acc + k, (unsigned long long)(clk[k + 1] - clk[k]));
          atomicAdd(acc + 6, (unsigned long long)(end - clk[6]));
          atomicAdd(acc + 7, 1ull);
          atomicAdd(acc + 8, (unsigned long long)clk[9]);
        }
#endif
      }
      else
      { // not evaluated: it cannot win.  Reported like an unsolved candidate, iters = -3 marks the reason.
        if (a.sorted_dt)
        { // ascending dt: every candidate after this one is beaten too -- take them all at once
          int old = 0;
          if (lane == 0) old = atomicExch(counters + prob, count + 1);
          old = __shfl_sync(FULL, old, 0);
          if (old < count) n_done += count - old;
          if (old < count)
            for (int i = c_begin + old + lane; i < c_begin + count; i += 32)
            {
              a.feasible[i] = 0; a.cost[i] = INFINITY;
              if (a.iters) a.iters[i] = -3;
              if (a.coeffs) for (int k = 0; k < 12 * D::N; k++) a.coeffs[(size_t)i * D::N * 12 + k] = 0.0;
            }
        }
        if (lane == 0)
        {
          a.feasible[cand] = 0; a.cost[cand] = INFINITY;
          if (a.iters) a.iters[cand] = -3;
        }
        if (a.coeffs)
          for (int idx = lane; idx < 12 * D::N; idx += 32) a.coeffs[(size_t)cand * D::N * 12 + idx] = 0.0;
      }
      if (a.sweep_done)
      { // single-problem sweep: whoever finishes the last candidate selects the winner (all results are published first)
        __threadfence();
        int fin = 0;
        if (lane == 0) fin = atomicAdd(a.sweep_done, n_done) + n_done;
        fin = __shfl_sync(FULL, fin, 0);
        if (fin == count)
        {
          __threadfence();
          sweep_tail_select<N_>(a, c_begin, count, lane);
        }
      }
      c = __shfl_sync(FULL, cn, 0);
    }
    __syncwarp();
  }
}

template <int N_, bool WHOLE_>
size_t smem_bytes_t(int max_faces, int item_cap, int sab_copies = W)
{
  using D = Dims<N_, WHOLE_>;
  return (size_t)8 * ((size_t)sab_copies * 4 * max_faces + D::NY * D::TZLD + D::NY) + (size_t)W * per_warp_bytes<D>(item_cap) +
         (40 * sab_copies + W * 32) * 4 + 16;
}

#ifndef FQ_EMULATE_ON_HOST
// `counters`: a.n_prob ints of device memory, zeroed here on `stream`
template <int N_, bool WHOLE_>
cudaError_t launch_t(const FqKernelArgs& a, long long total_cand_hint, cudaStream_t stream, int* counters, int sm_count)
{
  const size_t smem = smem_bytes_t<N_, WHOLE_>(a.max_faces, a.item_cap);
  if (smem > 227 * 1024) return cudaErrorInvalidConfiguration;   // caller falls back to the size-generic kernel
  auto kern = fq_solve_kernel_t<N_, WHOLE_>;
  // the shared-memory attribute and the occupancy query cost a few microseconds each: remembered per device (a replan
  // calls this with the same sizes every 10 ms; the chained replan four times per batch)
  struct Cached { size_t smem_set = 0, smem_occ = (size_t)-1; int per_sm = 0; };
  static Cached cache[64];
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  Cached local;
  Cached& cc = (dev >= 0 && dev < 64) ? cache[dev] : local;
  if (smem > cc.smem_set)
  {
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    cc.smem_set = smem;
  }
  if (smem != cc.smem_occ)
  {
    int q = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&q, kern, W * 32, smem);
    if (e != cudaSuccess) return e;
    cc.per_sm = q < 1 ? 1 : q;
    cc.smem_occ = smem;
  }
  const long long resident = (long long)cc.per_sm * sm_count;
  long long grid = resident;
  const long long need = (total_cand_hint + W - 1) / W;      // no point in more CTAs than candidates / warps
  if (grid > need) grid = need;
  if (a.first_feasible && a.sorted_dt && a.ee_width > 0 && need > resident)
  { // early exit on an ascending sweep that does not fit the GPU at once: keep only ~two time allocations per problem in
    // flight, so that the larger ones -- which cannot win once a smaller one is feasible -- are mostly never started.
    // A sweep that fits (one genNewTraj: a few hundred candidates) starts everything: a cap would only serialise it
    // (a capped sweep of one cfg4 corridor measured slower than an uncapped one).
    const long long cap = ((long long)a.n_prob * 2 * a.ee_width + W - 1) / W;
    if (grid > cap) grid = cap;
  }
  if (grid < 1) grid = 1;
  e = cudaMemsetAsync(counters, 0, sizeof(int) * ((size_t)a.n_prob + (a.sweep_done ? 1 : 0)), stream);
  if (e != cudaSuccess) return e;
  kern<<<(unsigned)grid, W * 32, smem, stream>>>(a, counters);
  return cudaGetLastError();
}
#endif
}  // namespace fqt
