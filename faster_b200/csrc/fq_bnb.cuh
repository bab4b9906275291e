// Exact MIQP for one corridor problem: branch-and-bound over the interval->polytope assignment (the binaries b[t][p]
// of the reference, solverGurobi.cpp:217-246) on the GPU, for several time allocations at once.
//
// A node fixes the polytopes of segments 0..k-1; its relaxation keeps every box row and the corridor rows of those
// segments only, so a child (one more segment fixed) only ADDS rows: the parent's optimum stays dual feasible and the
// dual active-set iteration continues from the parent's factorisation (w, J, R, multipliers), which a node stores in
// global memory.  One level of the tree is one launch (one warp per child): load the parent's state (7-8 KB, coalesced),
// build the row list of segments 0..k, iterate, then either drop the child (infeasible, or relaxation cost >= the
// incumbent of its time allocation) or store it for the next level; children at depth N are full assignments and lower
// the incumbent (atomicMin on the ordered bit pattern of the non-negative cost).  The incumbents start from the best
// non-decreasing assignment (evaluated beforehand by the ordinary batch solve), which is almost always optimal, so the
// tree only has to prove it.
//
// Several corridors at once (the chained replan, fq_pair_capi.cu): corridor c of the launch is problem c of the plan
// arguments; its nodes, leaves, counters and incumbents live in slices of their own, so a cut tree only affects its own
// corridor.  A level reads each corridor's parent count from device memory, so the levels of a sweep are enqueued without
// a host read in between.  CTAs are bound to one corridor (cpc of them per corridor), stage its rows once and stride over
// its children.  fq_gen_new_traj_exact runs the same kernel with one corridor and one warp per child.
#pragma once
#include "fq_assign.h"
#include "fq_presolve.h"

namespace fqb
{
constexpr int W = fqt::W;
constexpr unsigned FULL = fqt::FULL;
using fqt::build_items;
using fqt::Dims;
using fqt::gi_loop;
using fqt::per_warp_bytes;
using fqt::setup_rows;
using fqt::smem_bytes_t;
using fqt::update_Y;
using fqt::WarpState;

struct NodeHdr
{
  int dt_idx, depth, q, pad;
  unsigned char sigma[16];
};

struct LeafRec
{
  int dt_idx, pad;
  double cost;
  unsigned char sigma[16];
};

template <class D>
__host__ __device__ constexpr int node_doubles() { return D::JR + 3 * D::NW + ((D::JR + 3 * D::NW) & 1); }
template <class D>
__host__ __device__ constexpr size_t node_bytes() { return sizeof(NodeHdr) + sizeof(double) * node_doubles<D>(); }

struct BnbArgs
{
  FqKernelArgs k;                  // plan tables + the corridors (k.n_prob; corridor c is problem c); k.dt/k.sigma/outputs unused
  int n_dt;                        // time allocations per corridor: row length of dts, roots and incumbent
  const double* dts;               // device, n_prob x n_dt
  int depth;                       // depth of the parents of this launch (0: roots, state = identity)
  int cpc;                         // CTAs per corridor
  const int* n_parents;            // device, n_prob: parents of each corridor (depth 0: its roots)
  const unsigned char* parents;    // n_prob slices of cap nodes (ignored at depth 0: parent i is the root of dt index roots[i])
  const int* roots;                // depth 0 only: n_prob x n_dt dt indices
  unsigned char* children;         // n_prob slices of cap nodes
  int* n_children;                 // device, n_prob
  int cap;                         // nodes per corridor slice
  unsigned long long* incumbent;   // n_prob x n_dt: ordered bits of the best full-assignment cost so far
  LeafRec* leaves;                 // n_prob slices of leaf_cap
  int* n_leaves;                   // n_prob
  int leaf_cap;
  int* flags;                      // n_prob x 2: [0] overflow of children/leaves or rows, [1] numeric failures
  long long* nodes;                // n_prob: nodes evaluated, summed over the levels, or nullptr
  int keep_ties;                   // 0: prune at cost >= incumbent (> at the last level) and keep the leaves that
                                   //    lower or equal it;
                                   // 1: prune at cost > incumbent (1 + 1e-9) and keep every leaf within that bound
  // keep_ties only (nullptr otherwise), n_prob x n_dt each.  lbound: the smallest relaxation cost of depth 0 (segment 0
  // fixed), a lower bound on every assignment of that time allocation.  closed: set after level 0 (fq_bnb_certify_kernel)
  // where the list winner is certain to stand; no child of that time allocation is evaluated afterwards.  Both are final
  // before level 1 starts, so no pruning decision depends on the order in which warps finish except the incumbent's.
  unsigned long long* lbound;
  unsigned char* closed;
};

template <int N_, bool WHOLE_>
__global__ void __launch_bounds__(W * 32, (N_ <= 10 ? 4 : (N_ <= 15 ? 3 : 2))) fq_bnb_level_kernel(const BnbArgs b)
{
  using D = Dims<N_, WHOLE_>;
  constexpr int NW = D::NW, LD = D::LD, SLOTS = D::SLOTS, N = D::N, NYP = D::NYP;
  // N <= 10: 4 CTAs per SM at 128 registers.  As in the solve kernel (fqt::solve_candidate), the box scales and limits are
  // read or recomputed where they are needed, bit for bit, instead of held through the node solve
  constexpr bool LEAN = N <= 10;
  const FqKernelArgs& a = b.k;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* sm = reinterpret_cast<double*>(smem_raw);
  double* sAb = sm;            sm += 4 * a.max_faces;
  double* TZ = sm;             sm += D::NY * D::TZLD;
  double* SY = sm;             sm += D::NY;
  unsigned char* wraw = reinterpret_cast<unsigned char*>(sm);
  const int pwb = per_warp_bytes<D>(a.item_cap);
  int* sfo = reinterpret_cast<int*>(wraw + (size_t)W * pwb);

  const int c = blockIdx.x / b.cpc, sub = blockIdx.x - c * b.cpc;
  if (c >= a.n_prob) return;
  int* flg = b.flags + 2 * c;
  // one read of the parent count and the cut flag for the whole CTA (other CTAs may set the flag meanwhile), broadcast
  // through the unused word 36 of the face-offset block
  if (threadIdx.x == 0)
  {
    const int np = b.n_parents[c];
    sfo[36] = flg[0] != 0 ? 0 : (np < b.cap ? np : b.cap);   // a cut tree stops growing: its corridor falls back anyway
  }
  __syncthreads();
  const int n_par = sfo[36];
  const int p0 = a.poly_ofs[c], P = a.poly_ofs[c + 1] - p0;
  if (n_par <= 0 || P <= 0 || (long long)sub * W >= (long long)n_par * P) return;    // nothing for this CTA
  for (int i = threadIdx.x; i < D::NY * D::NZ; i += blockDim.x)
  {
    const int y = i / D::NZ, k = i - y * D::NZ;
    TZ[y * D::TZLD + k] = a.TZ[i];
  }
  for (int y = threadIdx.x; y < D::NY; y += blockDim.x)
  {
    double s = 0;
    for (int k = 0; k < D::NZ; k++) { const double t = a.TZ[y * D::NZ + k]; s = fma(t, t, s); }
    SY[y] = s > 1e-30 ? rsqrt(s) : 1e15;
  }
  const int f0 = a.face_ofs[p0];
  const int nf = a.face_ofs[p0 + P] - f0;
  bool rows_bad = false;
  {
    const double2* src = reinterpret_cast<const double2*>(a.Ab + (size_t)4 * f0);
    int bad = 0;
    const bool fits = nf >= 0 && nf <= a.max_faces;      // never overrun the staging area: cut the tree instead
    for (int i = threadIdx.x; fits && i < 2 * nf; i += blockDim.x)
    {
      double2 v = src[i];
      bad |= !(fabs(v.x) < 1e300) || !(fabs(v.y) < 1e300);
      if (i & 1) v.y += a.row_tol;
      fqt::row_store(sAb, i, v);
    }
    for (int i = threadIdx.x; i <= P && i < 36; i += blockDim.x) sfo[i] = a.face_ofs[p0 + i] - f0;
    rows_bad = __syncthreads_or(bad) != 0;
    if (!fits) { if (threadIdx.x == 0) flg[0] = 1; return; }
  }
  if (sub == 0 && threadIdx.x == 0 && b.nodes) b.nodes[c] += (long long)n_par * P;   // CTA 0 of a corridor always runs
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t slice = (size_t)c * b.cap;
  const int k = b.depth;
  unsigned long long* inc_row = b.incumbent + (size_t)c * b.n_dt;
  unsigned long long* lb_row = b.keep_ties && b.lbound ? b.lbound + (size_t)c * b.n_dt : nullptr;
  const unsigned char* closed_row = b.keep_ties && b.closed ? b.closed + (size_t)c * b.n_dt : nullptr;

  WarpState<D> m;
  {
    double* p = reinterpret_cast<double*>(wraw + (size_t)warp * pwb);
    m.J = p;   p += NW * LD;
    m.R = p;   p += D::RSZ;
    m.Y = p;   p += 3 * NYP;
    m.w = p;   p += NW;
    m.d = p;   p += NW + 2;
    m.zb = p;  p += NW;
    m.items = reinterpret_cast<unsigned short*>(p);
  }
  const long long n_child = (long long)n_par * P;
  for (long long child = (long long)sub * W + warp; child < n_child; child += (long long)b.cpc * W)
  {
    const int pi = (int)(child / P), pnew = (int)(child - (long long)pi * P);
    // ---- parent
    int dt_idx, q = 0;
    unsigned char sig[16];
    const unsigned char* pn = b.parents + (slice + pi) * node_bytes<D>();
    if (k == 0) dt_idx = b.roots[(size_t)c * b.n_dt + pi];
    else
    {
      const NodeHdr* h = reinterpret_cast<const NodeHdr*>(pn);
      dt_idx = h->dt_idx; q = h->q;
#pragma unroll
      for (int t = 0; t < 16; t++) sig[t] = h->sigma[t];
    }
    sig[k] = (unsigned char)pnew;
    if (closed_row && closed_row[dt_idx]) continue;     // the list winner stands at this time allocation (fixed since level 0)
    const double* dtp = b.dts + (size_t)c * b.n_dt + dt_idx;
    const double dt = *dtp;
    const double inv1 = 1.0 / dt, inv2 = inv1 * inv1, inv3 = inv2 * inv1;
    const double lim0 = a.lim[3 * c], lim1 = a.lim[3 * c + 1], lim2 = a.lim[3 * c + 2];
    double Yeq[D::RPL][3], bthr[D::RPL];
    setup_rows<D>(a, c, dt, lim0, lim1, lim2, lane, Yeq, bthr);
    {
      bool okc = dt > 0 && dt < 1e100 && lim0 > 0 && lim0 < 1e300 && lim1 > 0 && lim1 < 1e300 && lim2 > 0 && lim2 < 1e300 && !rows_bad;
#pragma unroll
      for (int r = 0; r < D::RPL; r++)
#pragma unroll
        for (int ax = 0; ax < 3; ax++) okc = okc && fabs(Yeq[r][ax]) < 1e300;
      if (!__all_sync(FULL, okc)) continue;      // non-finite input: the subtree is dropped (treated as infeasible)
    }
    // ---- state: identity at the roots, the parent's factorisation otherwise
    double lam[SLOTS], rdinv[SLOTS];
#pragma unroll
    for (int s = 0; s < SLOTS; s++) { lam[s] = 0; rdinv[s] = 0; }
    if (k == 0)
    { // roots: empty factorisation
#pragma unroll
      for (int s = 0; s < SLOTS; s++)
      {
        const int j = lane + 32 * s;
        if (j < NW) m.w[j] = 0.0;
      }
    }
    else
    {
      const double* st = reinterpret_cast<const double*>(pn + sizeof(NodeHdr));
      for (int idx = lane; idx < D::JR; idx += 32) m.J[idx] = st[idx];          // J then R (contiguous in both)
      const double* v = st + D::JR;
#pragma unroll
      for (int s = 0; s < SLOTS; s++)
      {
        const int j = lane + 32 * s;
        if (j < NW) { m.w[j] = v[j]; lam[s] = v[NW + j]; rdinv[s] = v[2 * NW + j]; }
      }
    }
    __syncwarp();
    // ---- rows of segments 0..k
    int run = 0;
    {
      int p = 0;
      if (lane <= k) p = sig[0];
#pragma unroll
      for (int t = 1; t < 16; t++)
        if (lane == t && t <= k) p = sig[t];
      run = build_items<D>(m, sfo, lane, k + 1, p, a.item_cap);
      if (run < 0) { if (lane == 0) flg[0] = 1; continue; }
    }
    int it = 0, bkey = 0;
    unsigned bcode = 0;
    if (k == 0) update_Y<D, true>(m, TZ, Yeq, bthr, SY, lane, bkey, bcode);
    else update_Y<D, false>(m, TZ, Yeq, bthr, SY, lane, bkey, bcode);
    const int status = gi_loop<D, LEAN>(m, TZ, SY, sAb, Yeq, bthr, lane, run, inv1, inv2, inv3, lim0, lim1, lim2, a.row_tol,
                                        lam, rdinv, q, it, bkey, bcode, dtp, a.lim + 3 * c);
    if (status != 1)
    {
      if (status == -1 && lane == 0) atomicAdd(flg + 1, 1);
      continue;
    }
    double cp = 0;
    for (int i = lane; i < 3 * N; i += 32)
    {
      const int ax = i / N, t = i - ax * N;
      const double u = m.Y[ax * NYP + 3 * N + 1 + t];
      cp = fma(u, u, cp);
    }
    const double oinv1 = LEAN ? 1.0 / dt : inv1, oinv3 = LEAN ? oinv1 * oinv1 * oinv1 : inv3;
    const double cost = fqt::warp_sum(cp) * (oinv3 * oinv3);
    const unsigned long long cbits = (unsigned long long)__double_as_longlong(cost);
    if (k == 0 && lb_row && lane == 0) atomicMin(lb_row + dt_idx, cbits);
    const unsigned long long inc = *reinterpret_cast<volatile unsigned long long*>(inc_row + dt_idx);
    // bound: children only add rows, the cost cannot decrease.  Without keep_ties a full assignment whose cost equals the
    // incumbent's is kept as well: the sweep then chooses among equal-cost leaves by assignment, not by which warp finished
    // first
    if (b.keep_ties ? !(cost <= __longlong_as_double((long long)inc) * (1.0 + 1e-9)) : (k + 1 == N ? cbits > inc : cbits >= inc))
      continue;
    if (k + 1 == N)
    { // a full assignment that beats or equals (or, keeping ties, comes within 1e-9 of) the incumbent
      if (lane == 0)
      {
        const unsigned long long old = atomicMin(inc_row + dt_idx, cbits);
        if (b.keep_ties || cbits <= old)
        {
          const int slot = atomicAdd(b.n_leaves + c, 1);
          if (slot < b.leaf_cap)
          {
            LeafRec* L = b.leaves + (size_t)c * b.leaf_cap + slot;
            L->dt_idx = dt_idx; L->pad = c; L->cost = cost;
            for (int t = 0; t < 16; t++) L->sigma[t] = t < N ? sig[t] : 0;
          }
          else flg[0] = 1;
        }
      }
      continue;
    }
    int slot = 0;
    if (lane == 0) slot = atomicAdd(b.n_children + c, 1);
    slot = __shfl_sync(FULL, slot, 0);
    if (slot >= b.cap) { if (lane == 0) flg[0] = 1; continue; }
    unsigned char* cn = b.children + (slice + slot) * node_bytes<D>();
    if (lane == 0)
    {
      NodeHdr* h = reinterpret_cast<NodeHdr*>(cn);
      h->dt_idx = dt_idx; h->depth = k + 1; h->q = q; h->pad = c;
      for (int t = 0; t < 16; t++) h->sigma[t] = t <= k ? sig[t] : 0;
    }
    double* st = reinterpret_cast<double*>(cn + sizeof(NodeHdr));
    for (int idx = lane; idx < D::JR; idx += 32) st[idx] = m.J[idx];
    double* v = st + D::JR;
#pragma unroll
    for (int s = 0; s < SLOTS; s++)
    {
      const int j = lane + 32 * s;
      if (j < NW) { v[j] = m.w[j]; v[NW + j] = lam[s]; v[2 * NW + j] = rdinv[s]; }
    }
    __syncwarp();
  }
}

template <int N_, bool WHOLE_>
size_t level_smem(int max_faces, int item_cap) { return smem_bytes_t<N_, WHOLE_>(max_faces, item_cap, 1); }   // one CTA-wide copy of the rows

#ifndef FQ_EMULATE_ON_HOST
template <int N_, bool WHOLE_>
cudaError_t launch_level(const BnbArgs& b, cudaStream_t stream)
{
  const size_t smem = level_smem<N_, WHOLE_>(b.k.max_faces, b.k.item_cap);
  if (smem > 227 * 1024) return cudaErrorInvalidConfiguration;
  auto kern = fq_bnb_level_kernel<N_, WHOLE_>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const long long blocks = (long long)b.k.n_prob * b.cpc;
  if (blocks <= 0) return cudaSuccess;
  if (blocks > 0x7fffffffLL) return cudaErrorInvalidValue;
  kern<<<(unsigned)blocks, W * 32, smem, stream>>>(b);
  return cudaGetLastError();
}
#endif

// ---- the chained replan's exact stage (fq_replan_pairs_exact*): roots before the levels, resolve after them.  One thread
//      per corridor each, so the roots and the chosen leaf do not depend on the order in which warps finish.

// Corridor c's list winner (win_idx / win_cost of fq_select_multi_kernel) fixes f*, the first factor with a feasible
// list candidate.  Every factor f <= f* (all of F_c without f*) whose presolve passes gets a root; the incumbents start
// at +inf, and at the list winner's cost at f*.  status[c]: 0 no tree needed (the list holds every assignment, or there
// are no candidates), 1 tree, 2 too large for the level kernel (more faces than the staging area holds, or N unsupported).
__global__ void fq_bnb_roots_kernel(const FqBnbChainArgs a)
{
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.n_prob) return;
  a.n_par[c] = 0; a.n_par[a.n_prob + c] = 0; a.n_leaves[c] = 0; a.flags[2 * c] = 0; a.flags[2 * c + 1] = 0; a.nodes[c] = 0;
  const int p0 = a.poly_ofs[c], P = a.poly_ofs[c + 1] - p0;
  const long long L = fqa::list_len(a.N, P, a.all_limit);
  const int c0 = a.cand_ofs[c], n = a.cand_ofs[c + 1] - c0;
  const int nf = a.n_fac_j ? a.n_fac_j[c] : a.n_fac;
  if (P <= 1 || fqa::use_all(a.N, P, a.all_limit) || n <= 0 || L <= 0 || nf <= 0 || nf > a.stride || (long long)n != L * nf)
  {
    a.status[c] = 0;
    return;
  }
  if (!a.tree_ok || a.face_ofs[p0 + P] - a.face_ofs[p0] > a.max_faces)
  {
    a.status[c] = 2;
    return;
  }
  a.status[c] = 1;
  const int w = a.win_idx[c];
  const int fstar = w >= 0 ? (int)(w / L) : -1;
  const int n_search = fstar >= 0 ? fstar + 1 : nf;
  const double inf = __longlong_as_double(0x7ff0000000000000ll);
  int nr = 0;
  for (int f = 0; f < n_search; f++)
  {
    const double t = a.cand_dt[c0 + (long long)f * L];
    const size_t at = (size_t)c * a.stride + f;
    a.dts[at] = t;
    a.incumbent[at] = (unsigned long long)__double_as_longlong(f == fstar ? a.win_cost[c] : inf);
    a.lbound[at] = (unsigned long long)__double_as_longlong(inf);
    a.closed[at] = 0;
    if (fqs::root_possible(P, a.face_ofs + p0, a.Ab, a.x0 + 9 * (size_t)c, a.xf + 9 * (size_t)c, a.force_final, t, a.row_tol))
      a.roots[(size_t)c * a.stride + nr++] = f;
  }
  a.n_par[c] = nr;
}

// After level 0, when the lower bounds are final: a list winner within lbound (1 + 1e-9) at f* cannot be beaten by more
// than a relative 1e-9 (every assignment costs at least lbound > win_cost (1 - 1e-9)), so it stands and f*'s tree is
// closed: no child of f* is evaluated at the later levels.
__global__ void fq_bnb_certify_kernel(const FqBnbChainArgs a)
{
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.n_prob || a.status[c] != 1 || a.win_idx[c] < 0) return;
  const int P = a.poly_ofs[c + 1] - a.poly_ofs[c];
  const long long L = fqa::list_len(a.N, P, a.all_limit);
  const size_t at = (size_t)c * a.stride + a.win_idx[c] / L;
  if (a.win_cost[c] <= __longlong_as_double((long long)a.lbound[at]) * (1.0 + 1e-9)) a.closed[at] = 1;
}

// The winner of corridor c: the first factor f <= f* whose incumbent is finite.  At f* the list winner stays unless the
// tree found a cost below it by more than a relative 1e-9; otherwise the winner is the lexicographically smallest stored
// leaf of that factor within 1e-9 of the minimum (every such leaf was stored: pruning keeps ties).  A cut tree (flags)
// keeps the list winner and reports exact = 0.  A new winner overwrites win_idx (f |L_c|: the factor), win_dt, win_cost
// (the tree's cost) and win_sig, and sets changed[c] for fq_pair_final_kernel.
__global__ void fq_bnb_resolve_kernel(const FqBnbChainArgs a)
{
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.n_prob) return;
  const int st = a.status[c];
  a.changed[c] = 0;
  const bool cut = st == 2 || (st == 1 && (a.flags[2 * c] != 0 || a.flags[2 * c + 1] != 0));
  if (a.exact_out) a.exact_out[c] = cut ? 0 : 1;
  if (a.nodes_out) a.nodes_out[c] = st == 1 ? a.nodes[c] : 0;
  if (st != 1 || cut) return;
  const int P = a.poly_ofs[c + 1] - a.poly_ofs[c];
  const long long L = fqa::list_len(a.N, P, a.all_limit);
  const int nf = a.n_fac_j ? a.n_fac_j[c] : a.n_fac;
  const int w = a.win_idx[c];
  const int fstar = w >= 0 ? (int)(w / L) : -1;
  const int n_search = fstar >= 0 ? fstar + 1 : nf;
  a.keep_idx[c] = w; a.keep_cost[c] = a.win_cost[c]; a.keep_dt[c] = a.win_dt[c];
  for (int t = 0; t < a.N; t++) a.keep_sig[(size_t)c * a.N + t] = a.win_sig[(size_t)c * a.N + t];
  const int nl = min(a.n_leaves[c], a.leaf_cap);
  const fqb::LeafRec* lv = reinterpret_cast<const fqb::LeafRec*>(a.leaves) + (size_t)c * a.leaf_cap;
  for (int f = 0; f < n_search; f++)
  {
    const double m = __longlong_as_double((long long)a.incumbent[(size_t)c * a.stride + f]);
    if (!(m < INFINITY)) continue;
    if (f == fstar && !(m < a.win_cost[c] * (1.0 - 1e-9))) return;      // the list winner stays
    const double lim = m * (1.0 + 1e-9);
    int best = -1;
    for (int i = 0; i < nl; i++)
    {
      if (lv[i].dt_idx != f || !(lv[i].cost <= lim)) continue;
      bool less = best < 0;
      for (int t = 0; t < a.N && !less; t++)
      {
        if (lv[i].sigma[t] != lv[best].sigma[t]) { less = lv[i].sigma[t] < lv[best].sigma[t]; break; }
      }
      if (less) best = i;
    }
    if (best < 0) return;
    a.win_idx[c] = (int)(f * L);
    a.win_dt[c] = a.dts[(size_t)c * a.stride + f];
    a.win_cost[c] = lv[best].cost;
    for (int t = 0; t < a.N; t++) a.win_sig[(size_t)c * a.N + t] = lv[best].sigma[t];
    a.changed[c] = 1;
    return;
  }
}

// The winners' coefficients come from the ordinary solve kernel, cold, while the tree proved its winner warm-started over
// N launches: the two can disagree (the cold solve hits the iteration cap, or calls the candidate infeasible).  Such a
// corridor gets its list winner back and exact = 0, and redo_dt[c] its dt (NaN elsewhere, and NaN when the list had no
// winner either) for a second coefficient solve; fq_bnb_adopt_kernel then takes those coefficients.
__global__ void fq_bnb_fallback_kernel(const FqBnbChainArgs a, const uint8_t* __restrict__ feasible, double* __restrict__ redo_dt)
{
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.n_prob) return;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  redo_dt[c] = nan;
  if (!a.changed[c] || feasible[c]) return;
  a.win_idx[c] = a.keep_idx[c]; a.win_cost[c] = a.keep_cost[c]; a.win_dt[c] = a.keep_dt[c];
  for (int t = 0; t < a.N; t++) a.win_sig[(size_t)c * a.N + t] = a.keep_sig[(size_t)c * a.N + t];
  a.changed[c] = 0;
  if (a.exact_out) a.exact_out[c] = 0;
  if (a.keep_idx[c] >= 0) redo_dt[c] = a.keep_dt[c];
}

__global__ void fq_bnb_adopt_kernel(int n_prob, int N, const double* __restrict__ redo_dt, const double* __restrict__ redo_coeffs,
                                    double* __restrict__ coeffs)
{
  const int c = blockIdx.x;
  if (c >= n_prob || !(redo_dt[c] == redo_dt[c])) return;
  for (int i = threadIdx.x; i < 12 * N; i += blockDim.x) coeffs[(size_t)c * 12 * N + i] = redo_coeffs[(size_t)c * 12 * N + i];
}
}  // namespace fqb
