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
#pragma once

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
  FqKernelArgs k;                  // plan tables + the ONE problem (n_prob = 1); k.dt/k.sigma/outputs unused
  int n_dt, P;                     // P = polytopes of the problem (children per parent)
  const double* dts;               // device, n_dt
  int depth;                       // depth of the parents of this launch (0: roots, state = identity)
  int n_parents;
  const unsigned char* parents;    // n_parents nodes (ignored at depth 0: parent i is the root of dt index roots[i])
  const int* roots;                // depth 0 only: dt index of each root
  unsigned char* children;         // capacity `cap` nodes
  int* n_children;
  int cap;
  unsigned long long* incumbent;   // n_dt: ordered bits of the best full-assignment cost so far
  LeafRec* leaves;
  int* n_leaves;
  int leaf_cap;
  int* flags;                      // [0] overflow of children/leaves, [1] numeric failures
};

template <int N_, bool WHOLE_>
__global__ void __launch_bounds__(W * 32, (N_ <= 10 ? 4 : (N_ <= 15 ? 3 : 2))) fq_bnb_level_kernel(const BnbArgs b)
{
  using D = Dims<N_, WHOLE_>;
  constexpr int NW = D::NW, LD = D::LD, SLOTS = D::SLOTS, N = D::N, NYP = D::NYP;
  const FqKernelArgs& a = b.k;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* sm = reinterpret_cast<double*>(smem_raw);
  double* sAb = sm;            sm += 4 * a.max_faces;
  double* TZ = sm;             sm += D::NY * D::TZLD;
  double* SY = sm;             sm += D::NY;
  unsigned char* wraw = reinterpret_cast<unsigned char*>(sm);
  const int pwb = per_warp_bytes<D>(a.item_cap);
  int* sfo = reinterpret_cast<int*>(wraw + (size_t)W * pwb);

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
  const int p0 = a.poly_ofs[0], P = a.poly_ofs[1] - p0;
  const int f0 = a.face_ofs[p0];
  const int nf = P > 0 ? a.face_ofs[p0 + P] - f0 : 0;
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
    if (!fits) { if (threadIdx.x == 0) b.flags[0] = 1; return; }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long child = (long long)blockIdx.x * W + warp;
  if (child >= (long long)b.n_parents * P) return;
  const int pi = (int)(child / P), pnew = (int)(child - (long long)pi * P);

  WarpState<D> m;
  int* seg_ofs;
  {
    double* p = reinterpret_cast<double*>(wraw + (size_t)warp * pwb);
    m.J = p;   p += NW * LD;
    m.R = p;   p += D::RSZ;
    m.Y = p;   p += 3 * NYP;
    m.w = p;   p += NW;
    m.d = p;   p += NW + 2;
    m.zb = p;  p += NW;
    m.items = reinterpret_cast<unsigned short*>(p);
    seg_ofs = sfo + 40 + warp * 32;
  }
  // ---- parent
  const int k = b.depth;
  int dt_idx, q = 0;
  unsigned char sig[16];
  const unsigned char* pn = b.parents + (size_t)pi * node_bytes<D>();
  if (k == 0) dt_idx = b.roots[pi];
  else
  {
    const NodeHdr* h = reinterpret_cast<const NodeHdr*>(pn);
    dt_idx = h->dt_idx; q = h->q;
#pragma unroll
    for (int t = 0; t < 16; t++) sig[t] = h->sigma[t];
  }
  sig[k] = (unsigned char)pnew;
  const double dt = b.dts[dt_idx];
  const double inv1 = 1.0 / dt, inv2 = inv1 * inv1, inv3 = inv2 * inv1;
  const double lim0 = a.lim[0], lim1 = a.lim[1], lim2 = a.lim[2];
  double Yeq[D::RPL][3], bthr[D::RPL];
  setup_rows<D>(a, 0, dt, lim0, lim1, lim2, lane, Yeq, bthr);
  {
    bool okc = dt > 0 && dt < 1e100 && lim0 > 0 && lim0 < 1e300 && lim1 > 0 && lim1 < 1e300 && lim2 > 0 && lim2 < 1e300 && !rows_bad;
#pragma unroll
    for (int r = 0; r < D::RPL; r++)
#pragma unroll
      for (int ax = 0; ax < 3; ax++) okc = okc && fabs(Yeq[r][ax]) < 1e300;
    if (!__all_sync(FULL, okc)) return;        // non-finite input: the subtree is dropped (treated as infeasible)
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
  int total_rows = 0;
  {
    int p = 0;
    if (lane <= k) p = sig[0];
#pragma unroll
    for (int t = 1; t < 16; t++)
      if (lane == t && t <= k) p = sig[t];
    total_rows = build_items<D>(m, sfo, seg_ofs, lane, k + 1, p, a.item_cap);
    if (total_rows < 0) { if (lane == 0) b.flags[0] = 1; return; }
  }
  int it = 0, bkey = 0;
  unsigned bcode = 0;
  if (k == 0) update_Y<D, true>(m, TZ, Yeq, bthr, SY, lane, bkey, bcode);
  else update_Y<D, false>(m, TZ, Yeq, bthr, SY, lane, bkey, bcode);
  const int status = gi_loop<D>(m, TZ, SY, sAb, Yeq, bthr, lane, total_rows, inv1, inv2, inv3, lim0, lim1, lim2, a.row_tol,
                                lam, rdinv, q, it, bkey, bcode);
  if (status != 1)
  {
    if (status == -1 && lane == 0) atomicAdd(b.flags + 1, 1);
    return;
  }
  double cp = 0;
  for (int i = lane; i < 3 * N; i += 32)
  {
    const int ax = i / N, t = i - ax * N;
    const double u = m.Y[ax * NYP + 3 * N + 1 + t];
    cp = fma(u, u, cp);
  }
  const double cost = fqt::warp_sum(cp) * (inv3 * inv3);
  const unsigned long long cbits = (unsigned long long)__double_as_longlong(cost);
  const unsigned long long inc = *reinterpret_cast<volatile unsigned long long*>(b.incumbent + dt_idx);
  if (cbits >= inc) return;                      // bound: children only add rows, the cost cannot decrease
  if (k + 1 == N)
  { // a full assignment that beats the incumbent
    if (lane == 0)
    {
      const unsigned long long old = atomicMin(b.incumbent + dt_idx, cbits);
      if (cbits < old)
      {
        const int slot = atomicAdd(b.n_leaves, 1);
        if (slot < b.leaf_cap)
        {
          LeafRec* L = b.leaves + slot;
          L->dt_idx = dt_idx; L->cost = cost;
          for (int t = 0; t < 16; t++) L->sigma[t] = t < N ? sig[t] : 0;
        }
        else b.flags[0] = 1;
      }
    }
    return;
  }
  int slot = 0;
  if (lane == 0) slot = atomicAdd(b.n_children, 1);
  slot = __shfl_sync(FULL, slot, 0);
  if (slot >= b.cap) { if (lane == 0) b.flags[0] = 1; return; }
  unsigned char* cn = b.children + (size_t)slot * node_bytes<D>();
  if (lane == 0)
  {
    NodeHdr* h = reinterpret_cast<NodeHdr*>(cn);
    h->dt_idx = dt_idx; h->depth = k + 1; h->q = q; h->pad = 0;
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
}

template <int N_, bool WHOLE_>
cudaError_t launch_level(const BnbArgs& b, cudaStream_t stream)
{
  const size_t smem = smem_bytes_t<N_, WHOLE_>(b.k.max_faces, b.k.item_cap, 1);   // one CTA-wide copy of the rows
  if (smem > 227 * 1024) return cudaErrorInvalidConfiguration;
  auto kern = fq_bnb_level_kernel<N_, WHOLE_>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const long long children = (long long)b.n_parents * b.P;
  if (children <= 0) return cudaSuccess;
  const long long blocks = (children + W - 1) / W;
  if (blocks > 0x7fffffffLL) return cudaErrorInvalidValue;
  kern<<<(unsigned)blocks, W * 32, smem, stream>>>(b);
  return cudaGetLastError();
}
}  // namespace fqb
