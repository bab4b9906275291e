// Device side of the chained replan that decomposes its own corridors (fq_replan_pairs_decomp*, include/faster_b200.h):
// fq_ellipsoid_decomp (fq_decomp.cpp) for every (corridor, segment) of a sweep at once, on the arithmetic of fq_decomp.h.
//
//   fq_decomp_kernel      one CTA per (corridor j, segment s): scan j's cloud (AABB reject, exact bbox test), compact the
//                         survivors in cloud order (ballots + a block prefix) and inflate them -- or, with an indexed map
//                         (fq_map.h), the same test on the points of the cells the AABB overlaps, the survivors in gather
//                         order, each with its index in the cloud; the two ellipsoid-shrink loops and the carving loop, each
//                         round a block-wide arg-min (lowest cloud index on ties: the host's "first strict minimum") plus
//                         one filter; then the six bbox faces and the ground face.  The rows go to slot j * max_poly + s of
//                         a staging array (cap_pf rows), their count or -status beside it.
//   fq_decomp_csr_kernel  one CTA: per-corridor status and rows, a block scan into the gap-free CSR (face_ofs absolute over
//                         poly_ofs, Ab packed), and the final state E / M of every corridor.
//
// Survivors beyond the kFitPts held in shared memory go to the CTA's slice of a global spill array, sized from the largest
// cloud of one corridor (max_obs), so nothing is ever truncated: a cloud above max_obs is refused (FQ_DECOMP_CLOUD).  With
// a map, max_obs caps the survivors of one segment instead, and a segment above it is refused the same way.
#pragma once
#include "fq_decomp.h"
#include "fq_map.h"

namespace fqd
{
constexpr int kThreads = 256;
constexpr int kFitPts = 1024;
constexpr double kNone = 1.7976931348623157e308;   // the host's starting "best distance"

// block-wide arg-min of per-thread (d, key, i): smallest d, then lowest key (the point's index in the cloud); returns the
// storage position i of the winner, or -1.  (kNone, 0x7fffffff) stands for "no candidate".  Every thread of the CTA calls it.
__device__ __forceinline__ int block_argmin(double d, int key, int i, double* s_d, int* s_k, int* s_i, int* s_best)
{
  for (int o = 16; o > 0; o >>= 1)
  {
    const double od = __shfl_xor_sync(0xffffffffu, d, o);
    const int ok = __shfl_xor_sync(0xffffffffu, key, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (od < d || (od == d && ok < key)) { d = od; key = ok; i = oi; }
  }
  if ((threadIdx.x & 31) == 0) { s_d[threadIdx.x >> 5] = d; s_k[threadIdx.x >> 5] = key; s_i[threadIdx.x >> 5] = i; }
  __syncthreads();
  if (threadIdx.x == 0)
  {
    double bd = s_d[0];
    int bk = s_k[0], bi = s_i[0];
    for (int k = 1; k < kThreads / 32; k++)
      if (s_d[k] < bd || (s_d[k] == bd && s_k[k] < bk)) { bd = s_d[k]; bk = s_k[k]; bi = s_i[k]; }
    *s_best = bk == 0x7fffffff ? -1 : bi;
  }
  __syncthreads();
  return *s_best;
}

__global__ void __launch_bounds__(kThreads) fq_decomp_kernel(const FqDecompArgs a)
{
  __shared__ double s_x[kFitPts], s_y[kFitPts], s_z[kFitPts], s_dist[kFitPts];
  __shared__ uint8_t s_flag[kFitPts];     // bit 0: inside the first ellipsoid, bit 1: in the current shrink loop, bit 2: not cut off
  __shared__ int s_idx[kFitPts];          // each survivor's index in the cloud: the arg-min's tie-break
  __shared__ int s_cnt[kThreads / 32], s_bk[kThreads / 32], s_bi[kThreads / 32], s_best;
  __shared__ double s_bd[kThreads / 32];
  const int slot = blockIdx.x, j = slot / a.max_poly, s = slot - j * a.max_poly;
  if (j >= a.n_prob) return;
  const int P = a.poly_ofs[j + 1] - a.poly_ofs[j];
  if (s >= P || P > a.max_poly) return;                  // (more than max_poly polytopes: fq_decomp_csr_kernel refuses it)
  const int tid = threadIdx.x;
  double* rows = a.stage + (size_t)slot * a.cap_pf * 4;
  const double* pv = a.path + 3 * ((size_t)a.poly_ofs[j] + j + s);
  V3 p1 = { pv[0], pv[1], pv[2] };
  const V3 p2 = { pv[3], pv[4], pv[5] };
  if (a.first)
  { // the safe path starts at R (faster.cpp:485); without a whole winner there is no R
    const double* r = a.first + 9 * (size_t)j;
    if (!(isfinite(r[0]) && isfinite(r[1]) && isfinite(r[2]))) { if (tid == 0) a.stage_n[slot] = -FQ_DECOMP_NOT_RUN; return; }
    if (s == 0) p1 = { r[0], r[1], r[2] };
  }
  const int map_id = a.maps ? (a.map_index ? a.map_index[j] : 0) : 0;
  const int o0 = a.maps ? 0 : a.obs_ofs[j], n_obs = a.maps ? 0 : a.obs_ofs[j + 1] - o0;
  if (n_obs < 0 || n_obs > a.max_obs || map_id < 0 || (a.maps && map_id >= a.n_maps))
  { if (tid == 0) a.stage_n[slot] = -FQ_DECOMP_CLOUD; return; }
  if (norm(sub(p2, p1)) == 0) { if (tid == 0) a.stage_n[slot] = -FQ_DECOMP_ZERO_SEGMENT; return; }

  Plane bb[6];
  local_bbox(p1, p2, a.bbox, bb);
  double lo[3], hi[3];
  bbox_aabb(p1, bb, lo, hi);
  Ellip E;
  M3 Ri;
  double f;
  ellipsoid_start(p1, p2, &E, &Ri, &f);
  double* sp = a.spill + (size_t)slot * a.spill_n * 4;
  uint8_t* sf = a.spill_flag + (size_t)slot * a.spill_n;
  auto at = [&](int i) -> V3 {
    if (i < kFitPts) return { s_x[i], s_y[i], s_z[i] };
    const double* q = sp + 4 * (size_t)(i - kFitPts);
    return { q[0], q[1], q[2] };
  };
  auto dist_of = [&](int i) -> double& { return i < kFitPts ? s_dist[i] : sp[4 * (size_t)(i - kFitPts) + 3]; };
  auto flag = [&](int i) -> uint8_t& { return i < kFitPts ? s_flag[i] : sf[i - kFitPts]; };
  int* si = a.spill_idx ? a.spill_idx + (size_t)slot * a.spill_n : nullptr;
  auto key = [&](int i) { return i < kFitPts ? s_idx[i] : (si ? si[i - kFitPts] : i); };

  // set_obs, the survivors inflated (line_segment.h:178-190) as they are stored: the points pts[b .. e), whose indices in
  // the cloud are idx[i] + shift (idx NULL: the points are the whole cloud in its order, and a survivor's key is its
  // position, so that the spilled ones need no key of their own)
  const int lane = tid & 31, w = tid >> 5, room = kFitPts + a.spill_n;
  int n = 0;
  auto take = [&](const double* pts, const int* idx, int shift, int b, int e) {
    for (int c0 = b; c0 < e; c0 += kThreads)
    {
      const int i = c0 + tid;
      V3 pt = { 0, 0, 0 };
      bool keep = false;
      if (i < e)
      {
        const double* q = pts + 3 * (size_t)i;
        pt = { q[0], q[1], q[2] };
        keep = !outside_aabb(lo, hi, pt.x, pt.y, pt.z) && inside_bbox(bb, pt);
      }
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (lane == 0) s_cnt[w] = __popc(m);
      __syncthreads();
      int before = n, total = n;
      for (int k = 0; k < kThreads / 32; k++) { before += k < w ? s_cnt[k] : 0; total += s_cnt[k]; }
      if (keep)
      {
        const int k = before + __popc(m & ((1u << lane) - 1u));
        const V3 q = inflate_point(Ri, E.d, pt, a.inflate);
        const int id = idx ? idx[i] + shift : k;        // a cloud in cloud order: the position is the index
        if (k < kFitPts) { s_x[k] = q.x; s_y[k] = q.y; s_z[k] = q.z; s_idx[k] = id; }
        else if (k < room)
        {
          double* r = sp + 4 * (size_t)(k - kFitPts);
          r[0] = q.x; r[1] = q.y; r[2] = q.z;
          if (si) si[k - kFitPts] = id;
        }
      }
      n = total;
      __syncthreads();
    }
  };
  if (!a.maps) take(a.obs + 3 * (size_t)o0, nullptr, 0, 0, n_obs);   // the corridor's cloud, in cloud order
  else
  { // the map's cells that overlap the AABB, a run of cells along x at a time: O, or U then O (O's indices after U's)
    const FqMapDev& M = *a.maps[map_id];
    const FqMapGrid g = M.grid;
    int c0[3], c1[3];
    fq_map_range(g, lo, hi, c0, c1);
    const int rows = (c1[1] - c0[1] + 1) * (c1[2] - c0[2] + 1);
    for (int side = a.map_unk ? 0 : 1; side < 2; side++)
    {
      const FqMapCloud& c = side ? M.occ : M.unk;
      for (int r = 0; r < rows; r++)
      {
        int b, e;
        fq_map_row(g, c, c0, c1, r, &b, &e);
        take(c.xyz, c.idx, side ? M.unk.n : 0, b, e);
      }
    }
    if (n > a.max_obs) { if (tid == 0) a.stage_n[slot] = -FQ_DECOMP_CLOUD; return; }
  }

  // find_ellipsoid (line_segment.h:191-247): the points inside the first ellipsoid, then the two shrink loops
  for (int i = tid; i < n; i += kThreads) flag(i) = E.dist(at(i)) <= 1 ? 3 : 0;
  __syncthreads();
  for (;;)
  {
    double bd = kNone;
    int bk = 0x7fffffff, bi = 0;
    for (int i = tid; i < n; i += kThreads)
      if (flag(i) & 2)
      {
        const double d = E.dist(at(i));
        if (d < bd || (d == bd && key(i) < bk)) { bd = d; bk = key(i); bi = i; }
      }
    const int best = block_argmin(bd, bk, bi, s_bd, s_bk, s_bi, &s_best);
    if (best < 0) break;
    shrink_short_axes(&E, Ri, at(best));
    for (int i = tid; i < n; i += kThreads)
      if ((flag(i) & 2) && !still_inside(E, at(i))) flag(i) &= (uint8_t)~2;
    __syncthreads();
  }
  E.ax[2] = f;
  for (int i = tid; i < n; i += kThreads)
    if (flag(i) & 1) flag(i) = E.dist(at(i)) <= 1 ? 3 : 1;
  __syncthreads();
  for (;;)
  {
    double bd = kNone;
    int bk = 0x7fffffff, bi = 0;
    for (int i = tid; i < n; i += kThreads)
      if (flag(i) & 2)
      {
        const double d = E.dist(at(i));
        if (d < bd || (d == bd && key(i) < bk)) { bd = d; bk = key(i); bi = i; }
      }
    const int best = block_argmin(bd, bk, bi, s_bd, s_bk, s_bi, &s_best);
    if (best < 0) break;
    shrink_third_axis(&E, at(best));
    for (int i = tid; i < n; i += kThreads)
      if ((flag(i) & 2) && !still_inside(E, at(i))) flag(i) &= (uint8_t)~2;
    __syncthreads();
  }

  // find_polyhedron (decomp_base.h:83-115): the ellipsoid is final, every distance is evaluated once
  for (int i = tid; i < n; i += kThreads) { dist_of(i) = E.dist(at(i)); flag(i) = 4; }
  __syncthreads();
  const V3 mid = scale(add(p1, p2), 0.5);
  int nf = 0;
  for (;;)
  {
    double bd = kNone;
    int bk = 0x7fffffff, bi = 0;
    for (int i = tid; i < n; i += kThreads)
      if ((flag(i) & 4) && (dist_of(i) < bd || (dist_of(i) == bd && key(i) < bk))) { bd = dist_of(i); bk = key(i); bi = i; }
    const int best = block_argmin(bd, bk, bi, s_bd, s_bk, s_bi, &s_best);
    if (best < 0) break;
    if (nf + 1 + 7 > a.cap_pf) { if (tid == 0) a.stage_n[slot] = -FQ_DECOMP_POLY_FACES; return; }
    const V3 cp = at(best);
    const V3 nrm = tangent_normal(E, cp);
    if (tid == 0) oriented_row(Plane{ cp, nrm }, mid, rows + 4 * (size_t)nf);
    nf++;
    for (int i = tid; i < n; i += kThreads)
      if ((flag(i) & 4) && !before_plane(nrm, cp, at(i))) flag(i) &= (uint8_t)~4;
    __syncthreads();
  }
  if (tid != 0) return;
  if (nf + 7 > a.cap_pf) { a.stage_n[slot] = -FQ_DECOMP_POLY_FACES; return; }
  for (int k = 0; k < 6; k++) oriented_row(bb[k], mid, rows + 4 * (size_t)(nf + k));   // add_local_bbox (line_segment.h:33-38)
  ground_row(a.z_ground, rows + 4 * (size_t)(nf + 6));
  a.stage_n[slot] = nf + 7;
}

// corridor j's status and rows from the staged counts (no R, then the first failing segment's status, then the corridor cap)
__device__ __forceinline__ void corridor_rows(const FqDecompArgs& a, int j, int* status, int* n_rows)
{
  const int P = a.poly_ofs[j + 1] - a.poly_ofs[j];
  *status = 0;
  *n_rows = 0;
  if (P < 0 || P > a.max_poly) { *status = FQ_DECOMP_NOT_RUN; return; }
  if (a.first)
  { // no R (no whole winner): not run, also for a corridor without segments, where no decomposition CTA looked at R
    const double* f = a.first + 9 * (size_t)j;
    if (!(isfinite(f[0]) && isfinite(f[1]) && isfinite(f[2]))) { *status = FQ_DECOMP_NOT_RUN; return; }
  }
  int r = 0;
  for (int s = 0; s < P; s++)
  {
    const int c = a.stage_n[(size_t)j * a.max_poly + s];
    if (c < 0) { *status = -c; return; }
    r += c;
  }
  if (r > a.max_faces) { *status = FQ_DECOMP_CORRIDOR_FACES; return; }
  *n_rows = r;
}

// One CTA (any size up to 1024): every thread takes a contiguous run of corridors, as fq_assign_offsets_kernel
__global__ void __launch_bounds__(1024) fq_decomp_csr_kernel(const FqDecompArgs a)
{
  __shared__ int s_run[1024];
  const int T = blockDim.x, tid = threadIdx.x;
  const int per = (a.n_prob + T - 1) / T;
  const int j0 = min(a.n_prob, tid * per), j1 = min(a.n_prob, j0 + per);
  int sum = 0;
  for (int j = j0; j < j1; j++)
  {
    int st, r;
    corridor_rows(a, j, &st, &r);
    sum += r;
  }
  s_run[tid] = sum;
  __syncthreads();
  if (tid == 0)
  {
    int run = 0;
    for (int i = 0; i < T; i++) { const int x = s_run[i]; s_run[i] = run; run += x; }
    a.face_ofs[0] = 0;
  }
  __syncthreads();
  int run = s_run[tid];
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  for (int j = j0; j < j1; j++)
  {
    int st, r;
    corridor_rows(a, j, &st, &r);
    const int p0 = a.poly_ofs[j], P = a.poly_ofs[j + 1] - p0;
    for (int s = 0; s < P && p0 + s + 1 <= a.face_cap; s++)
    {
      const int c = st == 0 ? a.stage_n[(size_t)j * a.max_poly + s] : 0;
      const double* src = a.stage + ((size_t)j * a.max_poly + s) * a.cap_pf * 4;
      for (int k = 0; k < 4 * c; k++) a.Ab[4 * (size_t)run + k] = src[k];
      run += c;
      a.face_ofs[p0 + s + 1] = run;
    }
    // E / M (faster.cpp:395-403, :495-504): the last vertex, or G when the last polytope contains it (d > 0: outside)
    double* x = a.xf + 9 * (size_t)j;
    double pos[3] = { nan, nan, nan };
    if (st == 0)
    {
      const double* last = (P == 0 && a.first) ? a.first + 9 * (size_t)j : a.path + 3 * ((size_t)p0 + j + P);
      pos[0] = last[0]; pos[1] = last[1]; pos[2] = last[2];
      if (a.goal && P > 0)
      {
        const double* g = a.goal + 3 * (size_t)j;
        const double* lr = a.stage + ((size_t)j * a.max_poly + P - 1) * a.cap_pf * 4;
        bool inside = true;
        for (int k = 0; k < a.stage_n[(size_t)j * a.max_poly + P - 1] && inside; k++)
        {
          const double* q = lr + 4 * (size_t)k;
          inside = !(FQ_SUB(FQ_ADD(FQ_ADD(FQ_MUL(q[0], g[0]), FQ_MUL(q[1], g[1])), FQ_MUL(q[2], g[2])), q[3]) > 0);
        }
        if (inside) { pos[0] = g[0]; pos[1] = g[1]; pos[2] = g[2]; }
      }
    }
    for (int i = 0; i < 3; i++) x[i] = pos[i];
    for (int i = 3; i < 9; i++) x[i] = st == 0 ? 0.0 : nan;
    if (a.pos_out)
      for (int i = 0; i < 3; i++) a.pos_out[3 * (size_t)j + i] = pos[i];
    if (a.status) a.status[j] = st;
  }
}
}  // namespace fqd
