// The batch JPS kernels behind fq_jps_batch / fq_jps_batch_dev (fq_jps.cu): fq_jps3d_plan_world's search and
// post-processing (fq_jps.h) and fq_jps_in (fq_paths.h) for every planner, one warp each, then one CTA that packs the
// JPS_in rows in fq_map_paths_args' layout.  Kernel source only (tests/cpp/jps_batch_emu.cpp runs it under the block
// emulation).
//
// Work inside a warp.  An expansion's candidate directions (host order: natural, then forced with an occupied blocker)
// go one to a lane, and each lane runs its candidate's jump.  Lane 0 then creates, relaxes and pushes the successors in
// candidate order, exactly as the host does: the node set, the heap layout and every tie are the host's.  Only lane 0
// touches the node pool, the heap and the hash, so nothing there needs a barrier; the other lanes receive the expanded
// node by shuffle.  The line-of-sight test of removeCornerPts splits its ray samples over the lanes (the answer is "a
// blocked sample before the first sample outside the grid"); the chain around it runs on every lane with lane 0
// writing.
#pragma once
#include "../../include/faster_b200.h"
#include "fq_jps.h"
#include "fq_paths.h"

struct FqJpsArgs
{
  int n_prob, n_grids;
  const int8_t* cells;
  const long long* cell_ofs;
  const int* dims;
  const double* origin;
  const double* res;
  const int* grid_index;
  const double *x0, *goal, *pos;
  double Ra, dist_max;
  int use_jps, max_nodes, max_in;
  char* scratch;          // n_prob x per bytes (fq_jps_scratch_layout)
  size_t per;
  int *cnt, *st;          // per planner: JPS_in rows in its slot, status
  int* in_ofs;
  double* in;
  int *status, *k_end;
};

// Byte offsets of one planner's scratch: node pool, heap, hash keys and values (2 max_nodes slots), two path buffers,
// the JPS_in slot; returns the total
struct FqJpsLayout
{
  size_t nodes, heap, key, val, pa, pb, slot, total;
};
FQ_HD size_t fq_jps_a16(size_t x) { return (x + 15) & ~(size_t)15; }
FQ_HD FqJpsLayout fq_jps_scratch_layout(int max_nodes, int max_in)
{
  FqJpsLayout L;
  const size_t m = (size_t)max_nodes;
  L.nodes = 0;
  L.heap = L.nodes + fq_jps_a16(sizeof(fqjps::Node) * m);
  L.key = L.heap + fq_jps_a16(sizeof(int) * m);
  L.val = L.key + fq_jps_a16(sizeof(long long) * 2 * m);
  L.pa = L.val + fq_jps_a16(sizeof(int) * 2 * m);
  L.pb = L.pa + fq_jps_a16(sizeof(double) * 3 * m);
  L.slot = L.pb + fq_jps_a16(sizeof(double) * 3 * m);
  L.total = L.slot + fq_jps_a16(sizeof(double) * 3 * (size_t)max_in);
  return L;
}

// one planner's node storage on the device: a pool of max_nodes nodes, their heap, and an open-addressing hash (linear
// probing, 2 max_nodes slots, key -1 empty) from linear cell id to node
struct FqJpsStore
{
  fqjps::Node* n;
  int* h;
  long long* key;
  int* val;
  int slots, max_nodes, count;
  FQ_HD fqjps::Node& node(int k) { return n[k]; }
  FQ_HD int& heap(int i) { return h[i]; }
  FQ_HD int home(long long c) const { return (int)(((unsigned long long)c * 0x9E3779B97F4A7C15ull >> 32) % (unsigned)slots); }
  FQ_HD int lookup(long long c) const
  {
    for (int s = home(c);; s = s + 1 == slots ? 0 : s + 1)
    {
      if (key[s] == c) return val[s];
      if (key[s] < 0) return -1;
    }
  }
  FQ_HD int add(long long c)
  {
    if (count == max_nodes) return -1;
    int s = home(c);
    while (key[s] >= 0) s = s + 1 == slots ? 0 : s + 1;
    key[s] = c;
    val[s] = count;
    return count++;
  }
};

// One warp per planner: blockDim.x = 32 W (W <= kFqJpsMaxWarps) serves planners blockIdx.x W .. + W - 1.  Writes the
// planner's JPS_in into its slot and cnt / st.
constexpr int kFqJpsMaxWarps = 4;
__global__ void __launch_bounds__(32 * kFqJpsMaxWarps) fq_jps_search_kernel(const FqJpsArgs a)
{
  __shared__ fqjps::Rules s_rules;
  if (threadIdx.x == 0) fqjps::rules_build(&s_rules);
  __syncthreads();
  const fqjps::Rules& R = s_rules;
  const unsigned FULL = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (j >= a.n_prob) return;
  char* base = a.scratch + a.per * (size_t)j;
  const FqJpsLayout L = fq_jps_scratch_layout(a.max_nodes, a.max_in);
  double* slot = (double*)(base + L.slot);
  double* pa = (double*)(base + L.pa);
  double* pb = (double*)(base + L.pb);

  // ---- inputs (every lane reads the same)
  const int gi = a.grid_index ? a.grid_index[j] : 0;
  double A[3], G[3], P[3];
  bool ok = true;
  for (int k = 0; k < 3; k++)
  {
    A[k] = a.x0[9 * (size_t)j + k];
    G[k] = a.goal[3 * (size_t)j + k];
    P[k] = a.pos ? a.pos[3 * (size_t)j + k] : A[k];
    ok = ok && isfinite(A[k]) && isfinite(G[k]) && isfinite(P[k]);
  }
  fqjps::World w;
  ok = ok && gi >= 0 && gi < a.n_grids;
  if (ok)
  {
    const int xd = a.dims[3 * gi], yd = a.dims[3 * gi + 1], zd = a.dims[3 * gi + 2];
    w.g.m = a.cells + a.cell_ofs[gi];
    w.g.xd = xd; w.g.yd = yd; w.g.zd = zd;
    w.res = a.res[gi];
    for (int k = 0; k < 3; k++) w.origin[k] = a.origin[3 * gi + k];
    ok = xd > 0 && yd > 0 && zd > 0 && (double)xd * yd * zd <= 2147483648.0 && a.cell_ofs[gi] >= 0 && isfinite(w.res) && w.res > 0 &&
         isfinite(w.origin[0]) && isfinite(w.origin[1]) && isfinite(w.origin[2]);
  }
  int status = ok ? FQ_JPS_NO_PATH : FQ_JPS_INPUT;
  int m = 0;                                       // vertices of the post-processed path in pb
  if (ok)
  {
    const double As[3] = { A[0], A[1], A[2] < 0.0 ? 0.0 : A[2] };
    const double Gs[3] = { G[0], G[1], G[2] < 0.0 ? 0.0 : G[2] };
    int sc[3], gc[3];
    w.to_int(As, sc);
    w.to_int(Gs, gc);
    const fqjps::Grid& g = w.g;
    if (g.free_(sc[0], sc[1], sc[2]) && g.free_(gc[0], gc[1], gc[2]))
    {
      FqJpsStore st;
      st.n = (fqjps::Node*)(base + L.nodes); st.h = (int*)(base + L.heap);
      st.key = (long long*)(base + L.key); st.val = (int*)(base + L.val);
      st.slots = 2 * a.max_nodes; st.max_nodes = a.max_nodes; st.count = 0;
      for (int s = lane; s < st.slots; s += 32) st.key[s] = -1;
      __syncwarp();
      const bool use_jps = a.use_jps != 0;
      fqjps::Search<FqJpsStore> S(st, fqjps::v3(gc[0], gc[1], gc[2]));
      if (lane == 0) S.start(g, fqjps::v3(sc[0], sc[1], sc[2]));
      int found = -1;
      for (;;)
      {
        int k = -1, flag = 0;                      // 1: open list empty, 2: goal popped
        fqjps::Node cur;
        if (lane == 0)
        {
          if (S.heap_n == 0) flag = 1;
          else
          {
            k = S.pop();
            cur = st.node(k);
            if (S.is_goal(k)) flag = 2;
          }
        }
        flag = __shfl_sync(FULL, flag, 0);
        k = __shfl_sync(FULL, k, 0);
        if (flag == 1) break;
        if (flag == 2) { found = k; break; }
        cur.x = __shfl_sync(FULL, cur.x, 0); cur.y = __shfl_sync(FULL, cur.y, 0); cur.z = __shfl_sync(FULL, cur.z, 0);
        cur.dir = __shfl_sync(FULL, cur.dir, 0);
        const int d = fqjps::candidate(R, g, cur, use_jps, lane);
        fqjps::V3i jp = fqjps::v3(0, 0, 0);
        double cost = 0;
        const bool has = d >= 0 && fqjps::successor(R, g, S.goal, cur, use_jps, d, &jp, &cost);
        unsigned todo = __ballot_sync(FULL, has);
        int full = 0;
        while (todo)
        { // lane 0 applies the successors in candidate order
          const int i = __ffs(todo) - 1;
          todo &= todo - 1;
          const int x = __shfl_sync(FULL, jp.x, i), y = __shfl_sync(FULL, jp.y, i), z = __shfl_sync(FULL, jp.z, i);
          const int di = __shfl_sync(FULL, d, i);
          const double ci = __shfl_sync(FULL, cost, i);
          if (lane == 0 && !full)
          {
            const int c = S.node_at(g, x, y, z, di);
            if (c < 0) full = 1;
            else S.relax(k, c, ci);
          }
        }
        if (__shfl_sync(FULL, full, 0)) { status = FQ_JPS_NODES; break; }
      }
      if (found >= 0)
      { // the raw path in world coordinates (pa), line points out (pb), corner points out forwards and backwards
        if (lane == 0)
        {
          int n = 0;
          for (int i = found; i >= 0; i = st.node(i).parent) n++;
          int at = n;
          for (int i = found; i >= 0; i = st.node(i).parent)
          {
            const fqjps::Node& q = st.node(i);
            const int c[3] = { q.x, q.y, q.z };
            w.to_float(c, pa + 3 * --at);
          }
          m = fqjps::remove_line_pts(pa, n, pb);
        }
        m = __shfl_sync(FULL, m, 0);
        __syncwarp();
        auto blocked = [&](const double* p1, const double* p2) -> bool {
          double diff[3], s;
          const int md = w.ray(p1, p2, diff, &s);
          for (int b = 1; b < md; b += 32)
          {
            int c[3];
            const int r = b + lane < md ? w.sample(p1, diff, s, b + lane, c) : 0;
            const unsigned out = __ballot_sync(FULL, r == 2), blk = __ballot_sync(FULL, r == 1);
            if (blk && (!out || __ffs(blk) < __ffs(out))) return true;
            if (out) return false;
          }
          return false;
        };
        m = fqjps::remove_corner_pts(blocked, pb, m, pa, lane == 0);
        __syncwarp();
        if (lane == 0) fqjps::reverse_into(pa, m, pb);
        __syncwarp();
        m = fqjps::remove_corner_pts(blocked, pb, m, pa, lane == 0);
        __syncwarp();
        if (lane == 0) fqjps::reverse_into(pa, m, pb);
        status = FQ_JPS_OK;
      }
    }
  }
  if (lane != 0) return;
  int rows = 1;
  if (status == FQ_JPS_OK || status == FQ_JPS_NO_PATH)
  { // ra = min(|G - P| - 0.001, Ra) (faster.cpp:327-329), then fq_jps_in of the path, or of [A] when there is none
    const double dg = FQ_SUB(fqpath::dist3(G, P), 0.001);
    const double ra = a.Ra < dg ? a.Ra : dg;
    const fqpath::JpsIn jin(status == FQ_JPS_OK ? pb : A, status == FQ_JPS_OK ? m : 1, A, G, ra);
    if (jin.count(a.dist_max) > (double)a.max_in) status = FQ_JPS_LONG;
    else rows = jin.write(a.dist_max, slot, a.max_in);
  }
  if (status != FQ_JPS_OK && status != FQ_JPS_NO_PATH)
  {
    const unsigned long long qnan = 0x7ff8000000000000ull;   // the host's NAN, whatever the device's conversions give
    for (int k = 0; k < 3; k++) memcpy(slot + k, &qnan, sizeof(double));
  }
  a.cnt[j] = rows;
  a.st[j] = status;
}

// One CTA (any size up to 1024): in_ofs = the exclusive scan of the row counts, the rows packed from the slots, status,
// and k_end = -1 where the status is not FQ_JPS_OK.  Every thread takes a contiguous run of planners; thread 0 scans the
// runs' sums.
__global__ void __launch_bounds__(1024) fq_jps_write_kernel(const FqJpsArgs a)
{
  __shared__ int s_sum[1024];
  const int T = blockDim.x, tid = threadIdx.x;
  const int per = (a.n_prob + T - 1) / T;
  const int j0 = min(a.n_prob, tid * per), j1 = min(a.n_prob, j0 + per);
  int sum = 0;
  for (int j = j0; j < j1; j++) sum += a.cnt[j];
  s_sum[tid] = sum;
  __syncthreads();
  if (tid == 0)
  {
    int r = 0;
    for (int i = 0; i < T; i++)
    {
      const int x = s_sum[i];
      s_sum[i] = r;
      r += x;
    }
    a.in_ofs[a.n_prob] = r;
  }
  __syncthreads();
  int o = s_sum[tid];
  for (int j = j0; j < j1; j++)
  {
    a.in_ofs[j] = o;
    o += a.cnt[j];
    const int s = a.st[j];
    a.status[j] = s;
    if (a.k_end && s != FQ_JPS_OK) a.k_end[j] = -1;
  }
  __syncthreads();
  for (int j = 0; j < a.n_prob; j++)
  {
    const double* src = (const double*)(a.scratch + a.per * (size_t)j + fq_jps_scratch_layout(a.max_nodes, a.max_in).slot);
    double* dst = a.in + 3 * (size_t)a.in_ofs[j];
    for (int i = tid; i < 3 * a.cnt[j]; i += T) dst[i] = src[i];
  }
}
