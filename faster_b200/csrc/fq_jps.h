// The path search on a voxel grid as ONE source for the host and the device: the host planner (fq_jps3d_plan /
// fq_jps3d_plan_world, fq_jps.cpp) and the batch kernel (fq_jps_search_kernel, fq_jps.cuh) run the same code.  What it
// restates: jps_manager_.solveJPS3D (faster/src/faster.cpp:361 -> jps_manager.cpp:141 -> thirdparty/jps3d
// JPSPlanner<3>::plan, jps_planner.cpp:196-295 over GraphSearch, graph_search.cpp:123-219 A* loop, :272-470 jump-point
// successors): jump point search in 3D (26-connected, Euclidean step costs and heuristic) plus plain A*, and the path
// post-processing (removeLinePts / removeCornerPts with ray-traced line of sight, jps_planner.cpp:36-105,
// map_util.h:334-383).
//
// Cell values follow the reference's map (map_util.h): 0 free, > 0 occupied, < 0 unknown.  Only free cells can be
// entered; only OCCUPIED cells create forced neighbours (graph_search.cpp:58-66, :420-470).
//
// Pruning rules (what the reference tabulates in JPS3DNeib, graph_search.h:104-136; generated here from the geometric
// rule, checked against the reference's tables in tests/test_jps_cpu.py).  For a move d = a + b + c (axis components):
//   natural neighbours: every non-empty sub-sum of the components (1, 3 or 7 directions);
//   forced pairs (blocker f1 -> successor f2):
//     straight  d:      o -> o + d                       for the 8 offsets o perpendicular to d
//     planar    a+b:    -b -> a-b,  -a -> b-a,  and for both normals n:  n -> d+n,  -b+n -> a-b+n,  -a+n -> b-a+n,
//                       n -> a+n,  n -> b+n
//     spatial   a+b+c:  -a -> d-2a (and cyclic),  -b-c -> a-b-c (and cyclic),  -a -> -a+c, -a -> -a+b (and cyclic)
//
// Every floating operation is spelled through FQ_ADD / FQ_MUL / ... (fq_dtinit.h) in the host's order, so the device
// evaluates the same expression tree with round-to-nearest intrinsics and never contracts; std::round / round and floor
// are exact on both.  Host and device agree bit for bit.
#pragma once
#include "fq_dtinit.h"

#include <stdint.h>

namespace fqjps
{
struct V3i
{
  int x, y, z;
};
FQ_HD V3i v3(int x, int y, int z) { V3i v; v.x = x; v.y = y; v.z = z; return v; }
FQ_HD int dir_id(int dx, int dy, int dz) { return (dx + 1) + 3 * (dy + 1) + 9 * (dz + 1); }
FQ_HD V3i dir_of(int id) { return v3(id % 3 - 1, id / 3 % 3 - 1, id / 9 - 1); }

// the pruning rules per direction id: natural neighbours (direction ids, in jump()'s order: single components, pairs,
// the move itself last), forced (blocker, successor) pairs as offsets, and the distinct blockers
struct Rules
{
  int8_t n_nat[27], n_forced[27], n_blk[27];
  int8_t nat[27][26];
  int8_t f1[27][12][3], f2[27][12][3];
  int8_t blk[27][12][3];
};

FQ_HD void rules_build(Rules* R)
{
  for (int id = 0; id < 27; id++)
  {
    const V3i d = dir_of(id);
    R->n_nat[id] = R->n_forced[id] = R->n_blk[id] = 0;
    V3i comp[3];
    int n = 0;
    if (d.x) comp[n++] = v3(d.x, 0, 0);
    if (d.y) comp[n++] = v3(0, d.y, 0);
    if (d.z) comp[n++] = v3(0, 0, d.z);
    auto nat = [&](V3i v) { R->nat[id][R->n_nat[id]++] = (int8_t)dir_id(v.x, v.y, v.z); };
    auto add = [&](V3i a, V3i b) {
      const int k = R->n_forced[id]++;
      R->f1[id][k][0] = (int8_t)a.x; R->f1[id][k][1] = (int8_t)a.y; R->f1[id][k][2] = (int8_t)a.z;
      R->f2[id][k][0] = (int8_t)b.x; R->f2[id][k][1] = (int8_t)b.y; R->f2[id][k][2] = (int8_t)b.z;
    };
    if (n == 0)
    { // start node: all 26 directions
      for (int z = -1; z <= 1; z++)
        for (int y = -1; y <= 1; y++)
          for (int x = -1; x <= 1; x++)
            if (x || y || z) nat(v3(x, y, z));
      continue;
    }
    for (int k = 0; k < n; k++) nat(comp[k]);
    if (n == 3)
      for (int k = 0; k < 3; k++)
      {
        const V3i a = comp[k], b = comp[(k + 1) % 3];
        nat(v3(a.x + b.x, a.y + b.y, a.z + b.z));
      }
    if (n >= 2) nat(d);
    if (n == 1)
    {
      for (int z = -1; z <= 1; z++)
        for (int y = -1; y <= 1; y++)
          for (int x = -1; x <= 1; x++)
            if ((x || y || z) && x * d.x + y * d.y + z * d.z == 0) add(v3(x, y, z), v3(x + d.x, y + d.y, z + d.z));
    }
    else if (n == 2)
    {
      const V3i a = comp[0], b = comp[1];
      const V3i e = v3(d.x == 0 ? 1 : 0, d.y == 0 ? 1 : 0, d.z == 0 ? 1 : 0);   // normal of the move's plane
      add(v3(-b.x, -b.y, -b.z), v3(a.x - b.x, a.y - b.y, a.z - b.z));
      add(v3(-a.x, -a.y, -a.z), v3(b.x - a.x, b.y - a.y, b.z - a.z));
      for (int s = -1; s <= 1; s += 2)
      {
        const V3i m = v3(e.x * s, e.y * s, e.z * s);
        add(m, v3(d.x + m.x, d.y + m.y, d.z + m.z));
        add(v3(m.x - b.x, m.y - b.y, m.z - b.z), v3(a.x - b.x + m.x, a.y - b.y + m.y, a.z - b.z + m.z));
        add(v3(m.x - a.x, m.y - a.y, m.z - a.z), v3(b.x - a.x + m.x, b.y - a.y + m.y, b.z - a.z + m.z));
        add(m, v3(a.x + m.x, a.y + m.y, a.z + m.z));
        add(m, v3(b.x + m.x, b.y + m.y, b.z + m.z));
      }
    }
    else
    {
      const V3i* c = comp;
      for (int k = 0; k < 3; k++) add(v3(-c[k].x, -c[k].y, -c[k].z), v3(d.x - 2 * c[k].x, d.y - 2 * c[k].y, d.z - 2 * c[k].z));
      for (int k = 0; k < 3; k++)
      {
        const V3i p = c[(k + 1) % 3], q = c[(k + 2) % 3];
        add(v3(-p.x - q.x, -p.y - q.y, -p.z - q.z), v3(c[k].x - p.x - q.x, c[k].y - p.y - q.y, c[k].z - p.z - q.z));
      }
      for (int k = 0; k < 3; k++)
      {
        const V3i p = c[(k + 1) % 3], q = c[(k + 2) % 3];
        add(v3(-c[k].x, -c[k].y, -c[k].z), v3(p.x - c[k].x, p.y - c[k].y, p.z - c[k].z));
        add(v3(-c[k].x, -c[k].y, -c[k].z), v3(q.x - c[k].x, q.y - c[k].y, q.z - c[k].z));
      }
    }
    for (int k = 0; k < R->n_forced[id]; k++)
    {
      bool seen = false;
      for (int b = 0; b < R->n_blk[id]; b++)
        seen = seen || (R->blk[id][b][0] == R->f1[id][k][0] && R->blk[id][b][1] == R->f1[id][k][1] && R->blk[id][b][2] == R->f1[id][k][2]);
      if (!seen)
      {
        const int b = R->n_blk[id]++;
        for (int i = 0; i < 3; i++) R->blk[id][b][i] = R->f1[id][k][i];
      }
    }
  }
}

struct Grid
{
  const int8_t* m;
  int xd, yd, zd;
  FQ_HD bool inside(int x, int y, int z) const { return x >= 0 && x < xd && y >= 0 && y < yd && z >= 0 && z < zd; }
  FQ_HD long long id(int x, int y, int z) const { return x + (long long)xd * (y + (long long)yd * z); }
  FQ_HD bool free_(int x, int y, int z) const { return inside(x, y, z) && m[id(x, y, z)] == 0; }
  FQ_HD bool occupied(int x, int y, int z) const { return inside(x, y, z) && m[id(x, y, z)] > 0; }
};

struct Node
{
  int x, y, z;
  int dir;        // arrival direction id
  int parent;
  int heap_pos;   // -1 not in heap; -2 closed
  double g, h;
};

FQ_HD bool has_forced(const Rules& R, const Grid& g, int x, int y, int z, int d)
{
  for (int b = 0; b < R.n_blk[d]; b++)
    if (g.occupied(x + R.blk[d][b][0], y + R.blk[d][b][1], z + R.blk[d][b][2])) return true;
  return false;
}

// advance from (x,y,z) along d until a jump point: the goal, a cell with a forced neighbour, or a cell from which a
// sub-move (every natural neighbour but the move itself) finds one; false if blocked first.  The reference recurses; the
// recursion is at most three deep (3D diagonal -> 2D -> 1D, a 1D move has no sub-moves), so it runs here as a loop over
// a fixed stack in the same order.
FQ_HD bool jump(const Rules& R, const Grid& g, V3i goal, int x, int y, int z, int d, V3i* out)
{
  struct Frame
  {
    int x, y, z, d, k;   // k: next sub-move, -1: step first
  } st[3];
  int sp = 0;
  st[0].x = x; st[0].y = y; st[0].z = z; st[0].d = d; st[0].k = -1;
  int ret = -1;          // -1: nothing returned; 0 / 1: what the frame above returned
  for (;;)
  {
    Frame& f = st[sp];
    if (ret >= 0)
    {
      const bool found = ret == 1;
      ret = -1;
      if (found)
      { // a sub-move found a jump point: this cell is one
        if (sp == 0) { *out = v3(f.x, f.y, f.z); return true; }
        sp--; ret = 1;
        continue;
      }
      f.k++;
    }
    else if (f.k < 0)
    {
      const V3i dv = dir_of(f.d);
      f.x += dv.x; f.y += dv.y; f.z += dv.z;
      int r = -1;
      if (!g.free_(f.x, f.y, f.z)) r = 0;
      else if ((f.x == goal.x && f.y == goal.y && f.z == goal.z) || has_forced(R, g, f.x, f.y, f.z, f.d)) r = 1;
      if (r >= 0)
      {
        if (sp == 0)
        {
          if (r) *out = v3(f.x, f.y, f.z);
          return r == 1;
        }
        sp--; ret = r;
        continue;
      }
      f.k = 0;
    }
    if (f.k + 1 < R.n_nat[f.d])
    {
      Frame& c = st[sp + 1];
      c.x = f.x; c.y = f.y; c.z = f.z; c.d = R.nat[f.d][f.k]; c.k = -1;
      sp++;
      continue;
    }
    f.k = -1;            // no sub-move found one: continue straight
  }
}

// Candidate i (host order) of an expansion from `cur`: with JPS the natural directions, then the forced successors
// whose blocker is occupied; plain A* the 26 neighbours.  -> the candidate's direction id, or -1 past the last one.
FQ_HD int candidate(const Rules& R, const Grid& g, const Node& cur, bool use_jps, int i)
{
  if (!use_jps) return i < 26 ? R.nat[13][i] : -1;
  const int d = cur.dir;
  if (i < R.n_nat[d]) return R.nat[d][i];
  i -= R.n_nat[d];
  for (int k = 0; k < R.n_forced[d]; k++)
    if (g.occupied(cur.x + R.f1[d][k][0], cur.y + R.f1[d][k][1], cur.z + R.f1[d][k][2]) && i-- == 0)
      return dir_id(R.f2[d][k][0], R.f2[d][k][1], R.f2[d][k][2]);
  return -1;
}

// Successor of `cur` along candidate direction d: *jp the cell, *cost the step cost in cells.  false: none.
FQ_HD bool successor(const Rules& R, const Grid& g, V3i goal, const Node& cur, bool use_jps, int d, V3i* jp, double* cost)
{
  const V3i dv = dir_of(d);
  if (!use_jps)
  {
    *jp = v3(cur.x + dv.x, cur.y + dv.y, cur.z + dv.z);
    if (!g.free_(jp->x, jp->y, jp->z)) return false;
    *cost = FQ_SQRT((double)(dv.x * dv.x + dv.y * dv.y + dv.z * dv.z));
    return true;
  }
  if (!jump(R, g, goal, cur.x, cur.y, cur.z, d, jp)) return false;
  const int ex = jp->x - cur.x, ey = jp->y - cur.y, ez = jp->z - cur.z;
  *cost = FQ_SQRT((double)(ex * ex + ey * ey + ez * ez));
  return true;
}

// The A* open list and node bookkeeping over caller storage S, which provides
//   Node& node(int k); int& heap(int i); int lookup(long long cell) (-1: none); int add(long long cell) (-1: full).
template <class S>
struct Search
{
  S& s;
  V3i goal;
  int heap_n = 0;
  FQ_HD Search(S& store, V3i g) : s(store), goal(g) {}

  // priority: smaller f first; equal f (within 1e-6): larger g first (graph_search.h:19-27)
  FQ_HD bool lower(int a, int b)
  {
    const Node& na = s.node(a);
    const Node& nb = s.node(b);
    const double fa = FQ_ADD(na.g, na.h), fb = FQ_ADD(nb.g, nb.h);
    if (fa >= FQ_SUB(fb, 0.000001) && fa <= FQ_ADD(fb, 0.000001)) return na.g < nb.g;
    return fa > fb;
  }
  FQ_HD void swap_at(int i, int j)
  {
    const int t = s.heap(i);
    s.heap(i) = s.heap(j);
    s.heap(j) = t;
    s.node(s.heap(i)).heap_pos = i;
    s.node(s.heap(j)).heap_pos = j;
  }
  FQ_HD void up(int i)
  {
    while (i > 0)
    {
      const int p = (i - 1) / 2;
      if (!lower(s.heap(p), s.heap(i))) break;
      swap_at(p, i);
      i = p;
    }
  }
  FQ_HD void down(int i)
  {
    for (;;)
    {
      int best = i;
      const int l = 2 * i + 1, r = l + 1;
      if (l < heap_n && lower(s.heap(best), s.heap(l))) best = l;
      if (r < heap_n && lower(s.heap(best), s.heap(r))) best = r;
      if (best == i) break;
      swap_at(best, i);
      i = best;
    }
  }
  FQ_HD void push(int k)
  {
    s.node(k).heap_pos = heap_n;
    s.heap(heap_n++) = k;
    up(s.node(k).heap_pos);
  }
  FQ_HD int pop()
  {
    const int k = s.heap(0);
    s.heap(0) = s.heap(heap_n - 1);
    s.node(s.heap(0)).heap_pos = 0;
    heap_n--;
    if (heap_n > 0) down(0);
    s.node(k).heap_pos = -2;
    return k;
  }
  FQ_HD double heur(int x, int y, int z) const
  {
    return FQ_SQRT((double)((x - goal.x) * (x - goal.x) + (y - goal.y) * (y - goal.y) + (z - goal.z) * (z - goal.z)));
  }
  // the node of cell (x,y,z) in grid g, created with arrival direction d; -1 when the storage is full
  FQ_HD int node_at(const Grid& g, int x, int y, int z, int d)
  {
    const long long cid = g.id(x, y, z);
    int k = s.lookup(cid);
    if (k >= 0) return k;
    k = s.add(cid);
    if (k < 0) return -1;
    Node& n = s.node(k);
    n.x = x; n.y = y; n.z = z; n.dir = d; n.parent = -1; n.heap_pos = -1;
    n.g = INFINITY; n.h = heur(x, y, z);
    return k;
  }
  FQ_HD void start(const Grid& g, V3i a)
  {
    const int k = node_at(g, a.x, a.y, a.z, 13);
    s.node(k).g = 0;
    push(k);
  }
  FQ_HD bool is_goal(int k) { const Node& n = s.node(k); return n.x == goal.x && n.y == goal.y && n.z == goal.z; }
  // a successor c of k reached at `cost`: a better path re-parents it, re-derives an open node's arrival direction
  // and sifts it up, and opens a new node
  FQ_HD void relax(int k, int c, double cost)
  {
    Node& n = s.node(c);
    const Node& p = s.node(k);
    const double tg = FQ_ADD(p.g, cost);
    if (!(tg < n.g)) return;
    n.parent = k; n.g = tg;
    if (n.heap_pos >= 0)
    {
      const int dx = n.x - p.x, dy = n.y - p.y, dz = n.z - p.z;
      n.dir = dir_id((dx > 0) - (dx < 0), (dy > 0) - (dy < 0), (dz > 0) - (dz < 0));
      up(n.heap_pos);
    }
    else if (n.heap_pos == -1)
      push(c);
  }
};

// ---- world coordinates (map_util.h:334-383) --------------------------------------------------------------------------
struct World
{
  Grid g;
  double origin[3], res;
  FQ_HD void to_int(const double* p, int* c) const
  {
    for (int i = 0; i < 3; i++) c[i] = (int)round(FQ_SUB(FQ_DIV(FQ_SUB(p[i], origin[i]), res), 0.5));
  }
  FQ_HD void to_float(const int* c, double* p) const
  {
    for (int i = 0; i < 3; i++) p[i] = FQ_ADD(FQ_MUL(FQ_ADD((double)c[i], 0.5), res), origin[i]);
  }
  // the ray samples of blocked(p1, p2): n = 1 .. count - 1 of p1 + diff * s * n; returns count (<= 1: none)
  FQ_HD int ray(const double* p1, const double* p2, double* diff, double* s) const
  {
    double mx = 0;
    for (int i = 0; i < 3; i++)
    {
      diff[i] = FQ_SUB(p2[i], p1[i]);
      const double a = fabs(FQ_DIV(diff[i], res));
      mx = mx < a ? a : mx;                                     // std::max(mx, a)
    }
    const int max_diff = (int)FQ_DIV(mx, 0.8);
    *s = max_diff > 0 ? FQ_DIV(1.0, (double)max_diff) : 0.0;
    return max_diff;
  }
  // sample n of the ray: 0 free or repeated, 1 a cell with value >= 100, 2 outside the grid
  FQ_HD int sample(const double* p1, const double* diff, double s, int n, int* c) const
  {
    double pt[3];
    for (int i = 0; i < 3; i++) pt[i] = FQ_ADD(p1[i], FQ_MUL(FQ_MUL(diff[i], s), (double)n));
    to_int(pt, c);
    if (!g.inside(c[0], c[1], c[2])) return 2;
    return g.m[g.id(c[0], c[1], c[2])] >= 100 ? 1 : 0;
  }
  // any ray-traced cell between p1 and p2 with value >= 100 before the ray leaves the grid (map_util.h:349-383; the
  // reference skips a sample in the cell of the one before it, which has the same value)
  FQ_HD bool blocked(const double* p1, const double* p2) const
  {
    double diff[3], s;
    const int max_diff = ray(p1, p2, diff, &s);
    for (int n = 1; n < max_diff; n++)
    {
      int c[3];
      const int r = sample(p1, diff, s, n, c);
      if (r == 2) break;
      if (r == 1) return true;
    }
    return false;
  }
};

// Eigen-free 3-vector distance in the host's order: sqrt((dx^2 + dy^2) + dz^2)
FQ_HD double dist3(const double* a, const double* b)
{
  const double dx = FQ_SUB(a[0], b[0]), dy = FQ_SUB(a[1], b[1]), dz = FQ_SUB(a[2], b[2]);
  return FQ_SQRT(FQ_ADD(FQ_ADD(FQ_MUL(dx, dx), FQ_MUL(dy, dy)), FQ_MUL(dz, dz)));
}

// removeLinePts (jps_planner.cpp:83-105): p (n xyz) -> out (may not alias p); returns the count
FQ_HD int remove_line_pts(const double* p, int n, double* out)
{
  if (n < 3)
  {
    for (int i = 0; i < 3 * n; i++) out[i] = p[i];
    return n;
  }
  int m = 0;
  for (int k = 0; k < 3; k++) out[k] = p[k];
  m = 1;
  for (int i = 1; i + 1 < n; i++)
  {
    double s = 0;
    for (int k = 0; k < 3; k++)
      s = FQ_ADD(s, fabs(FQ_SUB(FQ_SUB(p[3 * (i + 1) + k], p[3 * i + k]), FQ_SUB(p[3 * i + k], p[3 * (i - 1) + k]))));
    if (s > 1e-2)
    {
      for (int k = 0; k < 3; k++) out[3 * m + k] = p[3 * i + k];
      m++;
    }
  }
  for (int k = 0; k < 3; k++) out[3 * m + k] = p[3 * (n - 1) + k];
  return m + 1;
}

// removeCornerPts (jps_planner.cpp:36-80): p (n xyz) -> out (may not alias p); blocked(a, b) is the line-of-sight test
// (World::blocked, or a warp's split of it).  `write`: whether this caller stores (every caller computes the count).
template <class Blocked>
FQ_HD int remove_corner_pts(Blocked&& blocked, const double* p, int n, double* out, bool write)
{
  if (n < 2)
  {
    for (int i = 0; write && i < 3 * n; i++) out[i] = p[i];
    return n;
  }
  int m = 1;
  for (int k = 0; write && k < 3; k++) out[k] = p[k];
  const double* prev = p;
  double cost1 = blocked(p, p + 3) ? INFINITY : dist3(p, p + 3);
  for (int i = 1; i + 1 < n; i++)
  {
    const double* a = p + 3 * i;
    const double* b = p + 3 * (i + 1);
    const double cost2 = blocked(a, b) ? INFINITY : dist3(a, b);
    const double cost3 = blocked(prev, b) ? INFINITY : dist3(prev, b);
    if (cost3 < FQ_ADD(cost1, cost2)) cost1 = cost3;
    else
    {
      for (int k = 0; write && k < 3; k++) out[3 * m + k] = a[k];
      m++;
      cost1 = dist3(a, b);
      prev = a;
    }
  }
  for (int k = 0; write && k < 3; k++) out[3 * m + k] = p[3 * (n - 1) + k];
  return m + 1;
}

FQ_HD void reverse_into(const double* p, int n, double* out)
{
  for (int i = 0; i < n; i++)
    for (int k = 0; k < 3; k++) out[3 * i + k] = p[3 * (n - 1 - i) + k];
}
}  // namespace fqjps
