// Host-side path search on a voxel grid: the first input generator of Faster::replan() (jps_manager_.solveJPS3D,
// faster/src/faster.cpp:361).  The search, its pruning rules and the path post-processing are fq_jps.h's, shared with the
// batch kernel (fq_jps.cuh); this file gives them host storage.  Stays on the host (BASELINE north_star); the batch
// entries fq_jps_batch / _dev run the same code on the GPU.
#include "../../include/faster_b200.h"
#include "fq_jps.h"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace
{
using fqjps::Grid;
using fqjps::Node;
using fqjps::V3i;
using fqjps::World;

const fqjps::Rules& rules()
{
  static const fqjps::Rules r = [] { fqjps::Rules t; fqjps::rules_build(&t); return t; }();
  return r;
}

// Host storage of one search: growing node pool and heap.  The cell -> node index map is as large as the grid (a few
// hundred thousand cells) while a search touches a few hundred of them: it lives in a per-thread buffer whose entries
// carry the number of the search that wrote them, so nothing is cleared between searches.
struct HostStore
{
  std::vector<Node> n;
  std::vector<int> h;
  std::vector<int>& cell;
  std::vector<unsigned>& stamp;
  unsigned epoch;
  struct Scratch
  {
    std::vector<int> cell;
    std::vector<unsigned> stamp;
    unsigned epoch = 0;
  };
  static Scratch& scratch()
  {
    static thread_local Scratch s;
    return s;
  }
  explicit HostStore(size_t cells) : cell(scratch().cell), stamp(scratch().stamp)
  {
    Scratch& sc = scratch();
    if (sc.cell.size() < cells) { sc.cell.assign(cells, -1); sc.stamp.assign(cells, 0u); sc.epoch = 0; }
    if (++sc.epoch == 0) { std::fill(sc.stamp.begin(), sc.stamp.end(), 0u); sc.epoch = 1; }
    epoch = sc.epoch;
  }
  Node& node(int k) { return n[(size_t)k]; }
  int& heap(int i)
  {
    if ((size_t)i >= h.size()) h.resize((size_t)i + 1);
    return h[(size_t)i];
  }
  int lookup(long long c) const { return stamp[(size_t)c] == epoch ? cell[(size_t)c] : -1; }
  int add(long long c)
  {
    stamp[(size_t)c] = epoch;
    cell[(size_t)c] = (int)n.size();
    n.push_back(Node{});
    return cell[(size_t)c];
  }
};

typedef std::vector<double> Path;   // xyz triples
}  // namespace

// fq_jps3d_plan with the number of nodes its search created (*n_nodes, may be NULL)
static int plan(const int8_t* map, int xd, int yd, int zd, const int* start, const int* goal, int use_jps, int max_expand, int* path_out,
                int cap, double* cost, int* n_expanded, long long* n_nodes)
{
  if (n_nodes) *n_nodes = 0;
  if (!map || xd <= 0 || yd <= 0 || zd <= 0 || !start || !goal) return FQ_E_ARG;
  if (cost) *cost = INFINITY;
  if (n_expanded) *n_expanded = 0;
  const Grid g = { map, xd, yd, zd };
  if (!g.free_(start[0], start[1], start[2]) || !g.free_(goal[0], goal[1], goal[2])) return 0;
  const fqjps::Rules& R = rules();
  HostStore st(xd * (size_t)yd * zd);
  fqjps::Search<HostStore> s(st, fqjps::v3(goal[0], goal[1], goal[2]));
  s.start(g, fqjps::v3(start[0], start[1], start[2]));
  int it = 0, k = -1;
  while (s.heap_n > 0)
  {
    it++;
    const int cur = s.pop();
    if (s.is_goal(cur)) { k = cur; break; }
    const Node c = st.node(cur);
    for (int i = 0;; i++)
    {
      const int d = fqjps::candidate(R, g, c, use_jps != 0, i);
      if (d < 0) break;
      V3i jp;
      double step;
      if (!fqjps::successor(R, g, s.goal, c, use_jps != 0, d, &jp, &step)) continue;
      s.relax(cur, s.node_at(g, jp.x, jp.y, jp.z, d), step);
    }
    if (max_expand > 0 && it >= max_expand) break;
  }
  if (n_expanded) *n_expanded = it;
  if (n_nodes) *n_nodes = (long long)st.n.size();
  if (k < 0) return 0;
  std::vector<int> chain;
  for (int i = k; i >= 0; i = st.node(i).parent) chain.push_back(i);
  const int n = (int)chain.size();
  double c = 0;
  for (int i = 0; i < n; i++)
  {
    const Node& a = st.node(chain[n - 1 - i]);
    if (path_out && i < cap) { path_out[3 * i] = a.x; path_out[3 * i + 1] = a.y; path_out[3 * i + 2] = a.z; }
    if (i > 0)
    {
      const Node& b = st.node(chain[n - i]);
      c += std::sqrt((double)((a.x - b.x) * (a.x - b.x) + (a.y - b.y) * (a.y - b.y) + (a.z - b.z) * (a.z - b.z)));
    }
  }
  if (cost) *cost = c;
  return n;
}

extern "C" int fq_jps3d_plan(const int8_t* map, int xd, int yd, int zd, const int* start, const int* goal, int use_jps,
                             int max_expand, int* path_out, int cap, double* cost, int* n_expanded)
{
  return plan(map, xd, yd, zd, start, goal, use_jps, max_expand, path_out, cap, cost, n_expanded, nullptr);
}

extern "C" long long fq_jps3d_nodes(const int8_t* map, int xd, int yd, int zd, const int* start, const int* goal, int use_jps)
{
  long long n = 0;
  const int rc = plan(map, xd, yd, zd, start, goal, use_jps, -1, nullptr, 0, nullptr, nullptr, &n);
  return rc < 0 ? rc : n;
}

extern "C" int fq_jps3d_plan_world(const int8_t* map, int xd, int yd, int zd, const double* origin, double res,
                                   const double* start, const double* goal, int use_jps, double* path_out, int cap,
                                   double* raw_cost)
{
  if (!map || !origin || !(res > 0) || !start || !goal || !path_out) return FQ_E_ARG;
  World w;
  w.g = Grid{ map, xd, yd, zd };
  w.res = res;
  for (int i = 0; i < 3; i++) w.origin[i] = origin[i];
  int s[3], g[3];
  w.to_int(start, s);
  w.to_int(goal, g);
  std::vector<int> cells((size_t)3 * ((size_t)xd + yd + zd + 8) * 4);
  double c = INFINITY;
  int n = fq_jps3d_plan(map, xd, yd, zd, s, g, use_jps, -1, cells.data(), (int)(cells.size() / 3), &c, nullptr);
  if (raw_cost) *raw_cost = n > 0 ? c * res : INFINITY;
  if (n <= 0) return n;
  if (n > (int)(cells.size() / 3))
  { // very long raw path: fetch it again with enough room
    cells.assign((size_t)3 * n, 0);
    n = fq_jps3d_plan(map, xd, yd, zd, s, g, use_jps, -1, cells.data(), n, &c, nullptr);
  }
  Path raw((size_t)3 * n), a((size_t)3 * n), b((size_t)3 * n);
  for (int i = 0; i < n; i++) w.to_float(&cells[3 * i], &raw[3 * i]);
  // jps_planner.cpp:289-293: line points out, corner points out forwards and backwards
  auto blocked = [&](const double* p1, const double* p2) { return w.blocked(p1, p2); };
  int m = fqjps::remove_line_pts(raw.data(), n, a.data());
  m = fqjps::remove_corner_pts(blocked, a.data(), m, b.data(), true);
  fqjps::reverse_into(b.data(), m, a.data());
  m = fqjps::remove_corner_pts(blocked, a.data(), m, b.data(), true);
  fqjps::reverse_into(b.data(), m, a.data());
  a.resize((size_t)3 * m);
  const Path& p = a;
  if (m > cap) return FQ_E_NOMEM;
  std::memcpy(path_out, p.data(), sizeof(double) * p.size());
  return m;
}

// introspection for tests: the pruning rules as flat tables in the reference's layout
// (ns[27][3][26], f1[27][3][12], f2[27][3][12], counts[27][2])
extern "C" void fq_jps3d_rules(int* ns, int* f1, int* f2, int* counts)
{
  std::memset(ns, 0, sizeof(int) * 27 * 3 * 26);
  std::memset(f1, 0, sizeof(int) * 27 * 3 * 12);
  std::memset(f2, 0, sizeof(int) * 27 * 3 * 12);
  const fqjps::Rules& R = rules();
  for (int id = 0; id < 27; id++)
  {
    counts[2 * id] = R.n_nat[id];
    counts[2 * id + 1] = R.n_forced[id];
    for (int k = 0; k < R.n_nat[id]; k++)
    {
      const V3i d = fqjps::dir_of(R.nat[id][k]);
      ns[(id * 3 + 0) * 26 + k] = d.x; ns[(id * 3 + 1) * 26 + k] = d.y; ns[(id * 3 + 2) * 26 + k] = d.z;
    }
    for (int k = 0; k < R.n_forced[id]; k++)
      for (int i = 0; i < 3; i++)
      {
        f1[(id * 3 + i) * 12 + k] = R.f1[id][k][i];
        f2[(id * 3 + i) * 12 + k] = R.f2[id][k][i];
      }
  }
}
