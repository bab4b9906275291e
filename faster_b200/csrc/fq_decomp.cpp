// Host-side convex decomposition of a polyline path against an obstacle point cloud: the input generator that feeds
// SolverGurobi::setPolytopes in the reference (JPS_Manager::cvxEllipsoidDecomp, faster/src/jps_manager.cpp:80-127, over
// DecompUtil's EllipsoidDecomp3D: decomp_util/ellipsoid_decomp.h:96-123, line_segment.h:33-38,57-98,156-252,
// decomp_base.h:39-46,83-115, decomp_geometry/ellipsoid.h:24-73, polyhedron.h:13-92,131-152).
// Eigen-free restatement.  The ellipsoid is kept as (Rf, axes) so that C^-1 = Rf diag(1/axes) Rf' is exact by construction.
// The arithmetic is fq_decomp.h, shared with the device kernel of the chained replan (fq_decomp.cuh); the loops, the
// pre-filter and the vectorised distance pass below are the host's own.
#include "../../include/faster_b200.h"

#include "fq_decomp.h"

#include <cmath>
#include <vector>

namespace
{
using namespace fqd;

// E.dist for n points given as separate coordinate arrays: the same operations in the same order as Ellip::dist (packed
// IEEE divisions and square roots round like the scalar ones; the avx2 clone has no FMA), four points per instruction
__attribute__((target_clones("avx2", "default")))
void dist_batch(const Ellip& E, int n, const double* __restrict__ X, const double* __restrict__ Y, const double* __restrict__ Z,
                double* __restrict__ out)
{
  const double r00 = E.Rf.m[0][0], r01 = E.Rf.m[0][1], r02 = E.Rf.m[0][2], r10 = E.Rf.m[1][0], r11 = E.Rf.m[1][1],
               r12 = E.Rf.m[1][2], r20 = E.Rf.m[2][0], r21 = E.Rf.m[2][1], r22 = E.Rf.m[2][2];
  const double dx = E.d.x, dy = E.d.y, dz = E.d.z, a0 = E.ax[0], a1 = E.ax[1], a2 = E.ax[2];
  for (int i = 0; i < n; i++)
  {
    const double vx = X[i] - dx, vy = Y[i] - dy, vz = Z[i] - dz;
    const double qx = r00 * vx + r10 * vy + r20 * vz, qy = r01 * vx + r11 * vy + r21 * vz, qz = r02 * vx + r12 * vy + r22 * vz;
    const double a = qx / a0, b = qy / a1, c = qz / a2;
    out[i] = std::sqrt(a * a + b * b + c * c);
  }
}

// first strict minimum of dist over the listed indices (ellipsoid.h:46-60)
int closest(const Ellip& E, const std::vector<V3>& pts, const std::vector<int>& idx)
{
  int best = -1;
  double bd = 1.7976931348623157e308;
  for (int i : idx)
  {
    const double d = E.dist(pts[i]);
    if (d < bd) { bd = d; best = i; }
  }
  return best;
}

void decompose_segment(V3 p1, V3 p2, const double* obs, int n_obs, const double* bbox, double inflate, std::vector<Plane>* planes)
{
  Plane bb[6];
  local_bbox(p1, p2, bbox, bb);
  // set_obs (decomp_base.h:39-46 / polyhedron.h:65-76): keep points with signed_dist <= epsilon_ for every bbox face
  // A cheap conservative reject first: the axis-aligned box around the eight corners of the oriented one, padded well
  // beyond epsilon_ (most of a map's points fail it after one or two comparisons); survivors get the exact test.
  double lo[3], hi[3];
  bbox_aabb(p1, bb, lo, hi);
  std::vector<V3> O;
  for (int i = 0; i < n_obs; i++)
  {
    const double x = obs[3 * i], y = obs[3 * i + 1], z = obs[3 * i + 2];
    if (outside_aabb(lo, hi, x, y, z)) continue;
    const V3 pt = { x, y, z };
    if (inside_bbox(bb, pt)) O.push_back(pt);
  }
  // find_ellipsoid(0)  (line_segment.h:156-252)
  double f;
  M3 Ri;
  Ellip E;
  ellipsoid_start(p1, p2, &E, &Ri, &f);
  for (V3& it : O) it = inflate_point(Ri, E.d, it, inflate);   // in place: the polyhedron below sees the inflated points
  // coordinate arrays of the (inflated) points for the two passes that evaluate the distance of EVERY point
  const int nO = (int)O.size();
  std::vector<double> soa((size_t)4 * nO);
  double *OX = soa.data(), *OY = OX + nO, *OZ = OY + nO, *dist_of = OZ + nO;
  for (int i = 0; i < nO; i++) { OX[i] = O[i].x; OY[i] = O[i].y; OZ[i] = O[i].z; }
  dist_batch(E, nO, OX, OY, OZ, dist_of);
  std::vector<int> inside0, cur;
  for (int i = 0; i < nO; i++)
    if (dist_of[i] <= 1) inside0.push_back(i);
  cur = inside0;
  while (!cur.empty())
  { // shrink the two short axes together (:195-217)
    shrink_short_axes(&E, Ri, O[closest(E, O, cur)]);
    std::vector<int> nxt;
    for (int i : cur)
      if (still_inside(E, O[i])) nxt.push_back(i);
    cur.swap(nxt);
  }
  E.ax[2] = f;   // reset with the old axes(2) (:219-224)
  cur.clear();
  for (int i : inside0)
    if (E.dist(O[i]) <= 1) cur.push_back(i);
  while (!cur.empty())
  { // shrink the third axis (:226-247)
    shrink_third_axis(&E, O[closest(E, O, cur)]);
    std::vector<int> nxt;
    for (int i : cur)
      if (still_inside(E, O[i])) nxt.push_back(i);
    cur.swap(nxt);
  }
  // find_polyhedron (decomp_base.h:83-115): tangent half-spaces at successive closest points
  std::vector<int> remain(O.size());
  for (int i = 0; i < (int)O.size(); i++) remain[i] = i;
  // the ellipsoid is final here: every point's distance is evaluated once (the same value the reference recomputes in
  // every round), and a round is an arg-min over the survivors plus one half-space test per survivor
  dist_batch(E, nO, OX, OY, OZ, dist_of);
  while (!remain.empty())
  {
    int best = -1;
    double bd = 1.7976931348623157e308;
    for (int i : remain)
      if (dist_of[i] < bd) { bd = dist_of[i]; best = i; }     // first strict minimum, as closest()
    const V3 cp = O[best];
    const V3 n = tangent_normal(E, cp);
    planes->push_back({ cp, n });
    std::vector<int> nxt;
    for (int i : remain)
      if (before_plane(n, cp, O[i])) nxt.push_back(i);
    remain.swap(nxt);
  }
  for (int k = 0; k < 6; k++) planes->push_back(bb[k]);   // add_local_bbox (line_segment.h:33-38)
}
}  // namespace

extern "C" int fq_ellipsoid_decomp(const double* path, int n_seg, const double* obs, int n_obs, const double* bbox,
                                   double inflate, double z_ground, int* face_ofs, double* Ab, int cap_rows)
{
  if (!path || n_seg < 1 || n_obs < 0 || (n_obs > 0 && !obs) || !bbox || !face_ofs || !Ab) return FQ_E_ARG;
  int rows = 0;
  face_ofs[0] = 0;
  // With several segments every point would be looked at once per segment; one pass against the hull of ALL the
  // segments' boxes first leaves each segment a short list (a map is much larger than a corridor).
  std::vector<double> near_pts;
  if (n_seg > 1 && n_obs > 256)
  {
    double ulo[3] = { 1e300, 1e300, 1e300 }, uhi[3] = { -1e300, -1e300, -1e300 };
    for (int s = 0; s < n_seg; s++)
    {
      const V3 p1 = { path[3 * s], path[3 * s + 1], path[3 * s + 2] }, p2 = { path[3 * s + 3], path[3 * s + 4], path[3 * s + 5] };
      if (norm(sub(p2, p1)) == 0) return FQ_E_ARG;
      Plane bb[6];
      double lo[3], hi[3];
      local_bbox(p1, p2, bbox, bb);
      bbox_aabb(p1, bb, lo, hi);
      for (int k = 0; k < 3; k++) { ulo[k] = std::fmin(ulo[k], lo[k]); uhi[k] = std::fmax(uhi[k], hi[k]); }
    }
    near_pts.reserve((size_t)3 * (n_obs / 4 + 16));
    for (int i = 0; i < n_obs; i++)
    {
      const double x = obs[3 * i], y = obs[3 * i + 1], z = obs[3 * i + 2];
      if (outside_aabb(ulo, uhi, x, y, z)) continue;
      near_pts.push_back(x); near_pts.push_back(y); near_pts.push_back(z);      // order preserved
    }
    obs = near_pts.data();
    n_obs = (int)(near_pts.size() / 3);
  }
  std::vector<Plane> planes;
  for (int s = 0; s < n_seg; s++)
  {
    const V3 p1 = { path[3 * s], path[3 * s + 1], path[3 * s + 2] }, p2 = { path[3 * s + 3], path[3 * s + 4], path[3 * s + 5] };
    if (norm(sub(p2, p1)) == 0) return FQ_E_ARG;
    planes.clear();
    decompose_segment(p1, p2, obs, n_obs, bbox, inflate, &planes);
    if (rows + (int)planes.size() + 1 > cap_rows) return FQ_E_NOMEM;
    const V3 mid = scale(add(p1, p2), 0.5);
    for (const Plane& pl : planes) oriented_row(pl, mid, Ab + (size_t)4 * rows++);
    ground_row(z_ground, Ab + (size_t)4 * rows++);
    face_ofs[s + 1] = rows;
  }
  return rows;
}
