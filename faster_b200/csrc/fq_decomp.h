// The per-point and per-plane arithmetic of the convex decomposition (JPS_Manager::cvxEllipsoidDecomp over DecompUtil's
// EllipsoidDecomp3D; references in fq_decomp.cpp) as ONE source for the host (fq_ellipsoid_decomp, fq_decomp.cpp) and the
// device (fq_decomp_kernel, fq_decomp.cuh).  The loops that drive it live with each caller.
//
// Every double operation is spelled through FQ_MUL/FQ_ADD/... (fq_dtinit.h), so the device evaluates the same expression
// tree as the host with round-to-nearest intrinsics, never contracted into FMAs.  What can still differ between the two
// are atan2, hypot, sin and cos (vec3_to_rotation, rotx): CUDA's versions may differ from glibc's by a few ulp.  So the
// device's ellipsoid can differ from the host's in the last bits, and where two obstacle points are equally far from it to
// within that, the device may pick the other one (a different face order or count).  tests/test_pair_decomp_gpu.py
// compares the two.
#pragma once
#include "fq_dtinit.h"

namespace fqd
{
constexpr double kEps = 1e-10;   // decomp_basis/data_type.h:129

struct V3
{
  double x, y, z;
};
FQ_HD V3 add(V3 a, V3 b) { return { FQ_ADD(a.x, b.x), FQ_ADD(a.y, b.y), FQ_ADD(a.z, b.z) }; }
FQ_HD V3 sub(V3 a, V3 b) { return { FQ_SUB(a.x, b.x), FQ_SUB(a.y, b.y), FQ_SUB(a.z, b.z) }; }
FQ_HD V3 scale(V3 a, double s) { return { FQ_MUL(a.x, s), FQ_MUL(a.y, s), FQ_MUL(a.z, s) }; }
FQ_HD double dot(V3 a, V3 b) { return FQ_ADD(FQ_ADD(FQ_MUL(a.x, b.x), FQ_MUL(a.y, b.y)), FQ_MUL(a.z, b.z)); }
FQ_HD double norm(V3 a) { return FQ_SQRT(dot(a, a)); }

struct M3
{
  double m[3][3];
};
FQ_HD V3 mul(const M3& R, V3 v)
{
  return { FQ_ADD(FQ_ADD(FQ_MUL(R.m[0][0], v.x), FQ_MUL(R.m[0][1], v.y)), FQ_MUL(R.m[0][2], v.z)),
           FQ_ADD(FQ_ADD(FQ_MUL(R.m[1][0], v.x), FQ_MUL(R.m[1][1], v.y)), FQ_MUL(R.m[1][2], v.z)),
           FQ_ADD(FQ_ADD(FQ_MUL(R.m[2][0], v.x), FQ_MUL(R.m[2][1], v.y)), FQ_MUL(R.m[2][2], v.z)) };
}
FQ_HD V3 mulT(const M3& R, V3 v)
{
  return { FQ_ADD(FQ_ADD(FQ_MUL(R.m[0][0], v.x), FQ_MUL(R.m[1][0], v.y)), FQ_MUL(R.m[2][0], v.z)),
           FQ_ADD(FQ_ADD(FQ_MUL(R.m[0][1], v.x), FQ_MUL(R.m[1][1], v.y)), FQ_MUL(R.m[2][1], v.z)),
           FQ_ADD(FQ_ADD(FQ_MUL(R.m[0][2], v.x), FQ_MUL(R.m[1][2], v.y)), FQ_MUL(R.m[2][2], v.z)) };
}
FQ_HD M3 matmul(const M3& A, const M3& B)
{
  M3 C;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++)
      C.m[i][j] = FQ_ADD(FQ_ADD(FQ_MUL(A.m[i][0], B.m[0][j]), FQ_MUL(A.m[i][1], B.m[1][j])), FQ_MUL(A.m[i][2], B.m[2][j]));
  return C;
}
FQ_HD M3 rotx(double a)
{
  const double c = cos(a), s = sin(a);
  return { { { 1, 0, 0 }, { 0, c, -s }, { 0, s, c } } };
}
// geometric_utils.h:27-35: zero roll, R = Rz(yaw) Ry(pitch)
FQ_HD M3 vec3_to_rotation(V3 v)
{
  const double pitch = atan2(-v.z, hypot(v.x, v.y)), yaw = atan2(v.y, v.x);
  const double cp = cos(pitch), sp = sin(pitch), cy = cos(yaw), sy = sin(yaw);
  const M3 ry = { { { cp, 0, sp }, { 0, 1, 0 }, { -sp, 0, cp } } };
  const M3 rz = { { { cy, -sy, 0 }, { sy, cy, 0 }, { 0, 0, 1 } } };
  return matmul(rz, ry);
}
FQ_HD double sgn(double v) { return (0.0 < v) - (v < 0.0); }

struct Plane
{
  V3 p, n;
};

struct Ellip
{
  M3 Rf;
  double ax[3];
  V3 d;
  // |C^-1 (pt - d)| with C = Rf diag(ax) Rf'   (ellipsoid.h:24-27)
  FQ_HD double dist(V3 pt) const
  {
    const V3 q = mulT(Rf, sub(pt, d));
    const double a = FQ_DIV(q.x, ax[0]), b = FQ_DIV(q.y, ax[1]), c = FQ_DIV(q.z, ax[2]);
    return FQ_SQRT(FQ_ADD(FQ_ADD(FQ_MUL(a, a), FQ_MUL(b, b)), FQ_MUL(c, c)));
  }
};

FQ_HD void local_bbox(V3 p1, V3 p2, const double* bbox, Plane out[6])
{ // line_segment.h:57-98
  const V3 d = sub(p2, p1);
  const V3 dir = scale(d, FQ_DIV(1.0, norm(d)));
  V3 dir_h = { dir.y, -dir.x, 0.0 };
  if (norm(dir_h) == 0) dir_h = { -1.0, 0.0, 0.0 };
  dir_h = scale(dir_h, FQ_DIV(1.0, norm(dir_h)));
  const V3 dir_v = { FQ_SUB(FQ_MUL(dir.y, dir_h.z), FQ_MUL(dir.z, dir_h.y)), FQ_SUB(FQ_MUL(dir.z, dir_h.x), FQ_MUL(dir.x, dir_h.z)),
                     FQ_SUB(FQ_MUL(dir.x, dir_h.y), FQ_MUL(dir.y, dir_h.x)) };
  out[0] = { add(p1, scale(dir_h, bbox[1])), dir_h };
  out[1] = { sub(p1, scale(dir_h, bbox[1])), scale(dir_h, -1.0) };
  out[2] = { add(p2, scale(dir, bbox[0])), dir };
  out[3] = { sub(p1, scale(dir, bbox[0])), scale(dir, -1.0) };
  out[4] = { add(p1, scale(dir_v, bbox[2])), dir_v };
  out[5] = { sub(p1, scale(dir_v, bbox[2])), scale(dir_v, -1.0) };
}

// axis-aligned hull of the oriented box bb[0..5] of local_bbox (padded by 1e-6, far beyond the 1e-10 of the exact test)
FQ_HD void bbox_aabb(V3 p1, const Plane bb[6], double lo[3], double hi[3])
{
  for (int k = 0; k < 3; k++) { lo[k] = 1e300; hi[k] = -1e300; }
  for (int c = 0; c < 8; c++)
  { // a corner adds to p1 the displacement of one face point of each opposite pair (the three axes are orthogonal)
    const Plane& fh = bb[(c & 1) ? 0 : 1];
    const Plane& fd = bb[(c & 2) ? 2 : 3];
    const Plane& fv = bb[(c & 4) ? 4 : 5];
    const V3 corner = add(add(add(p1, sub(fh.p, p1)), sub(fd.p, p1)), sub(fv.p, p1));
    const double cc[3] = { corner.x, corner.y, corner.z };
    for (int k = 0; k < 3; k++) { lo[k] = fmin(lo[k], cc[k]); hi[k] = fmax(hi[k], cc[k]); }
  }
  for (int k = 0; k < 3; k++) { lo[k] = FQ_SUB(lo[k], 1e-6); hi[k] = FQ_ADD(hi[k], 1e-6); }
}

FQ_HD bool outside_aabb(const double lo[3], const double hi[3], double x, double y, double z)
{
  return x < lo[0] || x > hi[0] || y < lo[1] || y > hi[1] || z < lo[2] || z > hi[2];
}

// set_obs (decomp_base.h:39-46 / polyhedron.h:65-76): signed_dist <= epsilon_ for every bbox face
FQ_HD bool inside_bbox(const Plane bb[6], V3 pt)
{
  bool in = true;
  for (int k = 0; k < 6 && in; k++) in = !(dot(bb[k].n, sub(pt, bb[k].p)) > kEps);
  return in;
}

// find_ellipsoid's start (line_segment.h:156-177): the sphere of diameter |p2 - p1| around the midpoint; f = its radius
FQ_HD void ellipsoid_start(V3 p1, V3 p2, Ellip* E, M3* Ri, double* f)
{
  *f = FQ_DIV(norm(sub(p1, p2)), 2);
  *Ri = vec3_to_rotation(sub(p2, p1));
  E->Rf = *Ri;
  E->ax[0] = E->ax[1] = E->ax[2] = *f;
  E->d = scale(add(p1, p2), 0.5);
}

// obstacle inflation in the ellipsoid frame (line_segment.h:178-190)
FQ_HD V3 inflate_point(const M3& Ri, V3 d, V3 it, double inflate)
{
  V3 p = mulT(Ri, sub(it, d));
  p = { FQ_SUB(p.x, FQ_MUL(sgn(p.x), inflate)), FQ_SUB(p.y, FQ_MUL(sgn(p.y), inflate)), FQ_SUB(p.z, FQ_MUL(sgn(p.z), inflate)) };
  return add(mul(Ri, p), d);
}

// a point stays in a shrink loop while 1 - E.dist > epsilon_ (line_segment.h:210-216, :240-246)
FQ_HD bool still_inside(const Ellip& E, V3 pt) { return FQ_SUB(1.0, E.dist(pt)) > kEps; }

// shrink the two short axes together towards the closest point pw (line_segment.h:195-217)
FQ_HD void shrink_short_axes(Ellip* E, const M3& Ri, V3 pw)
{
  V3 p = mulT(Ri, sub(pw, E->d));
  const double roll = atan2(p.z, p.y);
  E->Rf = matmul(Ri, rotx(roll));
  p = mulT(E->Rf, sub(pw, E->d));
  if (p.x < E->ax[0]) E->ax[1] = FQ_DIV(fabs(p.y), FQ_SQRT(FQ_SUB(1.0, FQ_MUL(FQ_DIV(p.x, E->ax[0]), FQ_DIV(p.x, E->ax[0])))));
  E->ax[2] = E->ax[1];
}

// shrink the third axis towards the closest point pw (line_segment.h:226-247)
FQ_HD void shrink_third_axis(Ellip* E, V3 pw)
{
  const V3 p = mulT(E->Rf, sub(pw, E->d));
  const double dd = FQ_SUB(FQ_SUB(1.0, FQ_MUL(FQ_DIV(p.x, E->ax[0]), FQ_DIV(p.x, E->ax[0]))),
                           FQ_MUL(FQ_DIV(p.y, E->ax[1]), FQ_DIV(p.y, E->ax[1])));
  if (dd > kEps) E->ax[2] = FQ_DIV(fabs(p.z), FQ_SQRT(dd));
}

// the tangent half-space at cp: n = C^-1 C^-T (cp - d) = Rf diag(1/ax^2) Rf' (cp - d), normalised  (ellipsoid.h:65-73)
FQ_HD V3 tangent_normal(const Ellip& E, V3 cp)
{
  V3 q = mulT(E.Rf, sub(cp, E.d));
  q = { FQ_DIV(q.x, FQ_MUL(E.ax[0], E.ax[0])), FQ_DIV(q.y, FQ_MUL(E.ax[1], E.ax[1])), FQ_DIV(q.z, FQ_MUL(E.ax[2], E.ax[2])) };
  const V3 n = mul(E.Rf, q);
  return scale(n, FQ_DIV(1.0, norm(n)));
}

// find_polyhedron keeps the points strictly on the inner side of every face found so far (decomp_base.h:100-110)
FQ_HD bool before_plane(V3 n, V3 cp, V3 pt) { return dot(n, sub(pt, cp)) < 0; }

// LinearConstraint3D(pt_inside, hyperplanes): A x <= b with the segment midpoint inside (polyhedron.h:131-152)
FQ_HD void oriented_row(const Plane& pl, V3 mid, double* r)
{
  V3 n = pl.n;
  double c = dot(pl.p, n);
  if (FQ_SUB(dot(n, mid), c) > 0) { n = scale(n, -1.0); c = -c; }
  r[0] = n.x; r[1] = n.y; r[2] = n.z; r[3] = c;
}

// ground face (jps_manager.cpp:118-122)
FQ_HD void ground_row(double z_ground, double* r) { r[0] = 0; r[1] = 0; r[2] = -1; r[3] = -z_ground; }
}  // namespace fqd
