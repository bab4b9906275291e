// The reference's float queries of unknown space as ONE source for the host and the device: FLANN's squared distance
// (findIndexH's query, fq_pair.cuh) and the crop of JPS_in where it first nears unknown space (Faster::getFirstCollisionJPS
// with UNKNOWN_MAP and RETURN_INTERSECTION, faster.cpp:767-921), with the helpers it calls from utils.cpp.  Host:
// fq_paths_cloud and fq_jps_in (fq_paths.cu); device: fq_paths_crop_kernel (fq_paths.cu).
//
// Every operation is spelled through FQ_MUL/FQ_ADD/... (double, fq_dtinit.h) or FQ_FMUL/FQ_FADD/... (float, below), so the
// device evaluates the same expression tree as the host with round-to-nearest intrinsics, never contracted into FMAs, in
// the reference's own mix of float and double.  Nothing here calls a transcendental function: host and device agree bit
// for bit.
#pragma once
#include "fq_dtinit.h"

#if defined(__CUDA_ARCH__)
#define FQ_F2(x) __double2float_rn(x)
#define FQ_FMUL(a, b) __fmul_rn((a), (b))
#define FQ_FADD(a, b) __fadd_rn((a), (b))
#define FQ_FSUB(a, b) __fsub_rn((a), (b))
#define FQ_FDIV(a, b) __fdiv_rn((a), (b))
#define FQ_FSQRT(a) __fsqrt_rn(a)
#else
#define FQ_F2(x) ((float)(x))
#define FQ_FMUL(a, b) ((a) * (b))
#define FQ_FADD(a, b) ((a) + (b))
#define FQ_FSUB(a, b) ((a) - (b))
#define FQ_FDIV(a, b) ((a) / (b))
#define FQ_FSQRT(a) std::sqrt((float)(a))
#endif

namespace fqp
{
// squared float distance in FLANN's L2 order (flann/algorithms/dist.h, L2::operator() for 3 values)
FQ_HD float flann_l2(const float* q, const double* p)
{
  const float dx = FQ_FSUB(FQ_F2(p[0]), q[0]), dy = FQ_FSUB(FQ_F2(p[1]), q[1]), dz = FQ_FSUB(FQ_F2(p[2]), q[2]);
  return FQ_FADD(FQ_FADD(FQ_FADD(0.0f, FQ_FMUL(dx, dx)), FQ_FMUL(dy, dy)), FQ_FMUL(dz, dz));
}
}  // namespace fqp

namespace fqpath
{
constexpr int kMaxSteps = 4096;   // sphere steps of one crop before FQ_PATHS_STALL
constexpr int kMaxIn = 4096;      // vertices of one JPS_in (FQ_PATHS_MAX_IN)

// Eigen's (a - b).norm() for 3-vectors: sqrt((dx^2 + dy^2) + dz^2) in double
FQ_HD double dist3(const double* a, const double* b)
{
  const double dx = FQ_SUB(a[0], b[0]), dy = FQ_SUB(a[1], b[1]), dz = FQ_SUB(a[2], b[2]);
  return FQ_SQRT(FQ_ADD(FQ_ADD(FQ_MUL(dx, dx), FQ_MUL(dy, dy)), FQ_MUL(dz, dz)));
}

// pow(d0, 2) + pow(d1, 2) + pow(d2, 2) of floats: double squares and sums, rounded to float on assignment
FQ_HD float pow2_sum(float d0, float d1, float d2)
{
  const double a = d0, b = d1, c = d2;
  return FQ_F2(FQ_ADD(FQ_ADD(FQ_MUL(a, a), FQ_MUL(b, b)), FQ_MUL(c, c)));
}

// the quadratic of getIntersectionWithSphere (utils.cpp:732-736) for the line p1 -> p2 and the sphere (p3, r); p* are the
// float x1.., x2.., x3..; returns t = (-b + sqrt(b^2 - 4ac)) / (2a) and the discriminant
FQ_HD float sphere_t(const float* p1, const float* p2, const float* p3, double r, float* discrim)
{
  float d[3], e[3];
  for (int k = 0; k < 3; k++) { d[k] = FQ_FSUB(p2[k], p1[k]); e[k] = FQ_FSUB(p1[k], p3[k]); }
  const float a = pow2_sum(d[0], d[1], d[2]);
  const float b = FQ_FMUL(2.0f, FQ_FADD(FQ_FADD(FQ_FMUL(d[0], e[0]), FQ_FMUL(d[1], e[1])), FQ_FMUL(d[2], e[2])));
  float s = FQ_FMUL(p3[0], p3[0]);
  s = FQ_FADD(s, FQ_FMUL(p3[1], p3[1]));
  s = FQ_FADD(s, FQ_FMUL(p3[2], p3[2]));
  s = FQ_FADD(s, FQ_FMUL(p1[0], p1[0]));
  s = FQ_FADD(s, FQ_FMUL(p1[1], p1[1]));
  s = FQ_FADD(s, FQ_FMUL(p1[2], p1[2]));
  const float m = FQ_FMUL(2.0f, FQ_FADD(FQ_FADD(FQ_FMUL(p3[0], p1[0]), FQ_FMUL(p3[1], p1[1])), FQ_FMUL(p3[2], p1[2])));
  const float c = FQ_F2(FQ_SUB((double)FQ_FSUB(s, m), FQ_MUL(r, r)));          // `- r * r` is a double term
  *discrim = FQ_FSUB(FQ_FMUL(b, b), FQ_FMUL(FQ_FMUL(4.0f, a), c));
  return FQ_FDIV(FQ_FADD(-b, FQ_FSQRT(*discrim)), FQ_FMUL(2.0f, a));
}

// getIntersectionWithSphere (utils.cpp:713-776): A inside, B outside the sphere (center, r); when the discriminant is
// <= 0, the line from the center through A instead.  *fallback (may be NULL) tells which.
FQ_HD void sphere_point(const double* A, const double* B, double r, const double* center, double* out, bool* fallback = nullptr)
{
  float a[3], b[3], c[3], disc;
  for (int k = 0; k < 3; k++) { a[k] = FQ_F2(A[k]); b[k] = FQ_F2(B[k]); c[k] = FQ_F2(center[k]); }
  const float* p1 = a;
  const float* p2 = b;
  float t = sphere_t(p1, p2, c, r, &disc);
  const bool fb = disc <= 0;
  if (fb) { p1 = c; p2 = a; t = sphere_t(p1, p2, c, r, &disc); }
  if (fallback) *fallback = fb;
  for (int k = 0; k < 3; k++) out[k] = (double)FQ_FADD(p1[k], FQ_FMUL(FQ_FSUB(p2[k], p1[k]), t));
}

// The crop of one JPS_in: the cropped path is in[0 .. m-1] followed, when `extra`, by the vertex e.  A corridor whose
// status is not 0 (FQ_PATHS_*) has no paths.
struct Crop
{
  int status, crossed, m, extra;
  double e[3];
};

// reduceJPSbyDistance(in[0 .. idx-1] ++ [head], d) (utils.cpp:690-710) into c
FQ_HD void reduce_by_distance(const double* in, int idx, const double* head, double d, Crop* c)
{
  c->m = idx; c->extra = 1;
  for (int k = 0; k < 3; k++) c->e[k] = head[k];
  double so_far = 0;
  for (int ii = idx; ii > 0; ii--)
  {
    const double* p1 = in + 3 * (ii - 1);
    const double* p2 = ii == idx ? head : in + 3 * ii;
    double v[3];
    for (int k = 0; k < 3; k++) v[k] = FQ_SUB(p2[k], p1[k]);
    const double sq = FQ_ADD(FQ_ADD(FQ_MUL(v[0], v[0]), FQ_MUL(v[1], v[1])), FQ_MUL(v[2], v[2]));
    const double nv = FQ_SQRT(sq);
    so_far = FQ_ADD(so_far, nv);
    if (so_far > d)
    {
      const double want = FQ_SUB(so_far, d);
      c->m = ii;
      for (int k = 0; k < 3; k++) c->e[k] = FQ_ADD(p1[k], FQ_MUL(sq > 0 ? FQ_DIV(v[k], nv) : v[k], want));   // v.normalized()
      return;
    }
  }
}

// getFirstCollisionJPS's loop (faster.cpp:792-921) over JPS_in = in[0 .. n-1].  The working path is [head] ++ in[idx ..]:
// it never needs a copy.  Each step first needs the nearest unknown point of the head rounded to float (query()), but only
// up to need(): a nearest point farther than that gives the same answer as no point at all.
struct March
{
  double head[3];
  int idx = 1, iter = 0;
  FQ_HD explicit March(const double* in) { for (int k = 0; k < 3; k++) head[k] = in[k]; }
  FQ_HD void query(float* q) const { for (int k = 0; k < 3; k++) q[k] = FQ_F2(head[k]); }   // eigenPoint2pclPoint
  // the largest distance from the head to a vertex of the working path, and at least drone_radius
  FQ_HD double need(const double* in, int n, double drone_radius) const
  {
    double r = drone_radius;
    for (int i = idx; i < n; i++) { const double d = dist3(in + 3 * i, head); r = d > r ? d : r; }
    return r;
  }
  // one step with the squared distance d2 of the nearest unknown point (any: U has a point at all).  Returns true when the
  // crop is decided, then *c holds it (status 0).
  FQ_HD bool step(const double* in, int n, double drone_radius, bool any, float d2, Crop* c)
  {
    c->status = 0; c->crossed = 0; c->m = n; c->extra = 0;
    if (!any) return true;                                         // no neighbours: JPS_in as it is
    const double r = (double)FQ_FSQRT(d2);
    if (r < drone_radius)
    {
      c->crossed = 1;
      if (iter == 0)
      { // :833-841, the first point in collision: [orig0, orig0 + (0.01, 0, 0)]
        c->m = 1; c->extra = 1;
        c->e[0] = FQ_ADD(in[0], 0.01); c->e[1] = in[1]; c->e[2] = in[2];
      }
      else
        reduce_by_distance(in, idx, head, drone_radius, c);         // :846-858
      return true;
    }
    // getFirstIntersectionWithSphere(path, r, path[0]) (utils.cpp:782-866); path[i] = head (i = 0) or in[idx + i - 1]
    const int size = 1 + n - idx;
    int index = -1;
    for (int i = 0; i < size && index < 0; i++)
      if (dist3(i ? in + 3 * (idx + i - 1) : head, head) > r) index = i;
    if (index < 0) return true;                                    // no point outside the sphere: JPS_in as it is
    double inters[3];
    int last;
    if (index == 0)
    {
      for (int k = 0; k < 3; k++) inters[k] = head[k];
      last = 1;
    }
    else
    {
      const double* A = index == 1 ? head : in + 3 * (idx + index - 2);
      sphere_point(A, in + 3 * (idx + index - 1), r, head, inters);
      last = index - 1;
    }
    idx = idx + last < n ? idx + last : n;                         // path = [inters] ++ path[last + 1 ..]
    for (int k = 0; k < 3; k++) head[k] = inters[k];
    iter++;
    return false;
  }
};

// JPS_in from a path of n >= 1 vertices (faster.cpp:361-384), for fq_jps_in and the batch JPS kernel.  Vertex 0 := start
// and the last vertex := goal, both with z = std::max(z, 0.0) as solveJPS3D forces them (jps_manager.cpp:143-144,
// :172-186; a one-vertex path becomes [start, goal]); the path up to where it first leaves the sphere of radius ra around
// vertex 0 (getFirstIntersectionWithSphere, :373-382); then createMoreVertexes(dist_max) (:80-97): floor(dist / d)
// vertices on every segment longer than d, each d past the one before it.
struct JpsIn
{
  const double* jps;
  int n, m, li;            // the clipped path is path[0 .. li] ++ [E] (li >= 0), or the whole path (li < 0), m vertices
  double s[3], g[3], E[3];
  FQ_HD const double* path(int i) const { return i == 0 ? s : (i == (n < 2 ? 1 : n - 1) ? g : jps + 3 * i); }
  FQ_HD const double* jin(int i) const { return li >= 0 && i == li + 1 ? E : path(i); }

  FQ_HD JpsIn(const double* p, int count, const double* start, const double* goal, double ra) : jps(p), n(count)
  {
    for (int k = 0; k < 3; k++) { s[k] = start[k]; g[k] = goal[k]; }
    s[2] = start[2] < 0.0 ? 0.0 : start[2];
    g[2] = goal[2] < 0.0 ? 0.0 : goal[2];
    const int size = n < 2 ? 2 : n;
    int index = -1;
    for (int i = 0; i < size && index < 0; i++)
      if (dist3(path(i), s) > ra) index = i;
    li = -1; m = size;
    if (index >= 0)
    {
      li = index == 0 ? 1 : index - 1;
      for (int k = 0; k < 3; k++) E[k] = s[k];
      if (index > 0) sphere_point(path(index - 1), path(index), ra, s, E);
      m = li + 2;
    }
  }
  // the vertex count of createMoreVertexes's output, in double as the host counts it
  FQ_HD double count(double dist_max) const
  {
    double c = m;
    for (int j = 0; j + 1 < m; j++)
    {
      const double d = dist3(jin(j + 1), jin(j));
      if (d > dist_max) c = FQ_ADD(c, floor(FQ_DIV(d, dist_max)));
    }
    return c;
  }
  // writes the first min(count, cap) vertices to out; returns the count
  FQ_HD int write(double dist_max, double* out, int cap) const
  {
    int w = 0;
    auto emit = [&](const double* v) {
      if (w < cap) for (int k = 0; k < 3; k++) out[3 * (size_t)w + k] = v[k];
      w++;
    };
    for (int j = 0; j < m; j++)
    {
      const double* a = jin(j);
      emit(a);
      if (j + 1 == m) break;
      const double* b = jin(j + 1);
      double v[3];
      for (int k = 0; k < 3; k++) v[k] = FQ_SUB(b[k], a[k]);
      const double dist = FQ_SQRT(FQ_ADD(FQ_ADD(FQ_MUL(v[0], v[0]), FQ_MUL(v[1], v[1])), FQ_MUL(v[2], v[2])));
      if (!(dist > dist_max)) continue;
      const int add = (int)floor(FQ_DIV(dist, dist_max));
      for (int k = 0; k < 3; k++) v[k] = FQ_DIV(v[k], dist);             // (path[j + 1] - path[j]).normalized()
      double p[3] = { a[0], a[1], a[2] };
      for (int i = 0; i < add; i++)
      {
        for (int k = 0; k < 3; k++) p[k] = FQ_ADD(p[k], FQ_MUL(v[k], dist_max));
        emit(p);
      }
    }
    return w;
  }
};

// vertex counts of the outputs: deleteVertexes(path, max_poly) keeps max_poly + 1 vertices (utils.cpp:1117-1124); a
// corridor without paths (status != 0) gets one vertex of NaN
FQ_HD int whole_poly(const Crop& c, int n, int max_poly) { return c.status ? 0 : (n - 1 < max_poly ? n - 1 : max_poly); }
FQ_HD int safe_poly(const Crop& c, int max_poly)
{
  const int p = c.m + c.extra - 1;
  return c.status ? 0 : (p < max_poly ? p : max_poly);
}
// vertex i of the whole (JPS_in) or the safe (cropped) path of a corridor
FQ_HD void path_vertex(const Crop& c, bool safe, const double* in, int i, double* o)
{
  for (int k = 0; k < 3; k++) o[k] = c.status ? (double)NAN : (safe && i >= c.m ? c.e[k] : in[3 * i + k]);
}
}  // namespace fqpath
