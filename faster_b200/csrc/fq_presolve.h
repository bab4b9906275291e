// Presolve of the exact MIQP sweep (branch-and-bound over assignments, fq_bnb.cuh): ONE source for the host
// (fq_gen_new_traj_exact) and the device (the chained replan's roots kernel, fq_pair.cuh), so the two cannot drift.
//
// Segment 0 starts with three control points fixed by (x0, dt): cp0 = p0, cp1 = p0 + v0 dt / 3, cp2 = p0 + 2 v0 dt / 3 +
// a0 dt^2 / 6; with the final position pinned, the last control point is xf.  A time allocation for which no polytope holds
// all three of cp0..cp2 (or none holds xf) is infeasible for EVERY assignment and needs no tree; without the test such
// corridors make the tree explore every prefix.  A point is inside polytope p when every row satisfies
// a . x - b <= tol.  Products and sums are rounded one by one (FQ_MUL / FQ_ADD), so host and device agree bit for bit.
#pragma once
#include "fq_dtinit.h"

namespace fqs
{
// is pt inside the polytope of rows f0 .. f1-1 of Ab ([ax ay az b] per row)?
FQ_HD bool inside(const double* Ab, int f0, int f1, const double* pt, double tol)
{
  for (int f = f0; f < f1; f++)
  {
    const double* r = Ab + 4 * (size_t)f;
    const double s = FQ_SUB(FQ_ADD(FQ_ADD(FQ_MUL(r[0], pt[0]), FQ_MUL(r[1], pt[1])), FQ_MUL(r[2], pt[2])), r[3]);
    if (!(s <= tol)) return false;
  }
  return true;
}

// control point kk (0, 1, 2) of segment 0 for time allocation t
FQ_HD void start_point(const double* x0, double t, int kk, double* pt)
{
  for (int ax = 0; ax < 3; ax++)
  {
    double v = x0[ax];
    if (kk >= 1) v = FQ_ADD(v, FQ_MUL(FQ_MUL(x0[3 + ax], t), kk == 1 ? 1.0 / 3.0 : 2.0 / 3.0));
    if (kk == 2) v = FQ_ADD(v, FQ_DIV(FQ_MUL(FQ_MUL(x0[6 + ax], t), t), 6.0));
    pt[ax] = v;
  }
}

// can any assignment be feasible at time allocation t?  P polytopes, polytope p = rows face_ofs[p] .. face_ofs[p+1]-1.
FQ_HD bool root_possible(int P, const int* face_ofs, const double* Ab, const double* x0, const double* xf, int force_final,
                         double t, double tol)
{
  if (force_final)
  {
    bool any = false;
    for (int p = 0; p < P && !any; p++) any = inside(Ab, face_ofs[p], face_ofs[p + 1], xf, tol);
    if (!any) return false;
  }
  for (int p = 0; p < P; p++)
  {
    bool in = true;
    for (int kk = 0; kk < 3 && in; kk++)
    {
      double pt[3];
      start_point(x0, t, kk, pt);
      in = inside(Ab, face_ofs[p], face_ofs[p + 1], pt, tol);
    }
    if (in) return true;
  }
  return false;
}
}  // namespace fqs
