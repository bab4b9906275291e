// The committed plan of one planner (Faster::plan_, faster.hpp:70) as a ring row: ONE source for the host entries
// fq_queue_* (fq_pair_capi.cu) and the device (fq_pair.cuh: the select, pop and reset kernels and the chain's append).
//
// A row is `cap` states of 12 doubles in fq_fill_x's layout (pos vel accel jerk); its i-th state (0 = front) is at slot
// (head + i) % cap, and it holds `size` states.  A row whose head is outside 0 .. cap-1 or whose size is outside 0 .. cap
// is not a ring (ring_ok): the host entries refuse it and the device treats it as a row it may not touch.
#pragma once
#include "fq_dtinit.h"
#include "../../include/faster_b200.h"

namespace fqq
{
static const int kState = 12;

FQ_HD bool ring_ok(int head, int size, int cap) { return head >= 0 && head < cap && size >= 0 && size <= cap; }

// the slot of the row's i-th state
FQ_HD long long slot(int head, long long i, int cap) { return ((long long)head + i) % cap; }

FQ_HD double qnan()
{
#if defined(__CUDA_ARCH__)
  return __longlong_as_double(0x7ff8000000000000ll);
#else
  return NAN;
#endif
}

// updateState's first push (faster.cpp:253-266): the row becomes one state holding only pos
FQ_HD void reset(double* row, int* head, int* size, const double* pos)
{
  for (int q = 0; q < kState; q++) row[q] = q < 3 ? pos[q] : 0.0;
  *head = 0;
  *size = 1;
}

// faster.cpp:350-352: k_end_whole = max(size - deltaT_, 0) and A = plan_[size - 1 - k_end_whole] (pos, vel, accel to
// x0).  An empty row returns -1 and a NaN x0.
FQ_HD int select(const double* row, int head, int size, int cap, int delta_t, double* x0)
{
  if (size < 1)
  {
    for (int q = 0; q < 9; q++) x0[q] = qnan();
    return -1;
  }
  const int k = size - delta_t > 0 ? size - delta_t : 0;
  const double* A = row + kState * slot(head, size - 1 - k, cap);
  for (int q = 0; q < 9; q++) x0[q] = A[q];
  return k;
}

// getNextGoal (faster.cpp:699-723) `ticks` times: goal t = the front, then pop while more than one state is left.  An
// empty row publishes NaN states.
FQ_HD void pop(const double* row, int* head, int* size, int cap, int ticks, double* goals)
{
  for (int t = 0; t < ticks; t++)
  {
    double* g = goals + kState * (size_t)t;
    const double* f = row + kState * (size_t)*head;
    for (int q = 0; q < kState; q++) g[q] = *size > 0 ? f[q] : qnan();
    if (*size > 1)
    {
      *head = *head + 1 == cap ? 0 : *head + 1;
      *size = *size - 1;
    }
  }
}

// appendToPlan's decision (faster.cpp:606-648) for a piece of `rows` states (0: the replan appends nothing) on a row of
// `size` states, with k_end from the select before the replan (-1: none): FQ_QUEUE_*.  On FQ_QUEUE_OK, *keep is the
// number of states left after erasing the last k_end + 1, and the piece goes to states keep .. keep + rows - 1.
FQ_HD int append_status(int size, int cap, int k_end, long long rows, long long* keep)
{
  if (rows <= 0 || k_end < 0) return FQ_QUEUE_NONE;
  if (size - 1 - k_end < 0) return FQ_QUEUE_PUBLISHED;           // "Already publised the point A"
  const long long kept = (long long)size - 1 - k_end;
  if (kept + rows > cap) return FQ_QUEUE_CAPACITY;
  *keep = kept;
  return FQ_QUEUE_OK;
}

// faster.cpp:563-572: GOAL_SEEN when |G_term - plan_.back().pos| < goal_radius (the norm as ((dx^2 + dy^2) + dz^2))
FQ_HD bool goal_seen(const double* last, const double* G, double goal_radius)
{
  const double dx = FQ_SUB(G[0], last[0]), dy = FQ_SUB(G[1], last[1]), dz = FQ_SUB(G[2], last[2]);
  return FQ_SQRT(FQ_ADD(FQ_ADD(FQ_MUL(dx, dx), FQ_MUL(dy, dy)), FQ_MUL(dz, dz))) < goal_radius;
}
}  // namespace fqq
