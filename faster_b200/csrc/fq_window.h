// Per-corridor time-allocation windows of the chained replan (fq_replan_pairs_window*, include/faster_b200.h): ONE source
// for the host (fq_pair_window_factors, the host variant's validation and buffer sizes, the multi-GPU shards) and the
// device (fq_pair.cuh: the factor rows, the records' factors and the next windows).
//
// F(fi, ff, inc): the factors that genNewTraj's loop
//     for (double i = factor_initial_; i <= factor_final_; i = i + factor_increment_)       solverGurobi.cpp:445-446
// visits, in order.  They are accumulated exactly as that loop does (never fi + k * inc: with inc = 0.1 the two differ in
// count and in bits).  ff < fi gives the empty list (genNewTraj returns false with trials_ = 0).  Refused: fi, ff or inc not
// finite, fi <= 0, inc <= 0, more than kMaxFactors factors (the drop-in class's cap, include/solverGurobi.hpp:165), and an
// accumulation that stalls (i + inc == i), where the reference's loop would never end.
//
// Next window (faster.cpp:582-588), applied only when BOTH sweeps of the replan have a winner; otherwise Faster::replan
// returns before the update (:420-424, :529-533) and the window stays as it was:
//     init  = max(f* - gamma, 1.0)        final = f* + gammap
// appendToPlan's early return (:548) depends on the planner's plan_ deque: fq_replan_pairs_queue* keeps it on the device and
// gates the update on it (FqPairWindowArgs::gate); with the other families a caller whose plan could not be appended keeps
// its previous windows itself.
#pragma once
#include "fq_dtinit.h"

namespace fqw
{
static const int kMaxFactors = 4096;

FQ_HD bool finite(double x) { return fabs(x) <= 1.7976931348623157e308; }    // false for NaN and +-inf

// |F(fi, ff, inc)|, writing its first min(|F|, cap) factors to out (may be NULL); -1 when the window is refused
FQ_HD int factors(double fi, double ff, double inc, double* out, int cap)
{
  if (!finite(fi) || !finite(ff) || !finite(inc) || !(fi > 0) || !(inc > 0)) return -1;
  int n = 0;
  for (double i = fi; i <= ff;)
  {
    if (n == kMaxFactors) return -1;
    if (out && n < cap) out[n] = i;
    n++;
    const double next = FQ_ADD(i, inc);
    if (next == i) return -1;
    i = next;
  }
  return n;
}

// the window of the next replan: (init, final) from the winning factor f_star when both sweeps won, else unchanged
FQ_HD void next_window(bool both_won, double f_star, double gamma, double gammap, double init, double final_, double* next_init,
                       double* next_final)
{
  if (!both_won)
  {
    *next_init = init;
    *next_final = final_;
    return;
  }
  const double lo = FQ_SUB(f_star, gamma);
  *next_init = lo < 1.0 ? 1.0 : lo;                             // std::max(f* - gamma, 1.0)
  *next_final = FQ_ADD(f_star, gammap);
}
}  // namespace fqw
