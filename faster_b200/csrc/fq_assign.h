// Per-corridor interval -> polytope assignment lists of the chained replan (fq_replan_pairs_assign*, include/faster_b200.h):
// ONE source for the host (fq_pair_assign_count, the host variant's buffer sizes, the multi-GPU shards) and the device
// (fq_pair.cuh: the offsets and the unranking grid expansion).
//
// L(N, P, all_limit) of a corridor with P polytopes and a sweep of N segments:
//   P = 0                  the single all-zero assignment (no corridor rows: fq_gen_new_traj with P = 0)
//   P^N <= all_limit       all P^N assignments, lexicographic with segment 0 most significant (base-P digits; the order
//                          in which SolverGurobi::ensureAssignments enumerates ALL)
//   otherwise              the non-decreasing assignments in lexicographic order (fq_monotone_sigmas), C(N+P-1, N)
// Lists longer than 2^20 are refused.
#pragma once
#include "fq_dtinit.h"

#include <stdint.h>

namespace fqa
{
static const long long kMaxList = 1LL << 20;

// C(n, k) for n <= FQ_MAX_N + FQ_MAX_POLY - 1 = 47, k <= 16: at most C(47, 16) ~ 1.4e12, exact in 64 bits
FQ_HD long long binom(int n, int k)
{
  if (k < 0 || k > n) return 0;
  if (k > n - k) k = n - k;
  long long r = 1;
  for (int i = 0; i < k; i++) r = r * (n - i) / (i + 1);   // exact: r * (n - i) is divisible by i + 1 at every step
  return r;
}

// all_limit >= 0: does the corridor enumerate every assignment (P^N <= all_limit)?
FQ_HD bool use_all(int N, int P, long long all_limit)
{
  if (P <= 1) return false;                                 // 0 and 1 polytopes: one assignment either way
  long long pw = 1;
  for (int t = 0; t < N; t++)
  {
    if (pw > all_limit / P) return false;                   // pw * P > all_limit
    pw *= P;
  }
  return true;
}

// |L(N, P, all_limit)|, or -1 when it is longer than 2^20
FQ_HD long long list_len(int N, int P, long long all_limit)
{
  if (P <= 0) return 1;
  long long n;
  if (use_all(N, P, all_limit))
  {
    n = 1;
    for (int t = 0; t < N; t++) n *= P;
  }
  else
    n = binom(N + P - 1, N);
  return n <= kMaxList ? n : -1;
}

// assignment number `idx` of L(N, P, all_limit) into out[0 .. N-1].  binom_tab (may be NULL): C(n, k) at [n * 17 + k]
// for n < 48, k <= 16 (fq_pair.cuh keeps it in shared memory)
FQ_HD void unrank(int N, int P, bool all, long long idx, const long long* binom_tab, uint8_t* out)
{
  if (P <= 0)
  {
    for (int t = 0; t < N; t++) out[t] = 0;
    return;
  }
  if (all)
  { // base-P digits, segment 0 most significant
    for (int t = N - 1; t >= 0; t--) { out[t] = (uint8_t)(idx % P); idx /= P; }
    return;
  }
  // non-decreasing sequences in lexicographic order: at segment t with lower bound v, the sequences that put value c at t
  // number C(m + (P - c) - 1, m) with m = N - t - 1 segments left (non-decreasing over the P - c values c .. P-1)
  int v = 0;
  for (int t = 0; t < N; t++)
  {
    const int m = N - t - 1;
    for (int c = v; c < P; c++)
    {
      const int n = m + (P - c) - 1;
      const long long cnt = binom_tab ? binom_tab[n * 17 + m] : binom(n, m);
      if (idx < cnt) { v = c; break; }
      idx -= cnt;
    }
    out[t] = (uint8_t)v;
  }
}

// the index of s[0 .. N-1] in L(N, P, all_limit) (the inverse of unrank), or -1 when s is not in the list
FQ_HD long long rank(int N, int P, bool all, const uint8_t* s)
{
  long long idx = 0;
  if (P <= 0)
  {
    for (int t = 0; t < N; t++)
      if (s[t] != 0) return -1;
    return 0;
  }
  if (all)
  {
    for (int t = 0; t < N; t++)
    {
      if (s[t] >= P) return -1;
      idx = idx * P + s[t];
    }
    return idx;
  }
  int v = 0;
  for (int t = 0; t < N; t++)
  {
    if (s[t] < v || s[t] >= P) return -1;
    const int m = N - t - 1;
    for (int c = v; c < s[t]; c++) idx += binom(m + (P - c) - 1, m);
    v = s[t];
  }
  return idx;
}
}  // namespace fqa
