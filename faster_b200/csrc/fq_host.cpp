// Host-side pieces of the hot path that need no GPU: plan tables, getDTInitial, resetX/fillX, sigma lists.
#include "fq_plan.h"
#include "fq_dtinit.h"
#include "fq_assign.h"
#include "fq_window.h"
#include "../../include/faster_b200.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

typedef long double ld;

namespace
{
// coefficient of ubar_s in (P,V,A) at knot t (s < t), k = t-1-s
inline ld cP(int k) { return (3.0L * k * k + 3.0L * k + 1.0L) / 6.0L; }
inline ld cV(int k) { return k + 0.5L; }

// functional y -> (row over ubar [N], free response on (P0,V0,A0) [3])
void functional(int N, int y, std::vector<ld>& c, ld f[3])
{
  c.assign(N, 0.0L);
  f[0] = f[1] = f[2] = 0.0L;
  auto addP = [&](int t, ld w) {
    for (int s = 0; s < t; s++) c[s] += w * cP(t - 1 - s);
    f[0] += w; f[1] += w * t; f[2] += w * (ld)t * t / 2.0L;
  };
  auto addV = [&](int t, ld w) {
    for (int s = 0; s < t; s++) c[s] += w * cV(t - 1 - s);
    f[1] += w; f[2] += w * t;
  };
  auto addA = [&](int t, ld w) {
    for (int s = 0; s < t; s++) c[s] += w;
    f[2] += w;
  };
  if (y <= N) addP(y, 1);
  else if (y < 2 * N + 1) addV(y - (N + 1), 1);
  else if (y < 3 * N + 1) addA(y - (2 * N + 1), 1);
  else if (y < 4 * N + 1) c[y - (3 * N + 1)] = 1;
  else if (y < 5 * N + 1) { int t = y - (4 * N + 1); addP(t, 1); addV(t, 1.0L / 3.0L); }
  else { int t = y - (5 * N + 1); addP(t, 1); addV(t, 2.0L / 3.0L); addA(t, 1.0L / 6.0L); }
}
}  // namespace

bool fq_build_plan(int N, int force_final, FqPlanHost* plan)
{
  const int ne = force_final ? 3 : 2;
  if (N < ne || N > FQ_MAX_N) return false;
  const int nz = N - ne, NY = 6 * N + 1;
  plan->N = N; plan->force_final = force_final; plan->ne = ne; plan->nz = nz; plan->NY = NY;

  // terminal rows at knot N
  std::vector<std::vector<ld>> C(ne, std::vector<ld>(N));
  std::vector<ld> FT(ne * 3, 0.0L);
  {
    int e = 0;
    if (force_final)
    {
      for (int s = 0; s < N; s++) C[e][s] = cP(N - 1 - s);
      FT[e * 3 + 0] = 1; FT[e * 3 + 1] = N; FT[e * 3 + 2] = (ld)N * N / 2.0L;
      e++;
    }
    for (int s = 0; s < N; s++) C[e][s] = cV(N - 1 - s);
    FT[e * 3 + 1] = 1; FT[e * 3 + 2] = N;
    e++;
    for (int s = 0; s < N; s++) C[e][s] = 1;
    FT[e * 3 + 2] = 1;
  }
  // Householder QR of C' (N x ne):  Q = H_0 H_1 .. H_{ne-1},  C' = Q [R; 0]
  std::vector<std::vector<ld>> A(N, std::vector<ld>(ne));
  for (int i = 0; i < N; i++)
    for (int e = 0; e < ne; e++) A[i][e] = C[e][i];
  std::vector<std::vector<ld>> Q(N, std::vector<ld>(N, 0.0L));
  for (int i = 0; i < N; i++) Q[i][i] = 1;
  for (int e = 0; e < ne; e++)
  {
    ld nrm = 0;
    for (int i = e; i < N; i++) nrm += A[i][e] * A[i][e];
    nrm = sqrtl(nrm);
    std::vector<ld> v(N, 0.0L);
    ld alpha = A[e][e] >= 0 ? -nrm : nrm;
    for (int i = e; i < N; i++) v[i] = A[i][e];
    v[e] -= alpha;
    ld vv = 0;
    for (int i = e; i < N; i++) vv += v[i] * v[i];
    if (vv == 0) continue;
    for (int c = 0; c < ne; c++)
    {
      ld s = 0;
      for (int i = e; i < N; i++) s += v[i] * A[i][c];
      s = 2 * s / vv;
      for (int i = e; i < N; i++) A[i][c] -= s * v[i];
    }
    for (int r = 0; r < N; r++)
    { // Q <- Q H
      ld s = 0;
      for (int i = e; i < N; i++) s += Q[r][i] * v[i];
      s = 2 * s / vv;
      for (int i = e; i < N; i++) Q[r][i] -= s * v[i];
    }
  }
  // Eplus = Q1 R^-T  (N x ne): minimum-norm solution of C ubar = rhs is Eplus rhs
  std::vector<std::vector<ld>> Ep(N, std::vector<ld>(ne, 0.0L));
  for (int i = 0; i < N; i++)
  { // solve R' x = e_k column by column: Ep[i][:] = Q1[i][:] R^-T  <=>  Ep R' = Q1
    // R' is lower triangular (ne x ne) with R'[a][b] = R[b][a] = A[b][a]
    for (int b = ne - 1; b >= 0; b--)
    {
      ld s = Q[i][b];
      for (int a = b + 1; a < ne; a++) s -= Ep[i][a] * A[b][a];
      Ep[i][b] = s / A[b][b];
    }
  }
  plan->TZ.assign((size_t)NY * std::max(nz, 1), 0.0);
  plan->T0.assign((size_t)NY * (3 + ne), 0.0);
  plan->FT.resize(ne * 3);
  for (int i = 0; i < ne * 3; i++) plan->FT[i] = (double)FT[i];
  std::vector<ld> c;
  for (int y = 0; y < NY; y++)
  {
    ld f[3];
    functional(N, y, c, f);
    ld nrm = 0, cn = 0;
    std::vector<ld> tz(nz, 0.0L);
    for (int m = 0; m < nz; m++)
    {
      ld s = 0;
      for (int i = 0; i < N; i++) s += c[i] * Q[i][ne + m];
      tz[m] = s; nrm += s * s;
    }
    for (int i = 0; i < N; i++) cn += c[i] * c[i];
    // rows that are pinned by the eliminated equalities (P_N when force_final) are exactly zero
    const bool zero = nrm <= 1e-24L * (cn > 1 ? cn : 1);
    for (int m = 0; m < nz; m++) plan->TZ[(size_t)y * nz + m] = zero ? 0.0 : (double)tz[m];
    for (int k = 0; k < 3; k++) plan->T0[(size_t)y * (3 + ne) + k] = (double)f[k];
    for (int e = 0; e < ne; e++)
    {
      ld s = 0;
      for (int i = 0; i < N; i++) s += c[i] * Ep[i][e];
      plan->T0[(size_t)y * (3 + ne) + 3 + e] = (double)s;
    }
  }
  return true;
}

// ---------------------------------------------------------------------------------------------------------
// getDTInitial (reference solverGurobi.cpp:659-759).  The reference mixes float temporaries with double
// arithmetic; the same conversions are made here.  Its roots come from Eigen's companion-matrix solver; here
// from closed forms refined by Newton steps, then rounded to float exactly as the reference's assignments do.
// ---------------------------------------------------------------------------------------------------------
extern "C" double fq_dt_initial(const double* x0, const double* xf, const double* lim, int N)
{
  return fqdt::dt_initial(x0, xf, lim, N);       // fq_dtinit.h: one source for host and device
}

extern "C" int fq_num_samples(int N, double dt, double DC) { return fqdt::num_samples(N, dt, DC); }

extern "C" void fq_fill_x(int N, const double* coeffs, double dt, double DC, int n_samples, double* out)
{ // fillX (:122-168): time accumulates by DC; the interval index advances by at most one per sample
  double t = 0;
  int interval = 0;
  for (int i = 0; i < n_samples; i++)
  {
    t = t + DC;
    if (t > dt * (interval + 1)) interval = std::min(interval + 1, N - 1);
    const double tau = t - interval * dt;
    fqdt::eval_sample(coeffs + 12 * interval, tau, out + (size_t)12 * i);
  }
  if (n_samples > 0)
    for (int k = 3; k < 12; k++) out[(size_t)12 * (n_samples - 1) + k] = 0.0;   // :165-167
}

extern "C" long fq_monotone_sigmas(int N, int P, uint8_t* out, long cap)
{
  if (N < 1 || P < 1 || N > FQ_MAX_N) return 0;
  std::vector<uint8_t> s(N, 0);
  long count = 0;
  for (;;)
  {
    if (out && count < cap) std::memcpy(out + (size_t)count * N, s.data(), N);
    count++;
    int i = N - 1;
    while (i >= 0 && s[i] == P - 1) i--;
    if (i < 0) break;
    uint8_t v = s[i] + 1;
    for (int j = i; j < N; j++) s[j] = v;
  }
  return count;
}

extern "C" long fq_pair_assign_count(int N, int P, long all_limit)
{
  if (N < 1 || N > FQ_MAX_N || P < 0 || P > FQ_MAX_POLY || all_limit < 0) return FQ_E_ARG;
  const long long n = fqa::list_len(N, P, all_limit);
  return n < 0 ? FQ_E_ARG : (long)n;
}

extern "C" long fq_pair_window_factors(double fi, double ff, double inc, double* out, long cap)
{
  const int n = fqw::factors(fi, ff, inc, out, (int)std::max(0L, std::min(cap, (long)fqw::kMaxFactors)));
  return n < 0 ? FQ_E_ARG : n;
}

extern "C" int fq_abi_version(void) { return FQ_ABI_VERSION; }

// Introspection for tests: copies the plan tables of (N, force_final).  Returns NY, or 0 if unsupported.
// Sizes: TZ NY*nz, T0 NY*(3+ne), FT ne*3 with ne = force_final ? 3 : 2, nz = N - ne, NY = 6N+1.
extern "C" int fq_plan_tables(int N, int force_final, double* TZ, double* T0, double* FT)
{
  FqPlanHost p;
  if (!fq_build_plan(N, force_final, &p)) return 0;
  if (TZ) std::memcpy(TZ, p.TZ.data(), sizeof(double) * (size_t)p.NY * p.nz);
  if (T0) std::memcpy(T0, p.T0.data(), sizeof(double) * p.T0.size());
  if (FT) std::memcpy(FT, p.FT.data(), sizeof(double) * p.FT.size());
  return p.NY;
}


// ---------------------------------------------------------------------------------------------------------
// Input validation scans used by the host-pointer entry points (fq_capi.cu).  Integer-only bodies so that they
// vectorise; compiled twice (AVX2 / baseline) with run-time dispatch -- a 65 536-candidate batch must not spend
// longer being validated than being copied.
// ---------------------------------------------------------------------------------------------------------
#if defined(__x86_64__) && defined(__GNUC__)
#define FQ_CLONES __attribute__((target_clones("avx2", "default")))
#else
#define FQ_CLONES
#endif

FQ_CLONES bool fq_scan_all_finite(const double* p, size_t n)
{
  if (!p) return n == 0;
  const uint64_t* w = reinterpret_cast<const uint64_t*>(p);
  uint64_t bad = 0;
  for (size_t i = 0; i < n; i++) bad |= (uint64_t)((w[i] & 0x7ff0000000000000ull) == 0x7ff0000000000000ull);
  return bad == 0;
}

FQ_CLONES bool fq_scan_all_positive_finite(const double* p, size_t n)
{
  if (!p) return n == 0;
  const uint64_t* w = reinterpret_cast<const uint64_t*>(p);
  uint64_t bad = 0;
  for (size_t i = 0; i < n; i++)
    bad |= (uint64_t)((w[i] & 0x7ff0000000000000ull) == 0x7ff0000000000000ull) | (w[i] >> 63) | (uint64_t)((w[i] << 1) == 0);
  return bad == 0;
}

FQ_CLONES int fq_scan_max_u8(const uint8_t* p, size_t n)
{
  uint8_t mx = 0;
  for (size_t i = 0; i < n; i++) mx = p[i] > mx ? p[i] : mx;
  return mx;
}
