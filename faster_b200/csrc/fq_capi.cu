// C ABI of faster_b200 (see include/faster_b200.h): context, plan cache, host<->device staging, launches.
#include "fq_ctx.h"

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

std::string g_create_error;

int fq_fail(fq_ctx* c, int code, const std::string& msg)
{
  if (c) c->err = msg; else g_create_error = msg;
  return code;
}
int fq_cuda_fail(fq_ctx* c, cudaError_t e, const char* what)
{
  return fq_fail(c, FQ_E_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

int fq_get_plan(fq_ctx* ctx, int N, int force_final, FqPlanDev** out)
{
  const int key = N * 2 + (force_final ? 1 : 0);
  auto it = ctx->plans.find(key);
  if (it == ctx->plans.end())
  {
    FqPlanDev pd;
    if (!fq_build_plan(N, force_final ? 1 : 0, &pd.h))
      return fq_fail(ctx, FQ_E_ARG, "unsupported N (need ne <= N <= FQ_MAX_N)");
    FQ_CUDA(cudaMalloc(&pd.TZ, sizeof(double) * (pd.h.TZ.size() + 1)));
    FQ_CUDA(cudaMalloc(&pd.T0, sizeof(double) * pd.h.T0.size()));
    FQ_CUDA(cudaMalloc(&pd.FT, sizeof(double) * pd.h.FT.size()));
    FQ_CUDA(cudaMemcpy(pd.TZ, pd.h.TZ.data(), sizeof(double) * pd.h.TZ.size(), cudaMemcpyHostToDevice));
    FQ_CUDA(cudaMemcpy(pd.T0, pd.h.T0.data(), sizeof(double) * pd.h.T0.size(), cudaMemcpyHostToDevice));
    FQ_CUDA(cudaMemcpy(pd.FT, pd.h.FT.data(), sizeof(double) * pd.h.FT.size(), cudaMemcpyHostToDevice));
    it = ctx->plans.emplace(key, pd).first;
  }
  *out = &it->second;
  return 0;
}

void fq_fill_plan_args(const FqPlanDev& pd, FqKernelArgs* a)
{
  a->N = pd.h.N; a->force_final = pd.h.force_final; a->ne = pd.h.ne; a->nz = pd.h.nz;
  a->nw = 3 * pd.h.nz; a->NY = pd.h.NY; a->ld = (3 * pd.h.nz) | 1;
  a->TZ = pd.TZ; a->T0 = pd.T0; a->FT = pd.FT;
}

const char* fq_scan_corridors(int n_prob, const int* poly_ofs, const int* face_ofs, FqCorridorSizes* sizes)
{
  *sizes = FqCorridorSizes();
  for (int j = 0; j < n_prob; j++)
  {
    const int P = poly_ofs[j + 1] - poly_ofs[j];
    if (P < 0 || P > FQ_MAX_POLY) return "polytope count out of range (0..FQ_MAX_POLY)";
    for (int p = poly_ofs[j]; p < poly_ofs[j + 1]; p++)
    {
      if (face_ofs[p + 1] < face_ofs[p]) return "face_ofs not monotone";
      sizes->max_poly_faces = std::max(sizes->max_poly_faces, face_ofs[p + 1] - face_ofs[p]);
    }
    sizes->max_faces = std::max(sizes->max_faces, face_ofs[poly_ofs[j + 1]] - face_ofs[poly_ofs[j]]);
  }
  sizes->n_poly = poly_ofs[n_prob];
  sizes->n_face = face_ofs[sizes->n_poly];
  return nullptr;
}

extern "C" int fq_create(fq_ctx** out, int device)
{
  if (!out) return fq_fail(nullptr, FQ_E_ARG, "out is NULL");
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0)
    return fq_fail(nullptr, FQ_E_NOGPU, std::string("no CUDA device: ") + (e != cudaSuccess ? cudaGetErrorString(e) : "count 0") +
                                            " (faster_b200 has no CPU fallback)");
  if (device < 0 || device >= n) return fq_fail(nullptr, FQ_E_ARG, "device index out of range");
  fq_ctx* ctx = new (std::nothrow) fq_ctx();
  if (!ctx) return fq_fail(nullptr, FQ_E_NOMEM, "out of host memory");
  ctx->device = device;
  e = cudaSetDevice(device);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->stream2, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->ev_head, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device);
  ctx->counters_cap = 4096;
  if (e == cudaSuccess) e = cudaMalloc(&ctx->d_counters, sizeof(int) * (size_t)kFqCounterSlots * ctx->counters_cap);
  if (e != cudaSuccess)
  {
    std::string msg = std::string("cuda init: ") + cudaGetErrorString(e);
    delete ctx;
    return fq_fail(nullptr, FQ_E_CUDA, msg);
  }
  *out = ctx;
  return 0;
}

extern "C" void fq_destroy(fq_ctx* ctx)
{
  if (!ctx) return;
  fq_comm_release(ctx);                            // NCCL communicator(s), if any (fq_multi.cu)
  for (fq_ctx* p : ctx->peers) fq_destroy(p);      // fq_create_multi: the other devices' contexts
  ctx->peers.clear();
  cudaSetDevice(ctx->device);
  for (auto& kv : ctx->plans) { cudaFree(kv.second.TZ); cudaFree(kv.second.T0); cudaFree(kv.second.FT); }
  ctx->d_in.release(); ctx->d_out.release(); ctx->d_bnb.release(); ctx->d_pair.release(); ctx->d_pair_io.release();
  ctx->h_in.release(); ctx->h_out.release();
  if (ctx->d_counters) cudaFree(ctx->d_counters);
  if (ctx->d_first) cudaFree(ctx->d_first);
  if (ctx->ev_head) cudaEventDestroy(ctx->ev_head);
  if (ctx->stream2) cudaStreamDestroy(ctx->stream2);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

extern "C" int fq_set_option(fq_ctx* ctx, const char* key, int value)
{
  if (!ctx || !key) return FQ_E_ARG;
  for (fq_ctx* p : ctx->peers)                     // a multi-GPU group: every member gets the option
    if (int rc = fq_set_option(p, key, value)) { ctx->err = p->err; return rc; }
  if (std::string(key) == "force_generic_kernel") { ctx->force_generic = value != 0; return 0; }
  if (std::string(key) == "throughput_slices") { ctx->throughput_slices = value > 0 && value <= 64 ? value : 0; return 0; }
  if (std::string(key) == "max_faces_per_polytope") { ctx->max_poly_faces_hint = value > 0 ? value : 0; return 0; }
  if (std::string(key) == "cert_memo") return 0;   // accepted and ignored: the GPU kernels have no certificate memo
  if (std::string(key) == "sweep_early_exit") { ctx->early_exit = value != 0; return 0; }
  if (std::string(key) == "row_tol_1e9")
  { // row tolerance in units of 1e-9 (10 = the default 1e-8, 1000 = Gurobi's default FeasibilityTol 1e-6).  0 is refused:
    // a row just made active can still be violated by rounding, is picked again and the active set cycles to the
    // iteration cap; 1e-9 is also the lowest FeasibilityTol Gurobi accepts
    if (value < 1 || value > 1000000) return fq_fail(ctx, FQ_E_ARG, "row_tol_1e9 out of range (1..1000000, i.e. 1e-9 to 1e-3)");
    ctx->row_tol = 1e-9 * (double)value;
    return 0;
  }
  return fq_fail(ctx, FQ_E_ARG, std::string("unknown option ") + key);
}

extern "C" int fq_has_feature(const char* name)
{
  if (!name) return 0;
  const std::string n(name);
  if (n == "sweep_early_exit" || n == "replan_pairs" || n == "multi_gpu" || n == "row_tol" || n == "certificates") return 1;
  return 0;
}

extern "C" const char* fq_last_error(const fq_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int fq_launch_solve_ctx(fq_ctx* ctx, FqKernelArgs a, int max_cand, int max_poly_faces, cudaStream_t stream, bool* tail,
                        bool early_exit_ok)
{
  if (tail) *tail = false;
  FqPlanDev* pd = nullptr;
  if (int rc = fq_get_plan(ctx, a.N, a.force_final, &pd)) return rc;
  fq_fill_plan_args(*pd, &a);
  if (a.max_faces <= 0) a.max_faces = 1;
  a.item_cap = a.N * (max_poly_faces > 0 && max_poly_faces <= a.max_faces ? max_poly_faces : a.max_faces);
  a.row_tol = ctx->row_tol;
  if (fq_solve_smem_bytes(a) > 227 * 1024)
    return fq_fail(ctx, FQ_E_ARG, "problem too large for shared memory (N / faces per problem)");
  const int n_prob = a.n_prob;
  if (n_prob > ctx->counters_cap)
  { // rare: grow the counter ring (needs the device idle because earlier launches may still use the old one)
    FQ_CUDA(cudaDeviceSynchronize());
    cudaFree(ctx->d_counters);
    ctx->d_counters = nullptr;
    if (ctx->d_first) { cudaFree(ctx->d_first); ctx->d_first = nullptr; }
    ctx->counters_cap = n_prob + n_prob / 2;
    FQ_CUDA(cudaMalloc(&ctx->d_counters, sizeof(int) * (size_t)kFqCounterSlots * ctx->counters_cap));
  }
  const unsigned slot = ctx->counters_pos++ % kFqCounterSlots;
  int* counters = ctx->d_counters + (size_t)slot * ctx->counters_cap;
  if (ctx->early_exit && early_exit_ok && max_cand > 1)
  {
    if (!ctx->d_first) FQ_CUDA(cudaMalloc(&ctx->d_first, sizeof(unsigned long long) * (size_t)kFqCounterSlots * ctx->counters_cap));
    a.first_feasible = ctx->d_first + (size_t)slot * ctx->counters_cap;
    FQ_CUDA(cudaMemsetAsync(a.first_feasible, 0xff, sizeof(unsigned long long) * (size_t)n_prob, stream));
  }
  const bool generic = ctx->force_generic || a.cert != nullptr;
  // the selection in the tail needs the specialised kernel, one problem and the coefficients of every candidate
  a.sweep_done = a.sweep_n_sigma > 0 && n_prob == 1 && a.coeffs && !generic ? counters + n_prob : nullptr;
  if (!a.sweep_done) { a.sweep_n_sigma = 0; a.sweep_idx = nullptr; a.sweep_win = nullptr; }
  bool spec = false;
  FQ_CUDA(fq_launch_solve(a, max_cand, stream, counters, ctx->sm_count, generic, &spec));
  if (tail) *tail = spec && a.sweep_done != nullptr;
  return 0;
}

extern "C" int fq_solve_multi_dev(fq_ctx* ctx, int N, int force_final, int n_prob, const double* d_x0,
                                  const double* d_xf, const double* d_lim, const int* d_poly_ofs,
                                  const int* d_face_ofs, const double* d_Ab, const int* d_cand_ofs,
                                  int max_cand_per_prob, int max_faces_per_prob, const double* d_dt,
                                  const uint8_t* d_sigma, uint8_t* d_feasible, double* d_cost, double* d_coeffs,
                                  int32_t* d_iters, void* stream)
{
  if (!ctx) return FQ_E_ARG;
  if (n_prob < 0 || max_cand_per_prob < 0) return fq_fail(ctx, FQ_E_ARG, "negative count");
  if (n_prob == 0 || max_cand_per_prob == 0) return 0;
  if (((uintptr_t)d_Ab & 15) != 0) return fq_fail(ctx, FQ_E_ARG, "Ab must be 16-byte aligned");
  FQ_CUDA(cudaSetDevice(ctx->device));
  FqKernelArgs a{};
  a.N = N; a.force_final = force_final; a.n_prob = n_prob; a.x0 = d_x0; a.xf = d_xf; a.lim = d_lim;
  a.poly_ofs = d_poly_ofs; a.face_ofs = d_face_ofs; a.Ab = d_Ab; a.max_faces = max_faces_per_prob;
  a.cand_ofs = d_cand_ofs; a.dt = d_dt; a.sigma = d_sigma;
  a.feasible = d_feasible; a.cost = d_cost; a.coeffs = d_coeffs; a.iters = d_iters;
  return fq_launch_solve_ctx(ctx, a, max_cand_per_prob, ctx->max_poly_faces_hint, stream ? (cudaStream_t)stream : ctx->stream);
}

int fq_settle(fq_ctx* ctx)
{
  for (fq_ctx* p : ctx->peers)                     // a multi-GPU group settles every member
    if (int rc = fq_settle(p)) { ctx->err = p->err; return rc; }
  if (!ctx->pending) return 0;
  ctx->pending = false;
  FQ_CUDA(cudaSetDevice(ctx->device));
  FQ_CUDA(cudaStreamSynchronize(ctx->stream2));
  FQ_CUDA(cudaStreamSynchronize(ctx->stream));
  return 0;
}

namespace
{
struct HostLayout
{ // byte offsets of each array inside the input / output arenas
  size_t x0, xf, lim, dt, Ab, poly_ofs, face_ofs, cand_ofs, sigma, in_bytes;
  size_t cost, coeffs, iters, feasible, win_cost, win_dt, win_idx, win_ofs, out_bytes;
};

// validates the host description and computes sizes
int describe(fq_ctx* ctx, int N, int force_final, int n_prob, const int* poly_ofs, const int* face_ofs,
             const int* cand_ofs, const uint8_t* sigma, bool want_coeffs, bool want_iters, HostLayout* L,
             FqCorridorSizes* cs, int* n_cand, int* max_cand)
{
  const int ne = force_final ? 3 : 2;
  if (N < ne || N > FQ_MAX_N) return fq_fail(ctx, FQ_E_ARG, "N out of range");
  if (n_prob <= 0) return fq_fail(ctx, FQ_E_ARG, "n_prob <= 0");
  if (poly_ofs[0] != 0 || cand_ofs[0] != 0 || face_ofs[0] != 0) return fq_fail(ctx, FQ_E_ARG, "offset arrays must start at 0");
  if (const char* why = fq_scan_corridors(n_prob, poly_ofs, face_ofs, cs)) return fq_fail(ctx, FQ_E_ARG, why);
  *max_cand = 0;
  for (int j = 0; j < n_prob; j++)
  {
    const int P = poly_ofs[j + 1] - poly_ofs[j], nc = cand_ofs[j + 1] - cand_ofs[j];
    if (nc < 0) return fq_fail(ctx, FQ_E_ARG, "cand_ofs not monotone");
    if (P > 0 && sigma)
    { // branch-free max over the bytes (vectorises); one compare per problem
      if (fq_scan_max_u8(sigma + (size_t)cand_ofs[j] * N, (size_t)nc * N) >= P)
        return fq_fail(ctx, FQ_E_ARG, "sigma entry >= number of polytopes");
    }
    if (nc > *max_cand) *max_cand = nc;
  }
  *n_cand = cand_ofs[n_prob];
  size_t o = 0;
  L->Ab = o;        o = fq_align16(o + sizeof(double) * 4 * (size_t)(cs->n_face > 0 ? cs->n_face : 1));
  L->x0 = o;        o += sizeof(double) * 9 * (size_t)n_prob;
  L->xf = o;        o += sizeof(double) * 9 * (size_t)n_prob;
  L->lim = o;       o += sizeof(double) * 3 * (size_t)n_prob;
  L->poly_ofs = o;  o += sizeof(int) * (size_t)(n_prob + 1);
  L->face_ofs = o;  o += sizeof(int) * (size_t)(cs->n_poly + 1);
  L->cand_ofs = o;  o = fq_align16(o + sizeof(int) * (size_t)(n_prob + 1));
  L->dt = o;        o += sizeof(double) * (size_t)*n_cand;      // per-candidate arrays last: [0, dt) is the
  L->sigma = o;     o += (size_t)*n_cand * N;                   // per-problem description
  L->in_bytes = fq_align16(o);
  o = 0;
  L->cost = o;      o += sizeof(double) * (size_t)*n_cand;
  L->win_cost = o;  o += sizeof(double) * (size_t)n_prob;       // per-problem winners (fq_solve_multi_sharded)
  L->win_dt = o;    o += sizeof(double) * (size_t)n_prob;
  L->coeffs = o;    o += want_coeffs ? sizeof(double) * 12 * (size_t)N * (size_t)*n_cand : 0;
  L->iters = o;     o += want_iters ? sizeof(int32_t) * (size_t)*n_cand : 0;
  L->win_idx = o;   o += sizeof(int) * (size_t)n_prob;
  L->win_ofs = o;   o += sizeof(int) * (size_t)(n_prob + 1);
  L->feasible = o;  o += (size_t)*n_cand;
  L->out_bytes = fq_align16(o);
  return 0;
}

constexpr size_t kPackThreshold = 512 * 1024;   // below this, inputs are packed into one pinned staging copy

struct Trace
{ // FQ_TRACE=1: host-side phase times of fq_solve_multi on stderr
  bool on;
  std::chrono::steady_clock::time_point t0;
  Trace() : on(std::getenv("FQ_TRACE") != nullptr), t0(std::chrono::steady_clock::now()) {}
  void mark(const char* what)
  {
    if (!on) return;
    const auto t1 = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[fq trace] %-10s %8.1f us\n", what, std::chrono::duration<double, std::micro>(t1 - t0).count());
    t0 = t1;
  }
};

// deferred: return once everything is enqueued (large batches only; small ones complete before returning either way).
// cert (device, cert_stride doubles per candidate): fq_solve_batch_cert's certificate buffer, or nullptr
int solve_multi_impl(fq_ctx* ctx, int N, int force_final, int n_prob, const double* x0, const double* xf,
                     const double* lim, const int* poly_ofs, const int* face_ofs, const double* Ab,
                     const int* cand_ofs, const double* dt, const uint8_t* sigma, uint8_t* feasible,
                     double* cost, double* coeffs, int32_t* iters, bool deferred, HostLayout* L_out = nullptr,
                     double* cert = nullptr, int cert_stride = 0)
{
  if (!ctx) return FQ_E_ARG;
  if (int src = fq_settle(ctx)) return src;
  Trace tr;
  if (!x0 || !xf || !lim || !poly_ofs || !face_ofs || !cand_ofs || !dt || !feasible || !cost)
    return fq_fail(ctx, FQ_E_ARG, "NULL argument");
  HostLayout L;
  FqCorridorSizes cs;
  int n_cand, max_cand;
  int rc = describe(ctx, N, force_final, n_prob, poly_ofs, face_ofs, cand_ofs, sigma, coeffs != nullptr,
                    iters != nullptr, &L, &cs, &n_cand, &max_cand);
  if (rc) return rc;
  if (L_out) *L_out = L;
  tr.mark("describe");
  if (n_cand == 0) return 0;
  const int n_poly = cs.n_poly;
  if (n_poly > 0 && (!Ab || !sigma)) return fq_fail(ctx, FQ_E_ARG, "polytopes given but Ab or sigma is NULL");
  // value checks (the kernels also refuse non-finite data, but an argument error is the better answer).  Small batches:
  // before anything is enqueued.  Large batches: while the GPU already works on the data (see the throughput path).
  auto values_ok = [&]() -> const char* {
    if (!fq_scan_all_finite(x0, 9 * (size_t)n_prob) || !fq_scan_all_finite(xf, 9 * (size_t)n_prob) ||
        !fq_scan_all_finite(Ab, 4 * (size_t)cs.n_face))
      return "non-finite value in x0/xf/Ab";
    if (!fq_scan_all_positive_finite(dt, (size_t)n_cand)) return "dt must be finite and > 0";
    if (!fq_scan_all_positive_finite(lim, 3 * (size_t)n_prob)) return "limits must be finite and > 0";
    return nullptr;
  };
  const bool big = L.in_bytes > kPackThreshold;
  if (!big)
    if (const char* why = values_ok()) return fq_fail(ctx, FQ_E_ARG, why);
  FQ_CUDA(cudaSetDevice(ctx->device));
  FQ_CUDA(ctx->d_in.reserve(L.in_bytes));
  FQ_CUDA(ctx->d_out.reserve(L.out_bytes));
  char* din = (char*)ctx->d_in.p;
  char* dout = (char*)ctx->d_out.p;
  FqKernelArgs a{};      // the whole batch; a slice of it offsets the per-problem pointers
  a.N = N; a.force_final = force_final; a.n_prob = n_prob;
  a.x0 = (const double*)(din + L.x0); a.xf = (const double*)(din + L.xf); a.lim = (const double*)(din + L.lim);
  a.poly_ofs = (const int*)(din + L.poly_ofs); a.face_ofs = (const int*)(din + L.face_ofs); a.Ab = (const double*)(din + L.Ab);
  a.max_faces = cs.max_faces; a.cand_ofs = (const int*)(din + L.cand_ofs); a.dt = (const double*)(din + L.dt);
  a.sigma = (const uint8_t*)(din + L.sigma); a.feasible = (uint8_t*)(dout + L.feasible); a.cost = (double*)(dout + L.cost);
  a.coeffs = coeffs ? (double*)(dout + L.coeffs) : nullptr; a.iters = iters ? (int32_t*)(dout + L.iters) : nullptr;
  a.cert = cert; a.cert_stride = cert_stride;
  cudaStream_t st = ctx->stream;
  const size_t sig_bytes = (size_t)n_cand * N;
  struct Piece { size_t off; const void* src; size_t bytes; };
  const Piece pieces[] = {
    { L.Ab, Ab, sizeof(double) * 4 * (size_t)cs.n_face }, { L.x0, x0, sizeof(double) * 9 * (size_t)n_prob },
    { L.xf, xf, sizeof(double) * 9 * (size_t)n_prob }, { L.lim, lim, sizeof(double) * 3 * (size_t)n_prob },
    { L.dt, dt, sizeof(double) * (size_t)n_cand },     { L.poly_ofs, poly_ofs, sizeof(int) * (size_t)(n_prob + 1) },
    { L.face_ofs, face_ofs, sizeof(int) * (size_t)(n_poly + 1) },
    { L.cand_ofs, cand_ofs, sizeof(int) * (size_t)(n_prob + 1) }, { L.sigma, sigma, n_poly > 0 ? sig_bytes : 0 },
  };
  if (L.in_bytes <= kPackThreshold)
  { // latency path: one pinned staging buffer, one H2D copy
    FQ_CUDA(ctx->h_in.reserve(L.in_bytes));
    for (const Piece& p : pieces)
      if (p.bytes) std::memcpy((char*)ctx->h_in.p + p.off, p.src, p.bytes);
    FQ_CUDA(cudaMemcpyAsync(din, ctx->h_in.p, L.in_bytes, cudaMemcpyHostToDevice, st));
  }
  else
  { // throughput path: the per-problem description is small and goes through one staged copy; the per-candidate arrays
    // (dt, sigma) are DMA'd straight from the caller's buffers (true async when they are pinned) in up to four slices
    // of whole problems, alternating between two streams: slice k+1 uploads while slice k computes and slice k-1
    // downloads, and the next slice's CTAs fill the SMs that the previous launch's tail leaves idle.
    const bool pack_head = L.dt <= kPackThreshold;
    if (pack_head) FQ_CUDA(ctx->h_in.reserve(L.dt));
    for (const Piece& p : pieces)
    {
      if (!p.bytes || p.off >= L.dt) continue;
      if (pack_head) std::memcpy((char*)ctx->h_in.p + p.off, p.src, p.bytes);
      else FQ_CUDA(cudaMemcpyAsync(din + p.off, p.src, p.bytes, cudaMemcpyHostToDevice, st));
    }
    if (pack_head) FQ_CUDA(cudaMemcpyAsync(din, ctx->h_in.p, L.dt, cudaMemcpyHostToDevice, st));
    FQ_CUDA(cudaEventRecord(ctx->ev_head, st));
    FQ_CUDA(cudaStreamWaitEvent(ctx->stream2, ctx->ev_head, 0));
    // chosen with bench.py (64 corridors x 1024 candidates) on the GPU the kernel was first tuned on: 4 slices are best for a blocking call (copies hide behind the
    // solves), 2 when another context's batch is in flight as well (fewer, deeper launches: shorter tails)
    const int want_slices = ctx->throughput_slices > 0 ? ctx->throughput_slices : (deferred ? 2 : 4);
    const int n_slices = n_prob < want_slices ? n_prob : want_slices;
    int p_lo = 0;
    for (int k = 0; k < n_slices; k++)
    {
      // slice boundaries balance the candidate counts
      const long long target = (long long)n_cand * (k + 1) / n_slices;
      int p_hi = p_lo;
      while (p_hi < n_prob && (cand_ofs[p_hi + 1] <= target || p_hi == p_lo)) p_hi++;
      if (k == n_slices - 1) p_hi = n_prob;
      if (p_hi == p_lo) continue;
      const size_t c_lo = (size_t)cand_ofs[p_lo], c_n = (size_t)cand_ofs[p_hi] - c_lo;
      cudaStream_t s2 = (k & 1) ? ctx->stream2 : st;
      int mc = 0;
      for (int j = p_lo; j < p_hi; j++) mc = std::max(mc, cand_ofs[j + 1] - cand_ofs[j]);
      if (c_n > 0)
      {
        FQ_CUDA(cudaMemcpyAsync(din + L.dt + sizeof(double) * c_lo, dt + c_lo, sizeof(double) * c_n, cudaMemcpyHostToDevice, s2));
        if (n_poly > 0)
          FQ_CUDA(cudaMemcpyAsync(din + L.sigma + c_lo * N, sigma + c_lo * N, c_n * N, cudaMemcpyHostToDevice, s2));
        else
          FQ_CUDA(cudaMemsetAsync(din + L.sigma + c_lo * N, 0, c_n * N, s2));
        FqKernelArgs slice = a;
        slice.n_prob = p_hi - p_lo; slice.x0 += 9 * (size_t)p_lo; slice.xf += 9 * (size_t)p_lo; slice.lim += 3 * (size_t)p_lo;
        slice.poly_ofs += p_lo; slice.cand_ofs += p_lo;
        rc = fq_launch_solve_ctx(ctx, slice, mc, cs.max_poly_faces, s2);
        if (rc) { cudaStreamSynchronize(st); cudaStreamSynchronize(ctx->stream2); return rc; }
        FQ_CUDA(cudaMemcpyAsync(cost + c_lo, dout + L.cost + sizeof(double) * c_lo, sizeof(double) * c_n, cudaMemcpyDeviceToHost, s2));
        FQ_CUDA(cudaMemcpyAsync(feasible + c_lo, dout + L.feasible + c_lo, c_n, cudaMemcpyDeviceToHost, s2));
        if (coeffs)
          FQ_CUDA(cudaMemcpyAsync(coeffs + 12 * (size_t)N * c_lo, dout + L.coeffs + sizeof(double) * 12 * (size_t)N * c_lo,
                                  sizeof(double) * 12 * (size_t)N * c_n, cudaMemcpyDeviceToHost, s2));
        if (iters)
          FQ_CUDA(cudaMemcpyAsync(iters + c_lo, dout + L.iters + sizeof(int32_t) * c_lo, sizeof(int32_t) * c_n, cudaMemcpyDeviceToHost, s2));
      }
      p_lo = p_hi;
    }
    tr.mark("enqueue");
    const char* why = values_ok();                 // overlaps with the GPU work enqueued above
    tr.mark("finite");
    if (deferred && !why) { ctx->pending = true; return 0; }     // fq_wait() (or the next call) completes it
    FQ_CUDA(cudaStreamSynchronize(ctx->stream2));
    FQ_CUDA(cudaStreamSynchronize(st));
    tr.mark("wait");
    if (why) return fq_fail(ctx, FQ_E_ARG, why);      // outputs were written but are not to be trusted
    return 0;
  }
  if (n_poly == 0) FQ_CUDA(cudaMemsetAsync(din + L.sigma, 0, sig_bytes, st));
  rc = fq_launch_solve_ctx(ctx, a, max_cand, cs.max_poly_faces, st);
  if (rc) return rc;
  if (L.out_bytes <= kPackThreshold)
  {
    FQ_CUDA(ctx->h_out.reserve(L.out_bytes));
    FQ_CUDA(cudaMemcpyAsync(ctx->h_out.p, dout, L.out_bytes, cudaMemcpyDeviceToHost, st));
    FQ_CUDA(cudaStreamSynchronize(st));
    const char* ho = (const char*)ctx->h_out.p;
    std::memcpy(cost, ho + L.cost, sizeof(double) * (size_t)n_cand);
    std::memcpy(feasible, ho + L.feasible, (size_t)n_cand);
    if (coeffs) std::memcpy(coeffs, ho + L.coeffs, sizeof(double) * 12 * (size_t)N * n_cand);
    if (iters) std::memcpy(iters, ho + L.iters, sizeof(int32_t) * (size_t)n_cand);
  }
  else
  {
    FQ_CUDA(cudaMemcpyAsync(cost, dout + L.cost, sizeof(double) * (size_t)n_cand, cudaMemcpyDeviceToHost, st));
    FQ_CUDA(cudaMemcpyAsync(feasible, dout + L.feasible, (size_t)n_cand, cudaMemcpyDeviceToHost, st));
    if (coeffs)
      FQ_CUDA(cudaMemcpyAsync(coeffs, dout + L.coeffs, sizeof(double) * 12 * (size_t)N * n_cand, cudaMemcpyDeviceToHost, st));
    if (iters)
      FQ_CUDA(cudaMemcpyAsync(iters, dout + L.iters, sizeof(int32_t) * (size_t)n_cand, cudaMemcpyDeviceToHost, st));
    FQ_CUDA(cudaStreamSynchronize(st));
  }
  return 0;
}

// fq_solve_batch's one problem as a multi-problem description (cert as in solve_multi_impl)
int solve_batch_impl(fq_ctx* ctx, int N, int force_final, const double* x0, const double* xf, const double* lim, int P,
                     const int* face_ofs, const double* Ab, int n_cand, const double* dt, const uint8_t* sigma,
                     uint8_t* feasible, double* cost, double* coeffs, int32_t* iters, double* cert, int cert_stride)
{
  if (P < 0 || n_cand < 0) return fq_fail(ctx, FQ_E_ARG, "negative count");
  const int poly_ofs[2] = { 0, P }, cand_ofs[2] = { 0, n_cand }, zero_face[1] = { 0 };
  return solve_multi_impl(ctx, N, force_final, 1, x0, xf, lim, poly_ofs, P > 0 ? face_ofs : zero_face, Ab, cand_ofs, dt, sigma,
                          feasible, cost, coeffs, iters, false, nullptr, cert, cert_stride);
}
}  // namespace

extern "C" int fq_solve_multi(fq_ctx* ctx, int N, int force_final, int n_prob, const double* x0, const double* xf,
                              const double* lim, const int* poly_ofs, const int* face_ofs, const double* Ab,
                              const int* cand_ofs, const double* dt, const uint8_t* sigma, uint8_t* feasible,
                              double* cost, double* coeffs, int32_t* iters)
{
  return solve_multi_impl(ctx, N, force_final, n_prob, x0, xf, lim, poly_ofs, face_ofs, Ab, cand_ofs, dt, sigma, feasible, cost,
                          coeffs, iters, false);
}

extern "C" int fq_solve_multi_async(fq_ctx* ctx, int N, int force_final, int n_prob, const double* x0, const double* xf,
                                    const double* lim, const int* poly_ofs, const int* face_ofs, const double* Ab,
                                    const int* cand_ofs, const double* dt, const uint8_t* sigma, uint8_t* feasible,
                                    double* cost, double* coeffs, int32_t* iters)
{
  return solve_multi_impl(ctx, N, force_final, n_prob, x0, xf, lim, poly_ofs, face_ofs, Ab, cand_ofs, dt, sigma, feasible, cost,
                          coeffs, iters, true);
}

int fq_solve_multi_host_ex(fq_ctx* ctx, int N, int force_final, int n_prob, const double* x0, const double* xf, const double* lim,
                           const int* poly_ofs, const int* face_ofs, const double* Ab, const int* cand_ofs, const double* dt,
                           const uint8_t* sigma, uint8_t* feasible, double* cost, double* coeffs, int32_t* iters, bool deferred,
                           int** d_win_idx, double** d_win_cost)
{
  HostLayout L;
  int rc = solve_multi_impl(ctx, N, force_final, n_prob, x0, xf, lim, poly_ofs, face_ofs, Ab, cand_ofs, dt, sigma, feasible, cost,
                            coeffs, iters, true, &L);
  if (rc) return rc;
  if (cand_ofs[n_prob] == 0) return fq_fail(ctx, FQ_E_ARG, "no candidates");
  FQ_CUDA(cudaSetDevice(ctx->device));
  // slices of a large batch alternate between the two streams: join before selecting
  FQ_CUDA(cudaEventRecord(ctx->ev_head, ctx->stream2));
  FQ_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_head, 0));
  char* din = (char*)ctx->d_in.p;
  char* dout = (char*)ctx->d_out.p;
  FqSelectMultiArgs sa;
  sa.n_prob = n_prob; sa.N = N; sa.n_sig = 0; sa.cand_ofs = (const int*)(din + L.cand_ofs); sa.dt = (const double*)(din + L.dt);
  sa.sigma = nullptr; sa.feasible = (const uint8_t*)(dout + L.feasible); sa.cost = (const double*)(dout + L.cost);
  sa.win_idx = (int*)(dout + L.win_idx); sa.win_cost = (double*)(dout + L.win_cost); sa.win_dt = (double*)(dout + L.win_dt);
  sa.win_sigma = nullptr; sa.win_ofs = (int*)(dout + L.win_ofs);
  FQ_CUDA(fq_launch_select_multi(sa, ctx->stream));
  if (d_win_idx) *d_win_idx = sa.win_idx;
  if (d_win_cost) *d_win_cost = sa.win_cost;
  ctx->pending = true;
  if (!deferred) return fq_settle(ctx);
  return 0;
}

extern "C" int fq_wait(fq_ctx* ctx)
{
  if (!ctx) return FQ_E_ARG;
  ctx->pending = true;          // also drains device-pointer launches made on the context's own stream
  for (fq_ctx* p : ctx->peers) p->pending = true;
  return fq_settle(ctx);
}

// fq_solve_batch through the size-generic kernel, which also exports, for every candidate it finds infeasible, the Farkas
// certificate it stopped on (include/faster_b200.h)
extern "C" int fq_solve_batch_cert(fq_ctx* ctx, int N, int force_final, const double* x0, const double* xf, const double* lim,
                                   int P, const int* face_ofs, const double* Ab, int n_cand, const double* dt,
                                   const uint8_t* sigma, uint8_t* feasible, double* cost, double* cert, int cert_stride)
{
  if (!ctx) return FQ_E_ARG;
  if (!cert || cert_stride < 4 + 2 * 3 * FQ_MAX_N || n_cand <= 0) return fq_fail(ctx, FQ_E_ARG, "cert buffer: stride >= 4 + 6 FQ_MAX_N doubles per candidate");
  if (int rc = fq_settle(ctx)) return rc;
  FQ_CUDA(cudaSetDevice(ctx->device));
  FqArena arena;
  FQ_CUDA(arena.reserve(sizeof(double) * (size_t)cert_stride * n_cand));
  FQ_CUDA(cudaMemset(arena.p, 0, sizeof(double) * (size_t)cert_stride * n_cand));
  const int rc = solve_batch_impl(ctx, N, force_final, x0, xf, lim, P, face_ofs, Ab, n_cand, dt, sigma, feasible, cost, nullptr,
                                  nullptr, (double*)arena.p, cert_stride);
  cudaError_t e = cudaMemcpy(cert, arena.p, sizeof(double) * (size_t)cert_stride * n_cand, cudaMemcpyDeviceToHost);
  arena.release();
  if (rc) return rc;
  FQ_CUDA(e);
  return 0;
}

extern "C" int fq_solve_batch(fq_ctx* ctx, int N, int force_final, const double* x0, const double* xf,
                              const double* lim, int P, const int* face_ofs, const double* Ab, int n_cand,
                              const double* dt, const uint8_t* sigma, uint8_t* feasible, double* cost,
                              double* coeffs, int32_t* iters)
{
  if (!ctx) return FQ_E_ARG;
  return solve_batch_impl(ctx, N, force_final, x0, xf, lim, P, face_ofs, Ab, n_cand, dt, sigma, feasible, cost, coeffs, iters,
                          nullptr, 0);
}

namespace
{
int gen_new_traj_impl(fq_ctx* ctx, int N, int force_final, const double* x0, const double* xf, const double* lim, int P,
                      const int* face_ofs, const double* Ab, int n_dt, const double* dts, int n_sigma,
                      const uint8_t* sigmas, int* dt_index, int* sigma_index, double* cost, double* coeffs, double DC,
                      int max_samples, double* samples, int* n_samples)
{
  if (!ctx) return FQ_E_ARG;
  if (int src = fq_settle(ctx)) return src;
  Trace tr;
  if (!x0 || !xf || !lim || !dts) return fq_fail(ctx, FQ_E_ARG, "NULL argument");
  if (P < 0 || P > FQ_MAX_POLY || n_dt <= 0) return fq_fail(ctx, FQ_E_ARG, "bad P or n_dt");
  if (P == 0) n_sigma = 1;
  if (n_sigma <= 0 || (P > 0 && (!sigmas || !face_ofs || !Ab))) return fq_fail(ctx, FQ_E_ARG, "bad sigma list / polytopes");
  if (n_sigma > (1 << 20)) return fq_fail(ctx, FQ_E_ARG, "n_sigma > 2^20");
  const int ne = force_final ? 3 : 2;
  if (N < ne || N > FQ_MAX_N) return fq_fail(ctx, FQ_E_ARG, "N out of range");
  const int poly_ofs[2] = { 0, P }, zero_face[1] = { 0 };
  FqCorridorSizes cs;
  if (const char* why = fq_scan_corridors(1, poly_ofs, P > 0 ? face_ofs : zero_face, &cs)) return fq_fail(ctx, FQ_E_ARG, why);
  const int n_face = cs.n_face;
  if (!fq_scan_all_finite(x0, 9) || !fq_scan_all_finite(xf, 9) || !fq_scan_all_positive_finite(lim, 3) ||
      !fq_scan_all_positive_finite(dts, (size_t)n_dt) || (P > 0 && !fq_scan_all_finite(Ab, 4 * (size_t)n_face)))
    return fq_fail(ctx, FQ_E_ARG, "non-finite input, dt <= 0 or limit <= 0");
  const long long n_cand_ll = (long long)n_dt * n_sigma;
  if (n_cand_ll > (1LL << 30)) return fq_fail(ctx, FQ_E_ARG, "too many candidates");
  const int n_cand = (int)n_cand_ll;
  if (P > 0 && fq_scan_max_u8(sigmas, (size_t)n_sigma * N) >= P) return fq_fail(ctx, FQ_E_ARG, "sigma entry >= number of polytopes");
  FQ_CUDA(cudaSetDevice(ctx->device));
  // ---- pack the (small) problem description; the dt x sigma grid is expanded on the host side of the copy
  size_t o = 0;
  const size_t oAb = o;   o = fq_align16(o + sizeof(double) * 4 * (size_t)(n_face > 0 ? n_face : 1));
  const size_t ox0 = o;   o += sizeof(double) * 9;
  const size_t oxf = o;   o += sizeof(double) * 9;
  const size_t olim = o;  o += sizeof(double) * 3;
  const size_t odt = o;   o += sizeof(double) * (size_t)n_cand;
  const size_t opo = o;   o += sizeof(int) * 2;
  const size_t ofo = o;   o += sizeof(int) * (size_t)(P + 1);
  const size_t oco = o;   o += sizeof(int) * 2;
  const size_t osig = o;  o = fq_align16(o + (size_t)n_cand * N);
  const size_t odts = o;  o += sizeof(double) * (size_t)n_dt;      // the n_dt distinct time allocations (for fillX)
  const size_t in_bytes = fq_align16(o);
  o = 0;
  const size_t ocost = o;   o += sizeof(double) * (size_t)n_cand;
  const size_t ocoef = o;   o += sizeof(double) * 12 * (size_t)N * n_cand;
  const size_t owin = o;    o += sizeof(double) * (1 + 12 * (size_t)N);     // winner: cost + coeffs
  const size_t oidx = o;    o += sizeof(int) * 2;
  const size_t onsamp = o;  o += sizeof(int) * 2;
  const size_t osamp = o;   o += samples ? sizeof(double) * 12 * (size_t)max_samples : 0;
  const size_t ofeas = o;   o += (size_t)n_cand;
  const size_t out_bytes = fq_align16(o);
  FQ_CUDA(ctx->d_in.reserve(in_bytes));
  FQ_CUDA(ctx->d_out.reserve(out_bytes));
  FQ_CUDA(ctx->h_in.reserve(in_bytes));
  FQ_CUDA(ctx->h_out.reserve(sizeof(double) * (1 + 12 * (size_t)N) + 4 * sizeof(int) +
                             (samples ? sizeof(double) * 12 * (size_t)max_samples : 0)));
  char* hi = (char*)ctx->h_in.p;
  if (n_face) std::memcpy(hi + oAb, Ab, sizeof(double) * 4 * (size_t)n_face);
  std::memcpy(hi + ox0, x0, sizeof(double) * 9);
  std::memcpy(hi + oxf, xf, sizeof(double) * 9);
  std::memcpy(hi + olim, lim, sizeof(double) * 3);
  {
    double* hd = (double*)(hi + odt);
    uint8_t* hs = (uint8_t*)(hi + osig);
    for (int d = 0; d < n_dt; d++)
      for (int s = 0; s < n_sigma; s++)
      {
        hd[(size_t)d * n_sigma + s] = dts[d];
        if (P > 0) std::memcpy(hs + ((size_t)d * n_sigma + s) * N, sigmas + (size_t)s * N, N);
        else std::memset(hs + ((size_t)d * n_sigma + s) * N, 0, N);
      }
    std::memcpy(hi + odts, dts, sizeof(double) * (size_t)n_dt);
    int* po = (int*)(hi + opo); po[0] = 0; po[1] = P;
    int* fo = (int*)(hi + ofo); fo[0] = 0; for (int p = 0; p < P; p++) fo[p + 1] = face_ofs[p + 1];
    int* co = (int*)(hi + oco); co[0] = 0; co[1] = n_cand;
  }
  tr.mark("pack");
  cudaStream_t st = ctx->stream;
  char* din = (char*)ctx->d_in.p;
  char* dout = (char*)ctx->d_out.p;
  cudaEvent_t tev[5] = { nullptr, nullptr, nullptr, nullptr, nullptr };      // FQ_TRACE: device-side phase times
  if (tr.on)
    for (auto& e : tev) cudaEventCreate(&e);
  if (tr.on) cudaEventRecord(tev[0], st);
  FQ_CUDA(cudaMemcpyAsync(din, hi, in_bytes, cudaMemcpyHostToDevice, st));
  if (tr.on) cudaEventRecord(tev[1], st);
  FqKernelArgs a{};
  a.N = N; a.force_final = force_final; a.n_prob = 1;
  a.x0 = (const double*)(din + ox0); a.xf = (const double*)(din + oxf); a.lim = (const double*)(din + olim);
  a.poly_ofs = (const int*)(din + opo); a.face_ofs = (const int*)(din + ofo); a.Ab = (const double*)(din + oAb);
  a.max_faces = n_face; a.cand_ofs = (const int*)(din + oco); a.dt = (const double*)(din + odt);
  a.sigma = (const uint8_t*)(din + osig); a.feasible = (uint8_t*)(dout + ofeas); a.cost = (double*)(dout + ocost);
  a.coeffs = (double*)(dout + ocoef);
  a.sorted_dt = 1;
  for (int d = 1; d < n_dt; d++) a.sorted_dt = a.sorted_dt && dts[d] >= dts[d - 1];
  a.ee_width = a.sorted_dt ? n_sigma : 0;
  char* ho = (char*)ctx->h_out.p;
  const size_t win_bytes = sizeof(double) * (1 + 12 * (size_t)N);
  if (!samples)
  { // the last warp to finish selects the winner and writes the record (cost, coefficients, indices) into this pinned,
    // device-visible host buffer: no selection launch and no device-to-host copy on the latency path
    void *dwin = nullptr;
    if (cudaHostGetDevicePointer(&dwin, ho, 0) == cudaSuccess)
    {
      a.sweep_n_sigma = n_sigma;
      a.sweep_win = (double*)dwin;
      a.sweep_idx = (int*)((char*)dwin + win_bytes);
      ((int*)(ho + win_bytes))[0] = -2;               // overwritten by the kernel
    }
  }
  bool tail = false;
  // the early exit skips candidates by dt VALUE, the selection picks the first dt INDEX with a feasible assignment: the
  // two agree only when the dt list is ascending, so a sweep over any other order evaluates every candidate
  int rc = fq_launch_solve_ctx(ctx, a, n_cand, cs.max_poly_faces, st, &tail, a.sorted_dt != 0);
  if (rc) return rc;
  if (tr.on) cudaEventRecord(tev[2], st);
  FqSelectArgs sa;
  sa.n_dt = n_dt; sa.n_sigma = n_sigma; sa.N = N;
  sa.feasible = (const uint8_t*)(dout + ofeas); sa.cost = (const double*)(dout + ocost);
  sa.coeffs = (const double*)(dout + ocoef);
  sa.out_idx = (int*)(dout + oidx); sa.out_cost = (double*)(dout + owin); sa.out_coeffs = (double*)(dout + owin) + 1;
  if (!tail) FQ_CUDA(fq_launch_select(sa, st));
  size_t tail_bytes = 2 * sizeof(int);
  if (samples)
  { // fillX on the device, chained on the same stream; samples travel back with the winner record
    FqFillArgs fa;
    fa.N = N; fa.n_dt = n_dt; fa.max_samples = max_samples; fa.DC = DC;
    fa.dts = (const double*)(din + odts); fa.win_idx = (const int*)(dout + oidx);
    fa.coeffs = (const double*)(dout + owin) + 1; fa.out = (double*)(dout + osamp); fa.n_samples = (int*)(dout + onsamp);
    FQ_CUDA(fq_launch_fill(fa, st));
    tail_bytes = 4 * sizeof(int) + sizeof(double) * 12 * (size_t)max_samples;
  }
  if (tr.on) cudaEventRecord(tev[3], st);
  if (!tail) FQ_CUDA(cudaMemcpyAsync(ho, dout + owin, win_bytes + tail_bytes, cudaMemcpyDeviceToHost, st));
  if (tr.on) cudaEventRecord(tev[4], st);
  tr.mark("enqueue");
  FQ_CUDA(cudaStreamSynchronize(st));
  tr.mark("wait");
  if (tr.on)
  {
    float a = 0, b = 0, c = 0, d = 0;
    cudaEventElapsedTime(&a, tev[0], tev[1]); cudaEventElapsedTime(&b, tev[1], tev[2]);
    cudaEventElapsedTime(&c, tev[2], tev[3]); cudaEventElapsedTime(&d, tev[3], tev[4]);
    std::fprintf(stderr, "[fq trace] device: h2d %.1f us, counters+solve %.1f us, select(+fill) %.1f us, d2h %.1f us\n", a * 1e3, b * 1e3,
                 c * 1e3, d * 1e3);
    for (auto& e : tev) cudaEventDestroy(e);
  }
  static_assert(sizeof(double) == 8, "layout");
  const int* idx = (const int*)(ho + win_bytes);
  const double* win = (const double*)ho;
  if (tail && idx[0] == -2) return fq_fail(ctx, FQ_E_CUDA, "internal: the sweep finished without its selection");
  if (dt_index) *dt_index = idx[0];
  if (sigma_index) *sigma_index = idx[1];
  if (n_samples) *n_samples = 0;
  if (idx[0] < 0) { if (cost) *cost = INFINITY; return 0; }
  if (cost) *cost = win[0];
  if (coeffs) std::memcpy(coeffs, win + 1, sizeof(double) * 12 * (size_t)N);
  if (samples)
  {
    const int ns = idx[2];
    if (n_samples) *n_samples = ns;
    std::memcpy(samples, ho + win_bytes + 4 * sizeof(int), sizeof(double) * 12 * (size_t)ns);
  }
  return 1;
}
}  // namespace

extern "C" int fq_gen_new_traj(fq_ctx* ctx, int N, int force_final, const double* x0, const double* xf,
                               const double* lim, int P, const int* face_ofs, const double* Ab, int n_dt,
                               const double* dts, int n_sigma, const uint8_t* sigmas, int* dt_index,
                               int* sigma_index, double* cost, double* coeffs)
{
  return gen_new_traj_impl(ctx, N, force_final, x0, xf, lim, P, face_ofs, Ab, n_dt, dts, n_sigma, sigmas, dt_index,
                           sigma_index, cost, coeffs, 0.0, 0, nullptr, nullptr);
}

extern "C" int fq_gen_new_traj_sampled(fq_ctx* ctx, int N, int force_final, const double* x0, const double* xf,
                                       const double* lim, int P, const int* face_ofs, const double* Ab, int n_dt,
                                       const double* dts, int n_sigma, const uint8_t* sigmas, double DC,
                                       int max_samples, int* dt_index, int* sigma_index, double* cost,
                                       double* coeffs, double* samples, int* n_samples)
{
  if (!ctx) return FQ_E_ARG;
  if (!samples || max_samples < 2 || !(DC > 0)) return fq_fail(ctx, FQ_E_ARG, "samples buffer, max_samples >= 2 and DC > 0 required");
  return gen_new_traj_impl(ctx, N, force_final, x0, xf, lim, P, face_ofs, Ab, n_dt, dts, n_sigma, sigmas, dt_index,
                           sigma_index, cost, coeffs, DC, max_samples, samples, n_samples);
}


// ---------------------------------------------------------------------------------------------------------------------
// Exact MIQP sweep: genNewTraj with the minimum over ALL P^N assignments (what Gurobi's branch-and-bound returns), by
// branch-and-bound on the GPU (fq_bnb.cuh).  Only the time allocations up to the first one that is feasible for a
// non-decreasing assignment can win (first feasible factor wins, solverGurobi.cpp:445-446), so only those are searched.
// ---------------------------------------------------------------------------------------------------------------------
extern "C" int fq_gen_new_traj_exact(fq_ctx* ctx, int N, int force_final, const double* x0, const double* xf,
                                     const double* lim, int P, const int* face_ofs, const double* Ab, int n_dt,
                                     const double* dts, int* dt_index, uint8_t* sigma_out, double* cost, double* coeffs,
                                     long* nodes_out, int* exact_out)
{
  if (!ctx) return FQ_E_ARG;
  if (int src = fq_settle(ctx)) return src;
  if (!x0 || !xf || !lim || !dts || n_dt <= 0) return fq_fail(ctx, FQ_E_ARG, "NULL argument or n_dt <= 0");
  if (P < 0 || P > FQ_MAX_POLY) return fq_fail(ctx, FQ_E_ARG, "bad P");
  if (N < (force_final ? 3 : 2) || N > FQ_MAX_N) return fq_fail(ctx, FQ_E_ARG, "N out of range");
  if (nodes_out) *nodes_out = 0;
  if (exact_out) *exact_out = 1;
  if (sigma_out) std::memset(sigma_out, 0, (size_t)N);
  if (P == 0)
    return gen_new_traj_impl(ctx, N, force_final, x0, xf, lim, 0, face_ofs, Ab, n_dt, dts, 1, nullptr, dt_index, nullptr, cost,
                             coeffs, 0.0, 0, nullptr, nullptr);
  if (!face_ofs || !Ab) return fq_fail(ctx, FQ_E_ARG, "polytopes missing");
  const int poly_ofs[2] = { 0, P };
  FqCorridorSizes cs;
  if (const char* why = fq_scan_corridors(1, poly_ofs, face_ofs, &cs)) return fq_fail(ctx, FQ_E_ARG, why);
  const int n_face = cs.n_face;
  const size_t nb = fq_bnb_node_bytes(N, force_final);
  // ---- 1. non-decreasing assignments for every time allocation: the ordinary sweep (one launch + selection).  Its winner
  //         is the first monotone-feasible time allocation `fstar` with that allocation's best monotone cost; earlier
  //         allocations have no feasible monotone assignment, later ones cannot win.
  // C(N+P-1, N) in closed form (enumerating to count would take hours for large N and P)
  long n_mono = 1;
  for (int i = 1; i <= N && n_mono <= (1L << 40); i++) n_mono = n_mono * (P - 1 + i) / i;
  if (n_mono <= 0 || n_mono > (1L << 20) || (long long)n_mono * n_dt > (1LL << 24))
    return fq_fail(ctx, FQ_E_ARG, "assignment list too long for the monotone pre-sweep (N, P, n_dt too large)");
  std::vector<uint8_t> mono((size_t)n_mono * N);
  fq_monotone_sigmas(N, P, mono.data(), n_mono);
  int m_dt = -1, m_sig = -1;
  double m_cost = INFINITY;
  std::vector<double> m_coeffs((size_t)12 * N, 0.0);
  int rc = gen_new_traj_impl(ctx, N, force_final, x0, xf, lim, P, face_ofs, Ab, n_dt, dts, (int)n_mono, mono.data(), &m_dt, &m_sig,
                             &m_cost, m_coeffs.data(), 0.0, 0, nullptr, nullptr);
  if (rc < 0) return rc;
  const int fstar = rc == 1 ? m_dt : -1;
  std::vector<double> best(n_dt, INFINITY);
  std::vector<long> best_k(n_dt, -1);
  if (fstar >= 0) { best[fstar] = m_cost; best_k[fstar] = m_sig; }
  const int n_search = fstar >= 0 ? fstar + 1 : n_dt;       // later time allocations cannot win
  bool exact = nb != 0 && n_face <= 2047;
  std::vector<uint8_t> win_sigma(N, 0);
  int win_dt = -1;
  if (exact)
  {
    // ---- 2. device buffers
    const int cap = 65536, leaf_cap = 4096;
    size_t o = 0;
    const size_t oAb = o;    o = fq_align16(o + sizeof(double) * 4 * (size_t)n_face);
    const size_t ox0 = o;    o += sizeof(double) * 9;
    const size_t oxf = o;    o += sizeof(double) * 9;
    const size_t olim = o;   o += sizeof(double) * 3;
    const size_t odts = o;   o += sizeof(double) * (size_t)n_dt;
    const size_t oinc = o;   o += sizeof(unsigned long long) * (size_t)n_dt;
    const size_t opo = o;    o += sizeof(int) * 2;
    const size_t ofo = o;    o += sizeof(int) * (size_t)(P + 1);
    const size_t oroot = o;  o += sizeof(int) * (size_t)n_dt;
    const size_t ocnt = o;   o = fq_align16(o + sizeof(int) * 8);   // [0] n_children [1] n_leaves [2..3] flags
    const size_t head = o;
    const size_t oleaf = o;  o = fq_align16(o + 32 * (size_t)leaf_cap);
    const size_t opoolA = o; o = fq_align16(o + nb * (size_t)cap);
    const size_t opoolB = o; o = fq_align16(o + nb * (size_t)cap);
    FQ_CUDA(cudaSetDevice(ctx->device));
    FQ_CUDA(ctx->d_bnb.reserve(o));
    FQ_CUDA(ctx->h_in.reserve(head));
    char* hi = (char*)ctx->h_in.p;
    char* db = (char*)ctx->d_bnb.p;
    std::memset(hi, 0, head);
    std::memcpy(hi + oAb, Ab, sizeof(double) * 4 * (size_t)n_face);
    std::memcpy(hi + ox0, x0, sizeof(double) * 9);
    std::memcpy(hi + oxf, xf, sizeof(double) * 9);
    std::memcpy(hi + olim, lim, sizeof(double) * 3);
    std::memcpy(hi + odts, dts, sizeof(double) * (size_t)n_dt);
    // presolve on the constant control points: segment 0 starts with cp0, cp1, cp2 fixed by (x0, dt) and, with the final
    // position pinned, the last control point is xf -- a time allocation for which no polytope holds them is infeasible
    // for EVERY assignment and needs no tree (otherwise such corridors make the tree explore all prefixes)
    auto inside_any = [&](const double* pt) {
      for (int p = 0; p < P; p++)
      {
        bool in = true;
        for (int f = face_ofs[p]; f < face_ofs[p + 1] && in; f++)
          in = Ab[4 * f] * pt[0] + Ab[4 * f + 1] * pt[1] + Ab[4 * f + 2] * pt[2] - Ab[4 * f + 3] <= ctx->row_tol;
        if (in) return true;
      }
      return false;
    };
    int n_roots = 0;
    for (int d = 0; d < n_dt; d++)
    {
      unsigned long long bits;
      const double c = best[d];
      std::memcpy(&bits, &c, 8);
      ((unsigned long long*)(hi + oinc))[d] = bits;              // +inf orders above every finite cost
      if (d >= n_search) continue;
      bool possible = true;
      if (force_final) possible = inside_any(xf);
      if (possible)
      { // all three constant points of segment 0 must share one polytope
        possible = false;
        const double t = dts[d];
        for (int p = 0; p < P && !possible; p++)
        {
          bool in = true;
          for (int kk = 0; kk < 3 && in; kk++)
          {
            double pt[3];
            for (int ax = 0; ax < 3; ax++)
              pt[ax] = x0[ax] + (kk >= 1 ? x0[3 + ax] * t * (kk == 1 ? 1.0 / 3.0 : 2.0 / 3.0) : 0.0) + (kk == 2 ? x0[6 + ax] * t * t / 6.0 : 0.0);
            for (int f = face_ofs[p]; f < face_ofs[p + 1] && in; f++)
              in = Ab[4 * f] * pt[0] + Ab[4 * f + 1] * pt[1] + Ab[4 * f + 2] * pt[2] - Ab[4 * f + 3] <= ctx->row_tol;
          }
          possible = in;
        }
      }
      if (possible) ((int*)(hi + oroot))[n_roots++] = d;
    }
    ((int*)(hi + opo))[0] = 0; ((int*)(hi + opo))[1] = P;
    for (int p = 0; p <= P; p++) ((int*)(hi + ofo))[p] = face_ofs[p];
    cudaStream_t st = ctx->stream;
    FQ_CUDA(cudaMemcpyAsync(db, hi, head, cudaMemcpyHostToDevice, st));
    FqPlanDev* pd = nullptr;
    rc = fq_get_plan(ctx, N, force_final, &pd);
    if (rc) return rc;
    FqBnbLevel L{};
    fq_fill_plan_args(*pd, &L.k);
    L.k.n_prob = 1; L.k.x0 = (const double*)(db + ox0); L.k.xf = (const double*)(db + oxf); L.k.lim = (const double*)(db + olim);
    L.k.poly_ofs = (const int*)(db + opo); L.k.face_ofs = (const int*)(db + ofo); L.k.Ab = (const double*)(db + oAb);
    L.k.max_faces = n_face; L.k.item_cap = N * cs.max_poly_faces; L.k.row_tol = ctx->row_tol;
    L.n_dt = n_dt; L.P = P; L.dts = (const double*)(db + odts); L.roots = (const int*)(db + oroot);
    L.incumbent = (unsigned long long*)(db + oinc); L.leaves = db + oleaf; L.n_leaves = (int*)(db + ocnt) + 1;
    L.leaf_cap = leaf_cap; L.flags = (int*)(db + ocnt) + 2; L.n_children = (int*)(db + ocnt); L.cap = cap;
    int n_par = n_roots;
    long nodes = 0;
    unsigned char* pools[2] = { (unsigned char*)(db + opoolA), (unsigned char*)(db + opoolB) };
    int cnt[4] = { 0, 0, 0, 0 };
    for (int depth = 0; depth < N && n_par > 0; depth++)
    {
      L.depth = depth; L.n_parents = n_par;
      L.parents = pools[depth & 1]; L.children = pools[(depth + 1) & 1];
      FQ_CUDA(cudaMemsetAsync(L.n_children, 0, sizeof(int), st));
      cudaError_t e = fq_launch_bnb_level(L, st);
      if (e == cudaErrorInvalidConfiguration) { exact = false; break; }
      FQ_CUDA(e);
      FQ_CUDA(cudaMemcpyAsync(cnt, db + ocnt, sizeof(cnt), cudaMemcpyDeviceToHost, st));
      FQ_CUDA(cudaStreamSynchronize(st));
      nodes += (long)n_par * P;
      if (cnt[2]) { exact = false; break; }                      // pool overflow: the tree was cut
      if (cnt[3]) { exact = false; break; }                      // a node hit the iteration cap / a NaN and its subtree was
                                                                 // dropped: the optimum may hide there, so not exact
      n_par = cnt[0];
    }
    if (nodes_out) *nodes_out = nodes;
    if (exact)
    {
      const int n_leaves = std::min(cnt[1], leaf_cap);
      struct Leaf { int dt_idx, pad; double cost; unsigned char sigma[16]; };
      std::vector<Leaf> leaves((size_t)std::max(n_leaves, 1));
      std::vector<unsigned long long> inc(n_dt);
      if (n_leaves) FQ_CUDA(cudaMemcpyAsync(leaves.data(), db + oleaf, sizeof(Leaf) * (size_t)n_leaves, cudaMemcpyDeviceToHost, st));
      FQ_CUDA(cudaMemcpyAsync(inc.data(), db + oinc, sizeof(unsigned long long) * (size_t)n_dt, cudaMemcpyDeviceToHost, st));
      FQ_CUDA(cudaStreamSynchronize(st));
      for (int d = 0; d < n_search && win_dt < 0; d++)
      {
        double c;
        std::memcpy(&c, &inc[d], 8);
        if (!(c < INFINITY)) continue;
        win_dt = d;
        bool from_leaf = false;
        for (int i = 0; i < n_leaves; i++)                         // the last improving leaf of this dt holds the incumbent
          if (leaves[i].dt_idx == d && leaves[i].cost == c) { std::memcpy(win_sigma.data(), leaves[i].sigma, N); from_leaf = true; }
        if (!from_leaf) std::memcpy(win_sigma.data(), &mono[(size_t)best_k[d] * N], N);
      }
    }
  }
  if (!exact)
  { // fall back to the non-decreasing optimum (reported through exact_out = 0)
    if (exact_out) *exact_out = 0;
    win_dt = fstar;
    if (fstar >= 0) std::memcpy(win_sigma.data(), &mono[(size_t)best_k[fstar] * N], N);
  }
  if (dt_index) *dt_index = win_dt;
  if (win_dt < 0) { if (cost) *cost = INFINITY; return 0; }
  if (sigma_out) std::memcpy(sigma_out, win_sigma.data(), N);
  // ---- 3. coefficients of the winner: the monotone sweep already has them unless the tree found something better
  if (win_dt == fstar && fstar >= 0 && std::memcmp(win_sigma.data(), &mono[(size_t)best_k[fstar] * N], N) == 0)
  {
    if (cost) *cost = m_cost;
    if (coeffs) std::memcpy(coeffs, m_coeffs.data(), sizeof(double) * 12 * (size_t)N);
    return 1;
  }
  uint8_t f1 = 0;
  double c1 = INFINITY;
  std::vector<double> co((size_t)12 * N);
  rc = fq_solve_batch(ctx, N, force_final, x0, xf, lim, P, face_ofs, Ab, 1, &dts[win_dt], win_sigma.data(), &f1, &c1, co.data(), nullptr);
  if (rc) return rc;
  if (!f1) return fq_fail(ctx, FQ_E_CUDA, "internal: the winning assignment did not re-solve");
  if (cost) *cost = c1;
  if (coeffs) std::memcpy(coeffs, co.data(), sizeof(double) * 12 * (size_t)N);
  return 1;
}
