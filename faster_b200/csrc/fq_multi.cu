// Multi-GPU behind the C ABI (SURVEY.md 8b/8e): the candidates of different corridors are independent, so a batch is
// sharded by corridor; the ONE exchange of the path is an all-gather of the per-corridor results (the winners of the
// genNewTraj selection: a few hundred bytes per corridor instead of every candidate's cost), done with NCCL inside the
// context.  Two ways to own several GPUs:
//   * one process per GPU (torchrun-style): fq_create + fq_comm_init(id, rank, world) on every rank;
//   * one process, several GPUs (what the reference's single planner process would do): fq_create_multi.
// NCCL is loaded lazily with dlopen (libnccl.so.2; FQ_NCCL_LIB overrides), so the library has no link-time dependency
// on it and single-GPU use needs no NCCL at all.
#include "fq_ctx.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <dlfcn.h>
#include <mutex>
#include <nccl.h>

namespace
{
struct NcclApi
{
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
  std::string why;
};
NcclApi g_nccl;
std::once_flag g_nccl_once;

const NcclApi* nccl()
{
  std::call_once(g_nccl_once, [] {
    const char* env = std::getenv("FQ_NCCL_LIB");
    const char* names[] = { env, "libnccl.so.2", "libnccl.so" };
    for (const char* n : names)
    {
      if (!n || !*n) continue;
      g_nccl.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (g_nccl.handle) break;
    }
    if (!g_nccl.handle) { g_nccl.why = std::string("cannot load NCCL (libnccl.so.2): ") + (dlerror() ? dlerror() : "not found"); return; }
    auto sym = [&](const char* s) { void* p = dlsym(g_nccl.handle, s); if (!p && g_nccl.why.empty()) g_nccl.why = std::string("NCCL lacks ") + s; return p; };
    g_nccl.GetUniqueId = (decltype(g_nccl.GetUniqueId))sym("ncclGetUniqueId");
    g_nccl.CommInitRank = (decltype(g_nccl.CommInitRank))sym("ncclCommInitRank");
    g_nccl.CommInitAll = (decltype(g_nccl.CommInitAll))sym("ncclCommInitAll");
    g_nccl.CommDestroy = (decltype(g_nccl.CommDestroy))sym("ncclCommDestroy");
    g_nccl.AllGather = (decltype(g_nccl.AllGather))sym("ncclAllGather");
    g_nccl.GroupStart = (decltype(g_nccl.GroupStart))sym("ncclGroupStart");
    g_nccl.GroupEnd = (decltype(g_nccl.GroupEnd))sym("ncclGroupEnd");
    g_nccl.GetErrorString = (decltype(g_nccl.GetErrorString))sym("ncclGetErrorString");
    g_nccl.GetVersion = (decltype(g_nccl.GetVersion))sym("ncclGetVersion");
  });
  return g_nccl.why.empty() ? &g_nccl : nullptr;
}

int nccl_fail(fq_ctx* ctx, ncclResult_t r, const char* what)
{
  return fq_fail(ctx, FQ_E_CUDA, std::string(what) + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "NCCL error"));
}
#define FQ_NCCL(call)                                        \
  do {                                                       \
    ncclResult_t r__ = (call);                               \
    if (r__ != ncclSuccess) return nccl_fail(ctx, r__, #call); \
  } while (0)
}  // namespace

struct FqComm
{
  ncclComm_t comm = nullptr;
};

void fq_comm_release(fq_ctx* ctx)
{
  if (!ctx || !ctx->comm) return;
  if (ctx->comm->comm && g_nccl.CommDestroy)
  {
    cudaSetDevice(ctx->device);
    g_nccl.CommDestroy(ctx->comm->comm);
  }
  delete ctx->comm;
  ctx->comm = nullptr;
}

extern "C" int fq_comm_unique_id(void* id128)
{
  if (!id128) return FQ_E_ARG;
  const NcclApi* n = nccl();
  if (!n) return fq_fail(nullptr, FQ_E_CUDA, g_nccl.why);
  ncclUniqueId id;
  if (n->GetUniqueId(&id) != ncclSuccess) return fq_fail(nullptr, FQ_E_CUDA, "ncclGetUniqueId failed");
  static_assert(sizeof(id) == 128, "ncclUniqueId is 128 bytes");
  std::memcpy(id128, &id, 128);
  return 0;
}

extern "C" int fq_comm_init(fq_ctx* ctx, const void* id128, int rank, int world)
{
  if (!ctx || !id128) return FQ_E_ARG;
  if (world < 1 || rank < 0 || rank >= world) return fq_fail(ctx, FQ_E_ARG, "bad rank / world");
  if (ctx->comm || ctx->is_group) return fq_fail(ctx, FQ_E_ARG, "context already belongs to a communicator");
  const NcclApi* n = nccl();
  if (!n) return fq_fail(ctx, FQ_E_CUDA, g_nccl.why);
  FQ_CUDA(cudaSetDevice(ctx->device));
  ncclUniqueId id;
  std::memcpy(&id, id128, 128);
  FqComm* c = new (std::nothrow) FqComm();
  if (!c) return fq_fail(ctx, FQ_E_NOMEM, "out of host memory");
  ncclResult_t r = n->CommInitRank(&c->comm, world, id, rank);
  if (r != ncclSuccess) { delete c; return nccl_fail(ctx, r, "ncclCommInitRank"); }
  ctx->comm = c; ctx->rank = rank; ctx->world = world;
  return 0;
}

extern "C" int fq_comm_info(const fq_ctx* ctx, int* rank, int* world, int* nccl_version)
{
  if (!ctx) return FQ_E_ARG;
  if (rank) *rank = ctx->rank;
  if (world) *world = ctx->world;
  if (nccl_version)
  {
    *nccl_version = 0;
    if (ctx->comm && g_nccl.GetVersion) g_nccl.GetVersion(nccl_version);
  }
  return 0;
}

extern "C" int fq_create_multi(fq_ctx** out, int n_gpus, const int* devices)
{
  if (!out) return fq_fail(nullptr, FQ_E_ARG, "out is NULL");
  *out = nullptr;
  if (n_gpus < 1 || n_gpus > 64) return fq_fail(nullptr, FQ_E_ARG, "n_gpus out of range (1..64)");
  std::vector<int> devs(n_gpus);
  for (int i = 0; i < n_gpus; i++) devs[i] = devices ? devices[i] : i;
  for (int i = 0; i < n_gpus; i++)
    for (int j = 0; j < i; j++)
      if (devs[i] == devs[j]) return fq_fail(nullptr, FQ_E_ARG, "duplicate device");
  fq_ctx* head = nullptr;
  int rc = fq_create(&head, devs[0]);
  if (rc) return rc;
  head->is_group = true; head->rank = 0; head->world = n_gpus;
  for (int i = 1; i < n_gpus; i++)
  {
    fq_ctx* p = nullptr;
    rc = fq_create(&p, devs[i]);
    if (rc) { fq_destroy(head); return rc; }
    p->rank = i; p->world = n_gpus;
    head->peers.push_back(p);
  }
  if (n_gpus > 1)
  {
    const NcclApi* n = nccl();
    if (!n) { fq_destroy(head); return fq_fail(nullptr, FQ_E_CUDA, g_nccl.why); }
    std::vector<ncclComm_t> comms(n_gpus, nullptr);
    ncclResult_t r = n->CommInitAll(comms.data(), n_gpus, devs.data());
    if (r != ncclSuccess) { fq_destroy(head); return nccl_fail(nullptr, r, "ncclCommInitAll"); }
    for (int i = 0; i < n_gpus; i++)
    {
      fq_ctx* c = i == 0 ? head : head->peers[i - 1];
      c->comm = new FqComm();
      c->comm->comm = comms[i];
    }
  }
  *out = head;
  return 0;
}

int fq_comm_allgather(fq_ctx* ctx, const void* d_send, void* d_recv, size_t bytes, cudaStream_t stream)
{
  if (!ctx->comm) return fq_fail(ctx, FQ_E_ARG, "no communicator attached (fq_comm_init / fq_create_multi)");
  FQ_NCCL(g_nccl.AllGather(d_send, d_recv, bytes, ncclChar, ctx->comm->comm, stream));
  return 0;
}

extern "C" int fq_allgather_dev(fq_ctx* ctx, const void* d_send, void* d_recv, long bytes, void* stream)
{
  if (!ctx || !d_send || !d_recv || bytes < 0) return FQ_E_ARG;
  FQ_CUDA(cudaSetDevice(ctx->device));
  if (!ctx->comm)
  { // a world of one: the gather is a copy
    FQ_CUDA(cudaMemcpyAsync(d_recv, d_send, (size_t)bytes, cudaMemcpyDeviceToDevice, stream ? (cudaStream_t)stream : ctx->stream));
    return 0;
  }
  return fq_comm_allgather(ctx, d_send, d_recv, (size_t)bytes, stream ? (cudaStream_t)stream : ctx->stream);
}

// Contiguous shard of problems for `rank` of `world`, balanced by candidate count (cand_ofs may be NULL: by problem
// count).  Every problem belongs to exactly one rank; ranks may be empty when world > n_prob.
extern "C" int fq_shard_range(int n_prob, const int* cand_ofs, int rank, int world, int* lo, int* hi)
{
  if (n_prob < 0 || world < 1 || rank < 0 || rank >= world || !lo || !hi) return FQ_E_ARG;
  auto cut = [&](int r) -> int {             // first problem of rank r
    if (r <= 0) return 0;
    if (r >= world) return n_prob;
    if (!cand_ofs) return (int)((long long)n_prob * r / world);
    const long long total = cand_ofs[n_prob], target = total * r / world;
    // the boundary j whose cand_ofs[j] is nearest to the target (monotone in r)
    int a = 0, b = n_prob;
    while (a < b) { const int m = (a + b) / 2; if (cand_ofs[m] >= target) b = m; else a = m + 1; }
    if (a > 0 && target - cand_ofs[a - 1] < cand_ofs[a] - target) a--;
    return a;
  };
  *lo = cut(rank); *hi = cut(rank + 1);
  if (*hi < *lo) *hi = *lo;
  return 0;
}

namespace
{
fq_ctx* member(fq_ctx* g, int i) { return i == 0 ? g : g->peers[i - 1]; }

struct SubCorridors
{ // rebased CSR description of problems [lo, hi)
  std::vector<int> poly_ofs, face_ofs;
  const double* Ab;
  void build(const int* po, const int* fo, const double* Ab_all, int lo, int hi)
  {
    poly_ofs.resize(hi - lo + 1);
    for (int j = lo; j <= hi; j++) poly_ofs[j - lo] = po[j] - po[lo];
    const int p0 = po[lo], p1 = po[hi];
    face_ofs.resize(p1 - p0 + 1);
    for (int p = p0; p <= p1; p++) face_ofs[p - p0] = fo[p] - fo[p0];
    Ab = Ab_all ? Ab_all + 4 * (size_t)fo[p0] : nullptr;
  }
};

// the one exchange of a sharded call: local member i (one for a rank context) sends `count` records from send[i] and
// receives every rank's, in rank order, into recv[i].  Over the members of a single-process group, over a rank's
// communicator, or a copy for a world of one.
template <class T>
int exchange(fq_ctx* g, const std::vector<T*>& send, const std::vector<T*>& recv, size_t count)
{
  fq_ctx* ctx = g;
  const size_t bytes = sizeof(T) * count;
  if (!g->is_group && g->comm) return fq_comm_allgather(g, send[0], recv[0], bytes, g->stream);
  // a context that is neither a group nor a communicator's rank keeps world == 1 (only fq_comm_init and fq_create_multi
  // set it), so past this point world > 1 means a group with world - 1 peers
  if (g->world == 1)
  {
    FQ_CUDA(cudaSetDevice(g->device));
    FQ_CUDA(cudaMemcpyAsync(recv[0], send[0], bytes, cudaMemcpyDeviceToDevice, g->stream));
    return 0;
  }
  FQ_NCCL(g_nccl.GroupStart());
  for (int i = 0; i < g->world; i++)
  {
    fq_ctx* c = member(g, i);
    cudaSetDevice(c->device);
    ncclResult_t r = g_nccl.AllGather(send[i], recv[i], bytes, ncclChar, c->comm->comm, c->stream);
    if (r != ncclSuccess) { g_nccl.GroupEnd(); return nccl_fail(g, r, "ncclAllGather"); }
  }
  FQ_NCCL(g_nccl.GroupEnd());
  return 0;
}
}  // namespace

// fq_replan_pairs on a multi-GPU context.  Group (one process): corridors [lo_i, hi_i) go to member i, every member runs
// its chain, the result records are all-gathered (padded to the largest shard) and read back once from member 0; the
// per-candidate arrays travel straight from each member into the caller's arrays.  Rank context (one process per GPU):
// every rank passes the SAME full description and solves its own shard; after the all-gather every rank holds every
// corridor's result record, while per-candidate outputs are filled for the rank's own corridors only.
int fq_replan_pairs_sharded(fq_ctx* g, const fq_pair_args* a, bool deferred)
{
  fq_ctx* ctx = g;
  if (!a || a->n_prob <= 0 || !a->results) return fq_fail(g, FQ_E_ARG, "bad arguments");
  // the shards' corridor descriptions are rebased on the host before the per-member validation runs: the arrays read
  // here must exist (everything else is checked by the member's own call)
  if (!a->x0 || !a->xf_whole || !a->xf_safe || !a->lim || !a->poly_ofs_whole || !a->face_ofs_whole || !a->poly_ofs_safe ||
      !a->face_ofs_safe)
    return fq_fail(g, FQ_E_ARG, "NULL argument");
  if (a->n_fac_whole <= 0 || a->n_fac_safe <= 0 || a->n_sig_whole <= 0 || a->n_sig_safe <= 0)
    return fq_fail(g, FQ_E_ARG, "empty factor / assignment grid");
  for (int j = 0; j < a->n_prob; j++)
    if (a->poly_ofs_whole[j + 1] < a->poly_ofs_whole[j] || a->poly_ofs_safe[j + 1] < a->poly_ofs_safe[j])
      return fq_fail(g, FQ_E_ARG, "poly_ofs not monotone");
  const int P = a->n_prob, world = g->world;
  const bool group = g->is_group;
  const int n_local = group ? world : 1;
  const size_t ncw1 = (size_t)a->n_fac_whole * a->n_sig_whole, ncs1 = (size_t)a->n_fac_safe * a->n_sig_safe;
  int pad = 0;
  std::vector<int> lo(world), hi(world);
  for (int r = 0; r < world; r++) { fq_shard_range(P, nullptr, r, world, &lo[r], &hi[r]); pad = std::max(pad, hi[r] - lo[r]); }
  std::vector<fq_pair_result*> d_res(n_local, nullptr), d_all(n_local, nullptr);
  for (int i = 0; i < n_local; i++)
  {
    fq_ctx* c = group ? member(g, i) : g;
    const int r = group ? i : g->rank;
    if (int rc = fq_settle(c)) return rc;
    cudaSetDevice(c->device);
    // gather buffers: [pad records to send | world x pad records received]
    cudaError_t e = c->d_out.reserve(sizeof(fq_pair_result) * (size_t)pad * (world + 1));
    if (e != cudaSuccess) return fq_cuda_fail(g, e, "gather buffer");
    d_res[i] = (fq_pair_result*)c->d_out.p;
    d_all[i] = d_res[i] + pad;
    e = cudaMemsetAsync(d_res[i], 0xff, sizeof(fq_pair_result) * (size_t)pad, c->stream);
    if (e != cudaSuccess) return fq_cuda_fail(g, e, "gather buffer");
    const int n = hi[r] - lo[r];
    if (n <= 0) continue;
    fq_pair_args s = *a;
    SubCorridors cw, cs;
    cw.build(a->poly_ofs_whole, a->face_ofs_whole, a->Ab_whole, lo[r], hi[r]);
    cs.build(a->poly_ofs_safe, a->face_ofs_safe, a->Ab_safe, lo[r], hi[r]);
    s.n_prob = n;
    s.x0 = a->x0 + 9 * (size_t)lo[r]; s.xf_whole = a->xf_whole + 9 * (size_t)lo[r]; s.xf_safe = a->xf_safe + 9 * (size_t)lo[r];
    s.lim = a->lim + 3 * (size_t)lo[r];
    s.poly_ofs_whole = cw.poly_ofs.data(); s.face_ofs_whole = cw.face_ofs.data(); s.Ab_whole = cw.Ab;
    s.poly_ofs_safe = cs.poly_ofs.data(); s.face_ofs_safe = cs.face_ofs.data(); s.Ab_safe = cs.Ab;
    if (a->feasible_whole) { s.feasible_whole = a->feasible_whole + ncw1 * lo[r]; s.cost_whole = a->cost_whole + ncw1 * lo[r]; }
    if (a->feasible_safe) { s.feasible_safe = a->feasible_safe + ncs1 * lo[r]; s.cost_safe = a->cost_safe + ncs1 * lo[r]; }
    if (a->coeffs_whole) s.coeffs_whole = a->coeffs_whole + 12 * (size_t)a->N_whole * lo[r];
    if (a->coeffs_safe) s.coeffs_safe = a->coeffs_safe + 12 * (size_t)a->N_safe * lo[r];
    s.results = a->results + lo[r];            // not copied back (copy_results = false): the gathered table is
    fq_pair_result* dr = nullptr;
    int rc = fq_replan_pairs_host_ex(c, &s, true, &dr, false);
    if (rc) { if (c != g) g->err = c->err; return rc; }
    e = cudaMemcpyAsync(d_res[i], dr, sizeof(fq_pair_result) * (size_t)n, cudaMemcpyDeviceToDevice, c->stream);
    if (e != cudaSuccess) return fq_cuda_fail(g, e, "gather staging");
  }
  if (int rc = exchange(g, d_res, d_all, (size_t)pad)) return rc;
  // ---- the gathered table, shard by shard, into the caller's results (from member 0 / this rank)
  FQ_CUDA(cudaSetDevice(g->device));
  for (int r = 0; r < world; r++)
    if (hi[r] > lo[r])
      FQ_CUDA(cudaMemcpyAsync(a->results + lo[r], d_all[0] + (size_t)r * pad, sizeof(fq_pair_result) * (size_t)(hi[r] - lo[r]),
                              cudaMemcpyDeviceToHost, g->stream));
  g->pending = true;
  if (deferred) return 0;
  for (int i = 0; i < n_local; i++)
    if (int rc = fq_settle(group ? member(g, i) : g)) return rc;
  return 0;
}

// fq_solve_multi on a multi-GPU context + the genNewTraj winner of every problem (the exchanged quantity)
extern "C" int fq_solve_multi_sharded(fq_ctx* g, int N, int force_final, int n_prob, const double* x0, const double* xf,
                                      const double* lim, const int* poly_ofs, const int* face_ofs, const double* Ab,
                                      const int* cand_ofs, const double* dt, const uint8_t* sigma, uint8_t* feasible,
                                      double* cost, int* win_idx, double* win_cost)
{
  if (!g) return FQ_E_ARG;
  fq_ctx* ctx = g;
  if (n_prob <= 0 || !x0 || !xf || !lim || !poly_ofs || !face_ofs || !cand_ofs || !dt || !feasible || !cost || !win_idx || !win_cost)
    return fq_fail(g, FQ_E_ARG, "bad arguments");
  if (poly_ofs[0] != 0 || face_ofs[0] != 0 || cand_ofs[0] != 0) return fq_fail(g, FQ_E_ARG, "offset arrays must start at 0");
  for (int j = 0; j < n_prob; j++)             // the shards are rebased on the host before the members validate theirs
    if (poly_ofs[j + 1] < poly_ofs[j] || cand_ofs[j + 1] < cand_ofs[j]) return fq_fail(g, FQ_E_ARG, "offset arrays not monotone");
  const int world = g->world;
  const bool group = g->is_group;
  const int n_local = group ? world : 1;
  struct Rec { double cost; int idx, pad; };
  int pad = 0;
  std::vector<int> lo(world), hi(world);
  for (int r = 0; r < world; r++) { fq_shard_range(n_prob, cand_ofs, r, world, &lo[r], &hi[r]); pad = std::max(pad, hi[r] - lo[r]); }
  std::vector<Rec*> d_res(n_local, nullptr), d_all(n_local, nullptr);
  std::vector<FqArena*> arenas(n_local, nullptr);
  for (int i = 0; i < n_local; i++)
  {
    fq_ctx* c = group ? member(g, i) : g;
    const int r = group ? i : g->rank;
    if (int rc = fq_settle(c)) return rc;
    cudaSetDevice(c->device);
    cudaError_t e = c->d_bnb.reserve(sizeof(Rec) * (size_t)pad * (world + 1));      // d_in / d_out belong to the solve
    if (e != cudaSuccess) return fq_cuda_fail(g, e, "gather buffer");
    d_res[i] = (Rec*)c->d_bnb.p;
    d_all[i] = d_res[i] + pad;
    e = cudaMemsetAsync(d_res[i], 0xff, sizeof(Rec) * (size_t)pad, c->stream);
    if (e != cudaSuccess) return fq_cuda_fail(g, e, "gather buffer");
    const int n = hi[r] - lo[r];
    if (n <= 0) continue;
    SubCorridors sc;
    sc.build(poly_ofs, face_ofs, Ab, lo[r], hi[r]);
    std::vector<int> co(n + 1);
    for (int j = 0; j <= n; j++) co[j] = cand_ofs[lo[r] + j] - cand_ofs[lo[r]];
    const size_t c0 = (size_t)cand_ofs[lo[r]];
    int* dwi = nullptr;
    double* dwc = nullptr;
    int rc = fq_solve_multi_host_ex(c, N, force_final, n, x0 + 9 * (size_t)lo[r], xf + 9 * (size_t)lo[r], lim + 3 * (size_t)lo[r],
                                    sc.poly_ofs.data(), sc.face_ofs.data(), sc.Ab, co.data(), dt + c0, sigma ? sigma + c0 * N : nullptr,
                                    feasible + c0, cost + c0, nullptr, nullptr, true, &dwi, &dwc);
    if (rc) { if (c != g) g->err = c->err; return rc; }
    // pack (cost, idx) records: two strided copies on the device
    e = cudaMemcpy2DAsync(&d_res[i][0].cost, sizeof(Rec), dwc, sizeof(double), sizeof(double), n, cudaMemcpyDeviceToDevice, c->stream);
    if (e == cudaSuccess)
      e = cudaMemcpy2DAsync(&d_res[i][0].idx, sizeof(Rec), dwi, sizeof(int), sizeof(int), n, cudaMemcpyDeviceToDevice, c->stream);
    if (e != cudaSuccess) return fq_cuda_fail(g, e, "winner records");
  }
  if (int rc = exchange(g, d_res, d_all, (size_t)pad)) return rc;
  FQ_CUDA(cudaSetDevice(g->device));
  std::vector<Rec> all((size_t)pad * world);
  FQ_CUDA(cudaMemcpyAsync(all.data(), d_all[0], sizeof(Rec) * all.size(), cudaMemcpyDeviceToHost, g->stream));
  g->pending = true;
  for (int i = 0; i < n_local; i++)
    if (int rc = fq_settle(group ? member(g, i) : g)) return rc;
  for (int r = 0; r < world; r++)
    for (int j = lo[r]; j < hi[r]; j++)
    {
      const Rec& q = all[(size_t)r * pad + (j - lo[r])];
      win_idx[j] = q.idx; win_cost[j] = q.cost;
    }
  return 0;
}
