// Internal (not installed): the solver context behind the opaque fq_ctx of include/faster_b200.h and the helpers shared
// by the translation units of the C ABI (fq_capi.cu, fq_pair_capi.cu, fq_multi.cu).
#pragma once
#include "../../include/faster_b200.h"
#include "fq_kernels.cuh"
#include "fq_plan.h"

#include <cstring>
#include <map>
#include <string>
#include <vector>

struct FqPlanDev
{
  FqPlanHost h;
  double *TZ = nullptr, *T0 = nullptr, *FT = nullptr;
};

template <cudaError_t (*Alloc)(void**, size_t), cudaError_t (*Free)(void*)>
struct FqGrowArena
{ // grow-only buffer: device memory (FqArena) or pinned host memory (FqHostArena)
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n)
  {
    if (n <= cap) return cudaSuccess;
    if (p) Free(p);
    p = nullptr; cap = 0;
    size_t want = n + n / 4 + 4096;
    cudaError_t e = Alloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) Free(p); p = nullptr; cap = 0; }
};
using FqArena = FqGrowArena<cudaMalloc, cudaFree>;
using FqHostArena = FqGrowArena<cudaMallocHost, cudaFreeHost>;

struct FqComm;                    // fq_multi.cu: NCCL communicator(s) of a context (loaded lazily with dlopen)

struct fq_ctx
{
  int device = 0;
  cudaStream_t stream = nullptr, stream2 = nullptr;
  cudaEvent_t ev_head = nullptr;
  std::map<int, FqPlanDev> plans; // key N*2+force_final
  FqArena d_in, d_out, d_bnb, d_pair, d_pair_io;
  FqHostArena h_in, h_out;
  std::string err;
  bool force_generic = false;
  int sm_count = 0;
  int* d_counters = nullptr;      // ring of per-problem claim counters (one slot per launch in flight)
  int counters_cap = 0;           // problems per slot
  unsigned counters_pos = 0;
  bool pending = false;           // a deferred host-pointer call is still using the arenas (settled by the next call / fq_wait)
  int throughput_slices = 0;      // option "throughput_slices": launches a large host batch is cut into (0 = default 4)
  int max_poly_faces_hint = 0;    // option "max_faces_per_polytope" (device-pointer API only)
  double row_tol = FQ_ROW_TOL;    // option "row_tol_1e9": absolute row tolerance of every solve of this context
  bool early_exit = false;        // option "sweep_early_exit": candidates that cannot win genNewTraj's selection are skipped
  unsigned long long* d_first = nullptr;   // ring (as d_counters) of per-problem "smallest feasible dt so far"
  // ---- multi-GPU (fq_multi.cu)
  FqComm* comm = nullptr;         // communicator this context belongs to (one process per GPU), or nullptr
  int rank = 0, world = 1;
  std::vector<fq_ctx*> peers;     // fq_create_multi: the per-device contexts of a single-process group (this = peers[0]'s owner)
  bool is_group = false;
};
static const int kFqCounterSlots = 64;

// ---- helpers implemented in fq_capi.cu
int fq_fail(fq_ctx* c, int code, const std::string& msg);
int fq_cuda_fail(fq_ctx* c, cudaError_t e, const char* what);
#define FQ_CUDA(call)                                             \
  do {                                                            \
    cudaError_t e__ = (call);                                     \
    if (e__ != cudaSuccess) return fq_cuda_fail(ctx, e__, #call); \
  } while (0)
int fq_get_plan(fq_ctx* ctx, int N, int force_final, FqPlanDev** out);
void fq_fill_plan_args(const FqPlanDev& pd, FqKernelArgs* a);
// a deferred call owns the context's arenas until it has drained: every entry point that reuses them settles first
int fq_settle(fq_ctx* ctx);
// common launch of the batch solve.  `a` comes value-initialised with N, force_final, the problems and outputs (device
// pointers), max_faces and this launch's options (sorted_dt, ee_width, sweep_*, cert); the launch adds the plan tables,
// row_tol, item_cap (max_poly_faces <= 0: unknown) and the context's state.  *tail: the selection ran in the kernel's tail.
// early_exit_ok = false: this launch evaluates every candidate even with option "sweep_early_exit" set.
int fq_launch_solve_ctx(fq_ctx* ctx, FqKernelArgs a, int max_cand, int max_poly_faces, cudaStream_t stream, bool* tail = nullptr,
                        bool early_exit_ok = true);
inline size_t fq_align16(size_t x) { return (x + 15) & ~(size_t)15; }
// Places arrays in an arena, each on a 16-byte boundary (so that any of them can be read as double2).  A layout is one
// piece of code run twice: over a default FqPack, the sizing pass, which only counts the bytes (`at`; its pointers are
// NULL), and, once the arena holds that many, over place(), which returns typed pointers into the arena and copies every
// input's host data into the arena's pinned host mirror or, without one, straight into the arena on `stream`.  done()
// refuses a placement that did not end where the sizing pass did (nothing is copied past that end).
struct FqPack
{
  char* base = nullptr;                 // the arena (nullptr: the sizing pass)
  char* host = nullptr;                 // its pinned host mirror, or nullptr
  cudaStream_t stream = nullptr;
  size_t at = 0, sized = 0;             // bytes placed so far; bytes the sizing pass counted
  cudaError_t err = cudaSuccess;        // the first direct upload that failed
  FqPack place(void* arena, void* mirror = nullptr, cudaStream_t st = nullptr) const
  {
    FqPack p;
    p.base = (char*)arena; p.host = (char*)mirror; p.stream = st; p.sized = at;
    return p;
  }
  // room for count T (count 0 takes none: the pointer is not NULL, and is the next array's)
  template <class T> T* scratch(size_t count)
  {
    T* r = base ? reinterpret_cast<T*>(base + at) : nullptr;
    at = fq_align16(at + sizeof(T) * count);
    return r;
  }
  // room for an output the caller wants (want == NULL: not wanted, NULL)
  template <class T> T* out(T* want, size_t count) { return want ? scratch<T>(count) : nullptr; }
  // the arena's copy of the input src (NULL: NULL)
  template <class T> T* in(const T* src, size_t count)
  {
    if (!src) return nullptr;
    const size_t o = at, bytes = sizeof(T) * count;
    T* r = scratch<T>(count);
    if (base && bytes && at <= sized)
    {
      if (host) std::memcpy(host + o, src, bytes);
      else if (err == cudaSuccess) err = cudaMemcpyAsync(r, src, bytes, cudaMemcpyHostToDevice, stream);
    }
    return r;
  }
  // the host mirror's copy of the array at arena address p
  template <class T> T* mirror(T* p) const { return reinterpret_cast<T*>(host + ((const char*)p - base)); }
  int done(fq_ctx* ctx) const
  {
    if (at != sized) return fq_fail(ctx, FQ_E_CUDA, "internal: an arena layout placed another size than it reserved");
    if (err != cudaSuccess) return fq_cuda_fail(ctx, err, "cudaMemcpyAsync (upload)");
    return 0;
  }
};
// corridors of n_prob problems (problem j: polytopes poly_ofs[j] .. poly_ofs[j+1]-1; polytope p: rows face_ofs[p] ..
// face_ofs[p+1]-1 of Ab).  fq_scan_corridors checks that every polytope count is in 0..FQ_MAX_POLY and that face_ofs is
// monotone, and returns why it refuses the description, or nullptr.  Entries that stage the arrays as given also
// require both offset arrays to start at 0; the single-problem sweeps do not (they stage rows 0 .. face_ofs[P]-1).
struct FqCorridorSizes
{
  int max_faces = 0, max_poly_faces = 0;    // largest total faces of one problem / faces of one polytope
  int n_poly = 0, n_face = 0;               // poly_ofs[n_prob], face_ofs[n_poly]
};
const char* fq_scan_corridors(int n_prob, const int* poly_ofs, const int* face_ofs, FqCorridorSizes* sizes);
// fq_solve_multi_async + the genNewTraj winner of every problem, selected on the device (the arrays stay in the context's
// output arena until the next call): what the multi-GPU path all-gathers
int fq_solve_multi_host_ex(fq_ctx* ctx, int N, int force_final, int n_prob, const double* x0, const double* xf, const double* lim,
                           const int* poly_ofs, const int* face_ofs, const double* Ab, const int* cand_ofs, const double* dt,
                           const uint8_t* sigma, uint8_t* feasible, double* cost, double* coeffs, int32_t* iters, bool deferred,
                           int** d_win_idx, double** d_win_cost);
// fq_map.cu: the device address of a map's descriptor (fixed for the map's life, rewritten by every update), its device,
// and whether its last update succeeded
const FqMapDev* fq_map_descriptor(const fq_map* m);
int fq_map_device(const fq_map* m);
bool fq_map_valid(const fq_map* m);
// ---- multi-GPU contexts (fq_multi.cu; the chained replan's sharding is in fq_pair_capi.cu).  A sharded host entry
// checks the whole description and then every shard of the world on the host before it writes or enqueues anything, so
// every rank of a communicator makes the same decision and none is left waiting in the all-gather.
void fq_comm_release(fq_ctx* ctx);
// all-gather on one context's communicator (one process per GPU): `bytes` from every rank, rank order
int fq_comm_allgather(fq_ctx* ctx, const void* d_send, void* d_recv, size_t bytes, cudaStream_t stream);
// member i of a single-process group (member 0 is the group's own context)
inline fq_ctx* fq_member(fq_ctx* g, int i) { return i == 0 ? g : g->peers[i - 1]; }
// the one exchange of a sharded call: local member i (one for a rank context) sends `bytes` from send[i] and receives
// every rank's, in rank order, into recv[i].  Over the members of a single-process group, over a rank's communicator, or
// a copy for a world of one.
int fq_exchange(fq_ctx* g, const std::vector<void*>& send, const std::vector<void*>& recv, size_t bytes);
struct FqSubCorridors
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
