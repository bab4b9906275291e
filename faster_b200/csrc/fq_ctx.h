// Internal (not installed): the solver context behind the opaque fq_ctx of include/faster_b200.h and the helpers shared
// by the translation units of the C ABI (fq_capi.cu, fq_pair_capi.cu, fq_multi.cu).
#pragma once
#include "../../include/faster_b200.h"
#include "fq_kernels.cuh"
#include "fq_plan.h"

#include <map>
#include <string>
#include <vector>

struct FqPlanDev
{
  FqPlanHost h;
  double *TZ = nullptr, *T0 = nullptr, *FT = nullptr;
};

struct FqArena
{ // grow-only device buffer
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n)
  {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    size_t want = n + n / 4 + 4096;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

struct FqPinnedArena
{
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t reserve(size_t n)
  {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFreeHost(p);
    p = nullptr; cap = 0;
    size_t want = n + n / 4 + 4096;
    cudaError_t e = cudaMallocHost(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
};

struct FqComm;                    // fq_multi.cu: NCCL communicator(s) of a context (loaded lazily with dlopen)

struct fq_ctx
{
  int device = 0;
  cudaStream_t stream = nullptr, stream2 = nullptr;
  cudaEvent_t ev_head = nullptr;
  std::map<int, FqPlanDev> plans; // key N*2+force_final
  FqArena d_in, d_out, d_bnb, d_pair, d_pair_io;
  FqPinnedArena h_in, h_out;
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
// fq_pair_capi.cu.  d_results (may be NULL): receives the device address of the result records; copy_results = false
// leaves the caller's `results` array untouched (the multi-GPU path reads the all-gathered table instead)
int fq_replan_pairs_host_ex(fq_ctx* ctx, const fq_pair_args* a, bool deferred, fq_pair_result** d_results, bool copy_results);
// fq_multi.cu
void fq_comm_release(fq_ctx* ctx);
// all-gather on one context's communicator (one process per GPU): `bytes` from every rank, rank order
int fq_comm_allgather(fq_ctx* ctx, const void* d_send, void* d_recv, size_t bytes, cudaStream_t stream);
// fq_replan_pairs on a multi-GPU context (a group or a rank of a communicator)
int fq_replan_pairs_sharded(fq_ctx* g, const fq_pair_args* a, bool deferred);
