// TEST INFRASTRUCTURE ONLY -- a lock-step emulation of one CUDA thread block on the host, so that the product's kernel SOURCE can be
// executed and checked in a container without a GPU (tests/test_kernel_emu_cpu.py).  Every CUDA thread is a fibre (ucontext) with
// its own stack; a fibre runs until it reaches a warp-collective (__shfl*_sync, __ballot_sync, __reduce_*_sync, __syncwarp, votes)
// or a block barrier (__syncthreads*), yields to the scheduler, and continues once every lane of its warp (every thread of the
// block) has arrived -- the semantics the kernel relies on with full masks.  Contributions are double-buffered per collective, so
// a lane that runs ahead to the next collective cannot overwrite what a slower lane still has to read.  Single OS thread: global
// "atomics" are plain read-modify-writes; shared memory is one static buffer (one block runs at a time).
#pragma once
#include <ucontext.h>

#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

#define __global__
#define __device__
#define __host__
#ifndef __shared__
#define __shared__            /* the dynamic shared array is one static buffer of the harness.  A translation unit whose
                                 kernels use static __shared__ variables defines it as `static`. */
#endif
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))

struct uint3 { unsigned x, y, z; };
struct dim3 { unsigned x = 1, y = 1, z = 1; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
struct alignas(16) double2 { double x, y; };
typedef int cudaError_t;
typedef void* cudaStream_t;
const cudaError_t cudaSuccess = 0, cudaErrorInvalidConfiguration = 9;

namespace simt
{
enum Wait { NONE = 0, WARP = 1, BLOCK = 2, DONE = 3 };
struct Fiber
{
  ucontext_t ctx;
  std::vector<char> stack;
  unsigned tid = 0;
  int wait = NONE;
  unsigned long long val[2] = { 0, 0 };     // contribution to the current / previous warp collective
  int phase = 0;
  int pred = 0;                             // contribution to __syncthreads_or
};
struct Block
{
  std::vector<Fiber> f;
  ucontext_t sched;
  int cur = 0;
  dim3 block, grid;
  uint3 bidx{ 0, 0, 0 };
  int block_or = 0;
  void (*entry)(void*) = nullptr;
  void* arg = nullptr;
};
inline Block* g = nullptr;
inline Fiber& self() { return g->f[(size_t)g->cur]; }
inline void yield(int kind)
{
  Fiber& me = self();
  me.wait = kind;
  swapcontext(&me.ctx, &g->sched);
}
// every lane stores `bits`, waits for its warp, then reads the lanes it needs from the same phase
inline int warp_arrive(unsigned long long bits)
{
  Fiber& me = self();
  const int ph = me.phase;
  me.val[ph] = bits;
  me.phase ^= 1;
  yield(WARP);
  return ph;
}
inline unsigned long long lane_val(int lane, int ph) { return g->f[(size_t)((g->cur & ~31) + (lane & 31))].val[ph]; }
inline int my_lane() { return g->cur & 31; }

}  // namespace simt

struct SimtIdx { unsigned x, y, z; };
inline SimtIdx simt_tid() { return SimtIdx{ simt::self().tid, 0, 0 }; }
#define threadIdx (simt_tid())
#define blockIdx (simt::g->bidx)
#define blockDim (simt::g->block)
#define gridDim (simt::g->grid)

// ---- warp collectives (full masks, as the kernel uses them)
template <class T>
inline unsigned long long simt_bits(T v) { unsigned long long b = 0; std::memcpy(&b, &v, sizeof(T)); return b; }
template <class T>
inline T simt_from(unsigned long long b) { T v; std::memcpy(&v, &b, sizeof(T)); return v; }
template <class T>
inline T __shfl_sync(unsigned, T v, int src) { const int ph = simt::warp_arrive(simt_bits(v)); return simt_from<T>(simt::lane_val(src, ph)); }
template <class T>
inline T __shfl_xor_sync(unsigned, T v, int m) { const int ph = simt::warp_arrive(simt_bits(v)); return simt_from<T>(simt::lane_val(simt::my_lane() ^ m, ph)); }
template <class T>
inline T __shfl_up_sync(unsigned, T v, unsigned d)
{
  const int ph = simt::warp_arrive(simt_bits(v));
  const int l = simt::my_lane();
  return l >= (int)d ? simt_from<T>(simt::lane_val(l - (int)d, ph)) : v;
}
inline unsigned __ballot_sync(unsigned, int p)
{
  const int ph = simt::warp_arrive((unsigned long long)(p != 0));
  unsigned r = 0;
  for (int l = 0; l < 32; l++) r |= (unsigned)(simt::lane_val(l, ph) & 1ull) << l;
  return r;
}
inline int __any_sync(unsigned m, int p) { return __ballot_sync(m, p) != 0; }
inline int __all_sync(unsigned m, int p) { return __ballot_sync(m, p) == 0xffffffffu; }
inline int __reduce_max_sync(unsigned, int v)
{
  const int ph = simt::warp_arrive(simt_bits(v));
  int r = v;
  for (int l = 0; l < 32; l++) { const int o = simt_from<int>(simt::lane_val(l, ph)); r = o > r ? o : r; }
  return r;
}
inline int __reduce_min_sync(unsigned, int v)
{
  const int ph = simt::warp_arrive(simt_bits(v));
  int r = v;
  for (int l = 0; l < 32; l++) { const int o = simt_from<int>(simt::lane_val(l, ph)); r = o < r ? o : r; }
  return r;
}
inline unsigned __reduce_min_sync(unsigned, unsigned v)
{
  const int ph = simt::warp_arrive(simt_bits(v));
  unsigned r = v;
  for (int l = 0; l < 32; l++) { const unsigned o = simt_from<unsigned>(simt::lane_val(l, ph)); r = o < r ? o : r; }
  return r;
}
inline unsigned __reduce_or_sync(unsigned, unsigned v)
{
  const int ph = simt::warp_arrive(simt_bits(v));
  unsigned r = 0;
  for (int l = 0; l < 32; l++) r |= simt_from<unsigned>(simt::lane_val(l, ph));
  return r;
}
inline void __syncwarp(unsigned = 0xffffffffu) { simt::warp_arrive(0); }
inline void __syncthreads() { simt::yield(simt::BLOCK); }
inline int __syncthreads_or(int p)
{
  simt::self().pred = p != 0;
  simt::yield(simt::BLOCK);
  return simt::g->block_or;
}
inline void __threadfence() {}
inline void __threadfence_system() {}

// ---- scalar intrinsics
inline int __ffs(unsigned v) { return v ? __builtin_ffs((int)v) : 0; }
inline int __double2hiint(double d) { return (int)(simt_bits(d) >> 32); }
inline int __double2loint(double d) { return (int)(simt_bits(d) & 0xffffffffull); }
inline double __hiloint2double(int hi, int lo) { return simt_from<double>(((unsigned long long)(unsigned)hi << 32) | (unsigned)lo); }
inline long long __double_as_longlong(double d) { return (long long)simt_bits(d); }
inline double __longlong_as_double(long long v) { return simt_from<double>((unsigned long long)v); }
template <class T>
inline T __ldg(const T* p) { return *p; }
inline double rsqrt(double x) { return 1.0 / std::sqrt(x); }
inline int max(int a, int b) { return a > b ? a : b; }
inline int min(int a, int b) { return a < b ? a : b; }
using std::fabs;
using std::fma;
using std::fmax;
using std::fmin;
inline int atomicAdd(int* p, int v) { const int o = *p; *p = o + v; return o; }
inline int atomicExch(int* p, int v) { const int o = *p; *p = v; return o; }
inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) { const unsigned long long o = *p; if (v < o) *p = v; return o; }
inline int atomicMin(int* p, int v) { const int o = *p; if (v < o) *p = v; return o; }
using std::isfinite;
inline unsigned long long atomicCAS(unsigned long long* p, unsigned long long c, unsigned long long v) { const unsigned long long o = *p; if (o == c) *p = v; return o; }

// ---- the scheduler: runs every fibre until it waits, releases warps / the block when all their live members have arrived
#include <cstdio>
namespace simt
{
inline void trampoline()
{
  Block* b = g;
  b->entry(b->arg);
  self().wait = DONE;
  swapcontext(&self().ctx, &b->sched);
}

inline void run_block(dim3 grid, dim3 block, uint3 bidx, void (*entry)(void*), void* arg, size_t stack_bytes = 512 * 1024)
{
  Block b;
  b.grid = grid; b.block = block; b.bidx = bidx; b.entry = entry; b.arg = arg;
  const int n = (int)block.x;
  b.f.resize((size_t)n);
  g = &b;
  for (int i = 0; i < n; i++)
  {
    Fiber& f = b.f[(size_t)i];
    f.tid = (unsigned)i;
    f.stack.resize(stack_bytes);
    getcontext(&f.ctx);
    f.ctx.uc_stack.ss_sp = f.stack.data();
    f.ctx.uc_stack.ss_size = f.stack.size();
    f.ctx.uc_link = &b.sched;
    makecontext(&f.ctx, trampoline, 0);
  }
  for (;;)
  {
    bool ran = false, all_done = true;
    for (int i = 0; i < n; i++)
    {
      if (b.f[(size_t)i].wait != NONE) continue;
      b.cur = i;
      swapcontext(&b.sched, &b.f[(size_t)i].ctx);
      ran = true;
    }
    // a warp whose live lanes all wait on a collective goes on
    for (int w = 0; w < n; w += 32)
    {
      int waiting = 0, live = 0;
      for (int l = w; l < w + 32 && l < n; l++) { live += b.f[(size_t)l].wait != DONE; waiting += b.f[(size_t)l].wait == WARP; }
      if (live && waiting == live)
        for (int l = w; l < w + 32 && l < n; l++) if (b.f[(size_t)l].wait == WARP) b.f[(size_t)l].wait = NONE;
    }
    int at_barrier = 0, live = 0, any = 0;
    for (int i = 0; i < n; i++)
    {
      const int wt = b.f[(size_t)i].wait;
      live += wt != DONE; at_barrier += wt == BLOCK; all_done = all_done && wt == DONE;
      if (wt == BLOCK) any |= b.f[(size_t)i].pred;
    }
    if (live && at_barrier == live)
    {
      b.block_or = any;
      for (int i = 0; i < n; i++) if (b.f[(size_t)i].wait == BLOCK) { b.f[(size_t)i].wait = NONE; b.f[(size_t)i].pred = 0; }
    }
    if (all_done) break;
    if (!ran)
    { // nobody could run and nothing was released in the previous round: a deadlock in the emulated code
      bool released = false;
      for (int i = 0; i < n; i++) released = released || b.f[(size_t)i].wait == NONE;
      if (!released) { std::fprintf(stderr, "simt_emu: deadlock (divergent collective?)\n"); std::abort(); }
    }
  }
  g = nullptr;
}
}  // namespace simt
