// Minimal CUDA-on-CPU execution layer (TEST INFRASTRUCTURE): lets g++ compile a .cu translation unit of this repo
// unchanged and run its kernels - every thread of a block is a host thread, so __syncthreads() and warp shuffles
// work; blocks run one after the other.  Only what lightkurve_b200/csrc/ls_nufft.cu needs is provided.
// Used by tests/native/nufft_emu_driver.cpp: the kernels AND the launch orchestration of the NUFFT Lomb-Scargle path
// are executed here and compared with the fp64 oracle (tests/test_nufft_emulated.py).
#pragma once
#define LKB_CUDA_EMU 1
#include <cuda_runtime.h>      // types only: float2/float4/dim3/uint3, cudaStream_t, cudaError_t, prototypes
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <condition_variable>
#include <mutex>
#include <thread>
#include <vector>

#undef __shared__
#define __shared__ static
#ifndef __launch_bounds__
#define __launch_bounds__(...)
#endif
#ifndef __noinline__
#define __noinline__ __attribute__((noinline))
#endif          // one block at a time: a function-local static IS the block's shared memory

namespace lkb_emu {

struct Barrier {                   // reusable barrier whose participants may leave (a thread that returns early)
  std::mutex m;
  std::condition_variable cv;
  int expected = 0, waiting = 0;
  long generation = 0;
  void reset(int n) { expected = n; waiting = 0; }
  void wait() {
    std::unique_lock<std::mutex> lk(m);
    const long gen = generation;
    if (++waiting >= expected) { waiting = 0; ++generation; cv.notify_all(); return; }
    cv.wait(lk, [&] { return gen != generation; });
  }
  void leave() {
    std::unique_lock<std::mutex> lk(m);
    --expected;
    if (expected > 0 && waiting >= expected) { waiting = 0; ++generation; cv.notify_all(); }
  }
};

struct Block {
  Barrier all;
  std::vector<Barrier> warp;
  std::vector<unsigned long long> scratch;      // 32 slots per warp
  std::vector<unsigned char> alive;             // per thread
  std::vector<int> vote;                        // per thread (__syncthreads_and)
  std::vector<unsigned long long> dyn;          // dynamic shared memory of the block
};

inline thread_local Block* t_block = nullptr;
inline thread_local int t_tid = 0;
inline std::mutex g_atomic_mu;

template <typename F>
struct Launcher {
  dim3 grid, block;
  size_t smem_bytes;
  F body;
  template <typename... Args>
  void operator()(Args... args);
};
template <typename F>
Launcher<F> make_launcher(dim3 grid, dim3 block, size_t smem, F body) { return Launcher<F>{grid, block, smem, body}; }

}  // namespace lkb_emu

inline thread_local uint3 threadIdx, blockIdx;
inline thread_local dim3 blockDim, gridDim;

template <typename F>
template <typename... Args>
void lkb_emu::Launcher<F>::operator()(Args... args) {
  const int nthreads = (int)(block.x * block.y * block.z);
  const int nwarps = (nthreads + 31) / 32;
  for (unsigned bz = 0; bz < grid.z; ++bz)
    for (unsigned by = 0; by < grid.y; ++by)
      for (unsigned bx = 0; bx < grid.x; ++bx) {
        Block blk;
        blk.all.reset(nthreads);
        blk.warp = std::vector<Barrier>(nwarps);
        for (int w = 0; w < nwarps; ++w) blk.warp[w].reset(std::min(32, nthreads - 32 * w));
        blk.scratch.assign((size_t)nwarps * 32, 0ull);
        blk.alive.assign(nthreads, 1);
        blk.vote.assign(nthreads, 1);
        blk.dyn.assign(smem_bytes / 8 + 2, 0ull);
        std::vector<std::thread> th;
        th.reserve(nthreads);
        for (int t = 0; t < nthreads; ++t)
          th.emplace_back([&, t] {
            t_block = &blk;
            t_tid = t;
            threadIdx.x = t % block.x;
            threadIdx.y = (t / block.x) % block.y;
            threadIdx.z = t / (block.x * block.y);
            blockIdx.x = bx; blockIdx.y = by; blockIdx.z = bz;
            blockDim = block;
            gridDim = grid;
            body(args...);
            blk.alive[t] = 0;
            blk.warp[t / 32].leave();
            blk.all.leave();
          });
        for (auto& x : th) x.join();
      }
}

#define LKB_LAUNCH(grid, block, stream, ...) \
  lkb_emu::make_launcher(dim3(grid), dim3(block), 0, [&](auto... emu_args) { __VA_ARGS__(emu_args...); })
#define LKB_LAUNCH_SMEM(grid, block, smem_bytes, stream, ...) \
  lkb_emu::make_launcher(dim3(grid), dim3(block), (smem_bytes), [&](auto... emu_args) { __VA_ARGS__(emu_args...); })
#define LKB_DYN_SMEM(type, name) type* name = reinterpret_cast<type*>(lkb_emu::t_block->dyn.data())

// ---- device built-ins ------------------------------------------------------------------------------------
inline void __syncthreads() { lkb_emu::t_block->all.wait(); }
// the AND of `pred` over the block's threads that have not returned
inline int __syncthreads_and(int pred) {
  lkb_emu::Block* b = lkb_emu::t_block;
  b->vote[lkb_emu::t_tid] = pred ? 1 : 0;
  b->all.wait();
  int out = 1;
  for (size_t t = 0; t < b->vote.size(); ++t)
    if (b->alive[t] && !b->vote[t]) out = 0;
  b->all.wait();
  return out;
}

template <typename T>
inline T __shfl_xor_sync(unsigned, T v, int lane_mask) {
  static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes");
  lkb_emu::Block* b = lkb_emu::t_block;
  const int t = lkb_emu::t_tid, w = t / 32, lane = t % 32, other = lane ^ lane_mask;
  unsigned long long bits = 0;
  memcpy(&bits, &v, sizeof(T));
  b->scratch[(size_t)w * 32 + lane] = bits;
  b->warp[w].wait();
  T out = v;
  const int ot = w * 32 + other;
  if (other < 32 && ot < (int)b->alive.size() && b->alive[ot]) {
    const unsigned long long ob = b->scratch[(size_t)w * 32 + other];
    memcpy(&out, &ob, sizeof(T));
  }
  b->warp[w].wait();
  return out;
}

template <typename T>
inline T __shfl_up_sync(unsigned, T v, int delta) {
  static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes");
  lkb_emu::Block* b = lkb_emu::t_block;
  const int t = lkb_emu::t_tid, w = t / 32, lane = t % 32, other = lane - delta;
  unsigned long long bits = 0;
  memcpy(&bits, &v, sizeof(T));
  b->scratch[(size_t)w * 32 + lane] = bits;
  b->warp[w].wait();
  T out = v;
  if (other >= 0 && b->alive[w * 32 + other]) {
    const unsigned long long ob = b->scratch[(size_t)w * 32 + other];
    memcpy(&out, &ob, sizeof(T));
  }
  b->warp[w].wait();
  return out;
}
template <typename T>
inline T __shfl_sync(unsigned, T v, int src_lane) {
  static_assert(sizeof(T) <= 8, "shuffle of at most 8 bytes");
  lkb_emu::Block* b = lkb_emu::t_block;
  const int t = lkb_emu::t_tid, w = t / 32, lane = t % 32;
  unsigned long long bits = 0;
  memcpy(&bits, &v, sizeof(T));
  b->scratch[(size_t)w * 32 + lane] = bits;
  b->warp[w].wait();
  T out = v;
  const unsigned long long ob = b->scratch[(size_t)w * 32 + (src_lane & 31)];
  memcpy(&out, &ob, sizeof(T));
  b->warp[w].wait();
  return out;
}
inline unsigned __ballot_sync(unsigned, int pred) {
  lkb_emu::Block* b = lkb_emu::t_block;
  const int t = lkb_emu::t_tid, w = t / 32, lane = t % 32;
  b->scratch[(size_t)w * 32 + lane] = pred ? 1ull : 0ull;
  b->warp[w].wait();
  unsigned out = 0;
  for (int l = 0; l < 32; ++l) {
    const int ot = w * 32 + l;
    if (ot < (int)b->alive.size() && b->alive[ot] && b->scratch[(size_t)w * 32 + l]) out |= 1u << l;
  }
  b->warp[w].wait();
  return out;
}
inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
inline unsigned __match_any_sync(unsigned, int value) {
  lkb_emu::Block* b = lkb_emu::t_block;
  const int t = lkb_emu::t_tid, w = t / 32, lane = t % 32;
  b->scratch[(size_t)w * 32 + lane] = (unsigned long long)(long long)value;
  b->warp[w].wait();
  unsigned out = 0;
  for (int l = 0; l < 32; ++l) {
    const int ot = w * 32 + l;
    if (ot < (int)b->alive.size() && b->alive[ot] && b->scratch[(size_t)w * 32 + l] == (unsigned long long)(long long)value)
      out |= 1u << l;
  }
  b->warp[w].wait();
  return out;
}
inline void __syncwarp(unsigned = 0xffffffffu) { lkb_emu::t_block->warp[lkb_emu::t_tid / 32].wait(); }
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline int __clz(int x) { return x == 0 ? 32 : __builtin_clz((unsigned)x); }
inline int __ffs(int x) { return __builtin_ffs(x); }
inline unsigned __fns(unsigned mask, unsigned base, int offset) {      // offset-th set bit at or above `base` (offset > 0)
  if (offset <= 0) return 0xffffffffu;
  for (unsigned bpos = base; bpos < 32; ++bpos)
    if ((mask >> bpos) & 1u) { if (--offset == 0) return bpos; }
  return 0xffffffffu;
}
inline long long __double_as_longlong(double v) { long long r; memcpy(&r, &v, 8); return r; }
inline double __longlong_as_double(long long v) { double r; memcpy(&r, &v, 8); return r; }
inline double atomicAdd(double* addr, double v) {
  std::lock_guard<std::mutex> lk(lkb_emu::g_atomic_mu);
  const double old = *addr;
  *addr = old + v;
  return old;
}
inline int atomicAdd(int* addr, int v) {
  std::lock_guard<std::mutex> lk(lkb_emu::g_atomic_mu);
  const int old = *addr;
  *addr = old + v;
  return old;
}

inline unsigned atomicMax(unsigned* addr, unsigned v) {
  std::lock_guard<std::mutex> lk(lkb_emu::g_atomic_mu);
  const unsigned old = *addr;
  if (v > old) *addr = v;
  return old;
}
inline int atomicMax(int* addr, int v) {
  std::lock_guard<std::mutex> lk(lkb_emu::g_atomic_mu);
  const int old = *addr;
  if (v > old) *addr = v;
  return old;
}

inline void sincospif(float x, float* s, float* c) { const double a = 3.14159265358979323846 * (double)x; *s = (float)sin(a); *c = (float)cos(a); }
inline void sincospi(double x, double* s, double* c) { const double a = 3.14159265358979323846 * x; *s = sin(a); *c = cos(a); }
inline float __sinf(float x) { return sinf(x); }
inline float __cosf(float x) { return cosf(x); }
inline float __expf(float x) { return expf(x); }
inline double __dadd_rn(double a, double b) { volatile double r = a + b; return r; }
inline double __dsub_rn(double a, double b) { volatile double r = a - b; return r; }
inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
inline float __int_as_float(int u) { float f; memcpy(&f, &u, 4); return f; }
inline int __float_as_int(float f) { int u; memcpy(&u, &f, 4); return u; }
inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
inline unsigned long long __double2ull_rd(double x) { return (unsigned long long)floor(x); }
template <typename A, typename B>
inline auto min(A a, B b) -> decltype(a + b) { return a < b ? a : b; }
template <typename A, typename B>
inline auto max(A a, B b) -> decltype(a + b) { return a > b ? a : b; }

// ---- the few runtime calls ls_nufft.cu makes: "device" memory is host memory ------------------------------------
extern "C" {
inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { memset(p, v, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) { memcpy(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaDeviceSynchronize(void) { return cudaSuccess; }
inline cudaError_t cudaGetLastError(void) { return cudaSuccess; }
inline const char* cudaGetErrorString(cudaError_t) { return "emulated"; }
inline cudaError_t cudaFuncSetAttribute(const void*, cudaFuncAttribute, int) { return cudaSuccess; }
}
template <typename T>
inline cudaError_t cudaFuncSetAttribute(T*, cudaFuncAttribute, int) { return cudaSuccess; }   // kernel-pointer form
extern "C" {
}
