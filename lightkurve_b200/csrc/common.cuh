// Shared host/device helpers for liblkb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <math.h>
#include "../../include/lkb200.h"

namespace lkb {

// ---- error plumbing ---------------------------------------------------------
void set_error(const char* fmt, ...);
extern int64_t g_launches;
extern int g_last_ls_algo;
extern int g_last_flatten_path;
// ls_nufft.cu: light curves of the current / last shared-grid NUFFT call that took the double-precision pass
void ls_nufft_begin_call(cudaStream_t st);
int ls_nufft_last_escalated();
void ls_nufft_last_plan(int* out);
extern int64_t g_epoch;

#define LKB_CUDA_CHECK(expr)                                                        \
  do {                                                                              \
    cudaError_t _e = (expr);                                                        \
    if (_e != cudaSuccess) {                                                        \
      lkb::set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__,           \
                     cudaGetErrorString(_e));                                       \
      return (_e == cudaErrorMemoryAllocation) ? LKB_E_OOM : LKB_E_CUDA;            \
    }                                                                               \
  } while (0)

#define LKB_LAUNCH_CHECK()                                                          \
  do {                                                                              \
    lkb::g_launches++;                                                              \
    cudaError_t _e = cudaGetLastError();                                            \
    if (_e != cudaSuccess) {                                                        \
      lkb::set_error("kernel launch failed at %s:%d: %s", __FILE__, __LINE__,       \
                     cudaGetErrorString(_e));                                       \
      return LKB_E_CUDA;                                                            \
    }                                                                               \
  } while (0)

#define LKB_REQUIRE(cond, msg)                                                      \
  do {                                                                              \
    if (!(cond)) {                                                                  \
      lkb::set_error("%s (%s:%d)", msg, __FILE__, __LINE__);                        \
      return LKB_E_ARG;                                                             \
    }                                                                               \
  } while (0)

// Kernel launch.  tests/native/cuda_emu.h redefines this to run the grid on host threads, which is how the whole
// translation unit ls_nufft.cu (kernels AND launch orchestration) is executed and checked on a machine without a GPU.
#ifndef LKB_LAUNCH
#define LKB_LAUNCH(grid, block, stream, ...) __VA_ARGS__<<<(grid), (block), 0, (stream)>>>
#define LKB_LAUNCH_SMEM(grid, block, smem_bytes, stream, ...) __VA_ARGS__<<<(grid), (block), (smem_bytes), (stream)>>>
// the kernel's dynamic shared memory as `type* name`
#define LKB_DYN_SMEM(type, name)                                   \
  extern __shared__ __align__(16) unsigned char lkb_dyn_smem_raw[]; \
  type* name = reinterpret_cast<type*>(lkb_dyn_smem_raw)
#endif

#define LKB_TRY(expr)                                                               \
  do {                                                                              \
    int _s = (expr);                                                                \
    if (_s != LKB_OK) return _s;                                                    \
  } while (0)

// ---- workspace pool -----------------------------------------------------------
// Grow-only device buffers keyed by slot; freed by lkb_shutdown().  Not
// re-entrant across host threads (one engine context per process/device).
enum Slot {
  WS_A = 0, WS_B, WS_C, WS_D, WS_E, WS_F, WS_G, WS_H, WS_I, WS_J, WS_K, WS_L, WS_M, WS_N, WS_O, WS_P,
  WS_IN0, WS_IN1, WS_IN2, WS_IN3, WS_IN4, WS_IN5, WS_IN6, WS_IN7,
  WS_OUT0, WS_OUT1, WS_OUT2, WS_OUT3, WS_OUT4, WS_OUT5, WS_OUT6, WS_OUT7,
  WS_X0, WS_X1, WS_X2, WS_X3, WS_X4, WS_X5, WS_X6, WS_X7,
  WS_Y0, WS_Y1, WS_Y2, WS_Y3, WS_Y4, WS_Y5, WS_Y6, WS_Y7,
  WS_NSLOTS
};
int ws_get(int slot, size_t bytes, void** out);
template <typename T>
inline int ws_get_t(int slot, size_t count, T** out) {
  void* p = nullptr;
  int s = ws_get(slot, count * sizeof(T), &p);
  *out = reinterpret_cast<T*>(p);
  return s;
}
int ensure_device();
int sm_count();
// optional per-launch timing of the dominant kernel of a call (bench.py roofline):
// CUDA events recorded on the launching stream around that kernel when profiling is enabled.
void prof_begin(cudaStream_t st);
void prof_end(cudaStream_t st);
// Library-owned side stream + fork/join events: lets a small independent kernel (the LS window
// terms) run concurrently with the long contraction kernel on the caller's stream.
int aux_stream_get(cudaStream_t* aux, cudaEvent_t* ev_fork, cudaEvent_t* ev_join);
int pipe_streams_get(cudaStream_t* h2d, cudaStream_t* d2h, cudaEvent_t** events, int* n_events);

// Large host<->device copies of PAGEABLE memory (numpy arrays): the driver's own staging path was measured at
// ~3.5 GB/s (13 GB of flatten/regression inputs+outputs in 3.6 s), so they go through two page-locked bounce
// buffers filled/drained by a few host threads while the previous chunk is on the wire.  Page-locked caller
// buffers and small copies use cudaMemcpyAsync directly.  h2d: returns once the source has been read; d2h: returns
// once the destination is complete.
int big_copy_h2d(void* dst_dev, const void* src_host, size_t bytes, cudaStream_t st);
int big_copy_d2h(void* dst_host, const void* src_dev, size_t bytes, cudaStream_t st);

// Stage a host buffer into the pool (or pass a device pointer through).
template <typename T>
inline int stage_in(int mem, int slot, const T* src, size_t count, const T** out, cudaStream_t st) {
  if (src == nullptr) { *out = nullptr; return LKB_OK; }
  if (mem == LKB_MEM_DEVICE) { *out = src; return LKB_OK; }
  T* d = nullptr;
  LKB_TRY(ws_get_t<T>(slot, count ? count : 1, &d));
  if (count) LKB_TRY(big_copy_h2d(d, src, count * sizeof(T), st));
  *out = d;
  return LKB_OK;
}
template <typename T>
inline int stage_out_alloc(int mem, int slot, T* dst, size_t count, T** out) {
  if (dst == nullptr) { *out = nullptr; return LKB_OK; }
  if (mem == LKB_MEM_DEVICE) { *out = dst; return LKB_OK; }
  return ws_get_t<T>(slot, count ? count : 1, out);
}
template <typename T>
inline int stage_out_copy(int mem, T* dst, const T* dev, size_t count, cudaStream_t st) {
  if (dst == nullptr || mem == LKB_MEM_DEVICE || count == 0) return LKB_OK;
  return big_copy_d2h(dst, dev, count * sizeof(T), st);
}

// ---- device helpers --------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum of doubles; result valid in all threads.  `red` needs 33 doubles.
__device__ __forceinline__ double block_sum(double v, double* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  if (w == 0) {
    double x = (lane < nw) ? red[lane] : 0.0;
    x = warp_sum(x);
    if (lane == 0) red[32] = x;
  }
  __syncthreads();
  return red[32];
}
__device__ __forceinline__ long long block_sum_ll(long long v, long long* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  if (w == 0) {
    long long x = (lane < nw) ? red[lane] : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if (lane == 0) red[32] = x;
  }
  __syncthreads();
  return red[32];
}

}  // namespace lkb
