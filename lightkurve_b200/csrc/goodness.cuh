// K9: the goodness metrics of CBVCorrector.correct (/root/reference/src/lightkurve/correctors/metrics.py).
//
// Under-fitting metric (underfit_metric_neighbors, metrics.py:178-255, and _compute_correlation): target b is compared
// with its M neighbours, rows of a pool [P, G] on a common cadence grid.  A cadence takes part when neither the target
// nor ANY of its neighbours is NaN there; over those n cadences
//   rms_i = sqrt(sum x_i^2 / n) (0 -> inf),   c_i = sum x_i t / (rms_i rms_t) / n,
//   C3 = nanmean(|c_0|^3 .. |c_{M-1}|^3, 0)   (the zeroed diagonal stays in the mean: divide by M + 1),
//   metric = 2 / (1 + exp(C3 log(2 / 0.95 - 1) / (0.0007 + 0.8083 n^-0.5023))).
//   gm_nan_bits_kernel   one bit per cadence, set where the value is not NaN, for every pool and target row
//                        (G / 8 bytes per row: the cadence union of M neighbours costs M G / 8 bytes, not 8 M G)
//   gm_underfit_kernel   one CTA per target: AND of the bit rows into shared memory, then warp i (mod 8) streams
//                        neighbour i once: dot and sum of squares over the surviving cadences
// Over-fitting terms (overfit_metric_lombscargle, metrics.py:23-123): per light curve, from fp32 power rows,
//   n_positive = #{corrected - original > 0},  sum_positive = sum of those differences (fp64),
//   noise_mean[s] = nanmean(noise power row s).
//   gm_overfit_kernel    one CTA per (light curve, row): y = 0 the differences, y = 1 + s noise row s
//
// Every sum is a fixed tree (per-thread strided partial sums, then warp_sum / block_sum), no atomics: results are
// bitwise repeatable and a light curve's results do not depend on the rest of the batch.  No inline PTX:
// tests/native/cuda_emu.h runs this file on the CPU (tests/test_goodness_emulated.py).
#pragma once
#include "common.cuh"

namespace lkb {

constexpr int GM_THREADS = 256;
constexpr size_t GM_SMEM_MAX = 227 * 1024;

__host__ __device__ inline int64_t gm_words(int64_t G) { return (G + 31) / 32; }

// bits[r, w] bit j: x[r, 32 w + j] is not NaN (bits past G are 0).  grid = (ceil(W / 8), rows), 8 warps = 8 words.
__global__ void __launch_bounds__(GM_THREADS)
gm_nan_bits_kernel(const double* __restrict__ x, int64_t G, uint32_t* __restrict__ bits) {
  const int64_t W = gm_words(G);
  const int64_t r = blockIdx.y;
  const int64_t w = (int64_t)blockIdx.x * (GM_THREADS / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int64_t g = w * 32 + lane;
  const bool ok = w < W && g < G && !isnan(x[r * G + g]);
  const unsigned m = __ballot_sync(0xffffffffu, ok);
  if (lane == 0 && w < W) bits[r * W + w] = m;
}

// Dynamic shared memory: valid [W] uint32 | dot [M] | ss [M] | nb [M] int32 (doubles first for alignment).
inline size_t gm_underfit_smem(int64_t G, int M) {
  return (size_t)M * 2 * sizeof(double) + (size_t)M * sizeof(int32_t) + (size_t)gm_words(G) * sizeof(uint32_t);
}

__global__ void __launch_bounds__(GM_THREADS)
gm_underfit_kernel(const double* __restrict__ pool, const uint32_t* __restrict__ pool_bits,
                   const double* __restrict__ target, const uint32_t* __restrict__ target_bits, int64_t G,
                   const int64_t* __restrict__ nb_off, const int32_t* __restrict__ nb_idx, double* __restrict__ metric,
                   int32_t* __restrict__ n_used, double* __restrict__ c3_mean) {
  LKB_DYN_SMEM(double, s_dot);
  __shared__ double s_red[33];
  __shared__ long long s_redl[33];
  const int b = blockIdx.x;
  const int64_t W = gm_words(G);
  const int M = (int)(nb_off[b + 1] - nb_off[b]);
  double* s_ss = s_dot + M;
  int32_t* s_nb = reinterpret_cast<int32_t*>(s_ss + M);
  uint32_t* s_valid = reinterpret_cast<uint32_t*>(s_nb + M);
  for (int i = threadIdx.x; i < M; i += blockDim.x) s_nb[i] = nb_idx[nb_off[b] + i];
  __syncthreads();
  // cadences where the target and every neighbour are present
  long long cnt = 0;
  for (int64_t w = threadIdx.x; w < W; w += blockDim.x) {
    uint32_t v = target_bits[(int64_t)b * W + w];
    for (int i = 0; i < M; ++i) v &= pool_bits[(int64_t)s_nb[i] * W + w];
    s_valid[w] = v;
    cnt += __popc(v);
  }
  const long long n = block_sum_ll(cnt, s_redl);          // (its barriers also publish s_valid)
  const double* t = target + (int64_t)b * G;
  double tt = 0.0;
  for (int64_t g = threadIdx.x; g < G; g += blockDim.x)
    if ((s_valid[g >> 5] >> (g & 31)) & 1u) tt = fma(t[g], t[g], tt);
  tt = block_sum(tt, s_red);
  // warp w: neighbours w, w + 8, ...; four independent partial sums per lane (unrolled loads), combined in order
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int i = warp; i < M; i += nw) {
    const double* x = pool + (int64_t)s_nb[i] * G;
    double d[4] = {0.0, 0.0, 0.0, 0.0}, q[4] = {0.0, 0.0, 0.0, 0.0};
    int64_t g0 = 0;
    for (; g0 + 128 <= G; g0 += 128) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t g = g0 + 32 * u + lane;
        if ((s_valid[g >> 5] >> (g & 31)) & 1u) {
          const double xv = x[g];
          d[u] = fma(xv, t[g], d[u]);
          q[u] = fma(xv, xv, q[u]);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {                      // the tail (< 128 cadences)
      const int64_t g = g0 + 32 * u + lane;
      if (g < G && ((s_valid[g >> 5] >> (g & 31)) & 1u)) {
        const double xv = x[g];
        d[u] = fma(xv, t[g], d[u]);
        q[u] = fma(xv, xv, q[u]);
      }
    }
    const double dd = warp_sum((d[0] + d[1]) + (d[2] + d[3]));
    const double qq = warp_sum((q[0] + q[1]) + (q[2] + q[3]));
    if (lane == 0) { s_dot[i] = dd; s_ss[i] = qq; }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const double nc = (double)n;
    double rt = sqrt(tt / nc);
    if (rt == 0.0) rt = INFINITY;
    double sum = 0.0;
    int cntc = 1;                                        // the zeroed diagonal entry
    for (int i = 0; i < M; ++i) {
      double ri = sqrt(s_ss[i] / nc);
      if (ri == 0.0) ri = INFINITY;
      const double c = s_dot[i] / (ri * rt) / nc;
      if (!isnan(c)) {
        const double a = fabs(c);
        sum = fma(a * a, a, sum);                        // explicit: nvcc contracts a * b + c, the host build does not
        ++cntc;
      }
    }
    const double c3 = sum / (double)cntc;
    const double wgn = fma(0.8083, pow(nc, -0.5023), 0.0007);
    const double scale = 1.0 / wgn * log(2.0 / 0.95 - 1.0);
    metric[b] = 2.0 / (1.0 + exp(scale * c3));
    if (n_used) n_used[b] = (int32_t)n;
    if (c3_mean) c3_mean[b] = c3;
  }
}

// grid = (B, 1 + S).  offsets [B + 1] on the device (row b of the corrected / original power at offsets[b]; noise row
// s of light curve b at S offsets[b] + s len_b).
__global__ void __launch_bounds__(GM_THREADS)
gm_overfit_kernel(const float* __restrict__ corrected, const float* __restrict__ original,
                  const float* __restrict__ noise, const int64_t* __restrict__ offsets, int S,
                  int32_t* __restrict__ n_positive, double* __restrict__ sum_positive, double* __restrict__ noise_mean) {
  __shared__ double s_red[33];
  __shared__ long long s_redl[33];
  const int b = blockIdx.x, row = blockIdx.y;
  const int64_t o = offsets[b], len = offsets[b + 1] - o;
  double acc = 0.0;
  long long cnt = 0;
  if (row == 0) {
    for (int64_t k = threadIdx.x; k < len; k += blockDim.x) {
      const double d = (double)corrected[o + k] - (double)original[o + k];
      if (d > 0.0) { acc += d; ++cnt; }
    }
  } else {
    const float* p = noise + (int64_t)S * o + (int64_t)(row - 1) * len;
    for (int64_t k = threadIdx.x; k < len; k += blockDim.x) {
      const double v = (double)p[k];
      if (!isnan(v)) { acc += v; ++cnt; }
    }
  }
  acc = block_sum(acc, s_red);
  cnt = block_sum_ll(cnt, s_redl);
  if (threadIdx.x == 0) {
    if (row == 0) {
      n_positive[b] = (int32_t)cnt;
      sum_positive[b] = acc;
    } else {
      noise_mean[(int64_t)b * S + row - 1] = acc / (double)cnt;
    }
  }
}

// Both launchers take device buffers (offsets and neighbour lists included); h_nb_off is the host copy of nb_off, used
// for the shared-memory size.  pool_bits [P, W] and target_bits [B, W] are scratch.
inline int gm_underfit_launch(const double* pool, int P, const double* target, int B, int64_t G, const int64_t* nb_off,
                              const int32_t* nb_idx, const int64_t* h_nb_off, uint32_t* pool_bits, uint32_t* target_bits,
                              double* metric, int32_t* n_used, double* c3_mean, cudaStream_t st) {
  int Mmax = 0;
  for (int b = 0; b < B; ++b) {
    const int64_t m = h_nb_off[b + 1] - h_nb_off[b];
    Mmax = m > Mmax ? (int)m : Mmax;
  }
  const size_t smem = gm_underfit_smem(G, Mmax);
  if (smem > GM_SMEM_MAX) {
    set_error("lkb_underfit_metric: %lld cadences and %d neighbours need %zu bytes of shared memory", (long long)G,
              Mmax, smem);
    return LKB_E_UNSUPPORTED;
  }
  static size_t attr = 0;
  if (smem > attr) {
    LKB_CUDA_CHECK(cudaFuncSetAttribute(gm_underfit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = smem;
  }
  const unsigned wblocks = (unsigned)((gm_words(G) + GM_THREADS / 32 - 1) / (GM_THREADS / 32));
  LKB_LAUNCH(dim3(wblocks, (unsigned)P), GM_THREADS, st, gm_nan_bits_kernel)(pool, G, pool_bits);
  LKB_LAUNCH_CHECK();
  LKB_LAUNCH(dim3(wblocks, (unsigned)B), GM_THREADS, st, gm_nan_bits_kernel)(target, G, target_bits);
  LKB_LAUNCH_CHECK();
  LKB_LAUNCH_SMEM((unsigned)B, GM_THREADS, smem, st, gm_underfit_kernel)(pool, pool_bits, target, target_bits, G, nb_off,
                                                                         nb_idx, metric, n_used, c3_mean);
  LKB_LAUNCH_CHECK();
  return LKB_OK;
}

inline int gm_overfit_launch(const float* corrected, const float* original, const float* noise, const int64_t* offsets,
                             int B, int S, int32_t* n_positive, double* sum_positive, double* noise_mean,
                             cudaStream_t st) {
  LKB_LAUNCH(dim3((unsigned)B, (unsigned)(1 + S)), GM_THREADS, st, gm_overfit_kernel)(
      corrected, original, noise, offsets, S, n_positive, sum_positive, noise_mean);
  LKB_LAUNCH_CHECK();
  return LKB_OK;
}

}  // namespace lkb
