// K7: windowed autocorrelation of periodogram windows (seismology ACF2D).
//   /root/reference/src/lightkurve/seismology/utils.py:137-160          autocorrelate
//   /root/reference/src/lightkurve/seismology/numax_estimators.py:170-182  the per-numax window loop
//   /root/reference/src/lightkurve/seismology/deltanu_estimators.py      its autocorrelate call
// For a window of n bins of one series, y = x[start:start+n] - nanmean(x[start:start+n]) and
//   acf_L = sum_{i < n-L} y_i y_{i+L},  L = 0 .. n-1       (np.correlate(y, y, "full")[n-1:])
//   metric = (sum_L |acf_L| - 1) / n
// Exact fp64 direct sums over the valid index pairs only, so a NaN in the window poisons exactly the lags numpy's
// do.  No atomics: every value is produced by a fixed sequence of operations that depends on the window alone, so
// a window's results are bitwise the same run to run and whatever else is in the batch.
//
// Kernels (one call):
//   acf_mean_kernel    one CTA per window: nanmean (sum and count of the non-NaN values, fixed reduction tree)
//   acf_corr_kernel    one CTA per (window, tile of ACF_TL lags), the dominant kernel.  The i range [0, n - L0) is
//                      walked in chunks of ACF_TI samples; a chunk stages y[i0 .. i0+TI) and y[i0+L0 .. i0+L0+TI+TL)
//                      in shared memory (windows of any length work).  Thread t owns the ACF_R consecutive lags
//                      L0 + t*R + r in registers and keeps a sliding window of 2R staged samples, so R broadcast
//                      loads and R strided loads feed R*R FMAs.  R is odd: the strided loads (R doubles apart)
//                      then fall in distinct banks within each half-warp.  Only the last steps of a thread's i
//                      range carry a predicate (the pairs with i + L >= n are skipped, not multiplied by zero).
//                      Writes sum_{lags of the tile} |acf_L| (fixed reduction tree) to its partial slot.
//   acf_metric_kernel  one thread per window: sums the window's partials in tile order into `metric`.
// Included by pgops.cu and by tests/native/acf_emu_driver.cpp (CPU emulator).
#pragma once
#include "common.cuh"

namespace lkb {

constexpr int ACF_THREADS = 128;
constexpr int ACF_R = 9;                          // lags per thread (odd, see above)
constexpr int ACF_TL = ACF_THREADS * ACF_R;       // lags per CTA: 1152
constexpr int ACF_TI = 64 * ACF_R;                // samples of i per staged chunk: 576

struct AcfWin {
  int64_t x0;        // first sample of the window in the concatenated series
  int64_t acf0;      // first lag of the window in the acf output (when requested)
  int64_t tile0;     // first lag tile of the window in the partial-sum array
  int64_t n;         // window length = lag count
};

__global__ void __launch_bounds__(256) acf_mean_kernel(const double* __restrict__ x, const AcfWin* __restrict__ win,
                                                       double* __restrict__ mean) {
  __shared__ double red[33];
  const AcfWin w = win[blockIdx.x];
  double s = 0.0, c = 0.0;
  for (int64_t i = threadIdx.x; i < w.n; i += blockDim.x) {
    const double v = x[w.x0 + i];
    if (v == v) { s += v; c += 1.0; }
  }
  s = block_sum(s, red);
  c = block_sum(c, red);
  if (threadIdx.x == 0) mean[blockIdx.x] = c > 0.0 ? s / c : __longlong_as_double(0x7ff8000000000000ll);
}

__global__ void __launch_bounds__(ACF_THREADS) acf_corr_kernel(const double* __restrict__ x,
                                                               const AcfWin* __restrict__ win,
                                                               const int64_t* __restrict__ tile_of, int W,
                                                               const double* __restrict__ mean,
                                                               double* __restrict__ partial, double* __restrict__ acf) {
  __shared__ double sa[ACF_TI];
  __shared__ double sb[ACF_TI + ACF_TL];
  __shared__ double red[33];
  const int64_t tile = blockIdx.x;
  int lo = 0, hi = W - 1;                         // the window of this tile: last w with tile_of[w] <= tile
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tile_of[mid] <= tile) lo = mid; else hi = mid - 1;
  }
  const AcfWin w = win[lo];
  const double mu = mean[lo];
  const int64_t n = w.n, L0 = (tile - w.tile0) * ACF_TL;
  const int t = threadIdx.x;
  const int64_t Lt = L0 + (int64_t)t * ACF_R;     // this thread's first lag
  double acc[ACF_R];
#pragma unroll
  for (int r = 0; r < ACF_R; ++r) acc[r] = 0.0;

  for (int64_t i0 = 0; i0 < n - L0; i0 += ACF_TI) {
    __syncthreads();
    for (int j = t; j < ACF_TI; j += ACF_THREADS) {
      const int64_t k = i0 + j;
      sa[j] = k < n ? x[w.x0 + k] - mu : 0.0;
    }
    for (int j = t; j < ACF_TI + ACF_TL; j += ACF_THREADS) {
      const int64_t k = i0 + L0 + j;
      sb[j] = k < n ? x[w.x0 + k] - mu : 0.0;
    }
    __syncthreads();
    // term (i0 + s*R + u, Lt + r) is valid iff s*R + u + r < lim
    const int64_t lim = n - i0 - Lt;
    if (lim <= 0) continue;
    const int steps = (int)min((int64_t)(ACF_TI / ACF_R), (lim + ACF_R - 1) / ACF_R);
    const int full = (int)min((int64_t)steps, max((int64_t)0, (lim - (2 * ACF_R - 2) + ACF_R - 1) / ACF_R));
    const double* bp = sb + t * ACF_R;
    double bcur[ACF_R], bnext[ACF_R];
#pragma unroll
    for (int k = 0; k < ACF_R; ++k) bcur[k] = bp[k];
    int s = 0;
    for (; s < full; ++s) {
      const double* ap = sa + s * ACF_R;
#pragma unroll
      for (int k = 0; k < ACF_R; ++k) bnext[k] = bp[(s + 1) * ACF_R + k];
#pragma unroll
      for (int u = 0; u < ACF_R; ++u) {
        const double av = ap[u];
#pragma unroll
        for (int r = 0; r < ACF_R; ++r) acc[r] = fma(av, u + r < ACF_R ? bcur[u + r] : bnext[u + r - ACF_R], acc[r]);
      }
#pragma unroll
      for (int k = 0; k < ACF_R; ++k) bcur[k] = bnext[k];
    }
    for (; s < steps; ++s) {                      // the last (at most two) steps: skip the pairs past the window
      const double* ap = sa + s * ACF_R;
      const int m = (int)(lim - (int64_t)s * ACF_R);
#pragma unroll
      for (int k = 0; k < ACF_R; ++k) bnext[k] = bp[(s + 1) * ACF_R + k];
#pragma unroll
      for (int u = 0; u < ACF_R; ++u) {
        const double av = ap[u];
#pragma unroll
        for (int r = 0; r < ACF_R; ++r)
          if (u + r < m) acc[r] = fma(av, u + r < ACF_R ? bcur[u + r] : bnext[u + r - ACF_R], acc[r]);
      }
#pragma unroll
      for (int k = 0; k < ACF_R; ++k) bcur[k] = bnext[k];
    }
  }

  double part = 0.0;
#pragma unroll
  for (int r = 0; r < ACF_R; ++r) {
    if (Lt + r < n) {
      part += fabs(acc[r]);
      if (acf) acf[w.acf0 + Lt + r] = acc[r];
    }
  }
  part = block_sum(part, red);
  if (t == 0) partial[tile] = part;
}

__global__ void __launch_bounds__(256) acf_metric_kernel(const AcfWin* __restrict__ win, int W,
                                                         const double* __restrict__ partial,
                                                         double* __restrict__ metric) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= W) return;
  const AcfWin v = win[w];
  const int64_t nt = (v.n + ACF_TL - 1) / ACF_TL;
  double s = 0.0;
  for (int64_t k = 0; k < nt; ++k) s += partial[v.tile0 + k];
  metric[w] = (s - 1.0) / (double)v.n;
}

// Launcher.  x/metric/acf follow `mem`; x_offsets [B+1], win_offsets [B+1], win_start [W], win_len [B] are host
// metadata.  Host mode stages through the workspace pool and returns with the outputs written.
inline int acf_windows_launch(const double* x, const int64_t* x_offsets, int B, const int64_t* win_offsets,
                              const int64_t* win_start, const int64_t* win_len, double* metric, double* acf,
                              int mem, cudaStream_t st) {
  LKB_REQUIRE(B >= 0, "lkb_acf_windows: negative batch size");
  if (B == 0) return LKB_OK;
  LKB_REQUIRE(x_offsets && win_offsets && win_len, "lkb_acf_windows: null metadata");
  LKB_REQUIRE(x_offsets[0] == 0 && win_offsets[0] == 0, "lkb_acf_windows: offsets must start at 0");
  for (int b = 0; b < B; ++b) {
    LKB_REQUIRE(x_offsets[b + 1] >= x_offsets[b] && win_offsets[b + 1] >= win_offsets[b],
                "lkb_acf_windows: negative series size or window count");
    LKB_REQUIRE(win_len[b] >= 1, "lkb_acf_windows: window length must be >= 1");
  }
  const int64_t W64 = win_offsets[B];
  LKB_REQUIRE(W64 < 2147483647, "lkb_acf_windows: too many windows");
  const int W = (int)W64;
  if (W == 0) return LKB_OK;
  LKB_REQUIRE(x && metric && win_start, "lkb_acf_windows: null argument");
  AcfWin* h_win = (AcfWin*)malloc(sizeof(AcfWin) * (size_t)W);
  int64_t* h_tile = (int64_t*)malloc(sizeof(int64_t) * (size_t)W);
  if (!h_win || !h_tile) {
    free(h_win);
    free(h_tile);
    set_error("lkb_acf_windows: host allocation failed");
    return LKB_E_OOM;
  }
  int64_t tiles = 0, lags = 0;
  int bad = -1;
  for (int b = 0; b < B && bad < 0; ++b) {
    const int64_t n = win_len[b], F = x_offsets[b + 1] - x_offsets[b];
    for (int64_t k = win_offsets[b]; k < win_offsets[b + 1]; ++k) {
      if (win_start[k] < 0 || win_start[k] > F - n) { bad = b; break; }
      h_win[k] = AcfWin{x_offsets[b] + win_start[k], lags, tiles, n};
      h_tile[k] = tiles;
      tiles += (n + ACF_TL - 1) / ACF_TL;
      lags += n;
    }
  }
  if (bad >= 0 || tiles >= 2147483647) {
    free(h_win);
    free(h_tile);
    if (bad >= 0) set_error("lkb_acf_windows: a window of series %d leaves the series (%s:%d)", bad, __FILE__, __LINE__);
    else set_error("lkb_acf_windows: too many lag tiles (%s:%d)", __FILE__, __LINE__);
    return LKB_E_ARG;
  }
  int rc = ensure_device();
  const double* d_x = nullptr;
  AcfWin* d_win = nullptr;
  int64_t* d_tile = nullptr;
  double *d_mean = nullptr, *d_part = nullptr, *d_metric = nullptr, *d_acf = nullptr;
  if (rc == LKB_OK) rc = stage_in<double>(mem, WS_IN0, x, (size_t)x_offsets[B], &d_x, st);
  if (rc == LKB_OK) rc = ws_get_t<AcfWin>(WS_A, (size_t)W, &d_win);
  if (rc == LKB_OK) rc = ws_get_t<int64_t>(WS_B, (size_t)W, &d_tile);
  if (rc == LKB_OK) rc = ws_get_t<double>(WS_C, (size_t)W, &d_mean);
  if (rc == LKB_OK) rc = ws_get_t<double>(WS_D, (size_t)tiles, &d_part);
  if (rc == LKB_OK) rc = stage_out_alloc<double>(mem, WS_OUT0, metric, (size_t)W, &d_metric);
  if (rc == LKB_OK) rc = stage_out_alloc<double>(mem, WS_OUT1, acf, (size_t)lags, &d_acf);
  // pageable sources: cudaMemcpyAsync returns once they have been read, so they can be freed right after
  if (rc == LKB_OK && cudaMemcpyAsync(d_win, h_win, sizeof(AcfWin) * W, cudaMemcpyHostToDevice, st) != cudaSuccess)
    rc = LKB_E_CUDA;
  if (rc == LKB_OK && cudaMemcpyAsync(d_tile, h_tile, sizeof(int64_t) * W, cudaMemcpyHostToDevice, st) != cudaSuccess)
    rc = LKB_E_CUDA;
  free(h_win);
  free(h_tile);
  if (rc == LKB_E_CUDA) set_error("lkb_acf_windows: metadata copy failed: %s", cudaGetErrorString(cudaGetLastError()));
  if (rc != LKB_OK) return rc;

  LKB_LAUNCH(W, 256, st, acf_mean_kernel)(d_x, d_win, d_mean);
  LKB_LAUNCH_CHECK();
  prof_begin(st);
  LKB_LAUNCH((unsigned)tiles, ACF_THREADS, st, acf_corr_kernel)(d_x, d_win, d_tile, W, d_mean, d_part, d_acf);
  LKB_LAUNCH_CHECK();
  prof_end(st);
  LKB_LAUNCH((W + 255) / 256, 256, st, acf_metric_kernel)(d_win, W, d_part, d_metric);
  LKB_LAUNCH_CHECK();
  LKB_TRY(stage_out_copy<double>(mem, metric, d_metric, (size_t)W, st));
  LKB_TRY(stage_out_copy<double>(mem, acf, d_acf, (size_t)lags, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

}  // namespace lkb
