// Periodogram post-processing for the step after Lomb-Scargle (asteroseismology chain):
//   /root/reference/src/lightkurve/periodogram.py:260-284  Periodogram.smooth(method="logmedian")
//   /root/reference/src/lightkurve/periodogram.py:381-429  Periodogram.flatten  (power / background)
// The reference walks a window of half-width filter_width in log10(frequency) across the spectrum in
// steps of filter_width / 2 and, for every window, adds nanmedian(power[window]) / (8/9)^3 to the bins in it;
// the background is that sum divided by the number of windows that covered the bin.
//
// The window list (start bin, end bin) is built on the host from the shared frequency grid with the
// reference's own expression (the x0 += 0.5 w accumulation must be reproduced in fp64); the GPU does the
// B x W exact medians (K6 radix select, one CTA per (window, periodogram)) and the per-bin combination
// in the reference's summation order (ascending window index).
//
// The seismology estimators that read the flattened periodogram (numax / deltanu ACF2D) run on the K7 windowed
// autocorrelation kernels of acf.cuh; lkb_acf_windows enters through acf_windows below.
#include "common.cuh"
#include "select.cuh"
#include "acf.cuh"

namespace lkb {

__global__ void __launch_bounds__(256)
pg_window_median_kernel(const double* __restrict__ power, int64_t F, const int32_t* __restrict__ win_lo,
                        const int32_t* __restrict__ win_hi, int W, double* __restrict__ med) {
  __shared__ SelSmem sm;
  const int w = blockIdx.x, b = blockIdx.y;
  const int lo = win_lo[w], n = win_hi[w] - lo;
  const double* p = power + (int64_t)b * F + lo;
  double m;
  if (n <= 0) {
    m = __longlong_as_double(0x7ff8000000000000ll);
  } else if (n <= 32) {
    // tiny windows (the low-frequency end of a linear grid): rank by counting inside warp 0
    m = 0.0;
    if (threadIdx.x < 32) {
      const int lane = threadIdx.x;
      const double v = lane < n ? p[lane] : __longlong_as_double(0x7ff8000000000000ll);
      const bool ok = v == v;
      const int cnt = __popc(__ballot_sync(0xffffffffu, ok));
      int rank = 0;
      for (int j = 0; j < 32; ++j) {
        const double u = __shfl_sync(0xffffffffu, v, j);
        if (u == u && (u < v || (u == v && j < lane))) rank++;
      }
      const int klo = (cnt - 1) / 2, khi = cnt / 2;
      const unsigned mlo = __ballot_sync(0xffffffffu, ok && rank == klo);
      const unsigned mhi = __ballot_sync(0xffffffffu, ok && rank == khi);
      double vlo = __shfl_sync(0xffffffffu, v, mlo ? __ffs(mlo) - 1 : 0);
      double vhi = __shfl_sync(0xffffffffu, v, mhi ? __ffs(mhi) - 1 : 0);
      m = cnt ? (vlo + vhi) / 2.0 : __longlong_as_double(0x7ff8000000000000ll);
    }
  } else {
    m = block_nanmedian([&](int64_t i) { return p[i]; }, n, sm);
  }
  if (threadIdx.x == 0) med[(int64_t)b * W + w] = m;
}

__global__ void __launch_bounds__(256)
pg_window_combine_kernel(const double* __restrict__ med, int64_t F, const int32_t* __restrict__ win_lo,
                         const int32_t* __restrict__ win_hi, int W, double inv_corr, double* __restrict__ bkg) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= F) return;
  // windows are ordered by start AND end bin: the ones covering bin i are a consecutive range
  int lo = 0, hi = W;                     // first window with win_hi > i
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (win_hi[mid] <= (int32_t)i) lo = mid + 1; else hi = mid;
  }
  double acc = 0.0;
  int count = 0;
  for (int w = lo; w < W && win_lo[w] <= (int32_t)i; ++w) {
    if (win_hi[w] > (int32_t)i) {
      acc += med[(int64_t)b * W + w] * inv_corr;       // reference: nanmedian(...) / corr_factor
      count++;
    }
  }
  bkg[(int64_t)b * F + i] = acc / (double)count;       // 0/0 -> NaN where no window covers the bin, like numpy
}

int pg_logmedian(const double* power, int B, int64_t F, const int32_t* h_win_lo, const int32_t* h_win_hi, int W,
                 double corr_factor, double* bkg, int mem, cudaStream_t st) {
  LKB_REQUIRE(power && bkg && h_win_lo && h_win_hi, "lkb_pg_logmedian: null argument");
  LKB_REQUIRE(B > 0 && B <= 65535 && F > 0 && F < ((int64_t)1 << 31) && W > 0 && W <= 2147483647,
              "lkb_pg_logmedian: bad sizes");
  LKB_REQUIRE(corr_factor > 0.0, "lkb_pg_logmedian: corr_factor must be positive");
  for (int w = 0; w < W; ++w) {
    LKB_REQUIRE(h_win_lo[w] >= 0 && h_win_hi[w] <= F && h_win_lo[w] <= h_win_hi[w], "lkb_pg_logmedian: bad window");
    LKB_REQUIRE(w == 0 || (h_win_lo[w] >= h_win_lo[w - 1] && h_win_hi[w] >= h_win_hi[w - 1]),
                "lkb_pg_logmedian: windows must be ordered (ascending frequency grid)");
  }
  LKB_TRY(ensure_device());
  const double* d_p = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, power, (size_t)B * F, &d_p, st));
  int32_t *d_lo = nullptr, *d_hi = nullptr;
  double* d_med = nullptr;
  LKB_TRY(ws_get_t<int32_t>(WS_A, W, &d_lo));
  LKB_TRY(ws_get_t<int32_t>(WS_B, W, &d_hi));
  LKB_TRY(ws_get_t<double>(WS_C, (size_t)B * W, &d_med));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_lo, h_win_lo, sizeof(int32_t) * W, cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_hi, h_win_hi, sizeof(int32_t) * W, cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaStreamSynchronize(st));      // the window arrays are caller-owned host memory
  double* d_b = nullptr;
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0, bkg, (size_t)B * F, &d_b));
  prof_begin(st);
  for (int w0 = 0; w0 < W; w0 += 65535 * 32) {     // grid.x limit is generous; keep one launch in practice
    const int wn = min(W - w0, 65535 * 32);
    pg_window_median_kernel<<<dim3((unsigned)wn, (unsigned)B), 256, 0, st>>>(d_p, F, d_lo + w0, d_hi + w0, W, d_med + w0);
    LKB_LAUNCH_CHECK();
  }
  prof_end(st);
  pg_window_combine_kernel<<<dim3((unsigned)((F + 255) / 256), (unsigned)B), 256, 0, st>>>(d_med, F, d_lo, d_hi, W,
                                                                                             1.0 / corr_factor, d_b);
  LKB_LAUNCH_CHECK();
  LKB_TRY(stage_out_copy<double>(mem, bkg, d_b, (size_t)B * F, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

int acf_windows(const double* x, const int64_t* x_offsets, int B, const int64_t* win_offsets, const int64_t* win_start,
                const int64_t* win_len, double* metric, double* acf, int mem, cudaStream_t st) {
  return acf_windows_launch(x, x_offsets, B, win_offsets, win_start, win_len, metric, acf, mem, st);
}

}  // namespace lkb
