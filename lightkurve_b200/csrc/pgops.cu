// Periodogram post-processing for the step after Lomb-Scargle (asteroseismology chain):
//   /root/reference/src/lightkurve/periodogram.py:260-284  Periodogram.smooth(method="logmedian")
//   /root/reference/src/lightkurve/periodogram.py:381-429  Periodogram.flatten  (power / background)
// The reference walks a window of half-width filter_width in log10(frequency) across the spectrum in
// steps of filter_width / 2 and, for every window, adds nanmedian(power[window]) / (8/9)^3 to the bins in it;
// the background is that sum divided by the number of windows that covered the bin.
//
// The window list (start bin, end bin) is built on the host from each frequency grid with the reference's own
// expression (the x0 += 0.5 w accumulation must be reproduced in fp64); the GPU does the exact medians of every
// (window, periodogram) (K6 radix select, one CTA each) and the per-bin combination in the reference's summation
// order (ascending window index).  One grid shared by B periodograms (lkb_pg_logmedian) and one grid per
// periodogram (lkb_pg_logmedian_ragged, which can also divide the power by its background) run the same kernels.
//
// The seismology estimators that read the flattened periodogram (numax / deltanu ACF2D) run on the K7 windowed
// autocorrelation kernels of acf.cuh; lkb_acf_windows enters through acf_windows below.
#include "common.cuh"
#include "select.cuh"
#include "acf.cuh"

namespace lkb {

// Where periodogram b's bins and windows are: one grid shared by all (bin_off == nullptr: F bins at b * F, the W
// windows [0, W) with their medians at b * W), or per-periodogram CSRs of bins and windows (the medians of window k
// at k, its bin range relative to the periodogram's first bin).
struct PgLayout {
  const int64_t* bin_off;   // [B + 1] or nullptr
  const int64_t* win_off;   // [B + 1] (when bin_off is set)
  int64_t F;
  int W;
  __device__ __forceinline__ int64_t bin0(int b) const { return bin_off ? bin_off[b] : (int64_t)b * F; }
  __device__ __forceinline__ int64_t nbins(int b) const { return bin_off ? bin_off[b + 1] - bin_off[b] : F; }
  __device__ __forceinline__ int64_t win0(int b) const { return bin_off ? win_off[b] : 0; }
  __device__ __forceinline__ int nwin(int b) const { return bin_off ? (int)(win_off[b + 1] - win_off[b]) : W; }
  __device__ __forceinline__ int64_t med0(int b) const { return bin_off ? win_off[b] : (int64_t)b * W; }
};

template <typename P>
__global__ void __launch_bounds__(256)
pg_window_median_kernel(const P* __restrict__ power, PgLayout g, const int32_t* __restrict__ win_lo,
                        const int32_t* __restrict__ win_hi, int w_base, double* __restrict__ med) {
  __shared__ SelSmem sm;
  const int w = w_base + blockIdx.x, b = blockIdx.y;
  if (w >= g.nwin(b)) return;
  const int64_t k = g.win0(b) + w;
  const int lo = win_lo[k], n = win_hi[k] - lo;
  const P* p = power + g.bin0(b) + lo;
  double m;
  if (n <= 0) {
    m = __longlong_as_double(0x7ff8000000000000ll);
  } else if (n <= 32) {
    // tiny windows (the low-frequency end of a linear grid): rank by counting inside warp 0
    m = 0.0;
    if (threadIdx.x < 32) {
      const int lane = threadIdx.x;
      const double v = lane < n ? (double)p[lane] : __longlong_as_double(0x7ff8000000000000ll);
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
    m = block_nanmedian([&](int64_t i) { return (double)p[i]; }, n, sm);
  }
  if (threadIdx.x == 0) med[g.med0(b) + w] = m;
}

// background = mean of the covering windows' medians / corr; with snr, also power / background (Periodogram.flatten)
template <typename P>
__global__ void __launch_bounds__(256)
pg_window_combine_kernel(const double* __restrict__ med, const P* __restrict__ power, PgLayout g,
                         const int32_t* __restrict__ win_lo, const int32_t* __restrict__ win_hi, double inv_corr,
                         double* __restrict__ bkg, double* __restrict__ snr) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= g.nbins(b)) return;
  const int32_t* wlo = win_lo + g.win0(b);
  const int32_t* whi = win_hi + g.win0(b);
  const double* mb = med + g.med0(b);
  const int W = g.nwin(b);
  // windows are ordered by start AND end bin: the ones covering bin i are a consecutive range
  int lo = 0, hi = W;                     // first window with win_hi > i
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (whi[mid] <= (int32_t)i) lo = mid + 1; else hi = mid;
  }
  double acc = 0.0;
  int count = 0;
  for (int w = lo; w < W && wlo[w] <= (int32_t)i; ++w) {
    if (whi[w] > (int32_t)i) {
      acc += mb[w] * inv_corr;                          // reference: nanmedian(...) / corr_factor
      count++;
    }
  }
  const double bg = acc / (double)count;                // 0/0 -> NaN where no window covers the bin, like numpy
  const int64_t j = g.bin0(b) + i;
  bkg[j] = bg;
  if (snr) snr[j] = (double)power[j] / bg;
}

// The windows of every periodogram (relative bin ranges, ordered, inside [0, F_b]) are checked on the host.
static int pg_check_windows(const int32_t* lo, const int32_t* hi, int W, int64_t F, int b) {
  for (int w = 0; w < W; ++w) {
    if (!(lo[w] >= 0 && hi[w] <= F && lo[w] <= hi[w]) ||
        !(w == 0 || (lo[w] >= lo[w - 1] && hi[w] >= hi[w - 1]))) {
      set_error("lkb_pg_logmedian: periodogram %d: window %d is out of range or out of order (windows must follow an "
                "ascending frequency grid)", b, w);
      return LKB_E_ARG;
    }
  }
  return LKB_OK;
}

template <typename P>
static int pg_logmedian_run(const P* d_p, int B, PgLayout g, int Wmax, int64_t Fmax, int64_t Wtot,
                            const int32_t* h_win_lo, const int32_t* h_win_hi, double corr_factor, double* bkg,
                            double* snr, int64_t total_bins, int mem, cudaStream_t st) {
  int32_t *d_lo = nullptr, *d_hi = nullptr;
  double* d_med = nullptr;
  LKB_TRY(ws_get_t<int32_t>(WS_A, Wtot, &d_lo));
  LKB_TRY(ws_get_t<int32_t>(WS_B, Wtot, &d_hi));
  LKB_TRY(ws_get_t<double>(WS_C, g.bin_off ? (size_t)Wtot : (size_t)B * Wtot, &d_med));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_lo, h_win_lo, sizeof(int32_t) * Wtot, cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_hi, h_win_hi, sizeof(int32_t) * Wtot, cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaStreamSynchronize(st));      // the window arrays are caller-owned host memory
  double *d_b = nullptr, *d_s = nullptr;
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0, bkg, total_bins, &d_b));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT1, snr, total_bins, &d_s));
  prof_begin(st);
  for (int w0 = 0; w0 < Wmax; w0 += 65535 * 32) {     // grid.x limit is generous; keep one launch in practice
    const int wn = min(Wmax - w0, 65535 * 32);
    pg_window_median_kernel<P><<<dim3((unsigned)wn, (unsigned)B), 256, 0, st>>>(d_p, g, d_lo, d_hi, w0, d_med);
    LKB_LAUNCH_CHECK();
  }
  prof_end(st);
  pg_window_combine_kernel<P><<<dim3((unsigned)((Fmax + 255) / 256), (unsigned)B), 256, 0, st>>>(
      d_med, d_p, g, d_lo, d_hi, 1.0 / corr_factor, d_b, d_s);
  LKB_LAUNCH_CHECK();
  LKB_TRY(stage_out_copy<double>(mem, bkg, d_b, total_bins, st));
  LKB_TRY(stage_out_copy<double>(mem, snr, d_s, total_bins, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

int pg_logmedian(const double* power, int B, int64_t F, const int32_t* h_win_lo, const int32_t* h_win_hi, int W,
                 double corr_factor, double* bkg, int mem, cudaStream_t st) {
  LKB_REQUIRE(power && bkg && h_win_lo && h_win_hi, "lkb_pg_logmedian: null argument");
  LKB_REQUIRE(B > 0 && B <= 65535 && F > 0 && F < ((int64_t)1 << 31) && W > 0 && W <= 2147483647,
              "lkb_pg_logmedian: bad sizes");
  LKB_REQUIRE(corr_factor > 0.0, "lkb_pg_logmedian: corr_factor must be positive");
  LKB_TRY(pg_check_windows(h_win_lo, h_win_hi, W, F, 0));
  LKB_TRY(ensure_device());
  const double* d_p = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, power, (size_t)B * F, &d_p, st));
  PgLayout g{nullptr, nullptr, F, W};
  return pg_logmedian_run<double>(d_p, B, g, W, F, W, h_win_lo, h_win_hi, corr_factor, bkg, nullptr, (int64_t)B * F,
                                  mem, st);
}

int pg_logmedian_ragged(const void* power, int p_dtype, const int64_t* h_bin_off, int B, const int32_t* h_win_lo,
                        const int32_t* h_win_hi, const int64_t* h_win_off, double corr_factor, double* bkg,
                        double* snr, int mem, cudaStream_t st) {
  LKB_REQUIRE(power && h_bin_off && h_win_lo && h_win_hi && h_win_off && bkg,
              "lkb_pg_logmedian_ragged: null argument");
  LKB_REQUIRE(p_dtype == LKB_DTYPE_F32 || p_dtype == LKB_DTYPE_F64, "lkb_pg_logmedian_ragged: bad power dtype");
  LKB_REQUIRE(B > 0 && B <= 65535 && h_bin_off[0] == 0 && h_win_off[0] == 0, "lkb_pg_logmedian_ragged: bad sizes");
  LKB_REQUIRE(corr_factor > 0.0, "lkb_pg_logmedian_ragged: corr_factor must be positive");
  int64_t Fmax = 0, Wmax = 0;
  for (int b = 0; b < B; ++b) {
    const int64_t F = h_bin_off[b + 1] - h_bin_off[b], W = h_win_off[b + 1] - h_win_off[b];
    if (F < 0 || F >= ((int64_t)1 << 31) || W < 0 || W > 65535 * 32) {
      set_error("lkb_pg_logmedian_ragged: periodogram %d has %lld bins and %lld windows", b, (long long)F,
                (long long)W);
      return LKB_E_ARG;
    }
    LKB_TRY(pg_check_windows(h_win_lo + h_win_off[b], h_win_hi + h_win_off[b], (int)W, F, b));
    Fmax = max(Fmax, F);
    Wmax = max(Wmax, W);
  }
  const int64_t total = h_bin_off[B], Wtot = h_win_off[B];
  if (total == 0) return LKB_OK;
  LKB_TRY(ensure_device());
  int64_t* d_csr = nullptr;
  LKB_TRY(ws_get_t<int64_t>(WS_D, 2 * ((size_t)B + 1), &d_csr));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_csr, h_bin_off, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_csr + B + 1, h_win_off, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  PgLayout g{d_csr, d_csr + B + 1, 0, 0};
  const int32_t one = 0;
  const int32_t* lo = Wtot ? h_win_lo : &one;
  const int32_t* hi = Wtot ? h_win_hi : &one;
  const int64_t Wn = Wtot ? Wtot : 1;
  if (p_dtype == LKB_DTYPE_F32) {
    const float* d_p = nullptr;
    LKB_TRY(stage_in<float>(mem, WS_IN0, (const float*)power, total, &d_p, st));
    return pg_logmedian_run<float>(d_p, B, g, (int)max(Wmax, (int64_t)1), Fmax, Wn, lo, hi, corr_factor, bkg, snr,
                                   total, mem, st);
  }
  const double* d_p = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, (const double*)power, total, &d_p, st));
  return pg_logmedian_run<double>(d_p, B, g, (int)max(Wmax, (int64_t)1), Fmax, Wn, lo, hi, corr_factor, bkg, snr,
                                  total, mem, st);
}

int acf_windows(const double* x, const int64_t* x_offsets, int B, const int64_t* win_offsets, const int64_t* win_start,
                const int64_t* win_len, double* metric, double* acf, int mem, cudaStream_t st) {
  return acf_windows_launch(x, x_offsets, B, win_offsets, win_start, win_len, metric, acf, mem, st);
}

}  // namespace lkb
