// K5: the per-light-curve kernels of RegressionCorrector that need no inline PTX - the model X w (rg_model_rows), the
// residuals and astropy's sigma_clip (rg_clip_kernel) and the median-subtracted final model (rg_final_kernel) - with the
// workspace they share with regress.cu.  Kept apart from regress.cu (mma.sync / cp.async) so that
// tests/native/cuda_emu.h can run them on the CPU (tests/test_regress_clip_emulated.py).
#pragma once
#include "common.cuh"
#include "select.cuh"

namespace lkb {

struct RgWs {
  int32_t* rows;      // [B, N] cadence list for the current accumulate pass
  int32_t* cnt;       // [B]
  uint8_t* used;      // [B, N] cadences currently inside A/rhs
  double* gram;       // [B, Ka, Ka], Ka = K + 1 (column K is y)
  double* resid;      // [B, N]
  double* wl;         // [B, N] 1/flux_err^2 of the listed cadences, in list order (ones without flux_err)
};

__device__ __forceinline__ const double* rg_xrow(const double* X, int x_batched, int b, int64_t N, int K, int64_t r) {
  return X + ((x_batched ? (int64_t)b * N : 0) + r) * K;
}

// ---- model + sigma clip ---------------------------------------------------------------------------
__device__ __forceinline__ void rg_model_rows(const double* X, int x_batched, int b, int64_t N, int K,
                                              const double* s_w, double* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int64_t r = warp; r < N; r += nw) {
    const double* xr = rg_xrow(X, x_batched, b, N, K, r);
    double acc = 0.0;
    for (int k = lane; k < K; k += 32) acc = fma(xr[k], s_w[k], acc);
    acc = warp_sum(acc);
    if (lane == 0) out[r] = acc;
  }
}

__global__ void __launch_bounds__(512)
rg_clip_kernel(const double* __restrict__ X, int x_batched, const double* __restrict__ y, int64_t N, int K,
               const double* __restrict__ coeff, double clip_sigma, RgWs ws, uint8_t* __restrict__ outlier,
               int model_ready) {
  LKB_DYN_SMEM(double, s_w);                          // [K] coefficients | FastSelSmem | FS_CAP + FS_SAMPLE candidates
  __shared__ SelSmem sm;
  __shared__ FastBracket s_br;
  const int b = blockIdx.x;
  for (int k = threadIdx.x; k < K; k += blockDim.x) s_w[k] = coeff[(int64_t)b * K + k];
  __syncthreads();
  double* res = ws.resid + (int64_t)b * N;
  const uint8_t* used = ws.used + (int64_t)b * N;
  uint8_t* om = outlier + (int64_t)b * N;
  const double* yb = y + (int64_t)b * N;
  const double qnan = __longlong_as_double(0x7ff8000000000000ll);
  if (!model_ready) rg_model_rows(X, x_batched, b, N, K, s_w, res);      // else ws.resid already holds X w
  __syncthreads();
  for (int64_t i = threadIdx.x; i < N; i += blockDim.x) res[i] = used[i] ? (yb[i] - res[i]) : qnan;
  __syncthreads();
  // astropy.stats.sigma_clip(residuals, sigma): maxiters=5, cenfunc=median, stdfunc=std.  One pass over the residuals
  // per round: the values outside the PREVIOUS round's bounds are struck out on the way into the median's partition
  // pass (select.cuh: block_nanmedian_fast, bracket carried from round to round), whose observer also gathers the sums
  // of the standard deviation.  (First version: 10-pass radix median + 2-pass std + clip pass per round, up to 65 sweeps
  // of the light curve - a quarter of the device time of correct().)
  FastSelSmem& fs = *reinterpret_cast<FastSelSmem*>(s_w + ((K + 1) & ~1));
  double* cand = reinterpret_cast<double*>(&fs + 1);
  if (threadIdx.x == 0) { fs.cand = cand; s_br.valid = false; }
  __syncthreads();
  const double inf = __longlong_as_double(0x7ff0000000000000ll);
  double lo_c = -inf, hi_c = inf;
  for (int round = 0; round <= 5; ++round) {
    long long changed = 0;
    double s1 = 0.0, s2 = 0.0;
    long long sc = 0;
    auto get = [&](int64_t i) {
      const double v = res[i];
      if (v == v && (v < lo_c || v > hi_c)) { res[i] = qnan; changed++; return qnan; }   // (idempotent: counted once)
      return v;
    };
    auto stats = [&](int64_t, double v, double lo, bool valid) {
      if (valid && v == v) { const double d = v - lo; s1 += d; s2 = fma(d, d, s2); sc++; }
    };
    bool observed = false;
    const double med = block_nanmedian_fast(get, N, sm, fs, -1, stats, &observed, &s_br,
                                            [&]() { s1 = 0.0; s2 = 0.0; sc = 0; });
    const long long tot = block_sum_ll(changed, sm.redll);
    if (round > 0 && tot == 0) break;             // the last clip removed nothing: converged
    if (round == 5 || !(med == med)) break;       // five clips done / nothing left
    double sd;
    if (observed) {
      const double t1 = block_sum(s1, sm.red), t2 = block_sum(s2, sm.red);
      const long long tc = block_sum_ll(sc, sm.redll);
      const double md = t1 / (double)tc, var = t2 / (double)tc - md * md;
      sd = (var == var) ? sqrt(var > 0.0 ? var : 0.0) : qnan;
    } else {
      sd = block_nanstd([&](int64_t i) { return res[i]; }, N, sm);
    }
    lo_c = med - sd * clip_sigma;
    hi_c = med + sd * clip_sigma;
  }
  __syncthreads();
  for (int64_t i = threadIdx.x; i < N; i += blockDim.x) {
    const double v = res[i];
    if (!(v == v)) om[i] = 1;          // .mask includes the cadences that were NaN on entry
  }
}

__global__ void __launch_bounds__(512)
rg_final_kernel(const double* __restrict__ X, int x_batched, int64_t N, int K, const double* __restrict__ coeff,
                double* __restrict__ model, int model_ready) {
  LKB_DYN_SMEM(double, s_w);
  __shared__ SelSmem sm;
  const int b = blockIdx.x;
  for (int k = threadIdx.x; k < K; k += blockDim.x) s_w[k] = coeff[(int64_t)b * K + k];
  __syncthreads();
  double* mo = model + (int64_t)b * N;
  if (!model_ready) rg_model_rows(X, x_batched, b, N, K, s_w, mo);
  __syncthreads();
  // np.median (NaN-propagating): a NaN model (singular fit) stays NaN
  long long cntv = 0;
  const double med = block_nanmedian([&](int64_t i) { return mo[i]; }, N, sm, &cntv);
  const double m = (cntv == N) ? med : __longlong_as_double(0x7ff8000000000000ll);
  for (int64_t i = threadIdx.x; i < N; i += blockDim.x) mo[i] -= m;
}

}  // namespace lkb
