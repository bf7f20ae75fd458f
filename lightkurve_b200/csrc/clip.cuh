// K11: astropy.stats.sigma_clip(x, sigma_lower, sigma_upper, maxiters).mask (cenfunc="median", stdfunc="std") over
// CSR-ragged fp64 light curves - LightCurve.remove_outliers, lightcurve.py:1429-1549.
// K12: the rest of LightCurve.estimate_cdpp (lightcurve.py:1764-1833) on the cleaned flattened flux: the normalize
// median, the running means of each transit duration and their standard deviation.
//
// One CTA per light curve; every clip round runs on the device with rg_clip_kernel's round structure
// (regress_clip.cuh): the previous round's bounds strike values out on the way into block_nanmedian_fast's partition
// pass, the bracket is carried from round to round, and the standard deviation's sums are gathered by the median's
// observer.  The light curve is copied once, non-finite values as NaN, into a working array: shared memory when it has
// at most CL_RES_CAP cadences (a TESS 2-minute sector, about 20 000 cadences, then never leaves the SM between the clip
// rounds and the CDPP finish), else a CSR scratch array in global memory that the rounds stream from L2/HBM (a 4-year
// Kepler light curve, 65 000 cadences, does not fit next to the median's 60 KB candidate buffer).  Both are the same
// code on a different pointer, so their results are bitwise equal.  Kept apart from the library's entry points so
// that tests/native/cuda_emu.h runs it on the CPU.
#pragma once
#include "common.cuh"
#include "select.cuh"

namespace lkb {

constexpr int CL_THREADS = 512;
// 160 KB of resident light curve + the 60 KB candidate buffer of block_nanmedian_fast + ~2 KB of static shared memory
// stay under the 227 KB an H100 CTA may have
constexpr int CL_RES_CAP = 20480;

struct ClipArgs {
  const double* x;          // [offsets[B]] values
  const int64_t* off;       // [B + 1] device CSR offsets
  double* work;             // [offsets[B]] scratch of the light curves longer than res_cap (may alias x); else unused
  double sigma_lower, sigma_upper;
  int maxiters;             // < 0: until a round clips nothing
  int res_cap;              // light curves with at most res_cap cadences work in shared memory
  int cand;                 // 1: the dynamic shared memory starts with the FS_CAP + FS_SAMPLE candidate buffer
  uint8_t* mask;            // [offsets[B]] 1 = clipped or non-finite (optional)
  double* center;           // [B] median of the kept values (optional)
  double* sd;               // [B] their standard deviation, ddof 0 (optional)
  int64_t* n_kept;          // [B] (optional)
  const int32_t* dur;       // [D] transit durations in cadences; NULL: no CDPP finish
  int D;
  double* cdpp;             // [B, D] ppm
};

// Resident capacity, candidate buffer and dynamic shared memory of one launch (host).
struct ClipPlan {
  int res_cap, cand;
  bool streams;             // some light curve works in global memory
  size_t smem;
};
inline ClipPlan clip_plan(const int64_t* h_off, int B, int64_t cap) {
  int64_t nres = 0, nmax = 0;
  for (int b = 0; b < B; ++b) {
    const int64_t n = h_off[b + 1] - h_off[b];
    nmax = n > nmax ? n : nmax;
    if (n <= cap && n > nres) nres = n;
  }
  ClipPlan p;
  p.res_cap = (int)nres;
  p.cand = nmax >= 4 * FS_SAMPLE;          // block_nanmedian_fast samples only from this length on
  p.streams = nmax > nres;
  p.smem = sizeof(double) * ((p.cand ? (size_t)(FS_CAP + FS_SAMPLE) : 0) + (size_t)nres);
  return p;
}

struct ClipScanSmem {
  int cnt[32];
  double sum[32];
};

// Block-wide scan of (flag, value): *excl = flags before this thread, *incl = values up to and including it (fixed
// order: lanes, then warps); *tot_c / *tot_s the block totals.  All threads must call.
__device__ __forceinline__ void clip_block_scan(int f, double y, int* excl, double* incl, int* tot_c, double* tot_s,
                                                ClipScanSmem& s) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int c = f;
  double v = y;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int cu = __shfl_up_sync(0xffffffffu, c, o);
    const double vu = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) { c += cu; v += vu; }
  }
  __syncthreads();                                   // the previous call's readers are done with s
  if (lane == 31) { s.cnt[wid] = c; s.sum[wid] = v; }
  __syncthreads();
  if (wid == 0) {
    int wc = lane < nw ? s.cnt[lane] : 0;
    double wv = lane < nw ? s.sum[lane] : 0.0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int cu = __shfl_up_sync(0xffffffffu, wc, o);
      const double vu = __shfl_up_sync(0xffffffffu, wv, o);
      if (lane >= o) { wc += cu; wv += vu; }
    }
    if (lane < nw) { s.cnt[lane] = wc; s.sum[lane] = wv; }
  }
  __syncthreads();
  *excl = (wid ? s.cnt[wid - 1] : 0) + c - f;
  *incl = (wid ? s.sum[wid - 1] : 0.0) + v;
  *tot_c = s.cnt[nw - 1];
  *tot_s = s.sum[nw - 1];
}

__global__ void __launch_bounds__(CL_THREADS) clip_cdpp_kernel(ClipArgs a) {
  LKB_DYN_SMEM(double, dyn);                 // [FS_CAP + FS_SAMPLE candidates if a.cand] [resident light curve]
  __shared__ SelSmem sm;
  __shared__ FastSelSmem fs;
  __shared__ FastBracket br;
  __shared__ ClipScanSmem scan;
  const int b = blockIdx.x;
  const int64_t o = a.off[b], n = a.off[b + 1] - o;
  double* w = n <= a.res_cap ? dyn + (a.cand ? FS_CAP + FS_SAMPLE : 0) : a.work + o;
  const double* xb = a.x + o;
  const double qnan = __longlong_as_double(0x7ff8000000000000ll), inf = __longlong_as_double(0x7ff0000000000000ll);
  long long fin = 0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {       // (in place when w aliases x: same thread, same i)
    const double v = xb[i];
    const bool ok = isfinite(v);
    w[i] = ok ? v : qnan;
    fin += ok ? 1 : 0;
  }
  if (threadIdx.x == 0) { fs.cand = dyn; br.valid = false; }
  long long kept = block_sum_ll(fin, sm.redll);                 // (its barriers publish w, fs and br)

  // ---- K11: round r strikes out the values outside round r - 1's bounds while it selects the median of the rest ----
  double lo_c = -inf, hi_c = inf, med = qnan, sd = qnan;
  for (int round = 0;; ++round) {
    long long changed = 0, sc = 0;
    double s1 = 0.0, s2 = 0.0;
    auto get = [&](int64_t i) {
      const double v = w[i];
      if (v == v && (v < lo_c || v > hi_c)) { w[i] = qnan; changed++; return qnan; }   // (idempotent: counted once)
      return v;
    };
    auto stats = [&](int64_t, double v, double lo, bool valid) {
      if (valid && v == v) { const double d = v - lo; s1 += d; s2 = fma(d, d, s2); sc++; }
    };
    bool observed = false;
    med = block_nanmedian_fast(get, n, sm, fs, -1, stats, &observed, &br, [&]() { s1 = 0.0; s2 = 0.0; sc = 0; });
    const long long tot = block_sum_ll(changed, sm.redll);
    kept -= tot;
    if (kept == 0) { med = qnan; sd = qnan; break; }
    if (observed) {
      const double t1 = block_sum(s1, sm.red), t2 = block_sum(s2, sm.red);
      const long long tc = block_sum_ll(sc, sm.redll);
      const double md = t1 / (double)tc, var = t2 / (double)tc - md * md;
      sd = (var == var) ? sqrt(var > 0.0 ? var : 0.0) : qnan;
    } else {
      sd = block_nanstd([&](int64_t i) { return w[i]; }, n, sm);
    }
    if (round > 0 && tot == 0) break;                           // the last clip removed nothing: converged
    if (a.maxiters >= 0 && round >= a.maxiters) break;          // maxiters clips done
    lo_c = med - sd * a.sigma_lower;                            // numpy's order: c - (s * sigma)
    hi_c = med + sd * a.sigma_upper;
  }
  if (threadIdx.x == 0) {
    if (a.center) a.center[b] = med;
    if (a.sd) a.sd[b] = sd;
    if (a.n_kept) a.n_kept[b] = kept;
  }
  __syncthreads();
  if (a.mask)
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) a.mask[o + i] = (w[i] == w[i]) ? 0 : 1;
  if (a.dur == nullptr) return;

  // ---- K12: running means over the kept values in their order, centred: y = (x / med - 1) 1e6 ppm.  The kept values
  // are compacted in place into their inclusive prefix sums (a write lands at or before the position its tile read) ----
  long long base = 0;
  double carry = 0.0;
  for (int64_t i0 = 0; i0 < n; i0 += blockDim.x) {
    const int64_t i = i0 + threadIdx.x;
    const double v = i < n ? w[i] : qnan;
    const int k = v == v ? 1 : 0;
    const double y = k ? (v / med - 1.0) * 1e6 : 0.0;
    int ex, tc;
    double inc, ts;
    clip_block_scan(k, y, &ex, &inc, &tc, &ts, scan);        // (barriers: the whole tile was read before any write)
    if (k) w[base + ex] = carry + inc;
    base += tc;
    carry += ts;
  }
  __syncthreads();
  for (int d = 0; d < a.D; ++d) {
    double res = qnan;
    if (kept > 0) {
      const long long dd = a.dur[d], win = dd < kept ? dd : kept, M = kept - win + 1;
      auto mean_at = [&](long long j) { return (w[j + win - 1] - (j > 0 ? w[j - 1] : 0.0)) / (double)win; };
      double s = 0.0;
      for (long long j = threadIdx.x; j < M; j += blockDim.x) s += mean_at(j);
      const double mu = block_sum(s, sm.red) / (double)M;
      double q = 0.0;
      for (long long j = threadIdx.x; j < M; j += blockDim.x) { const double e = mean_at(j) - mu; q += e * e; }
      res = sqrt(block_sum(q, sm.red) / (double)M);
    }
    if (threadIdx.x == 0) a.cdpp[(int64_t)b * a.D + d] = res;
  }
}

}  // namespace lkb
