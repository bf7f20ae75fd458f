// K3: Box Least Squares, the search lightkurve obtains from astropy at
//   /root/reference/src/lightkurve/periodogram.py:1161-1169
//   (BoxLeastSquares(t, y, dy).power(period, duration, objective, method="fast", oversample)).
// Algorithm = astropy bls.c (restated in oracle/bls_c.c): per trial period, fold the samples
// into bins of width min(duration)/oversample, wrap-pad, inclusive prefix sum, then scan every
// (duration, start bin) box and keep the FIRST strict maximum of the objective with y_out >= y_in.
//
// Mapping: one WARP per (light curve, period).  A CTA = BLS_WARPS warps working on
// consecutive periods of the SAME light curve, so the (t, w*y, w) sample tiles are staged into
// shared memory once per CTA and re-used by every warp.  Each warp owns a private
// shared-memory histogram (plain `+=`, no atomics): 32 consecutive samples have non-decreasing
// bin indices except at a period wrap, so a warp-segmented reduction leaves exactly one
// writer per bin (wrap blocks are split into monotone pieces).
//
// Densely sampled light curves (more cadences than bin boundaries over the baseline, e.g. TESS 2-min
// data with 7-min bins) take the BOUNDARY path instead: the exact (cycle, bin) index is monotone in
// time, so each bin of each cycle is a contiguous run of cadences; a lane finds the first cadence of
// its run with a table lookup + a short exact walk and adds the run's sum as a difference of a
// per-light-curve prefix sum - work per period ~ baseline / bin_duration instead of N, no scan.
//
// Bit-exactness: the bin index (int)(fabs(fmod(t - min_t, P)) / bin_duration) + 1 is evaluated
// with an exact fmod (fma remainder + fix-up) and an IEEE fp64 division, so it equals the C
// result bit for bit.  This file is compiled with -fmad=false so that no a*b+c is contracted
// where the C code (built with -ffp-contract=off) has two roundings.  The binned sums are
// accumulated in a different order than the sequential C loop => equal to ~1e-13 relative,
// not bitwise; exact ties between boxes that cover the same samples are preserved by the
// scan construction (see bls_cumsum).
#include "common.cuh"
#include "select.cuh"
#include "bls_plan.h"
#include "bls_stats.cuh"     // K10 (vetting statistics), and bls_fmod
#include <float.h>
#include <algorithm>
#include <vector>

namespace lkb {

// (int)(r / bd) with the IEEE division replaced, on the fast path, by a reciprocal multiply whose
// result is PROVEN equal: k = trunc(r * (1/bd)); rem = fma(-k, bd, r) is the (once rounded) remainder;
// if 0 <= rem < bd_safe = bd * (1 - (kmax + 2) 2^-51) with kmax >= k, the real quotient lies in
// [k, k + 1 - margin) and RN(r / bd) cannot reach k + 1, so trunc(RN(r/bd)) = k.  Anything else (a
// sample within ~1e-13 of a bin edge) takes the true division - a warp-uniform, out-of-line branch so
// that the ~25-instruction IEEE division is not if-converted into every iteration.
__device__ __noinline__ double bls_div_slow(double r, double bd) { return r / bd; }

__device__ __forceinline__ double bls_safe_width(double bd, int kmax) {
  return bd - bd * (((double)kmax + 2.0) * 4.440892098500626e-16);
}

// bin index of a sample at x >= 0 (time since the first cadence); `valid` lanes only.  Warp-collective.
__device__ __forceinline__ int bls_bin_warp(double x, bool valid, double period, double inv_period, double bd,
                                            double inv_bd, double bd_safe) {
  double q = trunc(x * inv_period);
  double r = fma(-q, period, x);
  if (r < 0.0) { q -= 1.0; r = fma(-q, period, x); }
  else if (r >= period) { q += 1.0; r = fma(-q, period, x); }
  double k = trunc(r * inv_bd);
  const double rem = fma(-k, bd, r);
  const bool slow = valid && !(rem >= 0.0 && rem < bd_safe);
  if (__any_sync(0xffffffffu, slow)) {
    if (slow) k = trunc(bls_div_slow(r, bd));
  }
  return valid ? (int)k + 1 : -1;
}

// exact (cycle q, bin k) of a sample at x >= 0; callable from divergent code
__device__ __forceinline__ void bls_cycle_bin(double x, double period, double inv_period, double bd, double inv_bd,
                                              double bd_safe, int& qi, int& ki) {
  double q = trunc(x * inv_period);
  double r = fma(-q, period, x);
  if (r < 0.0) { q -= 1.0; r = fma(-q, period, x); }
  else if (r >= period) { q += 1.0; r = fma(-q, period, x); }
  double k = trunc(r * inv_bd);
  const double rem = fma(-k, bd, r);
  if (!(rem >= 0.0 && rem < bd_safe)) k = trunc(bls_div_slow(r, bd));
  qi = (int)q;
  ki = (int)k;
}

__device__ __forceinline__ int bls_bin(double t, double min_t, double period, double inv_period, double bin_duration,
                                       double inv_bin) {
  const double r = fabs(bls_fmod(t - min_t, period, inv_period));
  const double k = trunc(r * inv_bin);
  const double rem = fma(-k, bin_duration, r);
  const double margin = bin_duration * ((k + 2.0) * 4.440892098500626e-16);
  if (rem >= 0.0 && rem < bin_duration - margin && k < 1073741824.0) return (int)k + 1;
  return (int)(r / bin_duration) + 1;
}

__global__ void bls_bin_index_kernel(const double* __restrict__ t, int64_t N, double min_t, double period,
                                     double bin_duration, int32_t* __restrict__ ind) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) ind[i] = bls_bin(t[i], min_t, period, 1.0 / fabs(period), bin_duration, 1.0 / bin_duration);
}

// ---- prologue: astropy core.py power(): t - min(t), y - median(y), ivar = 1/dy^2 ----------
struct BlsLcInfo {
  double t_ref, sum_y, sum_ivar, min_t, x_max;
  int sorted, pad;
};

// Also produces what the boundary path needs: sortedness, the baseline, and the exclusive prefix sums
// cpre[i] = sum_{i' < i} {w*y, w} (N + 1 entries per light curve, at offset o + b).
__global__ void __launch_bounds__(256)
bls_prep_kernel(const double* __restrict__ t, const double* __restrict__ y, const double* __restrict__ dy,
                const int64_t* __restrict__ offsets, double* __restrict__ trel, double* __restrict__ wy,
                double* __restrict__ iv, double2* __restrict__ cpre, BlsLcInfo* __restrict__ info) {
  __shared__ SelSmem sm;
  __shared__ double2 s_part[256];
  __shared__ int s_unsorted;
  const int b = blockIdx.x;
  const int64_t o = offsets[b], n = offsets[b + 1] - o;
  if (n <= 0) return;
  if (threadIdx.x == 0) s_unsorted = 0;
  // t_ref = min(t)
  double mn = __longlong_as_double(0x7ff0000000000000ll), mx = -mn;
  int unsorted = 0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const double v = t[o + i];
    mn = fmin(mn, v);
    mx = fmax(mx, v);
    if (i + 1 < n && !(t[o + i + 1] >= v)) unsorted = 1;
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, s));
    mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, s));
  }
  if ((threadIdx.x & 31) == 0) { sm.red[threadIdx.x >> 5] = mn; s_part[threadIdx.x >> 5].x = mx; }
  __syncthreads();
  if (unsorted) s_unsorted = 1;
  if (threadIdx.x == 0) {
    double x = sm.red[0], z = s_part[0].x;
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) { x = fmin(x, sm.red[w]); z = fmax(z, s_part[w].x); }
    sm.red[32] = x;
    sm.red[31] = z;
  }
  __syncthreads();
  const double t_ref = sm.red[32], t_max = sm.red[31];
  __syncthreads();
  const double* yy = y + o;
  const double med = block_nanmedian([&](int64_t i) { return yy[i]; }, n, sm);
  // each thread owns a contiguous chunk so that the prefix sums can be formed in two passes
  const int64_t L = (n + blockDim.x - 1) / blockDim.x;
  const int64_t lo = min((int64_t)threadIdx.x * L, n), hi = min(lo + L, n);
  double sy = 0.0, si = 0.0;
  for (int64_t i = lo; i < hi; ++i) {
    const double w = dy ? 1.0 / (dy[o + i] * dy[o + i]) : 1.0;
    const double v = (yy[i] - med) * w;
    trel[o + i] = t[o + i] - t_ref;
    wy[o + i] = v;
    iv[o + i] = w;
    sy += v;
    si += w;
  }
  s_part[threadIdx.x] = make_double2(sy, si);
  __syncthreads();
  if (threadIdx.x == 0) {
    double ax = 0.0, ay = 0.0;
    for (int k = 0; k < (int)blockDim.x; ++k) {
      const double2 p = s_part[k];
      s_part[k] = make_double2(ax, ay);
      ax += p.x; ay += p.y;
    }
    info[b].t_ref = t_ref;
    info[b].sum_y = ax;
    info[b].sum_ivar = ay;
    info[b].min_t = 0.0;   // min(t - t_ref)
    info[b].x_max = t_max - t_ref;
    info[b].sorted = s_unsorted ? 0 : 1;
    info[b].pad = 0;
  }
  __syncthreads();
  if (cpre) {
    double2* c = cpre + o + b;
    double ax = s_part[threadIdx.x].x, ay = s_part[threadIdx.x].y;
    for (int64_t i = lo; i < hi; ++i) {
      c[i] = make_double2(ax, ay);
      ax += wy[o + i]; ay += iv[o + i];
    }
    if (hi == n && lo <= n) c[n] = make_double2(ax, ay);   // (every thread with hi == n holds the full sum)
  }
}

// T[j] = first cadence with x >= j * delta (lower bound), j = 0 .. nT - 1, per light curve.
__global__ void __launch_bounds__(256)
bls_table_kernel(const double* __restrict__ trel, const int64_t* __restrict__ offsets,
                 const int64_t* __restrict__ tab_offsets, int b_base, double delta, int32_t* __restrict__ tab) {
  const int b = b_base + blockIdx.y;           // the launch covers light curves [b_base, b_base + gridDim.y)
  const int64_t o = offsets[b], n = offsets[b + 1] - o;
  const int64_t to = tab_offsets[b], nT = tab_offsets[b + 1] - to;
  const double* x = trel + o;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < nT; j += (int64_t)gridDim.x * blockDim.x) {
    const double target = (double)j * delta;
    int64_t lo = 0, hi = n;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (x[mid] < target) lo = mid + 1; else hi = mid;
    }
    tab[to + j] = (int32_t)lo;
  }
}

// ---- per-warp pieces ------------------------------------------------------------------------
// Add the 32 samples held one per lane into the warp's histogram h[bin] = {sum w*y, sum w}.
// key < 0 => lane inactive.  Equal keys are contiguous (bins are monotone between period wraps), so each
// run's sum is a difference of the light curve's exclusive prefix sums: c_i = prefix before this lane's
// sample, c_next = prefix after it; the run's last lane adds  c_next - c_(run head)  - one writer per bin.
__device__ __forceinline__ void bls_warp_bin(int key, double2 c_i, double2 c_next, double2* h, int lane) {
  const unsigned full = 0xffffffffu;
  const int prev = __shfl_up_sync(full, key, 1);
  const bool head = (lane == 0) || (key != prev);
  const bool wrap = (lane != 0) && (key < prev) && (key >= 0);
  const unsigned headmask = __ballot_sync(full, head);
  const unsigned wrapmask = __ballot_sync(full, wrap);
  const unsigned le = (lane == 31) ? 0xffffffffu : ((2u << lane) - 1u);
  const int start = 31 - __clz(headmask & le);          // lane of this run's head
  const double hy = __shfl_sync(full, c_i.x, start), hi = __shfl_sync(full, c_i.y, start);
  const bool tail = (((headmask >> 1) | 0x80000000u) >> lane & 1u) && key >= 0;
  const double vy = c_next.x - hy, vi = c_next.y - hi;
  if (wrapmask == 0) {
    if (tail) { double2 c = h[key]; c.x += vy; c.y += vi; h[key] = c; }
  } else {
    // split into monotone pieces so that equal keys are contiguous within a piece
    const int piece = __popc(wrapmask & le);
    const int npieces = __popc(wrapmask) + 1;
    for (int q = 0; q < npieces; ++q) {
      if (tail && piece == q) { double2 c = h[key]; c.x += vy; c.y += vi; h[key] = c; }
      __syncwarp();
    }
  }
  __syncwarp();
}

// Inclusive prefix sum over h[0..n] (n+1 entries, both components), in place.  Each lane scans a
// contiguous chunk sequentially; chunk offsets are a SEQUENTIAL prefix (lane 0) so that an empty bin
// leaves the running sum bitwise unchanged also across chunk boundaries (tie preservation).
__device__ __forceinline__ void bls_cumsum(double2* h, int n_entries, double2* scratch, int lane) {
  const int L = (n_entries + 31) / 32;
  const int lo = min(lane * L, n_entries), hi = min(lo + L, n_entries);
  double rx = 0.0, ry = 0.0;
  for (int i = lo; i < hi; ++i) {
    double2 c = h[i];
    rx += c.x; ry += c.y;
    h[i] = make_double2(rx, ry);
  }
  scratch[lane] = make_double2(rx, ry);
  __syncwarp();
  if (lane == 0) {
    double ox = 0.0, oy = 0.0;
    for (int l = 0; l < 32; ++l) {
      const double2 tot = scratch[l];
      scratch[l] = make_double2(ox, oy);
      ox += tot.x; oy += tot.y;
    }
  }
  __syncwarp();
  const double2 off = scratch[lane];
  if (lane > 0)
    for (int i = lo; i < hi; ++i) {
      double2 c = h[i];
      h[i] = make_double2(off.x + c.x, off.y + c.y);
    }
  __syncwarp();
}

// Everything after the histogram is filled: wrap-pad, prefix sums, box scan, first-max, outputs.
__device__ __forceinline__ void bls_finish_warp(double2* h, int n_bins, int oversample, double2* scr, int lane,
                                                const BlsLcInfo& li, const int* __restrict__ dur_bins, int D,
                                                double bin_duration, int objective, double per, double inv_per,
                                                int64_t oi, double* __restrict__ o_power,
                                                double* __restrict__ o_depth, double* __restrict__ o_depth_err,
                                                double* __restrict__ o_duration, double* __restrict__ o_ttime,
                                                double* __restrict__ o_snr, double* __restrict__ o_ll,
                                                int32_t* __restrict__ o_bins) {
  // wrap-pad: mean[n_bins - oversample + (n-1)] = mean[n], n = 1..oversample (no overlap, see DESIGN.md)
  for (int i = lane + 1; i <= oversample; i += 32) h[n_bins - oversample + (i - 1)] = h[i];
  __syncwarp();
  bls_cumsum(h, n_bins + 1, scr, lane);

  // search: only the objective is evaluated per box; the statistics of the winner are recomputed below
  double best_obj = -INFINITY;
  int best_k = 0x7fffffff, best_n = 0x7fffffff;
  for (int k = 0; k < D; ++k) {
    const int dur = dur_bins[k];
    const int n_max = n_bins - dur;
    for (int nn = lane; nn <= n_max; nn += 32) {
      const double2 hb = h[nn + dur], ha = h[nn];
      double y_in = hb.x - ha.x;
      const double ivar_in = hb.y - ha.y;
      double y_out = li.sum_y - y_in;
      const double ivar_out = li.sum_ivar - ivar_in;
      if ((ivar_in < DBL_EPSILON) || (ivar_out < DBL_EPSILON)) continue;
      y_in /= ivar_in;
      y_out /= ivar_out;
      if (!(y_out >= y_in)) continue;
      double obj;
      if (objective) obj = (y_out - y_in) / sqrt(1.0 / ivar_in + 1.0 / ivar_out);
      else obj = 0.5 * ivar_in * (y_out - y_in) * (y_out - y_in);
      if (obj > best_obj) { best_obj = obj; best_k = k; best_n = nn; }
    }
  }
  // first maximum in (duration-major, start-bin-minor) order across lanes
  double wobj = best_obj;
  int wk = best_k, wn = best_n;
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    const double oo = __shfl_xor_sync(0xffffffffu, wobj, s);
    const int ok = __shfl_xor_sync(0xffffffffu, wk, s);
    const int on = __shfl_xor_sync(0xffffffffu, wn, s);
    const bool take = (oo > wobj) || (oo == wobj && (ok < wk || (ok == wk && on < wn)));
    if (take) { wobj = oo; wk = ok; wn = on; }
  }
  if (lane == 0) {
    double depth = 0.0, depth_err = 0.0, snr = 0.0, ll = 0.0, bd = 0.0, ph = 0.0;
    int dur = -1;
    if (wk != 0x7fffffff) {
      dur = dur_bins[wk];
      const double2 hb = h[wn + dur], ha = h[wn];
      double y_in = hb.x - ha.x;
      const double ivar_in = hb.y - ha.y;
      double y_out = li.sum_y - y_in;
      const double ivar_out = li.sum_ivar - ivar_in;
      y_in /= ivar_in;
      y_out /= ivar_out;
      depth = y_out - y_in;
      depth_err = sqrt(1.0 / ivar_in + 1.0 / ivar_out);
      snr = depth / depth_err;
      ll = 0.5 * ivar_in * (y_out - y_in) * (y_out - y_in);
      bd = dur * bin_duration;
      ph = bls_fmod(wn * bin_duration + 0.5 * bd + li.min_t, per, inv_per);
    }
    o_power[oi] = wobj;
    o_depth[oi] = depth;
    o_depth_err[oi] = depth_err;
    o_snr[oi] = snr;
    o_ll[oi] = ll;
    o_duration[oi] = bd;
    o_ttime[oi] = ph + li.t_ref;
    if (o_bins) {
      o_bins[2 * oi] = dur >= 0 ? wn : -1;
      o_bins[2 * oi + 1] = dur;
    }
  }
}

struct BlsFast {            // boundary-path inputs (null tab => cadence path only)
  const double2* cpre;      // [total + B] exclusive prefix sums
  const int32_t* tab;       // lookup tables
  const int64_t* tab_offsets;  // [b] .. [b + 1]: light curve b's table (b in the current table group)
  double delta, inv_delta;
  double min_density;       // use the boundary path when N >= min_density * (x_max / bin_duration)
};

// GHIST = false: per-warp histograms in shared memory; true: in an (L2-resident) global workspace.
template <bool GHIST>
__global__ void __launch_bounds__(BLS_WARPS * 32)
bls_search_kernel(const double* __restrict__ trel, const double* __restrict__ wy, const double* __restrict__ iv,
                  const int64_t* __restrict__ offsets, const BlsLcInfo* __restrict__ info,
                  const double* __restrict__ period, const BlsCta* __restrict__ cta, int64_t out_stride,
                  const int* __restrict__ dur_bins, int D, double bin_duration,
                  int oversample, int objective, int hist_stride, double2* __restrict__ g_hist, BlsFast fast,
                  double* __restrict__ o_power, double* __restrict__ o_depth, double* __restrict__ o_depth_err,
                  double* __restrict__ o_duration, double* __restrict__ o_ttime, double* __restrict__ o_snr,
                  double* __restrict__ o_ll, int32_t* __restrict__ o_bins) {
  extern __shared__ __align__(16) unsigned char bls_smem[];
  double* s_t = reinterpret_cast<double*>(bls_smem);              // sample times of the tile
  double2* s_c = reinterpret_cast<double2*>(s_t + BLS_TILE);      // BLS_TILE + 1 exclusive prefix sums
  double2* s_scr = s_c + BLS_TILE + 1;                            // BLS_WARPS * 32
  double2* s_hist = s_scr + BLS_WARPS * 32;                       // BLS_WARPS * hist_stride (unless GHIST)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const BlsCta d = cta[blockIdx.x];             // this CTA: periods d.p .. d.p + d.n - 1 of light curve d.b
  const int b = d.b;
  const int64_t o = offsets[b], n = offsets[b + 1] - o;
  const int nwarps = blockDim.x >> 5;
  const int p = d.p + warp;                     // index into `period` (< 2^31); output at b * out_stride + p
  if (n <= 0) {      // empty light curve: every output NaN
    if (warp < d.n && lane == 0) {
      const double qn = __longlong_as_double(0x7ff8000000000000ll);
      const int64_t oi = (int64_t)b * out_stride + p;
      o_power[oi] = qn; o_depth[oi] = qn; o_depth_err[oi] = qn; o_duration[oi] = qn; o_ttime[oi] = qn;
      o_snr[oi] = qn; o_ll[oi] = qn;
      if (o_bins) { o_bins[2 * oi] = -1; o_bins[2 * oi + 1] = -1; }
    }
    return;
  }
  const bool active = warp < d.n;
  const double per = active ? period[p] : 1.0;
  const double inv_per = 1.0 / per;
  const double inv_bin = 1.0 / bin_duration;
  const int K1 = (int)ceil(per / bin_duration);
  const int n_bins = K1 + oversample;
  const double bd_safe = bls_safe_width(bin_duration, n_bins);
  const BlsLcInfo li = info[b];      // min(t - t_ref) = 0: the samples below are times since the first cadence

  double2* h;
  if constexpr (GHIST) {
    const size_t slot = (size_t)blockIdx.x * nwarps + warp;
    h = g_hist + slot * (size_t)hist_stride;
  } else {
    h = s_hist + (size_t)warp * hist_stride;
  }
  if (active)
    for (int i = lane; i <= n_bins; i += 32) h[i] = make_double2(0.0, 0.0);

  // boundary path?  CTA-uniform: sorted times, >= 33 bin slots per cycle (so that the 32 runs a warp
  // adds per step hit 32 different bins) and dense enough sampling for it to be the cheaper one.
  bool use_fast = false;
  if (fast.tab != nullptr && li.sorted) {
    const bool mine = !active || (K1 + 1 >= 33 && per < 1.0e9 * bin_duration &&
                                  (double)n >= fast.min_density * (li.x_max * inv_bin));
    use_fast = __syncthreads_and(mine ? 1 : 0) != 0;
  }

  if (use_fast) {
    if (!active) return;
    __syncwarp();
    const double* x = trel + o;
    const double2* c = fast.cpre + o + b;
    const int32_t* tab = fast.tab + fast.tab_offsets[b];
    const int nT = (int)(fast.tab_offsets[b + 1] - fast.tab_offsets[b]);
    const int kc = K1 + 1;                       // bin slots per cycle: k = 0 .. K1 (the last one normally empty)
    int q_last, k_last;
    bls_cycle_bin(x[n - 1], per, inv_per, bin_duration, inv_bin, bd_safe, q_last, k_last);
    const long long m_end = (long long)q_last * kc + k_last + 1;     // first boundary after the last cadence
    int q = 0, k = lane;                         // boundary m = it * 32 + lane  <->  (q, k); kc >= 33 > lane
    int carry_e = 0;
    double2 carry_c = make_double2(0.0, 0.0);
    for (long long m0 = 0; m0 <= m_end; m0 += 32) {
      int e = (int)n;
      if (m0 + lane <= m_end) {
        // (slot K1 starts at or after the end of the cycle: cap at the cycle end so that the walk starts before it)
        const double xb = fma((double)q, per, fmin((double)k * bin_duration, per));
        int j = (int)(xb * fast.inv_delta) - 1;
        j = max(0, min(j, nT - 1));
        const int e0 = tab[j];                   // every cadence before e0 is more than delta/2 before the boundary
        // Common case: the run starts at the first cadence with x >= xb (plain comparisons on three
        // speculatively loaded candidates).  Only when a cadence sits within ~1e-13 of the boundary can the
        // rounded fmod/division of bls.c disagree with real arithmetic: then walk with the exact function.
        const int nm1 = (int)n - 1;
        const double x0 = x[min(e0, nm1)], x1 = x[min(e0 + 1, nm1)], x2 = x[min(e0 + 2, nm1)];
        double xlo = -1.0e300, xhi = 1.0e300;
        if (x0 >= xb) { e = e0; xhi = x0; }
        else if (x1 >= xb) { e = e0 + 1; xlo = x0; xhi = x1; }
        else if (x2 >= xb) { e = e0 + 2; xlo = x1; xhi = x2; }
        else {
          e = e0 + 3;
          xlo = x2;
          while (e < n) {
            const double xv = x[e];
            if (xv >= xb) { xhi = xv; break; }
            xlo = xv;
            ++e;
          }
        }
        if (e > n) e = (int)n;                   // (the clamped candidates repeat the last cadence)
        const double tol = 1.0e-13 * (xb + per);
        if ((e < n && xhi - xb <= tol) || xb - xlo <= tol) {
          e = e0;
          while (e < n) {
            int qi, ki;
            bls_cycle_bin(x[e], per, inv_per, bin_duration, inv_bin, bd_safe, qi, ki);
            if (qi > q || (qi == q && ki >= k)) break;
            ++e;
          }
        }
      }
      const double2 ce = c[e];
      int e_prev = __shfl_up_sync(0xffffffffu, e, 1);
      double2 c_prev;
      c_prev.x = __shfl_up_sync(0xffffffffu, ce.x, 1);
      c_prev.y = __shfl_up_sync(0xffffffffu, ce.y, 1);
      if (lane == 0) { e_prev = carry_e; c_prev = carry_c; }
      if (e > e_prev) {                          // the run that ends at this boundary: bin slot k - 1 (cyclic)
        const int key = (k == 0 ? kc - 1 : k - 1) + 1;
        double2 cur = h[key];
        cur.x += ce.x - c_prev.x;
        cur.y += ce.y - c_prev.y;
        h[key] = cur;
      }
      carry_e = __shfl_sync(0xffffffffu, e, 31);
      carry_c.x = __shfl_sync(0xffffffffu, ce.x, 31);
      carry_c.y = __shfl_sync(0xffffffffu, ce.y, 31);
      k += 32;
      if (k >= kc) { k -= kc; ++q; }
      __syncwarp();
    }
  } else {
    const double2* cg = fast.cpre + o + b;
    for (int64_t c0 = 0; c0 < n; c0 += BLS_TILE) {
      const int cnt = (int)min((int64_t)BLS_TILE, n - c0);
      __syncthreads();
      for (int i = threadIdx.x; i <= cnt; i += blockDim.x) {
        if (i < cnt) s_t[i] = trel[o + c0 + i];
        s_c[i] = cg[c0 + i];
      }
      __syncthreads();
      if (active) {
        for (int i0 = 0; i0 < cnt; i0 += 32) {
          const int i = i0 + lane;
          const bool valid = i < cnt;
          const int ic = valid ? i : cnt - 1;
          const int key = bls_bin_warp(s_t[ic], valid, per, inv_per, bin_duration, inv_bin, bd_safe);
          bls_warp_bin(key, s_c[ic], s_c[ic + 1], h, lane);
        }
      }
    }
    if (!active) return;
  }
  __syncwarp();
  bls_finish_warp(h, n_bins, oversample, s_scr + warp * 32, lane, li, dur_bins, D, bin_duration, objective, per,
                  inv_per, (int64_t)b * out_stride + p, o_power, o_depth, o_depth_err, o_duration, o_ttime, o_snr, o_ll, o_bins);
}

// ---- host ------------------------------------------------------------------------------------
int bls_bin_index(const double* t_rel, int64_t N, double min_t, double period, double bin_duration, int32_t* ind,
                  int mem, cudaStream_t st) {
  LKB_REQUIRE(t_rel && ind && N > 0, "lkb_bls_bin_index: null/empty argument");
  LKB_REQUIRE(period > 0 && bin_duration > 0, "lkb_bls_bin_index: period and bin_duration must be positive");
  LKB_TRY(ensure_device());
  const double* d_t = nullptr;
  int32_t* d_i = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, t_rel, N, &d_t, st));
  LKB_TRY(stage_out_alloc<int32_t>(mem, WS_OUT0, ind, N, &d_i));
  bls_bin_index_kernel<<<(unsigned)((N + 255) / 256), 256, 0, st>>>(d_t, N, min_t, period, bin_duration, d_i);
  LKB_LAUNCH_CHECK();
  LKB_TRY(stage_out_copy<int32_t>(mem, ind, d_i, N, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

int bls_power(const double* t, const double* y, const double* dy, const int64_t* h_offsets, int B,
              const double* period, const int64_t* period_offsets, int64_t P, const double* duration, int D,
              int oversample, int objective, double* power, double* depth, double* depth_err, double* duration_out,
              double* transit_time, double* depth_snr, double* log_like, int32_t* best_bins, int mem,
              cudaStream_t st) {
  LKB_REQUIRE(t && y && h_offsets && period && duration, "lkb_bls_power: null input");
  LKB_REQUIRE(power && depth && depth_err && duration_out && transit_time && depth_snr && log_like,
              "lkb_bls_power: null output");
  LKB_REQUIRE(B > 0 && B <= 65535 && P > 0 && D > 0 && oversample > 0, "lkb_bls_power: bad sizes");
  LKB_REQUIRE(objective == 0 || objective == 1, "lkb_bls_power: bad objective");
  LKB_REQUIRE(P < ((int64_t)1 << 31), "lkb_bls_power: more than 2^31 - 1 periods");
  const int64_t* pofs = period_offsets;
  if (pofs) {
    LKB_REQUIRE(pofs[0] == 0 && pofs[B] == P, "lkb_bls_power: period_offsets[0] must be 0 and period_offsets[B] == P");
    for (int b = 0; b < B; ++b) {
      if (pofs[b + 1] < pofs[b]) { set_error("lkb_bls_power: period_offsets decrease at light curve %d", b); return LKB_E_ARG; }
      if (pofs[b + 1] == pofs[b]) { set_error("lkb_bls_power: light curve %d has an empty period grid", b); return LKB_E_ARG; }
    }
  }
  LKB_TRY(ensure_device());
  const int64_t total = h_offsets[B];

  // the period / duration grids are needed on the host for validation and launch shaping
  std::vector<double> h_per(P), h_dur(D);
  if (mem == LKB_MEM_HOST) {
    memcpy(h_per.data(), period, sizeof(double) * P);
    memcpy(h_dur.data(), duration, sizeof(double) * D);
  } else {
    LKB_CUDA_CHECK(cudaMemcpyAsync(h_per.data(), period, sizeof(double) * P, cudaMemcpyDeviceToHost, st));
    LKB_CUDA_CHECK(cudaMemcpyAsync(h_dur.data(), duration, sizeof(double) * D, cudaMemcpyDeviceToHost, st));
    LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  }
  // per grid (the shared one, or each light curve's own): finite periods, and its minimum
  const int n_grids = pofs ? B : 1;
  std::vector<double> grid_min(n_grids);
  for (int g = 0; g < n_grids; ++g) {
    const int64_t q0 = pofs ? pofs[g] : 0, q1 = pofs ? pofs[g + 1] : P;
    double mn = h_per[q0];
    for (int64_t i = q0; i < q1; ++i) {
      if (!(h_per[i] == h_per[i]) || isinf(h_per[i])) {
        if (pofs) set_error("lkb_bls_power: period of light curve %d contains nan/inf", g);
        else set_error("lkb_bls_power: period contains nan/inf");
        return LKB_E_ARG;
      }
      mn = fmin(mn, h_per[i]);
    }
    grid_min[g] = mn;
  }
  double min_dur = h_dur[0], max_dur = h_dur[0];
  for (int i = 0; i < D; ++i) {
    if (!(h_dur[i] == h_dur[i]) || isinf(h_dur[i])) { set_error("lkb_bls_power: duration contains nan/inf"); return LKB_E_ARG; }
    min_dur = fmin(min_dur, h_dur[i]);
    max_dur = fmax(max_dur, h_dur[i]);
  }
  for (int g = 0; g < n_grids; ++g) {
    if (grid_min[g] < DBL_EPSILON) {
      if (pofs) set_error("lkb_bls_power: periods of light curve %d must be positive", g);
      else set_error("lkb_bls_power: periods must be positive");
      return LKB_E_ARG;
    }
    if (max_dur >= grid_min[g] || min_dur < DBL_EPSILON) {
      set_error("The maximum transit duration must be shorter than the minimum period");
      return LKB_E_ARG;
    }
  }
  const double bin_duration = min_dur / (double)oversample;
  std::vector<int> h_durbins(D);
  for (int i = 0; i < D; ++i) h_durbins[i] = (int)round(h_dur[i] / bin_duration);

  const double *d_t = nullptr, *d_y = nullptr, *d_dy = nullptr, *d_per = nullptr, *d_dur = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, t, total, &d_t, st));
  LKB_TRY(stage_in<double>(mem, WS_IN1, y, total, &d_y, st));
  LKB_TRY(stage_in<double>(mem, WS_IN2, dy, total, &d_dy, st));
  LKB_TRY(stage_in<double>(mem, WS_IN3, period, P, &d_per, st));
  LKB_TRY(stage_in<double>(mem, WS_IN4, duration, D, &d_dur, st));
  int64_t* d_off = nullptr;
  int* d_durbins = nullptr;
  LKB_TRY(ws_get_t<int64_t>(WS_A, B + 1, &d_off));
  LKB_TRY(ws_get_t<int>(WS_B, D, &d_durbins));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_off, h_offsets, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_durbins, h_durbins.data(), sizeof(int) * D, cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaStreamSynchronize(st));   // h_durbins is a local

  double *d_trel = nullptr, *d_wy = nullptr, *d_iv = nullptr;
  BlsLcInfo* d_info = nullptr;
  LKB_TRY(ws_get_t<double>(WS_C, total, &d_trel));
  LKB_TRY(ws_get_t<double>(WS_D, total, &d_wy));
  LKB_TRY(ws_get_t<double>(WS_E, total, &d_iv));
  LKB_TRY(ws_get_t<BlsLcInfo>(WS_F, B, &d_info));

  // outputs: [B, P] for a shared grid, the CSR layout of `period` for per-light-curve grids
  const size_t outn = pofs ? (size_t)P : (size_t)B * P;
  const int64_t out_stride = pofs ? 0 : P;
  double *o0, *o1, *o2, *o3, *o4, *o5, *o6;
  int32_t* ob = nullptr;
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0, power, outn, &o0));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT1, depth, outn, &o1));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT2, depth_err, outn, &o2));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT3, duration_out, outn, &o3));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT4, transit_time, outn, &o4));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT5, depth_snr, outn, &o5));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT6, log_like, outn, &o6));
  LKB_TRY(stage_out_alloc<int32_t>(mem, WS_OUT7, best_bins, 2 * outn, &ob));

  double2* d_cpre = nullptr;
  LKB_TRY(ws_get_t<double2>(WS_H, total + B, &d_cpre));
  bls_prep_kernel<<<B, 256, 0, st>>>(d_t, d_y, d_dy, d_off, d_trel, d_wy, d_iv, d_cpre, d_info);
  LKB_LAUNCH_CHECK();

  // boundary path set-up: per-light-curve lookup tables "first cadence at or after j * delta", built per table
  // group (bls_plan.h) just before that group's search
  BlsFast fast;
  fast.cpre = d_cpre;
  fast.tab = nullptr;
  fast.tab_offsets = nullptr;
  fast.delta = bin_duration / 8.0;
  fast.inv_delta = 1.0 / fast.delta;
  fast.min_density = 0.8;
  if (const char* e = getenv("LKB_BLS_MIN_DENSITY")) fast.min_density = atof(e);
  std::vector<int64_t> h_to;
  std::vector<BlsTableGroup> groups;
  {
    std::vector<BlsLcInfo> h_info(B);
    LKB_CUDA_CHECK(cudaMemcpyAsync(h_info.data(), d_info, sizeof(BlsLcInfo) * B, cudaMemcpyDeviceToHost, st));
    LKB_CUDA_CHECK(cudaStreamSynchronize(st));
    std::vector<int64_t> n(B);
    std::vector<double> x_max(B);
    for (int b = 0; b < B; ++b) {
      n[b] = h_offsets[b + 1] - h_offsets[b];
      x_max[b] = h_info[b].x_max;
    }
    groups = bls_table_groups(n.data(), x_max.data(), B, fast.inv_delta, fast.min_density < 1e30, pofs == nullptr,
                              BLS_TABLE_BUDGET, h_to);
  }
  // search launches: CTA descriptors of every table group, uploaded once
  BlsPlanLimits lim;
  static const int ghist_bins = getenv("LKB_BLS_GHIST_BINS") ? atoi(getenv("LKB_BLS_GHIST_BINS")) : -1;
  lim.ghist_bins = ghist_bins;
  if (getenv("LKB_BLS_HIST_CAP_MB")) lim.hist_cap = (size_t)atoll(getenv("LKB_BLS_HIST_CAP_MB")) << 20;
  BlsPlan plan;
  std::vector<size_t> group_launch(groups.size() + 1, 0);
  for (size_t gi = 0; gi < groups.size(); ++gi) {
    char msg[256];
    if (!bls_plan(h_per.data(), pofs, P, groups[gi].b0, groups[gi].b1, bin_duration, oversample, lim, plan, msg,
                  sizeof msg)) {
      set_error("%s", msg);
      return LKB_E_UNSUPPORTED;
    }
    group_launch[gi + 1] = plan.launch.size();
  }
  int64_t tab_max = 0;
  for (const BlsTableGroup& g : groups)
    if (g.table) tab_max = std::max(tab_max, h_to[g.b1] - h_to[g.b0]);
  // table offsets relative to each group's first entry: group g's light curves b0 .. b1 (inclusive) at [b + g]
  std::vector<int64_t> h_torel(B + groups.size());
  for (size_t gi = 0; gi < groups.size(); ++gi)
    for (int b = groups[gi].b0; b <= groups[gi].b1; ++b) h_torel[b + gi] = h_to[b] - h_to[groups[gi].b0];
  int64_t* d_to = nullptr;
  int32_t* d_tab = nullptr;
  if (tab_max > 0) {
    LKB_TRY(ws_get_t<int64_t>(WS_I, h_torel.size(), &d_to));
    LKB_TRY(ws_get_t<int32_t>(WS_J, tab_max, &d_tab));
    LKB_CUDA_CHECK(cudaMemcpyAsync(d_to, h_torel.data(), sizeof(int64_t) * h_torel.size(), cudaMemcpyHostToDevice, st));
  }
  BlsCta* d_cta = nullptr;
  LKB_TRY(ws_get_t<BlsCta>(WS_K, plan.cta.size(), &d_cta));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_cta, plan.cta.data(), sizeof(BlsCta) * plan.cta.size(), cudaMemcpyHostToDevice, st));
  double2* g_hist = nullptr;
  if (plan.ghist_bytes > 0) LKB_TRY(ws_get_t<double2>(WS_G, plan.ghist_bytes / sizeof(double2), &g_hist));
  LKB_CUDA_CHECK(cudaStreamSynchronize(st));   // h_torel and plan.cta are locals

  static bool attr_set = false;
  if (!attr_set) {
    LKB_CUDA_CHECK(cudaFuncSetAttribute(bls_search_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    LKB_CUDA_CHECK(cudaFuncSetAttribute(bls_search_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  auto launch_tables = [&](size_t gi) {
    const BlsTableGroup& g = groups[gi];
    if (!g.table) {
      fast.tab = nullptr;
      fast.tab_offsets = nullptr;
      return;
    }
    int64_t nT_max = 0;
    for (int b = g.b0; b < g.b1; ++b) nT_max = std::max(nT_max, h_to[b + 1] - h_to[b]);
    const unsigned gxT = (unsigned)min((int64_t)64, (nT_max + 255) / 256);
    bls_table_kernel<<<dim3(gxT ? gxT : 1, (unsigned)(g.b1 - g.b0)), 256, 0, st>>>(d_trel, d_off, d_to + gi, g.b0,
                                                                                   fast.delta, d_tab);
    fast.tab = d_tab;
    fast.tab_offsets = d_to + gi;
  };
  launch_tables(0);
  LKB_LAUNCH_CHECK();
  prof_begin(st);
  for (size_t gi = 0; gi < groups.size(); ++gi) {
    if (gi > 0) launch_tables(gi);
    for (size_t li = group_launch[gi]; li < group_launch[gi + 1]; ++li) {
      const BlsLaunch& l = plan.launch[li];
      const unsigned gx = (unsigned)(l.cta_end - l.cta_begin);
      if (l.ghist)
        bls_search_kernel<true><<<gx, l.W * 32, l.smem, st>>>(d_trel, d_wy, d_iv, d_off, d_info, d_per,
                                                              d_cta + l.cta_begin, out_stride, d_durbins, D,
                                                              bin_duration, oversample, objective, l.stride, g_hist,
                                                              fast, o0, o1, o2, o3, o4, o5, o6, ob);
      else
        bls_search_kernel<false><<<gx, l.W * 32, l.smem, st>>>(d_trel, d_wy, d_iv, d_off, d_info, d_per,
                                                               d_cta + l.cta_begin, out_stride, d_durbins, D,
                                                               bin_duration, oversample, objective, l.stride, nullptr,
                                                               fast, o0, o1, o2, o3, o4, o5, o6, ob);
    }
    LKB_LAUNCH_CHECK();
  }
  prof_end(st);

  LKB_TRY(stage_out_copy<double>(mem, power, o0, outn, st));
  LKB_TRY(stage_out_copy<double>(mem, depth, o1, outn, st));
  LKB_TRY(stage_out_copy<double>(mem, depth_err, o2, outn, st));
  LKB_TRY(stage_out_copy<double>(mem, duration_out, o3, outn, st));
  LKB_TRY(stage_out_copy<double>(mem, transit_time, o4, outn, st));
  LKB_TRY(stage_out_copy<double>(mem, depth_snr, o5, outn, st));
  LKB_TRY(stage_out_copy<double>(mem, log_like, o6, outn, st));
  LKB_TRY(stage_out_copy<int32_t>(mem, best_bins, ob, 2 * outn, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

int bls_stats(const double* t, const double* y, const double* dy, const int64_t* h_offsets, int B,
              const double* period, const double* duration, const double* transit_time, const int64_t* h_toff,
              double* stats, int64_t* transit_first, int32_t* transit_n, int32_t* per_transit_count,
              double* per_transit_ll, uint8_t* in_transit, int32_t* status, int mem, cudaStream_t st) {
  LKB_REQUIRE(t && y && h_offsets && period && duration && transit_time && h_toff, "lkb_bls_stats: null input");
  LKB_REQUIRE(stats && transit_first && transit_n && status, "lkb_bls_stats: null output");
  LKB_REQUIRE(B > 0, "lkb_bls_stats: B must be > 0");
  LKB_REQUIRE(h_offsets[0] == 0 && h_toff[0] == 0, "lkb_bls_stats: offsets[0] and transit_offsets[0] must be 0");
  for (int b = 0; b < B; ++b) {
    const int64_t nb = h_offsets[b + 1] - h_offsets[b];
    if (nb < 1 || nb >= ((int64_t)1 << 31)) {
      set_error("lkb_bls_stats: light curve %d has %lld cadences (1 .. 2^31 - 1 supported)", b, (long long)nb);
      return LKB_E_ARG;
    }
    if (h_toff[b + 1] < h_toff[b]) {
      set_error("lkb_bls_stats: transit_offsets decrease at light curve %d", b);
      return LKB_E_ARG;
    }
  }
  const int64_t total = h_offsets[B], slots = h_toff[B];
  LKB_REQUIRE(slots == 0 || (per_transit_count && per_transit_ll), "lkb_bls_stats: null per-transit output");
  LKB_TRY(ensure_device());

  // the candidates are checked on the host
  std::vector<double> h_cand(3 * (size_t)B);
  const double* cand[3] = {period, duration, transit_time};
  for (int k = 0; k < 3; ++k) {
    if (mem == LKB_MEM_HOST) memcpy(h_cand.data() + (size_t)k * B, cand[k], sizeof(double) * B);
    else LKB_CUDA_CHECK(cudaMemcpyAsync(h_cand.data() + (size_t)k * B, cand[k], sizeof(double) * B,
                                        cudaMemcpyDeviceToHost, st));
  }
  if (mem != LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  for (int b = 0; b < B; ++b) {
    const double p = h_cand[b], d = h_cand[(size_t)B + b], tt = h_cand[2 * (size_t)B + b];
    if (!(p > 0.0) || isinf(p) || !(d > 0.0) || isinf(d)) {
      set_error("lkb_bls_stats: light curve %d: period (%g) and duration (%g) must be positive and finite", b, p, d);
      return LKB_E_ARG;
    }
    if (!isfinite(tt)) {
      set_error("lkb_bls_stats: light curve %d: transit_time is not finite", b);
      return LKB_E_ARG;
    }
  }

  const double *d_t = nullptr, *d_y = nullptr, *d_dy = nullptr, *d_p = nullptr, *d_d = nullptr, *d_tt = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, t, total, &d_t, st));
  LKB_TRY(stage_in<double>(mem, WS_IN1, y, total, &d_y, st));
  LKB_TRY(stage_in<double>(mem, WS_IN2, dy, total, &d_dy, st));
  LKB_TRY(stage_in<double>(mem, WS_IN3, period, B, &d_p, st));
  LKB_TRY(stage_in<double>(mem, WS_IN4, duration, B, &d_d, st));
  LKB_TRY(stage_in<double>(mem, WS_IN5, transit_time, B, &d_tt, st));
  int64_t *d_off = nullptr, *d_toff = nullptr;
  LKB_TRY(ws_get_t<int64_t>(WS_A, (size_t)B + 1, &d_off));
  LKB_TRY(ws_get_t<int64_t>(WS_B, (size_t)B + 1, &d_toff));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_off, h_offsets, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_toff, h_toff, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  double *o_st = nullptr, *o_ll = nullptr;
  int64_t* o_first = nullptr;
  int32_t *o_n = nullptr, *o_cnt = nullptr, *o_status = nullptr;
  uint8_t* o_mask = nullptr;
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0, stats, (size_t)B * LKB_BLS_STATS_NCOL, &o_st));
  LKB_TRY(stage_out_alloc<int64_t>(mem, WS_OUT1, transit_first, B, &o_first));
  LKB_TRY(stage_out_alloc<int32_t>(mem, WS_OUT2, transit_n, B, &o_n));
  LKB_TRY(stage_out_alloc<int32_t>(mem, WS_OUT3, slots ? per_transit_count : nullptr, slots, &o_cnt));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT4, slots ? per_transit_ll : nullptr, slots, &o_ll));
  LKB_TRY(stage_out_alloc<uint8_t>(mem, WS_OUT5, in_transit, total, &o_mask));
  LKB_TRY(stage_out_alloc<int32_t>(mem, WS_OUT6, status, B, &o_status));
  prof_begin(st);
  LKB_TRY(bls_stats_launch(d_t, d_y, d_dy, d_off, B, d_p, d_d, d_tt, d_toff, o_st, o_first, o_n, o_cnt, o_ll, o_mask,
                           o_status, st));
  prof_end(st);
  LKB_TRY(stage_out_copy<double>(mem, stats, o_st, (size_t)B * LKB_BLS_STATS_NCOL, st));
  LKB_TRY(stage_out_copy<int64_t>(mem, transit_first, o_first, B, st));
  LKB_TRY(stage_out_copy<int32_t>(mem, transit_n, o_n, B, st));
  LKB_TRY(stage_out_copy<int32_t>(mem, slots ? per_transit_count : nullptr, o_cnt, slots, st));
  LKB_TRY(stage_out_copy<double>(mem, slots ? per_transit_ll : nullptr, o_ll, slots, st));
  LKB_TRY(stage_out_copy<uint8_t>(mem, in_transit, o_mask, total, st));
  LKB_TRY(stage_out_copy<int32_t>(mem, status, o_status, B, st));
  // slot capacity: read the statuses (and the slots each light curve needed) back
  std::vector<int32_t> h_status(B), h_n(B);
  if (mem == LKB_MEM_HOST) {
    LKB_CUDA_CHECK(cudaStreamSynchronize(st));
    memcpy(h_status.data(), status, sizeof(int32_t) * B);
    memcpy(h_n.data(), transit_n, sizeof(int32_t) * B);
  } else {
    LKB_CUDA_CHECK(cudaMemcpyAsync(h_status.data(), status, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, st));
    LKB_CUDA_CHECK(cudaMemcpyAsync(h_n.data(), transit_n, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, st));
    LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  }
  for (int b = 0; b < B; ++b)
    if (h_status[b] == LKB_E_ARG) {
      set_error("lkb_bls_stats: light curve %d needs %d transit slots, transit_offsets gives it %lld", b, h_n[b],
                (long long)(h_toff[b + 1] - h_toff[b]));
      return LKB_E_ARG;
    }
  return LKB_OK;
}

}  // namespace lkb
