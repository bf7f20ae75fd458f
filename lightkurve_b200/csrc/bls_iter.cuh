// K14: the steps between the rounds of an iterative transit search (LightCurveCollection.find_transit_candidates), one CTA
// per light curve:
//
// bls_best_kernel: np.nanargmax of a light curve's segment of the K3 power - the first index of the largest non-NaN
//   value, -1 when every value is NaN - and the K3 outputs there.  Each thread keeps the best (value, index) of its
//   strided share; warps and then the block merge them by "larger value, else smaller index", a total order, so the
//   winner does not depend on the merge order.  The period is written as 1 / (1 / period[k]): the period_at_max_power
//   of BoxLeastSquaresPeriodogram, whose frequency axis is 1 / period.
//
// transit_count_kernel + transit_compact_kernel: lc[~get_transit_mask(P, D, T0)] from K10's in-transit flags and box
//   levels.  get_transit_mask is `model != median(model)` for the two-valued model (y_in in transit, y_out elsewhere):
//   with fewer than half the cadences in transit the median is y_out, with more it is y_in, with exactly half it is
//   (y_in + y_out) / 2, so whether an in-transit and whether an out-of-transit cadence is removed are two flags per
//   light curve (transit_count_kernel, one thread per light curve, which also counts the survivors).  The compaction
//   keeps the survivors in their order (a block scan per tile of BI_THREADS cadences), carries time, flux, flux_err
//   and the cadence's index in the original light curve, writes the round into masked_in at the removed cadences'
//   original positions, and reports what the next round's grid and weights need: the first, smallest and largest
//   surviving time, whether every surviving flux_err is finite (then the weights are flux_err, else unit weights, as
//   BoxLeastSquaresPeriodogram._prepare chooses them), and np.diff of the surviving times for the median step.
//
// Kept apart from the library's entry points (bls_iter.cu) so that tests/native/cuda_emu.h runs it on the CPU.
#pragma once
#include "common.cuh"

namespace lkb {

constexpr int BI_THREADS = 256;
constexpr int BI_STAT_COLS = 15;                  // LKB_BLS_STATS_NCOL

struct BestArgs {
  const double *power, *depth, *depth_err, *duration, *transit_time, *depth_snr;   // K3 outputs
  const double* period;     // the grid: [P] shared, or the CSR of pofs
  const int64_t* pofs;      // [B + 1] device CSR of the periods, or NULL: light curve b's outputs at b * P
  int64_t P;
  double *period_out, *duration_out, *transit_time_out, *depth_out, *depth_err_out, *depth_snr_out, *power_out;  // [B]
  int64_t* index_out;       // [B], -1: every power is NaN
};

// a before b in the nanargmax order (larger value first, then smaller index); index < 0 is "none"
__device__ __forceinline__ bool bi_better(double va, int64_t ia, double vb, int64_t ib) {
  if (ib < 0) return ia >= 0;
  if (ia < 0) return false;
  if (va != vb) return va > vb;
  return ia < ib;
}

__global__ void __launch_bounds__(BI_THREADS) bls_best_kernel(BestArgs a) {
  __shared__ double s_v[BI_THREADS / 32];
  __shared__ int64_t s_i[BI_THREADS / 32];
  const int b = blockIdx.x;
  const int64_t q0 = a.pofs ? a.pofs[b] : (int64_t)b * a.P;
  const int64_t n = a.pofs ? a.pofs[b + 1] - q0 : a.P;
  const double* pw = a.power + q0;
  double bv = 0.0;
  int64_t bi = -1;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const double v = pw[i];
    if (v == v && bi_better(v, i, bv, bi)) { bv = v; bi = i; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int64_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (bi_better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) { s_v[w] = bv; s_i[w] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < (int)(blockDim.x >> 5); ++k)
      if (bi_better(s_v[k], s_i[k], bv, bi)) { bv = s_v[k]; bi = s_i[k]; }
    const double qnan = nan("");
    a.index_out[b] = bi;
    if (bi < 0) {
      a.period_out[b] = a.duration_out[b] = a.transit_time_out[b] = a.depth_out[b] = a.depth_err_out[b] =
          a.depth_snr_out[b] = a.power_out[b] = qnan;
    } else {
      const int64_t k = q0 + bi;
      const double per = a.pofs ? a.period[k] : a.period[bi];
      a.period_out[b] = 1.0 / (1.0 / per);
      a.duration_out[b] = a.duration[k];
      a.transit_time_out[b] = a.transit_time[k];
      a.depth_out[b] = a.depth[k];
      a.depth_err_out[b] = a.depth_err[k];
      a.depth_snr_out[b] = a.depth_snr[k];
      a.power_out[b] = a.power[k];
    }
  }
}

// Flags (bit 0: remove the in-transit cadences, bit 1: the out-of-transit ones) and survivor count per light curve.
__global__ void transit_count_kernel(const int64_t* __restrict__ off, int B, const double* __restrict__ stats,
                                     int32_t* __restrict__ flags, int64_t* __restrict__ count) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int64_t n = off[b + 1] - off[b];
  const double* s = stats + (size_t)b * BI_STAT_COLS;
  const double y_in = s[12], y_out = s[13];
  const int64_t n_in = (int64_t)s[14];
  double med;
  if (2 * n_in < n) med = y_out;
  else if (2 * n_in > n) med = y_in;
  else med = (y_in + y_out) / 2.0;                 // np.mean of the two levels
  const bool drop_in = y_in != med, drop_out = y_out != med;
  flags[b] = (drop_in ? 1 : 0) | (drop_out ? 2 : 0);
  count[b] = n - (drop_in ? n_in : 0) - (drop_out ? n - n_in : 0);
}

struct CompactArgs {
  const double *t, *y, *dy;      // [off[B]] this round's cadences
  const int32_t* idx;            // [off[B]] their index in the original light curve
  const int64_t* off;            // [B + 1] device CSR
  const uint8_t* in_transit;     // [off[B]] K10's flags
  const int32_t* flags;          // [B] transit_count_kernel's
  const int64_t* noff;           // [B + 1] CSR of the survivors
  const int64_t* doff;           // [B + 1] CSR of their consecutive differences (max(n - 1, 0) each)
  const int64_t* orig_off;       // [B + 1] CSR of the original light curves (masked_in)
  int round;
  int8_t* masked_in;             // [orig_off[B]]
  double *t_out, *y_out, *dy_out, *w_out;   // [noff[B]]; w: dy, or 1 where a surviving dy is not finite
  int32_t* idx_out;              // [noff[B]]
  double* tinfo;                 // [B, 3]: first, smallest and largest surviving time (NaN without survivors)
  uint8_t* dy_finite;            // [B]
  double* dt;                    // [doff[B]]
};

__device__ __forceinline__ bool bi_keep(uint8_t in_tr, int flags) { return !(flags & (in_tr ? 1 : 2)); }

__global__ void __launch_bounds__(BI_THREADS) transit_compact_kernel(CompactArgs a) {
  __shared__ int s_wsum[33];
  __shared__ double s_red[33];
  const int b = blockIdx.x, tid = threadIdx.x, T = blockDim.x;
  const int64_t o = a.off[b], n = a.off[b + 1] - o, no = a.noff[b], cnt = a.noff[b + 1] - no;
  const int fl = a.flags[b];
  // pass 1: extremes of the surviving times and whether every surviving flux_err is finite
  double mn = INFINITY, mx = -INFINITY;
  int bad = 0;
  for (int64_t i = tid; i < n; i += T) {
    if (!bi_keep(a.in_transit[o + i], fl)) continue;
    const double t = a.t[o + i];
    mn = fmin(mn, t);
    mx = fmax(mx, t);
    bad |= isfinite(a.dy[o + i]) ? 0 : 1;
  }
  for (int k = 16; k > 0; k >>= 1) {
    mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, k));
    mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, k));
    bad |= __shfl_xor_sync(0xffffffffu, bad, k);
  }
  const int lane = tid & 31, wid = tid >> 5, nw = T >> 5;
  if (lane == 0) { s_red[wid] = mn; s_red[16 + wid] = mx; s_wsum[wid] = bad; }
  __syncthreads();
  if (tid == 0) {
    for (int k = 1; k < nw; ++k) { mn = fmin(mn, s_red[k]); mx = fmax(mx, s_red[16 + k]); bad |= s_wsum[k]; }
    s_red[32] = bad ? 0.0 : 1.0;
    const double qnan = nan("");
    a.tinfo[3 * (size_t)b + 1] = cnt ? mn : qnan;
    a.tinfo[3 * (size_t)b + 2] = cnt ? mx : qnan;
    a.dy_finite[b] = bad ? 0 : 1;
  }
  __syncthreads();
  const bool unit_w = s_red[32] == 0.0;
  __syncthreads();
  // pass 2: stable compaction, one tile of T cadences per step
  int64_t base = 0;
  for (int64_t i0 = 0; i0 < n; i0 += T) {
    const int64_t i = i0 + tid;
    const bool in = i < n;
    const bool keep = in && bi_keep(a.in_transit[o + i], fl);
    // exclusive scan of keep in thread order, and the tile's total
    int x = keep ? 1 : 0;
    for (int k = 1; k < 32; k <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, x, k);
      if (lane >= k) x += v;
    }
    if (lane == 31) s_wsum[wid] = x;
    __syncthreads();
    if (wid == 0) {
      int v = lane < nw ? s_wsum[lane] : 0;
      for (int k = 1; k < 32; k <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, v, k);
        if (lane >= k) v += u;
      }
      if (lane < nw) s_wsum[lane] = v;
    }
    __syncthreads();
    const int pos = (wid ? s_wsum[wid - 1] : 0) + x - (keep ? 1 : 0);
    const int tile = s_wsum[nw - 1];
    if (keep) {
      const int64_t d = no + base + pos;
      const double dyv = a.dy[o + i];
      a.t_out[d] = a.t[o + i];
      a.y_out[d] = a.y[o + i];
      a.dy_out[d] = dyv;
      a.w_out[d] = unit_w ? 1.0 : dyv;
      a.idx_out[d] = a.idx[o + i];
    } else if (in) {
      a.masked_in[a.orig_off[b] + a.idx[o + i]] = (int8_t)a.round;
    }
    base += tile;
    __syncthreads();                               // s_wsum is rewritten by the next tile
  }
  // the survivors are in place (a barrier makes this block's global writes visible to it): first time and steps
  if (tid == 0) a.tinfo[3 * (size_t)b] = cnt ? a.t_out[no] : nan("");
  const int64_t d0 = a.doff[b];
  for (int64_t i = tid; i + 1 < cnt; i += T) a.dt[d0 + i] = a.t_out[no + i + 1] - a.t_out[no + i];
}

}  // namespace lkb
