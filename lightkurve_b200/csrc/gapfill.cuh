// K15: LightCurve.fill_gaps (method="gaussian_noise", the variant without cadence numbers) for many light curves.
// Replaces the per-light-curve loop of /root/reference/src/lightkurve/lightcurve.py:1329-1427 as this repository's
// LightCurve.fill_gaps implements it:
//     dt = nanmedian(diff(t));  wherever t[i] - prev > 1.2 * dt insert prev += dt (prev restarting from t[i-1]);
//     flux_err at an inserted cadence = np.interp(x, t, flux_err);  flux = mean + std * z.
// Every gap restarts from an original time, so gaps are independent: one thread walks one gap with the loop's own
// sequential `prev + dt`, and a block scan of the per-gap counts gives every cadence its output position.  An
// inserted time lies strictly between its two original neighbours, so which cadences are original is positional.
// Compiled with -fmad=false (gapfill.cu; -ffp-contract=off in the emulator) so that 1.2 * dt, mean + std * z and the
// interpolation round like numpy's separate operations.
//
//   normalize_compact_kernel  normalize().remove_nans() before the gap filling (the seismology chain)
//   gap_steps_kernel  np.diff of the times (for the K6 median step) and the reject flags of each light curve
//   gap_plan_kernel   inserted cadences per light curve and the mean flux, given the median step
//   gap_fill_kernel   the filled time / flux / flux_err CSR, given the normal deviates z
#pragma once
#include "common.cuh"

namespace lkb {

constexpr int GF_THREADS = 256;
// A gap longer than this many median steps is refused (GF_LONG_GAP); it bounds every thread's walk.
constexpr int64_t GF_MAX_GAP = (int64_t)1 << 24;

// gap flags, per light curve
constexpr int GF_DECREASING = 1;    // some time step < 0
constexpr int GF_POSITIVE = 2;      // some time step > 0
constexpr int GF_LONG_GAP = 4;      // a gap of more than GF_MAX_GAP steps, or a step dt that does not advance prev

// Cadences the loop inserts between the original times tp < tn: while (tn - prev > 1.2 * dt) prev += dt.
// Returns -1 when the walk would exceed GF_MAX_GAP steps or stall (prev + dt == prev).
__host__ __device__ inline int64_t gf_gap_count(double tp, double tn, double dt) {
  if (!(dt > 0.0)) return 0;                       // the caller rejects a positive step with dt <= 0
  const double lim = 1.2 * dt;
  double prev = tp;
  int64_t k = 0;
  while (tn - prev > lim) {
    const double nx = prev + dt;
    if (!(nx > prev) || k >= GF_MAX_GAP) return -1;
    prev = nx;
    ++k;
  }
  return k;
}

// numpy's interp between (x0, f0) and (x1, f1) for x0 <= x < x1 (compiled_base.c, including its NaN second try).
__host__ __device__ inline double gf_interp(double x, double x0, double x1, double f0, double f1) {
  const double slope = (f1 - f0) / (x1 - x0);
  double r = slope * (x - x0) + f0;
  if (r != r) {
    r = slope * (x - x1) + f1;
    if (r != r && f0 == f1) r = f0;
  }
  return r;
}

// Inclusive block scan of v (every thread of the CTA calls it); *total gets the CTA's sum.  s: 33 int64 of shared.
__device__ inline int64_t gf_block_scan(int64_t v, int64_t* s, int64_t* total) {
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
  for (int k = 1; k < 32; k <<= 1) {
    const int64_t u = __shfl_up_sync(0xffffffffu, v, k);
    if (lane >= k) v += u;
  }
  if (lane == 31) s[wid] = v;
  __syncthreads();
  if (wid == 0) {
    int64_t w = lane < nw ? s[lane] : 0;
    for (int k = 1; k < 32; k <<= 1) {
      const int64_t u = __shfl_up_sync(0xffffffffu, w, k);
      if (lane >= k) w += u;
    }
    if (lane < nw) s[lane] = w;
  }
  __syncthreads();
  const int64_t r = v + (wid ? s[wid - 1] : 0);
  *total = s[nw - 1];
  __syncthreads();                                 // s is reused by the next call
  return r;
}

// LightCurve.normalize().remove_nans() (lightcurve.py:1216-1327): y / med[b] and e / med[b], keeping the cadences whose
// normalized flux is not NaN, in order.  One CTA per light curve.  Counting pass (t_out == nullptr): count[b] = the
// cadences kept, bad[b] = 1 when a kept time is not finite.  Writing pass: the kept cadences at noff[b], and
// ends[2b], ends[2b+1] = the first and last kept time.
struct NormArgs {
  const double *t, *y, *e;         // [off[B]] the raw light curves
  const int64_t* off;              // [B + 1]
  const double* med;               // [B] nanmedian of the flux (K6)
  int64_t* count;                  // [B]   counting pass
  int32_t* bad;                    // [B]   counting pass
  const int64_t* noff;             // [B + 1] writing pass: CSR of the kept cadences
  double *t_out, *y_out, *e_out;   // [noff[B]]
  double* ends;                    // [2 B]
};

__global__ void __launch_bounds__(GF_THREADS) normalize_compact_kernel(NormArgs a) {
  __shared__ int64_t s_c[33];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int64_t o = a.off[b], n = a.off[b + 1] - o;
  const double m = a.med[b];
  int64_t base = 0;
  int bad = 0;
  for (int64_t i0 = 0; i0 < n; i0 += blockDim.x) {
    const int64_t i = i0 + tid;
    double y = 0.0;
    bool keep = false;
    if (i < n) {
      y = a.y[o + i] / m;
      keep = !(y != y);
    }
    int64_t tile;
    const int64_t incl = gf_block_scan(keep ? 1 : 0, s_c, &tile);
    if (keep) {
      const double t = a.t[o + i];
      if (a.t_out) {
        const int64_t d = a.noff[b] + base + incl - 1;
        a.t_out[d] = t;
        a.y_out[d] = y;
        a.e_out[d] = a.e[o + i] / m;
      } else if (!isfinite(t)) {
        bad = 1;
      }
    }
    base += tile;
  }
  if (a.t_out) {
    __syncthreads();                               // the block's writes above are visible to thread 0
    if (tid == 0) {
      const int64_t no = a.noff[b], cnt = a.noff[b + 1] - no;
      a.ends[2 * (size_t)b] = cnt ? a.t_out[no] : nan("");
      a.ends[2 * (size_t)b + 1] = cnt ? a.t_out[no + cnt - 1] : nan("");
    }
    return;
  }
  for (int k = 16; k > 0; k >>= 1) bad |= __shfl_xor_sync(0xffffffffu, bad, k);
  if ((tid & 31) == 0) s_c[tid >> 5] = bad;
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) bad |= (int)s_c[w];
    a.count[b] = base;
    a.bad[b] = bad;
  }
}

// steps[doff[b] + i] = t[i + 1] - t[i]; flags[b] = GF_DECREASING | GF_POSITIVE as they occur.  One CTA per light curve.
__global__ void __launch_bounds__(GF_THREADS)
gap_steps_kernel(const double* __restrict__ t, const int64_t* __restrict__ off, const int64_t* __restrict__ doff,
                 double* __restrict__ steps, int32_t* __restrict__ flags) {
  __shared__ int s_f[32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int64_t o = off[b], n = off[b + 1] - o, d0 = doff[b];
  int f = 0;
  for (int64_t i = tid; i + 1 < n; i += blockDim.x) {
    const double d = t[o + i + 1] - t[o + i];
    steps[d0 + i] = d;
    f |= (d < 0.0 ? GF_DECREASING : 0) | (d > 0.0 ? GF_POSITIVE : 0);
  }
  for (int k = 16; k > 0; k >>= 1) f |= __shfl_xor_sync(0xffffffffu, f, k);
  if ((tid & 31) == 0) s_f[tid >> 5] = f;
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) f |= s_f[w];
    flags[b] = f;
  }
}

// n_ins[b] = cadences the loop inserts, mean[b] = sum(flux) / n (the flux is NaN-free), flags[b] |= GF_LONG_GAP.
// dt [B]: the median step (NaN for n < 2, where nothing is inserted).  One CTA per light curve.
__global__ void __launch_bounds__(GF_THREADS)
gap_plan_kernel(const double* __restrict__ t, const double* __restrict__ y, const int64_t* __restrict__ off,
                const double* __restrict__ dt, int64_t* __restrict__ n_ins, double* __restrict__ mean,
                int32_t* __restrict__ flags) {
  __shared__ int64_t s_c[33];
  __shared__ double s_y[32];
  __shared__ int s_f[32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
  const int64_t o = off[b], n = off[b + 1] - o;
  const double d = n >= 2 ? dt[b] : 0.0;
  int64_t c = 0;
  double sy = 0.0;
  int f = 0;
  for (int64_t i = tid; i < n; i += blockDim.x) {
    sy += y[o + i];
    if (i >= 1) {
      const int64_t k = gf_gap_count(t[o + i - 1], t[o + i], d);
      if (k < 0) f = GF_LONG_GAP; else c += k;
    }
  }
  for (int k = 16; k > 0; k >>= 1) {
    c += __shfl_xor_sync(0xffffffffu, c, k);
    sy += __shfl_xor_sync(0xffffffffu, sy, k);
    f |= __shfl_xor_sync(0xffffffffu, f, k);
  }
  if (lane == 0) { s_c[wid] = c; s_y[wid] = sy; s_f[wid] = f; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < nw; ++w) { c += s_c[w]; sy += s_y[w]; f |= s_f[w]; }
    n_ins[b] = f ? 0 : c;
    mean[b] = n ? sy / (double)n : nan("");
    flags[b] |= f;
  }
}

struct FillArgs {
  const double *t, *y, *e;         // [off[B]] sorted times, flux, flux_err of each light curve
  const int64_t* off;              // [B + 1]
  const int64_t* noff;             // [B + 1] CSR of the filled light curves (n_b + n_ins[b])
  const double *dt, *mean, *std;   // [B]
  const double* z;                 // [noff[B] - off[B]] normal deviates; light curve b's start at noff[b] - off[b]
  double *t_out, *y_out, *e_out;   // [noff[B]]
};

// One CTA per light curve, one tile of blockDim.x cadences per step.  Thread i writes original cadence i and, before
// it, the cadences inserted in the gap t[i-1] .. t[i]: positions from a scan of the per-gap counts.
__global__ void __launch_bounds__(GF_THREADS) gap_fill_kernel(FillArgs a) {
  __shared__ int64_t s_c[33];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int64_t o = a.off[b], n = a.off[b + 1] - o, no = a.noff[b], z0 = no - o;
  const double d = n >= 2 ? a.dt[b] : 0.0, m = a.mean[b], s = a.std[b];
  int64_t base = 0;                                // cadences inserted before this tile
  for (int64_t i0 = 0; i0 < n; i0 += blockDim.x) {
    const int64_t i = i0 + tid;
    const bool in = i < n;
    const int64_t k = (in && i >= 1) ? gf_gap_count(a.t[o + i - 1], a.t[o + i], d) : 0;
    const int64_t c = k > 0 ? k : 0;               // a refused gap (-1) never reaches here; keep the scan sane
    int64_t tile;
    const int64_t incl = gf_block_scan(c, s_c, &tile);
    if (in) {
      const int64_t before = base + incl;          // inserted cadences before original i
      a.t_out[no + i + before] = a.t[o + i];
      a.y_out[no + i + before] = a.y[o + i];
      a.e_out[no + i + before] = a.e[o + i];
      if (c > 0) {
        const double x0 = a.t[o + i - 1], x1 = a.t[o + i], f0 = a.e[o + i - 1], f1 = a.e[o + i];
        const int64_t first = before - c;          // index of this gap's first insert among the light curve's
        double prev = x0;
        for (int64_t k = 0; k < c; ++k) {
          prev = prev + d;
          const int64_t p = no + i - 1 + first + k + 1;
          a.t_out[p] = prev;
          a.e_out[p] = gf_interp(prev, x0, x1, f0, f1);
          a.y_out[p] = m + s * a.z[z0 + first + k];
        }
      }
    }
    base += tile;
  }
}

}  // namespace lkb
