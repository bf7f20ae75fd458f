// K10: the vetting step after a BLS search, for many light curves in one launch: the statistics of
// BoxLeastSquaresPeriodogram.compute_stats (periodogram.py:1194-1229, astropy BoxLeastSquares.compute_stats) and the
// transit mask of get_transit_mask (periodogram.py:1275-1296) of one candidate (period, duration, transit_time) per
// light curve.
//
// One CTA per light curve, two passes over its cadences (t, y, dy: 24 bytes per cadence per pass):
//   pass 1  with t = t_abs - t_abs[0] and tt = transit_time - t_abs[0] (the host code's origin), the masks
//           m_in, m_odd, m_even, m_phase, m_half and, on the unshifted times of get_transit_model, m_model; the sums
//           of ivar and y ivar over each mask and its complement, the weighted normal equations of
//           [sin 2 pi t / P, cos 2 pi t / P, 1], the counts, and the first and last transit id rint((t - tt) / P) of
//           the in-transit cadences.
//   finish  (thread 0) the _compute_depth pairs, y_in / y_out, and the 3x3 solve by LU with partial pivoting; an
//           exactly zero pivot is numpy's LinAlgError (status LKB_E_SINGULAR).
//   pass 2  full_ll, sin_ll, the per-transit counts and log-likelihoods and the in-transit mask.
//
// The masks and transit ids are bit-exact: the remainders are numpy's float `%` (an exact fmod plus numpy's sign
// fix-up) in numpy's operand order, the ids use an IEEE division and rint (round half to even, like np.round), and
// the translation unit that includes this header (bls.cu) is compiled with -fmad=false.
//
// Every sum has a fixed order: per-thread strided partial sums and a fixed tree for the block sums.  The per-transit
// sums go through chunks of BST_THREADS cadences in index order: each warp sums the runs of equal transit id among
// its 32 cadences in lane order, then warp 0 adds the run sums to the transit slots in (warp, lane) order.  So a
// light curve's results depend on its own data only - not on the batch, the launch or the run - and unsorted times
// are handled like sorted ones.  No inline PTX, no atomics: tests/native/cuda_emu.h runs this file on the CPU
// (tests/test_bls_stats_emulated.py).
#pragma once
#include "common.cuh"

namespace lkb {

constexpr int BST_THREADS = 256;
constexpr int BST_WARPS = BST_THREADS / 32;

// exact fmod for finite x, p != 0, |x/p| < 2^50 (true for any real light curve); inv_p = 1 / |p|
__device__ __forceinline__ double bls_fmod(double x, double p, double inv_p) {
  const double a = fabs(x), b = fabs(p);
  if (a < b) return x;
  double q = trunc(a * inv_p);
  double r = fma(-q, b, a);
  if (r < 0.0) { q -= 1.0; r = fma(-q, b, a); }
  else if (r >= b) { q += 1.0; r = fma(-q, b, a); }
  return copysign(r, x);
}

// numpy's float `x % p` for p > 0: fmod, then the result takes the sign of p
__device__ __forceinline__ double bst_npmod(double x, double p, double inv_p) {
  double r = bls_fmod(x, p, inv_p);
  if (r < 0.0) r += p;
  return r;
}

// accumulator slots of pass 1: (sum ivar, sum y ivar) per mask, then the normal equations
enum BstAcc {
  BA_OUT = 0, BA_IN = 2, BA_ODD = 4, BA_EVEN = 6, BA_PHASE = 8, BA_PHASE_OUT = 10, BA_HALF = 12, BA_NOT_HALF = 14,
  BA_MODEL_IN = 16, BA_MODEL_OUT = 18,
  BA_M00 = 20, BA_M01, BA_M02, BA_M11, BA_M12, BA_M22, BA_R0, BA_R1, BA_R2,
  BA_N
};
enum BstCnt { BC_IN = 0, BC_ODD, BC_EVEN, BC_PHASE, BC_PHASE_OUT, BC_HALF, BC_MODEL_IN, BC_N };

struct BstGeom {
  double P, iP, P2, iP2, Ph, iPh, hp, qp, hd, tt, tt_abs, t0;
};

// the masks of one cadence: bit 0 m_in, 1 m_odd, 2 m_even, 3 m_phase, 4 m_half, 5 m_model
// (trel = t_abs - t_abs[0], x = trel - tt)
__device__ __forceinline__ int bst_masks(double t_abs, const BstGeom& g, double& trel, double& x) {
  trel = t_abs - g.t0;
  x = trel - g.tt;
  const double xa = t_abs - g.tt_abs;
  int m = 0;
  if (fabs(bst_npmod(x + g.hp, g.P, g.iP) - g.hp) < g.hd) m |= 1;
  if (fabs(bst_npmod(x, g.P2, g.iP2) - g.P) < g.hd) m |= 2;
  if (fabs(bst_npmod(x + g.P, g.P2, g.iP2) - g.P) < g.hd) m |= 4;
  if (fabs(bst_npmod(x, g.P, g.iP) - g.hp) < g.hd) m |= 8;
  if (fabs(bst_npmod(x + g.qp, g.Ph, g.iPh) - g.qp) < g.hd) m |= 16;
  if (fabs(bst_npmod(xa + g.hp, g.P, g.iP) - g.hp) < g.hd) m |= 32;
  return m;
}

// what pass 2 needs from the finish step
struct BstShared {
  double y_in, y_out, w0, w1, w2;
  double first;            // first transit id (as a double: rint of it)
  int n_tr, slots_ok, solved;
};

__global__ void __launch_bounds__(BST_THREADS)
bls_stats_kernel(const double* __restrict__ t, const double* __restrict__ y, const double* __restrict__ dy,
                 const int64_t* __restrict__ offsets, const double* __restrict__ period,
                 const double* __restrict__ duration, const double* __restrict__ transit_time,
                 const int64_t* __restrict__ tr_offsets, double* __restrict__ stats, int64_t* __restrict__ tr_first,
                 int32_t* __restrict__ tr_n, int32_t* __restrict__ tr_count, double* __restrict__ tr_ll,
                 uint8_t* __restrict__ in_transit, int32_t* __restrict__ status) {
  __shared__ double s_red[BST_WARPS][BA_N + 2];
  __shared__ int s_redi[BST_WARPS][BC_N];
  __shared__ BstShared sh;
  __shared__ int s_key[2][BST_THREADS];
  __shared__ double s_val[2][BST_THREADS];
  __shared__ double s_rsum[2][BST_THREADS];
  __shared__ int s_rcnt[2][BST_THREADS];

  const int b = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t o = offsets[b], n = offsets[b + 1] - o;
  BstGeom g;
  g.t0 = t[o];
  g.P = period[b];
  g.iP = 1.0 / g.P;
  g.P2 = 2.0 * g.P;
  g.iP2 = 1.0 / g.P2;
  g.Ph = 0.5 * g.P;
  g.iPh = 1.0 / g.Ph;
  g.hp = 0.5 * g.P;
  g.qp = 0.25 * g.P;
  g.hd = 0.5 * duration[b];
  g.tt_abs = transit_time[b];
  g.tt = g.tt_abs - g.t0;
  const double two_pi = 6.283185307179586;       // 2 * np.pi

  // ---- pass 1 ----
  double acc[BA_N];
#pragma unroll
  for (int k = 0; k < BA_N; ++k) acc[k] = 0.0;
  int cnt[BC_N];
#pragma unroll
  for (int k = 0; k < BC_N; ++k) cnt[k] = 0;
  double id_min = INFINITY, id_max = -INFINITY;
  for (int64_t i = tid; i < n; i += BST_THREADS) {
    double trel, x;
    const int m = bst_masks(t[o + i], g, trel, x);
    const double yv = y[o + i];
    const double iv = dy ? 1.0 / (dy[o + i] * dy[o + i]) : 1.0;
    const double yiv = yv * iv;
    const bool in = m & 1, ph = m & 8, hf = m & 16, md = m & 32;
    const int sel[10] = {!in, in, (m >> 1) & 1, (m >> 2) & 1, ph, !ph && !in, hf, !hf, md, !md};
#pragma unroll
    for (int k = 0; k < 10; ++k)
      if (sel[k]) { acc[2 * k] += iv; acc[2 * k + 1] += yiv; }
    cnt[BC_IN] += in;
    cnt[BC_ODD] += (m >> 1) & 1;
    cnt[BC_EVEN] += (m >> 2) & 1;
    cnt[BC_PHASE] += ph;
    cnt[BC_PHASE_OUT] += !ph && !in;
    cnt[BC_HALF] += hf;
    cnt[BC_MODEL_IN] += md;
    double s, c;
    sincos(two_pi * trel / g.P, &s, &c);
    const double siv = s * iv, civ = c * iv;
    acc[BA_M00] += s * siv;
    acc[BA_M01] += s * civ;
    acc[BA_M02] += s * iv;
    acc[BA_M11] += c * civ;
    acc[BA_M12] += c * iv;
    acc[BA_M22] += iv;
    acc[BA_R0] += s * yiv;
    acc[BA_R1] += c * yiv;
    acc[BA_R2] += yiv;
    if (in) {
      const double id = rint(x / g.P);
      id_min = fmin(id_min, id);
      id_max = fmax(id_max, id);
    }
  }
  // fixed-tree block sums: xor butterfly in each warp, then the warps in order
#pragma unroll
  for (int k = 0; k < BA_N; ++k) acc[k] = warp_sum(acc[k]);
#pragma unroll
  for (int k = 0; k < BC_N; ++k) cnt[k] = warp_sum(cnt[k]);
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    id_min = fmin(id_min, __shfl_xor_sync(0xffffffffu, id_min, s));
    id_max = fmax(id_max, __shfl_xor_sync(0xffffffffu, id_max, s));
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < BA_N; ++k) s_red[warp][k] = acc[k];
    s_red[warp][BA_N] = id_min;
    s_red[warp][BA_N + 1] = id_max;
#pragma unroll
    for (int k = 0; k < BC_N; ++k) s_redi[warp][k] = cnt[k];
  }
  __syncthreads();

  // ---- finish ----
  if (tid == 0) {
    double a[BA_N];
    int c[BC_N];
    for (int k = 0; k < BA_N; ++k) a[k] = s_red[0][k];
    for (int k = 0; k < BC_N; ++k) c[k] = s_redi[0][k];
    double lo = s_red[0][BA_N], hi = s_red[0][BA_N + 1];
    for (int w = 1; w < BST_WARPS; ++w) {
      for (int k = 0; k < BA_N; ++k) a[k] += s_red[w][k];
      for (int k = 0; k < BC_N; ++k) c[k] += s_redi[w][k];
      lo = fmin(lo, s_red[w][BA_N]);
      hi = fmax(hi, s_red[w][BA_N + 1]);
    }
    const int nn = (int)n;
    // _compute_depth(m): (mean, variance) or (0, inf) for an empty mask
    auto mean_var = [&](int cm, int k, double& ym, double& vm) {
      if (cm > 0) { vm = 1.0 / a[k]; ym = a[k + 1] * vm; }
      else { ym = 0.0; vm = INFINITY; }
    };
    // _compute_depth(m, y_out, var_out): (y_out - mean, sqrt(var + var_out)) or (0, inf)
    auto depth = [&](int cm, int k, double yo, double vo, double& d, double& e) {
      if (cm > 0 && isfinite(vo)) {
        const double vm = 1.0 / a[k];
        const double ym = a[k + 1] * vm;
        d = yo - ym;
        e = sqrt(vm + vo);
      } else {
        d = 0.0;
        e = INFINITY;
      }
    };
    double* st = stats + (size_t)b * LKB_BLS_STATS_NCOL;
    double y_out, var_out, d, e, ym, vm;
    mean_var(nn - c[BC_IN], BA_OUT, y_out, var_out);
    depth(c[BC_IN], BA_IN, y_out, var_out, d, e);
    st[LKB_BLS_STATS_DEPTH] = d;
    st[LKB_BLS_STATS_DEPTH + 1] = e;
    const double y_in = y_out - d;
    depth(c[BC_ODD], BA_ODD, y_out, var_out, d, e);
    st[LKB_BLS_STATS_DEPTH_ODD] = d;
    st[LKB_BLS_STATS_DEPTH_ODD + 1] = e;
    depth(c[BC_EVEN], BA_EVEN, y_out, var_out, d, e);
    st[LKB_BLS_STATS_DEPTH_EVEN] = d;
    st[LKB_BLS_STATS_DEPTH_EVEN + 1] = e;
    mean_var(nn - c[BC_HALF], BA_NOT_HALF, ym, vm);
    depth(c[BC_HALF], BA_HALF, ym, vm, d, e);
    st[LKB_BLS_STATS_DEPTH_HALF] = d;
    st[LKB_BLS_STATS_DEPTH_HALF + 1] = e;
    mean_var(c[BC_PHASE_OUT], BA_PHASE_OUT, ym, vm);
    depth(c[BC_PHASE], BA_PHASE, ym, vm, d, e);
    st[LKB_BLS_STATS_DEPTH_PHASED] = d;
    st[LKB_BLS_STATS_DEPTH_PHASED + 1] = e;
    // the box model of get_transit_model: in- and out-of-transit weighted means (0 / 0 = NaN when empty)
    st[LKB_BLS_STATS_Y_IN] = a[BA_MODEL_IN + 1] / a[BA_MODEL_IN];
    st[LKB_BLS_STATS_Y_OUT] = a[BA_MODEL_OUT + 1] / a[BA_MODEL_OUT];
    st[LKB_BLS_STATS_N_IN] = (double)c[BC_MODEL_IN];

    // np.linalg.solve of the 3x3 normal equations: LU with partial pivoting, LinAlgError on an exactly zero pivot
    double M[3][3] = {{a[BA_M00], a[BA_M01], a[BA_M02]}, {a[BA_M01], a[BA_M11], a[BA_M12]},
                      {a[BA_M02], a[BA_M12], a[BA_M22]}};
    double r[3] = {a[BA_R0], a[BA_R1], a[BA_R2]};
    int solved = 1;
    for (int k = 0; k < 3 && solved; ++k) {
      int p = k;
      for (int i = k + 1; i < 3; ++i)
        if (fabs(M[i][k]) > fabs(M[p][k])) p = i;
      if (M[p][k] == 0.0) { solved = 0; break; }
      if (p != k) {
        for (int j = 0; j < 3; ++j) { const double tmp = M[k][j]; M[k][j] = M[p][j]; M[p][j] = tmp; }
        const double tmp = r[k]; r[k] = r[p]; r[p] = tmp;
      }
      for (int i = k + 1; i < 3; ++i) {
        const double f = M[i][k] / M[k][k];
        for (int j = k + 1; j < 3; ++j) M[i][j] -= f * M[k][j];
        r[i] -= f * r[k];
      }
    }
    double w[3] = {0.0, 0.0, 0.0};
    if (solved)
      for (int k = 2; k >= 0; --k) {
        double s = r[k];
        for (int j = k + 1; j < 3; ++j) s -= M[k][j] * w[j];
        w[k] = s / M[k][k];
      }
    st[LKB_BLS_STATS_HARMONIC_AMPLITUDE] = solved ? sqrt(w[0] * w[0] + w[1] * w[1]) : __longlong_as_double(0x7ff8000000000000ll);

    // transit slots used: last id - first id + 1 (kept below 2^31 so that a bad candidate cannot overflow it)
    const double n_tr_d = c[BC_IN] > 0 ? fmin(hi - lo + 1.0, 2147483647.0) : 0.0;
    const int n_tr = (int)n_tr_d;
    const int64_t cap = tr_offsets[b + 1] - tr_offsets[b];
    tr_first[b] = c[BC_IN] > 0 ? (int64_t)lo : 0;
    tr_n[b] = n_tr;
    const int ok = (int64_t)n_tr <= cap;
    status[b] = !ok ? LKB_E_ARG : solved ? LKB_OK : LKB_E_SINGULAR;
    sh.y_in = y_in;
    sh.y_out = y_out;
    sh.w0 = w[0];
    sh.w1 = w[1];
    sh.w2 = w[2];
    sh.first = lo;
    sh.n_tr = n_tr;
    sh.slots_ok = ok;
    sh.solved = solved;
  }
  __syncthreads();

  // ---- pass 2 ----
  const double y_in = sh.y_in, y_out = sh.y_out, w0 = sh.w0, w1 = sh.w1, w2 = sh.w2, first = sh.first;
  const bool slots = sh.slots_ok && sh.n_tr > 0;
  int32_t* cnt_b = tr_count + tr_offsets[b];
  double* ll_b = tr_ll + tr_offsets[b];
  for (int64_t j = tid; j < tr_offsets[b + 1] - tr_offsets[b]; j += BST_THREADS) { cnt_b[j] = 0; ll_b[j] = 0.0; }
  __syncthreads();
  double s_in = 0.0, s_out = 0.0, s_sin = 0.0;
  int buf = 0;
  for (int64_t c0 = 0; c0 < n; c0 += BST_THREADS, buf ^= 1) {
    const int64_t i = c0 + tid;
    int key = -1;
    double v = 0.0;
    if (i < n) {
      double trel, x;
      const int m = bst_masks(t[o + i], g, trel, x);
      const double yv = y[o + i];
      const double iv = dy ? 1.0 / (dy[o + i] * dy[o + i]) : 1.0;
      const double a = yv - y_in, bb = yv - y_out;
      if (m & 1) {
        s_in += iv * (a * a);
        v = -0.5 * iv * (a * a - bb * bb);
        key = (int)(rint(x / g.P) - first);
      } else {
        s_out += iv * (bb * bb);
      }
      double s, c;
      sincos(two_pi * trel / g.P, &s, &c);
      const double dm = yv - (s * w0 + c * w1 + w2);
      s_sin += (dm * dm) * iv;
      if (in_transit) in_transit[o + i] = (m & 32) ? 1 : 0;
    }
    if (slots) {
      // runs of equal transit id among the warp's 32 cadences, summed in lane order by the run's last lane
      s_key[buf][tid] = key;
      s_val[buf][tid] = v;
      __syncwarp();
      const int base = warp * 32;
      const int next = lane < 31 ? s_key[buf][tid + 1] : -2;
      int rc = 0;
      double rs = 0.0;
      if (key >= 0 && key != next) {
        int h = lane;
        while (h > 0 && s_key[buf][base + h - 1] == key) --h;
        for (int l = h; l <= lane; ++l) rs += s_val[buf][base + l];
        rc = lane - h + 1;
      }
      s_rsum[buf][tid] = rs;
      s_rcnt[buf][tid] = rc;
      // (the buffers alternate: the next chunk writes the other one, and the chunk after that starts behind
      // the barrier below, which warp 0 passes only once it has added this chunk's runs)
      __syncthreads();
      if (warp == 0) {
        for (int w = 0; w < BST_WARPS; ++w) {
          unsigned tails = __ballot_sync(0xffffffffu, s_rcnt[buf][w * 32 + lane] > 0);
          if (lane == 0)
            while (tails) {
              const int l = w * 32 + __ffs((int)tails) - 1;
              const int k = s_key[buf][l];
              cnt_b[k] += s_rcnt[buf][l];
              ll_b[k] += s_rsum[buf][l];
              tails &= tails - 1;
            }
        }
      }
    }
  }
  __syncthreads();
  s_in = warp_sum(s_in);
  s_out = warp_sum(s_out);
  s_sin = warp_sum(s_sin);
  if (lane == 0) {
    s_red[warp][0] = s_in;
    s_red[warp][1] = s_out;
    s_red[warp][2] = s_sin;
  }
  __syncthreads();
  if (tid == 0) {
    double a = s_red[0][0], bb = s_red[0][1], c = s_red[0][2];
    for (int w = 1; w < BST_WARPS; ++w) { a += s_red[w][0]; bb += s_red[w][1]; c += s_red[w][2]; }
    double full_ll = -0.5 * a;
    full_ll -= 0.5 * bb;
    const double sin_ll = -0.5 * c;
    stats[(size_t)b * LKB_BLS_STATS_NCOL + LKB_BLS_STATS_HARMONIC_DELTA_LOGLIKE] =
        sh.solved ? sin_ll - full_ll : __longlong_as_double(0x7ff8000000000000ll);
  }
}

// Launch on device (or, under the emulator, host) pointers; d_offsets / d_tr_offsets are [B + 1].
inline int bls_stats_launch(const double* t, const double* y, const double* dy, const int64_t* d_offsets, int B,
                            const double* period, const double* duration, const double* transit_time,
                            const int64_t* d_tr_offsets, double* stats, int64_t* tr_first, int32_t* tr_n,
                            int32_t* tr_count, double* tr_ll, uint8_t* in_transit, int32_t* status, cudaStream_t st) {
  LKB_LAUNCH((unsigned)B, BST_THREADS, st, bls_stats_kernel)(t, y, dy, d_offsets, period, duration, transit_time,
                                                             d_tr_offsets, stats, tr_first, tr_n, tr_count, tr_ll,
                                                             in_transit, status);
  LKB_LAUNCH_CHECK();
  return LKB_OK;
}

}  // namespace lkb
