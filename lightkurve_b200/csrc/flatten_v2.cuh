// K4 "v2": LightCurve.flatten (/root/reference/src/lightkurve/lightcurve.py:996-1070) as a small number of streaming
// passes per light curve instead of a 401-tap fp64 FIR over compacted copies (flatten.cu's first kernel: 0.017 of the
// HBM roofline, 7.4x wasted DRAM traffic).
//
// One CTA per light curve.  What changed:
//   * the kept-cadence set is a BITMASK in shared memory (n / 8 bytes) with a per-word prefix count: "the k-th kept
//     cadence" (select) and "how many kept cadences before i" (rank) are a few shared-memory operations, so there are
//     no compacted copies of time / flux (no cidx, fc, tc, xs, ys arrays), and segments / survivors are found by bit
//     scans instead of compaction + binary searches in global memory;
//   * Savitzky-Golay by SLIDING MOMENTS (SURVEY.md H7): the centre tap of a degree-p least-squares fit over a
//     symmetric window is an even polynomial in the offset j,  c_j = A0 + A2 j^2 (+ A4 j^4),  so
//     y_k = sum_s A_s sum_j j^s x_{k+j}  and the windowed power sums are differences of prefix sums of q^s x_q over a
//     tile (q measured from the tile centre) - O(1) per output instead of O(window).  Their rounding grows with the
//     tile and is amplified by the re-centring as the window shrinks, so short windows (flatten_plan.h: where the
//     predicted error exceeds F2_MOMENT_TOL) take the direct dot product of the centre taps with the staged inputs;
//   * the segment edges are the degree-p polynomial fitted to the first / last `window` samples (scipy
//     _fit_edges_polyfit) evaluated from its p + 1 moments (one block reduction per edge) instead of a
//     [window x window/2] table product;
//   * the trend is interpolated to all cadences only ONCE, after the last iteration (the reference overwrites the
//     intermediate ones, lightcurve.py:1053-1058), fused with flux / trend and flux_err / trend.
// Global memory per iteration: t once (gap statistics), f once + trend-at-kept written (filter), f + trend read
// (residual clip); order statistics by the radix select of select.cuh on functors that read through the bitmask.
// Supported: polyorder <= 5, a tile of >= 128 outputs, n <= F2_MAXN per light curve (flatten_plan.h), <= 1023 gap
// segments; anything else (and a light curve that overflows the segment list, status 2) runs flatten.cu's first kernel.
#pragma once
#include "common.cuh"
#include "select.cuh"
#include "flatten_plan.h"

namespace lkb {

constexpr int F2_THREADS = 512;
constexpr int F2_MAXWORDS = F2_MAXN / 32;
constexpr int F2_MAXSEG = 1024;
constexpr int F2_MAXQ = 6;                      // polyorder + 1

struct F2Coef {
  double A[3];                                  // centre taps c_j = A[0] + A[1] j^2 + A[2] j^4
  double Ginv[F2_MAXQ * F2_MAXQ];               // inverse normal matrix of the degree-p fit on u = (j - c) / c
  int q;                                        // polyorder + 1
};

struct F2Smem {
  FastSelSmem fs;                               // sampling select (median in two passes)
  unsigned keep[F2_MAXWORDS];                   // bit i: cadence i is used for the fit
  int wpre[F2_MAXWORDS + 1];                    // kept cadences before word w
  int cuts[F2_MAXSEG + 1];                      // segment starts (positions in the kept sequence), cuts[nseg] = m
  int ucuts[F2_MAXSEG];                         // the same, unordered (as found)
  SelSmem sel;
  double red[F2_MAXQ][17];
  double beta[F2_MAXQ];
  int scan_tmp[17];
  int misc[8];
  FastBracket br_dt;                            // the dt median's bracket, carried from one iteration to the next
};

// exclusive prefix of popc(keep[w]) over nw words -> wpre[0 .. nw]; returns the total.  All threads call.
__device__ inline int f2_prefix(F2Smem& sm, int nw) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  constexpr int PER = F2_MAXWORDS / F2_THREADS;           // 8 consecutive words per thread
  int loc[PER], tot = 0;
#pragma unroll
  for (int e = 0; e < PER; ++e) {
    const int w = t * PER + e;
    loc[e] = (w < nw) ? __popc(sm.keep[w]) : 0;
    tot += loc[e];
  }
  int incl = tot;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int u = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += u;
  }
  if (lane == 31) sm.scan_tmp[warp] = incl;
  __syncthreads();
  if (t == 0) {
    int run = 0;
    for (int w = 0; w < F2_THREADS / 32; ++w) { const int v = sm.scan_tmp[w]; sm.scan_tmp[w] = run; run += v; }
    sm.scan_tmp[16] = run;
  }
  __syncthreads();
  int run = sm.scan_tmp[warp] + incl - tot;
#pragma unroll
  for (int e = 0; e < PER; ++e) {
    const int w = t * PER + e;
    if (w <= nw) sm.wpre[w] = run;
    run += loc[e];
  }
  const int total = sm.scan_tmp[16];
  __syncthreads();
  return total;
}

__device__ __forceinline__ bool f2_kept(const F2Smem& sm, int i) { return (sm.keep[i >> 5] >> (i & 31)) & 1u; }
__device__ __forceinline__ int f2_rank(const F2Smem& sm, int i) {          // kept cadences with index < i
  return sm.wpre[i >> 5] + __popc(sm.keep[i >> 5] & ((1u << (i & 31)) - 1u));
}
__device__ __forceinline__ int f2_select(const F2Smem& sm, int nw, int k) {   // index of the k-th kept cadence (0-based)
  int lo = 0, hi = nw;                          // largest word with wpre[word] <= k
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (sm.wpre[mid] <= k) lo = mid; else hi = mid;
  }
  return lo * 32 + (int)__fns(sm.keep[lo], 0, k - sm.wpre[lo] + 1);
}
// f2_select for up to four ranks at once: threads 0..3 search, everyone reads the answers.  (Every thread running its
// own binary search over wpre was 25 % of the kernel's instructions - per-line profile of r02_flatten2_c.ncu-rep.)
// All threads call; two barriers.
__device__ inline void f2_select4(F2Smem& sm, int nw, int ka, int kb, int kc, int kd, int* out) {
  __syncthreads();
  if (threadIdx.x < 4) {
    const int k = threadIdx.x == 0 ? ka : threadIdx.x == 1 ? kb : threadIdx.x == 2 ? kc : kd;
    sm.misc[4 + threadIdx.x] = k >= 0 ? f2_select(sm, nw, k) : -1;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 4; ++j) out[j] = sm.misc[4 + j];
}
__device__ __forceinline__ int f2_prev(const F2Smem& sm, int i) {            // last kept cadence before i, or -1
  int w = i >> 5;
  unsigned bits = sm.keep[w] & ((1u << (i & 31)) - 1u);
  while (bits == 0u) {
    if (--w < 0) return -1;
    bits = sm.keep[w];
  }
  return w * 32 + 31 - __clz(bits);
}
__device__ __forceinline__ int f2_next(const F2Smem& sm, int nw, int i) {    // first kept cadence after i, or -1
  int w = i >> 5;
  unsigned bits = ((i & 31) == 31) ? 0u : (sm.keep[w] & ~((2u << (i & 31)) - 1u));
  while (bits == 0u) {
    if (++w >= nw) return -1;
    bits = sm.keep[w];
  }
  return w * 32 + __ffs(bits) - 1;
}
// segment of kept position k: cuts[s] <= k < cuts[s + 1]
__device__ __forceinline__ int f2_segment(const F2Smem& sm, int nseg, int k) {
  int lo = 0, hi = nseg;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (sm.cuts[mid] <= k) lo = mid; else hi = mid;
  }
  return lo;
}

// block sums of up to F2_MAXQ doubles per thread -> sm.beta[0 .. nq) (valid in all threads after the call)
__device__ inline void f2_block_sums(F2Smem& sm, const double* v, int nq) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  for (int s = 0; s < nq; ++s) {
    const double x = warp_sum(v[s]);
    if (lane == 0) sm.red[s][warp] = x;
  }
  __syncthreads();
  if (threadIdx.x < nq) {
    double x = 0.0;
    for (int w = 0; w < F2_THREADS / 32; ++w) x += sm.red[threadIdx.x][w];
    sm.beta[threadIdx.x] = x;
  }
  __syncthreads();
}

// NM = number of prefix-sum arrays (power sums q^0 .. q^(NM-1)): 1 for polyorder <= 1, 3 for <= 3, 5 for <= 5;
// DIRECT: the interior from the centre taps instead of the moments (flatten_plan.h), NM = 3 and 5 only
template <int NM, bool DIRECT = false>
__global__ void __launch_bounds__(F2_THREADS, 2)
flatten2_kernel(const double* __restrict__ time, const double* __restrict__ flux, const double* __restrict__ flux_err,
                const uint8_t* __restrict__ exclude, const int64_t* __restrict__ offsets, double* __restrict__ tro_ws,
                int window_length, double break_tolerance, int niters, double sigma, F2Coef cf, int tile_out,
                double* __restrict__ flat, double* __restrict__ flat_err, double* __restrict__ trend,
                int* __restrict__ status) {
  static_assert(!DIRECT || NM >= 3, "direct taps replace the moments of polyorder >= 2");
  LKB_DYN_SMEM(unsigned char, f2_dyn);
  F2Smem& sm = *reinterpret_cast<F2Smem*>(f2_dyn);
  double* P = reinterpret_cast<double*>(f2_dyn + ((sizeof(F2Smem) + 15) & ~(size_t)15));     // NM arrays of plen doubles
  if (threadIdx.x == 0) sm.fs.cand = P;        // the select's candidate buffer aliases the (then idle) prefix arrays
  __syncthreads();
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t o = offsets[b];
  const int n = (int)(offsets[b + 1] - o);
  if (n <= 0) return;
  const double* tt = time + o;
  const double* f = flux + o;
  double* tro = tro_ws + o;
  const int w = window_length, half = w / 2, nw = (n + 31) >> 5;
  const int plen = tile_out + 2 * half + 1;
  const double qnan = __longlong_as_double(0x7ff8000000000000ll);
  const double sc = half > 0 ? (double)half : 1.0;

  // ---- initial mask (:996-1010): finite, not excluded, within sigma * nanstd of the nanmedian ----
  // np.nanstd(flux) rides along in the median's partition pass: sums of d = flux - lo and d^2 (lo = the bracket's
  // lower value, within a few percent of a standard deviation of the mean) over the non-NaN values
  double is1 = 0.0, is2 = 0.0;
  int isc = 0;
  auto stats0 = [&](int64_t i, double, double lo, bool valid) {
    if (valid) {
      const double raw = f[i];                    // (infinities stay in, as in numpy: the result is then NaN)
      if (raw == raw) { const double d = raw - lo; is1 += d; is2 = fma(d, d, is2); isc++; }
    }
  };
  bool seen0 = false;
  const double med0 = block_nanmedian_fast([&](int64_t i) { const double v = f[i]; return isfinite(v) ? v : qnan; }, n,
                                           sm.sel, sm.fs, -1, stats0, &seen0);
  double std0;
  if (seen0) {
    const double t1 = block_sum(is1, sm.sel.red), t2 = block_sum(is2, sm.sel.red);
    const long long tc = block_sum_ll((long long)isc, sm.sel.redll);
    if (tc == 0) std0 = qnan;
    else {
      const double md = t1 / (double)tc, var = t2 / (double)tc - md * md;
      std0 = (var == var) ? sqrt(var > 0.0 ? var : 0.0) : qnan;
    }
  } else {
    std0 = block_nanstd([&](int64_t i) { return f[i]; }, n, sm.sel);
  }
  {
    const double thr = std0 * sigma;
    for (int w0 = warp; w0 < nw; w0 += F2_THREADS / 32) {
      const int i = w0 * 32 + lane;
      bool m = false;
      if (i < n) {
        const double v = f[i];
        double a = fabs(v - med0);
        if (a != a) a = 0.0;                      // nan_to_num
        m = (exclude ? (exclude[o + i] == 0) : true) && isfinite(v) && (a <= thr);
      }
      const unsigned bal = __ballot_sync(0xffffffffu, m);
      if (lane == 0) sm.keep[w0] = bal;
    }
    for (int w0 = nw + t; w0 < F2_MAXWORDS; w0 += F2_THREADS) sm.keep[w0] = 0u;
  }
  __syncthreads();

  bool ok = true;
  int m = 0;
  if (t == 0) sm.br_dt.valid = false;         // (the first f2_prefix's barriers publish it)
  for (int it = 0; it < niters && ok; ++it) {
    m = f2_prefix(sm, nw);
    if (m < 2) { ok = false; break; }
    // ---- gap segmentation (:1022-1027): cut where dt > break_tolerance * nanmedian(dt) over the kept cadences ----
    // The median's partition pass sees every dt once with a lower bound `lo` of the median: cadences with
    // dt > break_tolerance * lo (a superset of the cuts - a handful) are noted on the way, so that no second pass over
    // the time stamps is needed; they are filtered with the exact threshold afterwards.
    if (t == 0) { sm.misc[0] = 0; sm.misc[1] = 0; }          // misc[0] = cuts found, misc[1] = cut candidates noted
    __syncthreads();
    const bool bt_ok = break_tolerance >= 0.0;
    auto note = [&](int64_t i, double v, double lo, bool valid) {
      const bool c = valid && bt_ok && v > break_tolerance * lo;      // (NaN dt / NaN lo: false)
      const unsigned bal = __ballot_sync(0xffffffffu, c);
      if (bal) {
        int base = 0;
        if (lane == 0) base = atomicAdd(&sm.misc[1], __popc(bal));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (c) {
          const int pos = base + __popc(bal & ((1u << lane) - 1u));
          if (pos < F2_MAXSEG) sm.cuts[pos] = (int)i;
        }
      }
    };
#ifdef LKB_FS_TEST_BAD_BRACKET            // test hook (tests/test_flatten_emulated.py): a stale bracket that misses the median
    if (t == 0 && it > 0) { sm.br_dt.lo = -2.0; sm.br_dt.hi = -1.0; sm.br_dt.valid = true; }
    __syncthreads();
#endif
    bool observed = false;
    const double med_dt = block_nanmedian_fast([&](int64_t i) {
      if (!f2_kept(sm, (int)i)) return qnan;
      const int pv = f2_prev(sm, (int)i);
      return pv < 0 ? qnan : tt[i] - tt[pv];
    }, n, sm.sel, sm.fs, (long long)m - 1, note, &observed, &sm.br_dt, [&]() { if (t == 0) sm.misc[1] = 0; });
    const double thr_dt = break_tolerance * med_dt;
    __syncthreads();
    const int ncand = sm.misc[1];
    if (observed && bt_ok && ncand <= F2_MAXSEG) {
      // exact filter of the noted candidates (unordered append of the kept-sequence rank, as the full pass does)
      for (int e0 = 0; e0 < ncand; e0 += F2_THREADS) {
        const int e = e0 + t;
        bool cut = false;
        int i = 0;
        if (e < ncand) {
          i = sm.cuts[e];
          const int pv = f2_prev(sm, i);
          cut = pv >= 0 && (tt[i] - tt[pv]) > thr_dt;
        }
        const unsigned bal = __ballot_sync(0xffffffffu, cut);
        if (bal) {
          int base = 0;
          if (lane == 0) base = atomicAdd(&sm.misc[0], __popc(bal));
          base = __shfl_sync(0xffffffffu, base, 0);
          if (cut) {
            const int pos = base + __popc(bal & ((1u << lane) - 1u));
            if (pos < F2_MAXSEG - 1) sm.ucuts[pos] = f2_rank(sm, i);
          }
        }
      }
    } else {
    // (the median came from a fallback path, or too many candidates: one pass over the time stamps)
    // cuts are rare: unordered append (one atomic per warp that found any), then a rank sort of the short list
    for (int i0 = 0; i0 < n; i0 += 4 * F2_THREADS) {          // 4 independent (t[i], t[prev]) load pairs in flight
      double dd[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * F2_THREADS + t;
        dd[u] = qnan;                                         // no predecessor: never a cut
        if (i < n && f2_kept(sm, i)) {
          const int pv = f2_prev(sm, i);
          if (pv >= 0) dd[u] = tt[i] - tt[pv];
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * F2_THREADS + t;
        const bool cut = dd[u] > thr_dt;                      // (NaN threshold: no cuts, as in numpy)
        const unsigned bal = __ballot_sync(0xffffffffu, cut);
        if (bal) {
          int base = 0;
          if (lane == 0) base = atomicAdd(&sm.misc[0], __popc(bal));
          base = __shfl_sync(0xffffffffu, base, 0);
          if (cut) {
            const int pos = base + __popc(bal & ((1u << lane) - 1u));
            if (pos < F2_MAXSEG - 1) sm.ucuts[pos] = f2_rank(sm, i);
          }
        }
      }
    }
    }
    __syncthreads();
    const int ncut = sm.misc[0];
    if (ncut > F2_MAXSEG - 2) {                              // too many segments for the shared-memory list
      if (t == 0) status[b] = 2;
      return;
    }
    for (int e = t; e < ncut; e += F2_THREADS) {             // distinct values: rank = number of smaller entries
      const int v = sm.ucuts[e];
      int r = 0;
      for (int q = 0; q < ncut; ++q) r += (sm.ucuts[q] < v) ? 1 : 0;
      sm.cuts[1 + r] = v;
    }
    if (t == 0) sm.cuts[0] = 0;
    const int nseg = ncut + 1;
    if (t == 0) sm.cuts[nseg] = m;
    __syncthreads();

    // residual statistics of this iteration, gathered where the trend values are produced (no extra passes):
    // sum r, sum r^2, count over the kept cadences (np.nanstd semantics: NaN residuals are left out)
    double rs1 = 0.0, rs2 = 0.0;
    int rsc = 0;
    auto residual = [&](int i, double y) {
      const double r = f[i] - y;
      if (r == r) { rs1 += r; rs2 = fma(r, r, rs2); rsc++; }
    };
    // ---- Savitzky-Golay interior by tiles of `tile_out` kept positions ----
    // direct taps: c_j = A0 + A1 j^2 + A2 j^4 for j = 0 .. half in the second array (idle without moments; written
    // every iteration because the select's candidate buffer aliases it; the first f2_select4 publishes them)
    double* taps = P + plen;
    if (DIRECT)
      for (int j = t; j <= half; j += F2_THREADS) {
        const double j2 = (double)j * (double)j;
        taps[j] = fma(fma(cf.A[2], j2, cf.A[1]), j2, cf.A[0]);
      }
    for (int k0 = 0; k0 < m; k0 += tile_out) {
      const int kin0 = max(0, k0 - half), kin1 = min(m, k0 + tile_out + half);      // inputs [kin0, kin1)
      const int kout1 = min(m, k0 + tile_out);
      const int nin = kin1 - kin0;
      int sel4[4];
      f2_select4(sm, nw, kin0, kin1 - 1, k0, kout1 - 1, sel4);
      const int i_lo = sel4[0], i_hi = sel4[1] + 1;
      const double qc = 0.5 * (double)nin;
      // stage x_q in P[0][q + 1]
      for (int i0 = i_lo; i0 < i_hi; i0 += 4 * F2_THREADS) {       // 4 loads in flight per thread
        double xv[4];
        bool kp[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int i = i0 + u * F2_THREADS + t;
          kp[u] = i < i_hi && f2_kept(sm, i);
          xv[u] = kp[u] ? f[i] : 0.0;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int i = i0 + u * F2_THREADS + t;
          if (kp[u]) P[f2_rank(sm, i) - kin0 + 1] = xv[u];
        }
      }
      __syncthreads();
      // prefix sums P[s][q + 1] = sum_{q' <= q} (q' - qc)^s x_q'   (each thread owns PER consecutive q)
      if (!DIRECT) {
        const int PER = (nin + F2_THREADS - 1) / F2_THREADS;
        const int q0 = t * PER, q1 = min(nin, q0 + PER);
        double run[NM];
#pragma unroll
        for (int s = 0; s < NM; ++s) run[s] = 0.0;
        for (int q = q0; q < q1; ++q) {
          const double x = P[q + 1], d = (double)q - qc;
          double pw = x;
#pragma unroll
          for (int s = 0; s < NM; ++s) { run[s] += pw; pw *= d; }
        }
        // exclusive block scan of the thread totals
        double excl[NM];
#pragma unroll
        for (int s = 0; s < NM; ++s) {
          double incl = run[s];
#pragma unroll
          for (int oo = 1; oo < 32; oo <<= 1) {
            const double u = __shfl_up_sync(0xffffffffu, incl, oo);
            if (lane >= oo) incl += u;
          }
          if (lane == 31) sm.red[s][warp] = incl;
          excl[s] = incl - run[s];
        }
        __syncthreads();
        if (t < NM) {
          double r = 0.0;
          for (int ww = 0; ww < F2_THREADS / 32; ++ww) { const double v = sm.red[t][ww]; sm.red[t][ww] = r; r += v; }
        }
        __syncthreads();
        double acc[NM];
#pragma unroll
        for (int s = 0; s < NM; ++s) acc[s] = excl[s] + sm.red[s][warp];
        // second sweep: write the inclusive prefixes (x is still in P[0] for this thread's own range)
        double xs_loc[8];
        for (int q = q0; q < q1; ++q) xs_loc[q - q0] = P[q + 1];
        __syncthreads();
        for (int q = q0; q < q1; ++q) {
          const double x = xs_loc[q - q0], d = (double)q - qc;
          double pw = x;
#pragma unroll
          for (int s = 0; s < NM; ++s) { acc[s] += pw; P[s * plen + q + 1] = acc[s]; pw *= d; }
        }
        if (t == 0) {
#pragma unroll
          for (int s = 0; s < NM; ++s) P[s * plen] = 0.0;
        }
      }
      __syncthreads();
      // outputs of the tile that are interior points of a filtered segment
      const int o_lo = sel4[2], o_hi = sel4[3] + 1;
      int l = 0, h = -1;                                   // this thread's last segment (positions only grow)
      for (int i = o_lo + t; i < o_hi; i += F2_THREADS) {
        if (!f2_kept(sm, i)) continue;
        const int k = f2_rank(sm, i);
        if (k >= h) { const int s = f2_segment(sm, nseg, k); l = sm.cuts[s]; h = sm.cuts[s + 1]; }
        const int len = h - l;
        if ((w > len) || ((double)len < break_tolerance)) continue;          // median fallback (below)
        if (k - l < half || h - k <= half) continue;                           // edge (below)
        if (DIRECT) {
          const double* xk = P + (k - kin0 + 1);
          double y = taps[0] * xk[0];
          for (int j = 1; j <= half; ++j) y = fma(taps[j], xk[-j] + xk[j], y);
          tro[i] = y;
          residual(i, y);
          continue;
        }
        const int a = k - half - kin0, e = k + half - kin0 + 1;                // window [a, e) in tile coordinates
        const double kc = (double)(k - kin0) - qc;
        const double S0 = P[e] - P[a];
        double y = cf.A[0] * S0;
        if (NM >= 3) {
          const double S1 = P[plen + e] - P[plen + a], S2 = P[2 * plen + e] - P[2 * plen + a];
          const double S2c = S2 - 2.0 * kc * S1 + kc * kc * S0;
          y += cf.A[1] * S2c;
          if (NM >= 5) {
            const double S3 = P[3 * plen + e] - P[3 * plen + a], S4 = P[4 * plen + e] - P[4 * plen + a];
            const double k2 = kc * kc;
            const double S4c = S4 - 4.0 * kc * S3 + 6.0 * k2 * S2 - 4.0 * k2 * kc * S1 + k2 * k2 * S0;
            y += cf.A[2] * S4c;
          }
        }
        tro[i] = y;
        residual(i, y);
      }
    }
    __syncthreads();
    // ---- per segment: median fallback, or the polynomial edges ----
    for (int s = 0; s < nseg; ++s) {
      const int l = sm.cuts[s], h = sm.cuts[s + 1], len = h - l;
      if (len <= 0) continue;
      const bool fallback = (w > len) || ((double)len < break_tolerance);
      if (fallback) {
        int sel4[4];
        f2_select4(sm, nw, l, h - 1, -1, -1, sel4);
        const int i_lo = sel4[0], i_hi = sel4[1] + 1;
        const double md = block_nanmedian([&](int64_t j) { return f2_kept(sm, i_lo + (int)j) ? f[i_lo + j] : qnan; },
                                          i_hi - i_lo, sm.sel);
        for (int i = i_lo + t; i < i_hi; i += F2_THREADS)
          if (f2_kept(sm, i)) { tro[i] = md; residual(i, md); }
        continue;
      }
      if (half == 0) continue;
      for (int side = 0; side < 2; ++side) {
        const int kw0 = side == 0 ? l : h - w;                    // first kept position of the w-sample fit window
        const int kq0 = side == 0 ? l : h - half;                 // outputs: the first / last `half` positions of the window
        int sel4[4];
        f2_select4(sm, nw, kw0, kw0 + w - 1, kq0, kq0 + half - 1, sel4);
        const int i_lo = sel4[0], i_hi = sel4[1] + 1;
        double mom[F2_MAXQ];
#pragma unroll
        for (int r = 0; r < F2_MAXQ; ++r) mom[r] = 0.0;
        for (int i = i_lo + t; i < i_hi; i += F2_THREADS) {
          if (!f2_kept(sm, i)) continue;
          const double u = ((double)(f2_rank(sm, i) - kw0) - (double)half) / sc, x = f[i];
          double pw = x;
#pragma unroll
          for (int r = 0; r < F2_MAXQ; ++r) {
            if (r < cf.q) { mom[r] += pw; pw *= u; }
          }
        }
        f2_block_sums(sm, mom, cf.q);                              // sm.beta = moments
        // polynomial coefficients = Ginv * moments: q threads, one row each, then everyone reads them (all 512
        // threads indexing the parameter struct dynamically was 2.8 % of the kernel's instructions)
        __syncthreads();
        if (t < cf.q) {
          double acc = 0.0;
          for (int c2 = 0; c2 < cf.q; ++c2) acc += cf.Ginv[t * cf.q + c2] * sm.beta[c2];
          sm.red[0][t] = acc;
        }
        __syncthreads();
        double bet[F2_MAXQ];
#pragma unroll
        for (int r = 0; r < F2_MAXQ; ++r) bet[r] = (r < cf.q) ? sm.red[0][r] : 0.0;
        // outputs: the first (side 0) / last (side 1) `half` positions of the window
        const int j_lo = sel4[2], j_hi = sel4[3] + 1;
        for (int i = j_lo + t; i < j_hi; i += F2_THREADS) {
          if (!f2_kept(sm, i)) continue;
          const double u = ((double)(f2_rank(sm, i) - kw0) - (double)half) / sc;
          double y = 0.0;
#pragma unroll
          for (int r = F2_MAXQ - 1; r >= 0; --r)
            if (r < cf.q) y = y * u + bet[r];
          tro[i] = y;
          residual(i, y);
        }
        __syncthreads();
      }
    }
    __syncthreads();
    // ---- residual clip (:1049-1052, :1060-1063) ----
    // np.nanstd(flux - trend) from the running sums: var = <r^2> - <r>^2 (the residuals are centred on zero by
    // construction - |<r>| << std - so the one-pass form loses nothing; numpy's two-pass value differs by ~1e-16)
    double rstd;
    {
      const double t1 = block_sum(rs1, sm.sel.red), t2 = block_sum(rs2, sm.sel.red);
      const long long tc = block_sum_ll((long long)rsc, sm.sel.redll);
      if (tc == 0) rstd = qnan;
      else {
        const double mean = t1 / (double)tc, var = t2 / (double)tc - mean * mean;
        rstd = sqrt(var > 0.0 ? var : 0.0);
      }
    }
    const double rthr = rstd * sigma + 1e-14;
    for (int wb = warp; wb < nw; wb += 4 * (F2_THREADS / 32)) {   // 4 words per warp and trip: 8 loads in flight per lane
      double fv[4], tv4[4];
      bool kp[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int w0 = wb + u * (F2_THREADS / 32), i = w0 * 32 + lane;
        kp[u] = w0 < nw && i < n && f2_kept(sm, i);
        fv[u] = kp[u] ? f[i] : 0.0;
        tv4[u] = kp[u] ? tro[i] : 0.0;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int w0 = wb + u * (F2_THREADS / 32);
        bool keepit = false;
        if (kp[u]) {
          double a = fabs(fv[u] - tv4[u]);
          if (a != a) a = 0.0;
          keepit = a < rthr;
        }
        const unsigned bal = __ballot_sync(0xffffffffu, keepit);
        __syncwarp();
        if (lane == 0 && w0 < nw) sm.keep[w0] = bal;
      }
    }
    __syncthreads();
  }

  // ---- interp1d(kind="linear", fill_value="extrapolate") of the last trend onto every cadence (:1053-1058), fused
  // with flux / trend and flux_err / trend (:1065-1070) ----
  int ms = 0;
  if (ok) {
    ms = f2_prefix(sm, nw);
    if (ms < 2) ok = false;
  }
  double* tr = trend + o;
  if (!ok) {
    for (int g = t; g < n; g += F2_THREADS) {
      tr[g] = qnan;
      flat[o + g] = f[g] / qnan;
      if (flat_err) flat_err[o + g] = qnan;
    }
    if (t == 0) status[b] = 1;
    return;
  }
  int selE[4];
  f2_select4(sm, nw, 0, 1, ms - 1, ms - 2, selE);
  const int s_first = selE[0], s_second = selE[1], s_last = selE[2], s_prelast = selE[3];
  for (int g = t; g < n; g += F2_THREADS) {
    const int j = f2_rank(sm, g);                          // survivors before g = np.searchsorted(xs, t[g], "left")
    int il, ih;
    if (j == 0) { il = s_first; ih = s_second; }
    else if (j >= ms) { il = s_prelast; ih = s_last; }
    else {
      ih = f2_kept(sm, g) ? g : f2_next(sm, nw, g);
      il = f2_prev(sm, g);
    }
    const double xl = tt[il], xh = tt[ih], yl = tro[il], yh = tro[ih];
    const double slope = (yh - yl) / (xh - xl);
    const double tv = slope * (tt[g] - xl) + yl;
    tr[g] = tv;
    flat[o + g] = f[g] / tv;
    if (flat_err) flat_err[o + g] = (flux_err ? flux_err[o + g] : qnan) / tv;
  }
  if (t == 0) status[b] = 0;
}

}  // namespace lkb
