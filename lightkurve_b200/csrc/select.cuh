// K6: block-cooperative exact order statistics (np.nanmedian / np.median / np.nanstd semantics).
// Replaces np.nanmedian/np.nanstd at /root/reference/src/lightkurve/lightcurve.py:1003-1005,1035,1050,
// np.median at correctors/regressioncorrector.py:279 and the median/std inside astropy sigma_clip (:269).
// MSB-first 8-bit radix select over order-preserving uint64 keys of fp64 values; 8 passes,
// shared-memory integer histogram; exact (no approximation, no sorting of the payload).
#pragma once
#include "common.cuh"

namespace lkb {

struct SelSmem {
  int hist[256];
  double red[33];
  long long redll[33];
  unsigned long long prefix;
  long long k;
  int digit;
};

__device__ __forceinline__ unsigned long long f64_key(double v) {
  unsigned long long b = (unsigned long long)__double_as_longlong(v);
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double f64_unkey(unsigned long long k) {
  unsigned long long b = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
  return __longlong_as_double((long long)b);
}

// k-th smallest (0-based) among the non-NaN values get(0..n-1).  All threads must call.
// Precondition: 0 <= k < (number of non-NaN values).  Result valid in all threads.
template <class Get>
__device__ unsigned long long block_select_key(Get get, int64_t n, long long k, SelSmem& sm) {
  unsigned long long prefix = 0, mask = 0;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) sm.hist[i] = 0;
    __syncthreads();
    for (int64_t i0 = 0; i0 < n; i0 += blockDim.x) {         // warp-uniform trip count
      const int64_t i = i0 + threadIdx.x;
      int digit = -1;
      if (i < n) {
        const double v = get(i);
        if (v == v) {
          const unsigned long long key = f64_key(v);
          if ((key & mask) == prefix) digit = (int)((key >> shift) & 255ull);
        }
      }
      // warp-aggregated update: one atomic per distinct digit per warp (a regular cadence makes every
      // dt identical - a naive per-lane atomicAdd would serialise 32-way on one counter)
      const unsigned peers = __match_any_sync(0xffffffffu, digit);
      if (digit >= 0 && (threadIdx.x & 31) == (__ffs(peers) - 1)) atomicAdd(&sm.hist[digit], __popc(peers));
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      // warp 0: find the digit whose cumulative count first exceeds k
      const int lane = threadIdx.x;
      int loc[8], tot = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) { loc[j] = sm.hist[lane * 8 + j]; tot += loc[j]; }
      int incl = tot;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        int u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
      }
      const long long excl = (long long)incl - tot;
      if (k >= excl && k < (long long)incl) {
        long long kk = k - excl;
        int d = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (kk >= loc[j]) { kk -= loc[j]; d = j + 1; } else break;
        }
        sm.digit = lane * 8 + d;
        sm.k = kk;
      }
    }
    __syncthreads();
    prefix |= ((unsigned long long)sm.digit) << shift;
    mask |= 255ull << shift;
    k = sm.k;
    __syncthreads();
  }
  return prefix;
}

// np.nanmedian over get(0..n-1) (NaN entries ignored; all-NaN -> NaN).  `count_out` (optional)
// receives the number of non-NaN entries.
template <class Get>
__device__ double block_nanmedian(Get get, int64_t n, SelSmem& sm, long long* count_out = nullptr) {
  long long cnt = 0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const double v = get(i);
    cnt += (v == v) ? 1 : 0;
  }
  const long long m = block_sum_ll(cnt, sm.redll);
  if (count_out) *count_out = m;
  if (m == 0) return __longlong_as_double(0x7ff8000000000000ll);
  const long long klo = (m - 1) / 2, khi = m / 2;
  const unsigned long long key_lo = block_select_key(get, n, klo, sm);
  const double vlo = f64_unkey(key_lo);
  if (khi == klo) return vlo;
  // the next order statistic: equal to vlo if enough duplicates, else the smallest value above it
  long long le = 0;
  double mn = __longlong_as_double(0x7ff0000000000000ll);   // +inf
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const double v = get(i);
    if (v == v) {
      const unsigned long long key = f64_key(v);
      if (key <= key_lo) le++;
      else mn = fmin(mn, v);
    }
  }
  const long long le_tot = block_sum_ll(le, sm.redll);
  // block min
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sm.red[threadIdx.x >> 5] = mn;
  __syncthreads();
  if (threadIdx.x == 0) {
    double x = sm.red[0];
    for (int w = 1; w < (int)((blockDim.x + 31) >> 5); ++w) x = fmin(x, sm.red[w]);
    sm.red[32] = x;
  }
  __syncthreads();
  const double vnext = sm.red[32];
  __syncthreads();
  const double vhi = (le_tot >= khi + 1) ? vlo : vnext;
  return (vlo + vhi) / 2.0;
}

// ---- exact median in TWO passes over the data (Floyd-Rivest style) -----------------------------------------------
// The radix select above reads the data once per key byte (8 passes + count + tie pass).  Here a strided sample of
// FS_SAMPLE values brackets the wanted order statistics [lo, hi] (sample ranks +- FS_GAP around the target), ONE
// pass over the data counts the values below lo / equal lo / equal hi and collects those strictly between into a
// shared-memory buffer, and the order statistics are selected inside that buffer (radix select over shared memory).
// Exact; if the bracket misses (probability ~1e-3 per call for random data) or more than FS_CAP values fall between
// (heavily skewed duplicates), the caller's answer comes from block_nanmedian above - same result, just slower.
// Sizing: the bracket spans 2 FS_GAP of the FS_SAMPLE sample ranks, i.e. a fraction 2 FS_GAP / FS_SAMPLE = 1/16 of the data
// (65 000 cadences: 4060 +- 350 candidates, FS_CAP is 4.5 sigma above); the median's rank in the sample has standard
// deviation sqrt(FS_SAMPLE) / 2 = 22.6, so the bracket misses it with probability 0.5 %.  (Round 2's first version used
// 1024 / 56 / 6144: 7100 +- 630 expected candidates for 65 000 cadences - it overflowed the buffer and fell back to the
// 8-pass select 93 % of the time; found in a per-line ncu profile.)
constexpr int FS_SAMPLE = 2048, FS_GAP = 64, FS_CAP = 5632;
struct FastSelSmem {
  double* cand;                 // FS_CAP + FS_SAMPLE doubles of shared memory provided by the caller (may alias idle
                                // scratch): candidates first, then the sample
  int n_cand, c_lt, c_eqlo, c_eqhi, ok;
};

// value of rank r (0-based) among {lt block | eq-lo block | cand (sorted logically) | eq-hi block}; valid iff inside
template <class GetC>
__device__ inline double fs_rank_value(long long r, long long c_lt, long long c_eqlo, long long n_cand, long long c_eqhi,
                                       double lo, double hi, GetC getc, SelSmem& sm, bool* valid) {
  *valid = true;
  if (r < c_lt) { *valid = false; return 0.0; }
  r -= c_lt;
  if (r < c_eqlo) return lo;
  r -= c_eqlo;
  if (r < n_cand) return f64_unkey(block_select_key(getc, n_cand, r, sm));
  r -= n_cand;
  if (r < c_eqhi) return hi;
  *valid = false;
  return 0.0;
}

struct FsNoObserver {
  __device__ __forceinline__ void operator()(int64_t, double, double, bool) const {}
};
// A bracket [lo, hi] that held the median of an earlier, nearly identical data set (flatten: the time differences of
// the kept cadences change by a few hundred entries per iteration).  When given and valid, the sampling stage and its
// two selects are skipped; if the median turns out to lie outside, the call starts over with a fresh sample.
struct FastBracket {
  double lo, hi;
  bool valid;
};
// np.nanmedian over get(0..n-1); m = number of non-NaN values if known (>= 0), else -1 (counted in the sample pass).
// obs(i, v, lo, valid): called convergently (all 32 lanes of a warp, `valid` false for lanes past the end) for every
// element during the ONE partition pass, with the bracket's lower value `lo` <= median - a caller can piggy-back work
// that only needs a bound of the median (flatten: the gap-cut candidates).  *observed tells whether that pass ran
// (false on the small-n / fallback paths, where obs was never called or the pass was abandoned).
struct FsNoReset {
  __device__ __forceinline__ void operator()() const {}
};
// br (optional, in memory every thread of the block sees - shared memory): bracket to try first / to leave behind.  reset(): called (by all threads, followed by a barrier) before
// the partition pass is REPEATED with a fresh bracket, so that obs can start over.
template <class Get, class Obs = FsNoObserver, class Reset = FsNoReset>
__device__ double block_nanmedian_fast(Get get, int64_t n, SelSmem& sm, FastSelSmem& fs, long long m_known = -1,
                                       Obs obs = Obs(), bool* observed = nullptr, FastBracket* br = nullptr,
                                       Reset reset = Reset()) {
  if (observed) *observed = false;
  const double qnan = __longlong_as_double(0x7ff8000000000000ll);
  if (n < 4 * FS_SAMPLE) { if (br && threadIdx.x == 0) br->valid = false; return block_nanmedian(get, n, sm); }
  bool reuse = br != nullptr && br->valid;                       // (block-uniform: every thread holds the same copy)
  for (;;) {
    // ---- bracket: the caller's, or from a sample (every stride-th element; NaNs are dropped from the sample).  The
    // number of non-NaN values is only needed for the final rank: when the caller does not know it, it is counted
    // in the partition pass itself ----
    long long m = m_known;
    double lo, hi;
    if (reuse) {
      lo = br->lo;
      hi = br->hi;
    } else {
      const int64_t stride = n / FS_SAMPLE;
      double* const sample = fs.cand + FS_CAP;
      long long scnt = 0;
      for (int sidx = threadIdx.x; sidx < FS_SAMPLE; sidx += blockDim.x) {
        const double v = get((int64_t)sidx * stride);
        sample[sidx] = v;
        scnt += (v == v) ? 1 : 0;
      }
      const long long ns = block_sum_ll(scnt, sm.redll);         // (its barriers also publish the sample)
      if (ns < 4 * FS_GAP) { if (br && threadIdx.x == 0) br->valid = false; return block_nanmedian(get, n, sm); }
      auto gets = [&](int64_t i) { return sample[i]; };
      long long rlo = ns / 2 - FS_GAP, rhi = ns / 2 + FS_GAP;
      if (rlo < 0) rlo = 0;
      if (rhi > ns - 1) rhi = ns - 1;
      lo = f64_unkey(block_select_key(gets, FS_SAMPLE, rlo, sm));
      hi = f64_unkey(block_select_key(gets, FS_SAMPLE, rhi, sm));
    }
    // ---- the one pass: partition counts + candidates strictly between lo and hi ----
    if (threadIdx.x == 0) { fs.n_cand = 0; fs.c_lt = 0; fs.c_eqlo = 0; fs.c_eqhi = 0; fs.ok = 0; }
    __syncthreads();
    int c_lt = 0, c_eqlo = 0, c_eqhi = 0, c_ge = 0;               // c_ge: values >= hi (only the total is needed)
    for (int64_t i0 = 0; i0 < n; i0 += 4 * (int64_t)blockDim.x) { // warp-uniform trip count; 4 loads in flight per thread
      double vv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int64_t i = i0 + (int64_t)u * blockDim.x + threadIdx.x;
        vv[u] = (i < n) ? get(i) : qnan;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const double v = vv[u];
        obs(i0 + (int64_t)u * blockDim.x + threadIdx.x, v, lo, i0 + (int64_t)u * blockDim.x + threadIdx.x < n);
        bool between = false;
        if (v == v) {
          if (v < lo) c_lt++;
          else if (v == lo) c_eqlo++;
          else if (v < hi) between = true;
          else { c_ge++; if (v == hi) c_eqhi++; }
        }
        const unsigned bal = __ballot_sync(0xffffffffu, between);
        if (bal) {
          int base = 0;
          if ((threadIdx.x & 31) == 0) base = atomicAdd(&fs.n_cand, __popc(bal));
          base = __shfl_sync(0xffffffffu, base, 0);
          if (between) {
            const int pos = base + __popc(bal & ((1u << (threadIdx.x & 31)) - 1u));
            if (pos < FS_CAP) fs.cand[pos] = v;
          }
        }
      }
    }
    if (lo == hi) c_eqhi = 0;                                     // (one value: counted once, as eq-lo)
    c_lt = warp_sum(c_lt); c_eqlo = warp_sum(c_eqlo); c_eqhi = warp_sum(c_eqhi); c_ge = warp_sum(c_ge);
    if ((threadIdx.x & 31) == 0) {
      atomicAdd(&fs.c_lt, c_lt); atomicAdd(&fs.c_eqlo, c_eqlo); atomicAdd(&fs.c_eqhi, c_eqhi); atomicAdd(&fs.ok, c_ge);
    }
    __syncthreads();
    const long long n_cand = fs.n_cand, t_lt = fs.c_lt, t_eqlo = fs.c_eqlo, t_eqhi = fs.c_eqhi;
    if (m < 0) m = t_lt + t_eqlo + n_cand + (long long)fs.ok;    // (lo == hi: the values equal to it were counted as eq-lo)
    __syncthreads();
    const long long klo = (m - 1) / 2, khi = m / 2;
    if (reuse) {
      // is the median still inside the old bracket, and the candidate buffer large enough?  If not: fresh sample
      const bool inside = m > 0 && klo >= t_lt && khi < t_lt + t_eqlo + n_cand + t_eqhi && n_cand <= FS_CAP;
      if (!inside) {
        reuse = false;
        if (threadIdx.x == 0) br->valid = false;
        reset();
        __syncthreads();
        continue;
      }
    }
    // every element went past obs exactly once; but a fresh sample's bracket may miss above the median (lo > median:
    // more than klo values below lo), and then obs was not given a lower bound of the median
    if (observed) *observed = m > 0 && klo >= t_lt;
    if (br && threadIdx.x == 0) { br->lo = lo; br->hi = hi; br->valid = n_cand <= FS_CAP; }   // (barriers follow)
    if (n_cand > FS_CAP) return block_nanmedian(get, n, sm);
    auto getc = [&](int64_t i) { return fs.cand[i]; };
    bool v1, v2;
    const double a = fs_rank_value(klo, t_lt, t_eqlo, n_cand, t_eqhi, lo, hi, getc, sm, &v1);
    const double b = (khi == klo) ? a : fs_rank_value(khi, t_lt, t_eqlo, n_cand, t_eqhi, lo, hi, getc, sm, &v2);
    if (khi == klo) v2 = v1;
    if (!(v1 && v2)) {                                           // the bracket missed: full radix select
      if (br && threadIdx.x == 0) br->valid = false;
      return block_nanmedian(get, n, sm);
    }
    return (a + b) / 2.0;
  }
}

// np.nanstd (ddof = 0): two-pass (mean, then squared deviations), NaN ignored.
template <class Get>
__device__ double block_nanstd(Get get, int64_t n, SelSmem& sm, double* mean_out = nullptr) {
  double s = 0.0;
  long long c = 0;
#pragma unroll 4
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const double v = get(i);
    if (v == v) { s += v; c++; }
  }
  const double tot = block_sum(s, sm.red);
  const long long m = block_sum_ll(c, sm.redll);
  if (m == 0) return __longlong_as_double(0x7ff8000000000000ll);
  const double mean = tot / (double)m;
  if (mean_out) *mean_out = mean;
  double q = 0.0;
#pragma unroll 4
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const double v = get(i);
    if (v == v) { const double d = v - mean; q += d * d; }
  }
  const double qq = block_sum(q, sm.red);
  return sqrt(qq / (double)m);
}

}  // namespace lkb
