// K13: LightCurve.fold and LightCurve.bin (lightcurve.py:1089-1214, 1558-1763) over CSR-ragged fp64 light curves, one
// CTA per light curve, with the single-curve methods' exact semantics.
//
// Both rest on one primitive, fb_radix_sort: a stable LSD radix sort of (64- or 32-bit key, int32 payload) pairs, four
// bits per pass, in which every thread owns a contiguous chunk of the input, so that a digit's (digit, thread) prefix
// count is each element's stable rank - no atomics.  A pass whose digit is the same for every key moves nothing and is
// skipped.  Doubles are keyed by fb_key, whose unsigned order is np.argsort's: -0.0 and +0.0 are one key, NaN is the
// largest key, so with the cadence index as payload the sort equals np.argsort(kind="stable") bit for bit.
//
// fold_kernel: rel = ((t - t0) + shift + (P - wrap)) % P - (P - wrap) in the shim's operation order with numpy's float
//   remainder (fb_npmod), stably sorted; outputs the phase in sorted order (/ P when normalizing) and the permutation.
// bin_kernel: the cadences are stably sorted by time; each is put in bin searchsorted(starts, t, "right") - 1 and kept
//   when t < ends[bin] (t <= ends[-1] in the last bin).  Since starts ascend, each bin's kept cadences are one run of
//   the time-sorted order, whose start and end positions are all a bin needs.  nanmean is a fixed-order sum over the run;
//   nanmedian sorts by flux, then stably by the position of the bin's run (so each bin's cadences land on its run,
//   NaN last) and takes the middle value or the mean of the two middle values.  The error is the root mean square of
//   the errors when the light curve has any finite error, else the bin's nanstd of the flux.
//
// A light curve's sort buffers live in shared memory when it has at most res_cap cadences, else in a global workspace;
// both are the same code on a different pointer, so their results are bitwise equal.  Kept apart from the library's
// entry points so that tests/native/cuda_emu.h runs it on the CPU.
#pragma once
#include "common.cuh"

namespace lkb {

constexpr int FB_THREADS = 256;
constexpr int FB_RADIX = 16;                      // four bits per pass
// dynamic shared memory for the resident buffers: with the 16 KB digit histogram and the small static buffers it stays
// under the 227 KB an H100 CTA may have
constexpr size_t FB_SMEM_BYTES = 210 * 1024;
constexpr int FB_FOLD_BPC = 24;                   // bytes per cadence: two u64 key buffers, two int32 payload buffers
constexpr int FB_BIN_BPC = 32;                    // + the time-sorted permutation and each position's bin
constexpr int64_t FB_FOLD_CAP = FB_SMEM_BYTES / FB_FOLD_BPC;   // 8960 cadences
constexpr int64_t FB_BIN_CAP = FB_SMEM_BYTES / FB_BIN_BPC;     // 6720 cadences

enum FbAgg { FB_NANMEAN = 0, FB_NANMEDIAN = 1 };
enum FbStatus { FB_OK = 0, FB_BAD_STARTS = 1, FB_BAD_INDEX = 2 };

struct FoldArgs {
  const double* t;          // [off[B]]
  const int64_t* off;       // [B + 1] device CSR offsets
  const double* par;        // [4 B] device: t0, shift, period, wrap of each light curve
  int normalize;
  double* phase;            // [off[B]] in sorted order
  int32_t* perm;            // [off[B]] local cadence index of each sorted position
  uint64_t* work;           // global sort buffers of the light curves longer than res_cap
  const int64_t* woff;      // [B] their offsets into work, in cadences
  int res_cap;
};

struct BinArgs {
  const double *t, *f, *fe; // [off[B]] cadences; fe may be NULL (no errors)
  const int64_t* off;       // [B + 1]
  const int64_t* boff;      // [B + 1] device CSR offsets of the bins
  const double *starts, *ends;   // [boff[B]] edges as times, or NULL ...
  const int32_t *sidx, *eidx;    // ... as indices into the light curve's time-sorted cadences
  int agg;                  // FbAgg
  double *centre, *flux, *err;   // [boff[B]]
  int32_t* count;           // [boff[B]]
  int32_t* blo;             // [boff[B]] scratch: first time-sorted position of each bin's run
  int32_t* status;          // [B] FbStatus
  uint64_t* work;
  const int64_t* woff;
  int res_cap;
};

// Resident capacity, workspace offsets and dynamic shared memory of one launch (host).
struct FbPlan {
  int res_cap;
  int64_t work_cadences;    // cadences of the light curves that work in global memory
  size_t smem;
};
inline FbPlan fb_plan(const int64_t* h_off, int B, int64_t cap, int bpc, int64_t* h_woff) {
  FbPlan p{};
  int64_t nres = 0, w = 0;
  for (int b = 0; b < B; ++b) {
    const int64_t n = h_off[b + 1] - h_off[b];
    if (n <= cap) {
      if (n > nres) nres = n;
      h_woff[b] = 0;
    } else {
      h_woff[b] = w;
      w += n;
    }
  }
  p.res_cap = (int)nres;
  p.work_cadences = w;
  p.smem = (size_t)bpc * (size_t)nres;
  return p;
}

// numpy's less-than of its sorts and searchsorted: NaN is the largest value
__device__ __forceinline__ bool fb_less(double a, double b) { return a < b || (b != b && a == a); }

// order-preserving key: -0.0 is keyed as +0.0, every NaN as the largest key
__device__ __forceinline__ uint64_t fb_key(double v) {
  if (v != v) return ~0ull;
  if (v == 0.0) v = 0.0;
  const uint64_t u = (uint64_t)__double_as_longlong(v);
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

// numpy's float remainder x % p (npy_divmod): fmod, moved to the sign of p, and +0.0 (for p > 0) where fmod gives a
// zero - bst_npmod keeps fmod's -0.0 there, which survives fold's "- (P - wrap)" when wrap == P
__device__ __forceinline__ double fb_npmod(double x, double p) {
  double m = fmod(x, p);
  if (m != 0.0) {
    if ((p < 0.0) != (m < 0.0)) m += p;
  } else {
    m = copysign(0.0, p);
  }
  return m;
}

__device__ __forceinline__ double fb_fold_rel(double t, double t0, double shift, double period, double wrap) {
  const double c = period - wrap;
  return fb_npmod(((t - t0) + shift) + c, period) - c;
}

struct FbSortSmem {
  int hist[FB_RADIX * FB_THREADS];   // [digit][thread]
  int wsum[33];
  int skip;
};

// Block-wide exclusive scan of ints in thread order.  All threads must call.
__device__ __forceinline__ int fb_block_exscan(int v, int* wsum) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  __syncthreads();
  if (lane == 31) wsum[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int w = lane < nw ? wsum[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    if (lane < nw) wsum[lane] = w;
  }
  __syncthreads();
  return (wid ? wsum[wid - 1] : 0) + x - v;
}

// Stable sort of the n pairs (ka[i], va[i]) by the low `nbits` bits of the key; kb / vb are scratch of n entries.
// Returns 0 when the sorted pairs are in (ka, va), 1 when they are in (kb, vb).  All threads must call.
template <typename K>
__device__ int fb_radix_sort(K* ka, int32_t* va, K* kb, int32_t* vb, int n, int nbits, FbSortSmem& s) {
  const int T = blockDim.x, tid = threadIdx.x;
  const int chunk = (n + T - 1) / T;
  const int i0 = min(n, tid * chunk), i1 = min(n, i0 + chunk);
  int cur = 0;
  for (int sh = 0; sh < nbits; sh += 4) {
    const K* ks = cur ? kb : ka;
    const int32_t* vs = cur ? vb : va;
    K* kd = cur ? ka : kb;
    int32_t* vd = cur ? va : vb;
    for (int d = 0; d < FB_RADIX; ++d) s.hist[d * T + tid] = 0;
    if (tid == 0) s.skip = 0;
    for (int i = i0; i < i1; ++i) s.hist[(int)((ks[i] >> sh) & 15) * T + tid]++;
    __syncthreads();
    // exclusive scan of the counts in (digit, thread) order: thread tid scans entries [16 tid, 16 tid + 16)
    int sum = 0;
    for (int k = 0; k < FB_RADIX; ++k) sum += s.hist[FB_RADIX * tid + k];
    int run = fb_block_exscan(sum, s.wsum);
    for (int k = 0; k < FB_RADIX; ++k) {
      const int c = s.hist[FB_RADIX * tid + k];
      s.hist[FB_RADIX * tid + k] = run;
      run += c;
    }
    __syncthreads();
    if (tid < FB_RADIX) {                        // one digit holds every key: the pass would move nothing
      const int lo = s.hist[tid * T], hi = tid + 1 < FB_RADIX ? s.hist[(tid + 1) * T] : n;
      if (lo == 0 && hi == n) s.skip = 1;
    }
    __syncthreads();
    if (!s.skip) {
      for (int i = i0; i < i1; ++i) {
        const K k = ks[i];
        const int pos = s.hist[(int)((k >> sh) & 15) * T + tid]++;
        kd[pos] = k;
        vd[pos] = vs[i];
      }
      cur ^= 1;
    }
    __syncthreads();
  }
  return cur;
}

__global__ void __launch_bounds__(FB_THREADS) fold_kernel(FoldArgs a) {
  LKB_DYN_SMEM(uint64_t, dyn);
  __shared__ FbSortSmem ss;
  const int b = blockIdx.x;
  const int64_t o = a.off[b];
  const int n = (int)(a.off[b + 1] - o);
  uint64_t* K0 = n <= a.res_cap ? dyn : a.work + 3 * a.woff[b];
  uint64_t* K1 = K0 + n;
  int32_t* V0 = reinterpret_cast<int32_t*>(K1 + n);
  int32_t* V1 = V0 + n;
  const double t0 = a.par[4 * b], shift = a.par[4 * b + 1], P = a.par[4 * b + 2], wrap = a.par[4 * b + 3];
  const double* tb = a.t + o;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    K0[i] = fb_key(fb_fold_rel(tb[i], t0, shift, P, wrap));
    V0[i] = i;
  }
  __syncthreads();
  const int32_t* perm = fb_radix_sort<uint64_t>(K0, V0, K1, V1, n, 64, ss) ? V1 : V0;
  for (int j = threadIdx.x; j < n; j += blockDim.x) {
    const int i = perm[j];
    const double rel = fb_fold_rel(tb[i], t0, shift, P, wrap);
    a.phase[o + j] = a.normalize ? rel / P : rel;
    a.perm[o + j] = i;
  }
}

__global__ void __launch_bounds__(FB_THREADS) bin_kernel(BinArgs a) {
  LKB_DYN_SMEM(uint64_t, dyn);
  __shared__ FbSortSmem ss;
  __shared__ long long redll[33];
  const int b = blockIdx.x, T = blockDim.x, tid = threadIdx.x;
  const int64_t o = a.off[b], bo = a.boff[b];
  const int n = (int)(a.off[b + 1] - o), nb = (int)(a.boff[b + 1] - bo);
  const double qnan = __longlong_as_double(0x7ff8000000000000ll);

  // ---- the edges: starts ascend (numpy's order), indices are in range ----
  long long bad = 0;
  for (int j = tid; j < nb; j += T) {
    if (a.sidx) {
      const int s = a.sidx[bo + j], e = a.eidx[bo + j];
      if (s < 0 || s >= n || e < 0 || e >= n) bad |= FB_BAD_INDEX;
      else if (j > 0 && a.sidx[bo + j - 1] > s) bad |= FB_BAD_STARTS;
    } else if (j > 0 && fb_less(a.starts[bo + j], a.starts[bo + j - 1])) {
      bad |= FB_BAD_STARTS;
    }
  }
  bad = block_sum_ll(bad, redll);
  if (tid == 0) a.status[b] = bad == 0 ? FB_OK : ((bad & FB_BAD_INDEX) ? FB_BAD_INDEX : FB_BAD_STARTS);
  if (bad) return;

  uint64_t* K0 = n <= a.res_cap ? dyn : a.work + 4 * a.woff[b];
  uint64_t* K1 = K0 + n;
  int32_t* V0 = reinterpret_cast<int32_t*>(K1 + n);
  int32_t* V1 = V0 + n;
  int32_t* P = V1 + n;                       // time-sorted position -> cadence
  int32_t* G = P + n;                        // time-sorted position -> bin, -1 outside every bin
  const double *tb = a.t + o, *fb = a.f + o, *eb = a.fe ? a.fe + o : nullptr;

  // ---- stable sort by time; ts (in K0) = the sorted times ----
  long long efin = 0;
  for (int i = tid; i < n; i += T) {
    K0[i] = fb_key(tb[i]);
    V0[i] = i;
    if (eb && isfinite(eb[i])) efin++;
  }
  const bool have_err = block_sum_ll(efin, redll) > 0;     // (its barriers publish K0, V0)
  const int32_t* perm = fb_radix_sort<uint64_t>(K0, V0, K1, V1, n, 64, ss) ? V1 : V0;
  double* ts = reinterpret_cast<double*>(K0);
  for (int p = tid; p < n; p += T) {
    const int i = perm[p];
    P[p] = i;
    ts[p] = tb[i];
  }
  __syncthreads();

  auto start_of = [&](int j) { return a.sidx ? ts[a.sidx[bo + j]] : a.starts[bo + j]; };
  auto end_of = [&](int j) { return a.sidx ? ts[a.eidx[bo + j]] : a.ends[bo + j]; };

  // ---- each position's bin: searchsorted(starts, t, "right") - 1, kept when t < its end (<= in the last bin) ----
  for (int p = tid; p < n; p += T) {
    const double v = ts[p];
    int lo = 0, hi = nb;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (fb_less(v, start_of(mid))) hi = mid;
      else lo = mid + 1;
    }
    const int j = lo - 1;
    bool in = false;
    if (j >= 0) {
      const double e = end_of(j);
      in = v < e || (j == nb - 1 && v <= e);
    }
    G[p] = in ? j : -1;
  }
  for (int j = tid; j < nb; j += T) {
    const double s = start_of(j), e = end_of(j);
    a.centre[bo + j] = s + 0.5 * (e - s);
    a.blo[bo + j] = 0;
    a.count[bo + j] = 0;                     // (the end of the run until the finish)
  }
  __syncthreads();
  for (int p = tid; p < n; p += T) {         // a bin's kept cadences are one run of the time-sorted order
    const int g = G[p];
    if (g < 0) continue;
    if (p == 0 || G[p - 1] != g) a.blo[bo + g] = p;
    if (p == n - 1 || G[p + 1] != g) a.count[bo + g] = p + 1;
  }
  __syncthreads();

  // ---- nanmedian: sort by flux (NaN last), then stably by the start of the bin's run: each bin's cadences land on
  // its own run in flux order; a cadence outside every bin keeps its position ----
  const int32_t* med = nullptr;
  if (a.agg == FB_NANMEDIAN) {
    for (int p = tid; p < n; p += T) {
      K0[p] = fb_key(fb[P[p]]);
      V0[p] = p;
    }
    __syncthreads();
    const int r = fb_radix_sort<uint64_t>(K0, V0, K1, V1, n, 64, ss);
    uint64_t* Kr = r ? K1 : K0;
    int32_t* Vr = r ? V1 : V0;
    for (int q = tid; q < n; q += T) {
      const int p = Vr[q], g = G[p];
      Kr[q] = (uint64_t)(g >= 0 ? a.blo[bo + g] : p);
    }
    __syncthreads();
    const int r2 = fb_radix_sort<uint64_t>(Kr, Vr, r ? K0 : K1, r ? V0 : V1, n, 32, ss);
    med = r2 ? (r ? V0 : V1) : Vr;
  }

  // ---- per bin, one thread, in time-sorted order ----
  for (int j = tid; j < nb; j += T) {
    const int lo = a.blo[bo + j], cnt = a.count[bo + j] - lo;
    a.count[bo + j] = cnt;
    double fv = qnan, ev = qnan;
    if (cnt > 0) {
      double s = 0.0;
      int c = 0;
      bool anyfin = false;
      for (int q = lo; q < lo + cnt; ++q) {
        const double x = fb[P[q]];
        if (x == x) { s += x; c++; }
        anyfin |= (bool)isfinite(x);
      }
      const double mean = c ? s / (double)c : qnan;
      if (a.agg == FB_NANMEAN) {
        fv = mean;
      } else if (c > 0) {
        const int h = lo + c / 2;
        fv = (c & 1) ? fb[P[med[h]]] : (fb[P[med[h - 1]]] + fb[P[med[h]]]) / 2.0;
      }
      if (have_err) {
        double s2 = 0.0;
        int cf = 0;
        for (int q = lo; q < lo + cnt; ++q) {
          const double e = eb[P[q]];
          if (e == e) s2 += e * e;
          if (isfinite(e)) cf++;
        }
        if (cf) ev = sqrt(s2 / (double)cf);
      } else if (anyfin) {
        double q2 = 0.0;
        for (int q = lo; q < lo + cnt; ++q) {
          const double x = fb[P[q]];
          if (x == x) { const double d = x - mean; q2 += d * d; }
        }
        ev = sqrt(q2 / (double)c);
      }
    }
    a.flux[bo + j] = fv;
    a.err[bo + j] = ev;
  }
}

}  // namespace lkb
