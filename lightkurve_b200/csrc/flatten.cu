// K4: LightCurve.flatten, /root/reference/src/lightkurve/lightcurve.py:996-1070, on the device:
//   sigma-clip pre-mask (:1002-1010) -> per iteration: compaction of the kept cadences, gap
//   segmentation (:1022-1027), per segment Savitzky-Golay (scipy savgol_filter mode="interp",
//   :1040) or nanmedian fallback (:1034-1035), residual clip (:1049-1052), linear
//   interpolation/extrapolation back to every cadence (scipy interp1d, :1053-1058), mask update
//   (:1060-1063); finally flux/trend, flux_err/trend (:1065-1070).
// One CTA per light curve (the masks and segments are data dependent per light curve, H8 of
// SURVEY.md); all scratch lives in a CSR workspace in HBM; the FIR interior is a shared-memory
// tiled fp64 sliding-window filter (4 outputs per thread, skewed layout => conflict-free LDS.64).
// K6 entry lkb_nanmedian_std is here too.
#include "common.cuh"
#include "select.cuh"
#include "flatten_v2.cuh"
#include <vector>

namespace lkb {

int g_last_flatten_path = -1;      // kernel path of the last lkb_flatten call (LKB_FLATTEN_PATH_*; -1: none yet)

constexpr int FL_THREADS = 512;
constexpr int FL_R = 4;                          // outputs per thread per tile
constexpr int FL_TI = FL_THREADS * FL_R;         // outputs per tile

struct FlWs {
  uint8_t* mask;     // [total] 1 = cadence currently used for the fit
  int32_t* cidx;     // [total] compacted indices of used cadences
  double* fc;        // [total] flux at compacted cadences
  double* tc;        // [total] time at compacted cadences
  double* trc;       // [total] trend at compacted cadences
  uint8_t* mask1;    // [total]
  int32_t* sidx;     // [total] survivors (positions in the compacted list)
  int32_t* cuts;     // [total + B] segment start positions
  double* xs;        // [total] survivors' times (contiguous)
  double* ys;        // [total] survivors' trend values
};

__device__ __forceinline__ int fl_skew(int e) { return e + (e >> 4); }

// Order-preserving block compaction: out[k] = i for every i in [0,n) with pred(i); returns count.
template <class Pred>
__device__ int block_compact(Pred pred, int n, int32_t* out, int* s_warp_counts, int* s_base) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (threadIdx.x == 0) *s_base = 0;
  __syncthreads();
  for (int c0 = 0; c0 < n; c0 += blockDim.x) {
    const int i = c0 + threadIdx.x;
    const bool p = (i < n) && pred(i);
    const unsigned bal = __ballot_sync(0xffffffffu, p);
    if (lane == 0) s_warp_counts[warp] = __popc(bal);
    __syncthreads();
    int off = *s_base;
    for (int w = 0; w < warp; ++w) off += s_warp_counts[w];
    if (p) out[off + __popc(bal & ((1u << lane) - 1u))] = i;
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int w = 0; w < nw; ++w) tot += s_warp_counts[w];
      *s_base += tot;
    }
    __syncthreads();
  }
  return *s_base;
}

__global__ void __launch_bounds__(FL_THREADS, 2)
flatten_kernel(const double* __restrict__ time, const double* __restrict__ flux, const double* __restrict__ flux_err,
               const uint8_t* __restrict__ exclude, const int64_t* __restrict__ offsets, FlWs ws,
               int window_length, int polyorder, double break_tolerance, int niters, double sigma,
               const double* __restrict__ coeffs /*[w] correlation order*/,
               const double* __restrict__ edge /*[w][half]: edge[j*half+i] weight of x[j] for output i*/,
               double* __restrict__ flat, double* __restrict__ flat_err, double* __restrict__ trend) {
  extern __shared__ __align__(16) unsigned char fl_smem[];
  double* s_c = reinterpret_cast<double*>(fl_smem);                 // [w]
  double* s_x = s_c + ((window_length + 3) & ~3);                   // skewed [FL_TI + w]
  __shared__ SelSmem sm;
  __shared__ int s_wc[FL_THREADS / 32];
  __shared__ int s_base;
  __shared__ double s_val;

  const int b = blockIdx.x;
  const int64_t o = offsets[b];
  const int n = (int)(offsets[b + 1] - o);
  if (n <= 0) return;
  const double* t = time + o;
  const double* f = flux + o;
  uint8_t* mask = ws.mask + o;
  int32_t* cidx = ws.cidx + o;
  double* fc = ws.fc + o;
  double* tc = ws.tc + o;
  double* trc = ws.trc + o;
  uint8_t* mask1 = ws.mask1 + o;
  int32_t* sidx = ws.sidx + o;
  int32_t* cuts = ws.cuts + o + b;
  double* tr = trend + o;
  const int w = window_length, half = w / 2;
  const double qnan = __longlong_as_double(0x7ff8000000000000ll);

  for (int i = threadIdx.x; i < w; i += blockDim.x) s_c[i] = coeffs[i];

  // ---- initial mask (:996-1010) ----
  const double med0 = block_nanmedian([&](int64_t i) { const double v = f[i]; return isfinite(v) ? v : qnan; }, n, sm);
  // np.nanmedian/np.nanstd ignore NaN only; +-inf would poison them exactly as in numpy:
  // keep numpy semantics by feeding inf through the std (mean becomes inf/nan => std nan => mask all false).
  const double std0 = block_nanstd([&](int64_t i) { return f[i]; }, n, sm);
  {
    const double thr = std0 * sigma;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const double v = f[i];
      bool m = exclude ? (exclude[o + i] == 0) : true;
      double a = fabs(v - med0);
      if (a != a) a = 0.0;                      // nan_to_num
      m = m && isfinite(v) && (a <= thr);
      mask[i] = m ? 1 : 0;
    }
  }
  __syncthreads();

  bool ok = true;
  for (int it = 0; it < niters; ++it) {
    // ---- compaction ----
    const int m = block_compact([&](int i) { return mask[i] != 0; }, n, cidx, s_wc, &s_base);
    if (m < 2) { ok = false; break; }
    for (int i = threadIdx.x; i < m; i += blockDim.x) { const int g = cidx[i]; fc[i] = f[g]; tc[i] = t[g]; }
    __syncthreads();
    // ---- gap segmentation (:1022-1027) ----
    const double med_dt = block_nanmedian([&](int64_t i) { return tc[i + 1] - tc[i]; }, m - 1, sm);
    const double thr_dt = break_tolerance * med_dt;
    if (threadIdx.x == 0) cuts[0] = 0;
    const int ncut = block_compact([&](int i) { return (tc[i + 1] - tc[i]) > thr_dt; }, m - 1, cuts + 1, s_wc, &s_base);
    for (int i = threadIdx.x; i < ncut; i += blockDim.x) cuts[1 + i] += 1;    // cut = where(...) + 1
    __syncthreads();
    const int nseg = ncut + 1;
    // ---- per segment trend ----
    for (int s = 0; s < nseg; ++s) {
      const int l = cuts[s], h = (s + 1 < nseg) ? cuts[s + 1] : m;
      const int len = h - l;
      const bool fallback = (w > len) || ((double)len < break_tolerance);
      if (fallback) {
        const double* fs = fc + l;
        const double md = block_nanmedian([&](int64_t i) { return fs[i]; }, len, sm);
        for (int i = threadIdx.x; i < len; i += blockDim.x) trc[l + i] = md;
      } else {
        const double* x = fc + l;
        double* y = trc + l;
        // interior: y[i] = sum_j c[j] x[i - half + j], i in [half, len - half)
        const int i_end = len - half;
        for (int i0 = half; i0 < i_end; i0 += FL_TI) {
          const int nout = min(FL_TI, i_end - i0);
          const int nin = nout + w - 1;
          __syncthreads();
          for (int e = threadIdx.x; e < nin; e += blockDim.x) s_x[fl_skew(e)] = x[i0 - half + e];
          // zero the tail a thread may touch beyond nin
          for (int e = nin + threadIdx.x; e < FL_TI + w; e += blockDim.x) s_x[fl_skew(e)] = 0.0;
          __syncthreads();
          const int a = FL_R * threadIdx.x;
          if (a < nout) {
            double acc0 = 0.0, acc1 = 0.0, acc2 = 0.0, acc3 = 0.0;
            double x0 = s_x[fl_skew(a)], x1 = s_x[fl_skew(a + 1)], x2 = s_x[fl_skew(a + 2)], x3 = s_x[fl_skew(a + 3)];
            int j = 0;
            for (; j + 4 <= w; j += 4) {
              const double c0 = s_c[j], c1 = s_c[j + 1], c2 = s_c[j + 2], c3 = s_c[j + 3];
              const double x4 = s_x[fl_skew(a + j + 4)], x5 = s_x[fl_skew(a + j + 5)];
              const double x6 = s_x[fl_skew(a + j + 6)], x7 = s_x[fl_skew(a + j + 7)];
              acc0 = fma(c0, x0, acc0); acc0 = fma(c1, x1, acc0); acc0 = fma(c2, x2, acc0); acc0 = fma(c3, x3, acc0);
              acc1 = fma(c0, x1, acc1); acc1 = fma(c1, x2, acc1); acc1 = fma(c2, x3, acc1); acc1 = fma(c3, x4, acc1);
              acc2 = fma(c0, x2, acc2); acc2 = fma(c1, x3, acc2); acc2 = fma(c2, x4, acc2); acc2 = fma(c3, x5, acc2);
              acc3 = fma(c0, x3, acc3); acc3 = fma(c1, x4, acc3); acc3 = fma(c2, x5, acc3); acc3 = fma(c3, x6, acc3);
              x0 = x4; x1 = x5; x2 = x6; x3 = x7;
            }
            for (; j < w; ++j) {
              const double c0 = s_c[j];
              const double x4 = s_x[fl_skew(a + j + 4)];
              acc0 = fma(c0, x0, acc0); acc1 = fma(c0, x1, acc1); acc2 = fma(c0, x2, acc2); acc3 = fma(c0, x3, acc3);
              x0 = x1; x1 = x2; x2 = x3; x3 = x4;
            }
            if (a + 0 < nout) y[i0 + a + 0] = acc0;
            if (a + 1 < nout) y[i0 + a + 1] = acc1;
            if (a + 2 < nout) y[i0 + a + 2] = acc2;
            if (a + 3 < nout) y[i0 + a + 3] = acc3;
          }
        }
        // edges: polynomial fit of the first/last w samples (scipy _fit_edges_polyfit)
        for (int i = threadIdx.x; i < 2 * half; i += blockDim.x) {
          const bool left = i < half;
          const int ii = left ? i : (i - half);              // output within the edge
          double acc = 0.0;
          if (left) {
            for (int j = 0; j < w; ++j) acc = fma(edge[(size_t)j * half + ii], x[j], acc);
            y[ii] = acc;
          } else {
            // right edge by symmetry: weight of x[len-w+j] for output len-half+ii = edge[(w-1-j)][half-1-ii]
            const double* xr = x + (len - w);
            for (int j = 0; j < w; ++j) acc = fma(edge[(size_t)(w - 1 - j) * half + (half - 1 - ii)], xr[j], acc);
            y[len - half + ii] = acc;
          }
        }
      }
      __syncthreads();
    }
    // ---- residual clip (:1049-1052) ----
    const double rstd = block_nanstd([&](int64_t i) { return fc[i] - trc[i]; }, m, sm);
    const double rthr = rstd * sigma + 1e-14;
    for (int i = threadIdx.x; i < m; i += blockDim.x) {
      double a = fabs(fc[i] - trc[i]);
      if (a != a) a = 0.0;
      mask1[i] = (a < rthr) ? 1 : 0;
    }
    __syncthreads();
    const int ms = block_compact([&](int i) { return mask1[i] != 0; }, m, sidx, s_wc, &s_base);
    if (ms < 2) { ok = false; break; }
    // ---- interp1d(kind="linear", fill_value="extrapolate") onto every cadence (:1053-1058) ----
    // survivors' (time, trend) made contiguous first (re-using fc / the tail of tc is not possible:
    // both are still needed), so the binary search does one dependent load per step
    double* xs = ws.xs + o;
    double* ys = ws.ys + o;
    for (int k = threadIdx.x; k < ms; k += blockDim.x) { const int j = sidx[k]; xs[k] = tc[j]; ys[k] = trc[j]; }
    __syncthreads();
    for (int g = threadIdx.x; g < n; g += blockDim.x) {
      const double xq = t[g];
      // np.searchsorted(xp, xq, side="left"): the survivors are a thinned copy of the cadences, so the answer
      // sits next to g * ms / n - gallop out from there (2-4 dependent loads instead of log2(ms) = 16)
      int lo, hi;
      {
        const int g0 = min(ms - 1, (int)(((long long)g * ms) / n));
        int step = 1;
        if (xs[g0] < xq) {
          lo = g0 + 1;
          hi = min(ms, lo + step);
          while (hi < ms && xs[hi] < xq) { lo = hi + 1; step <<= 1; hi = min(ms, lo + step); }
        } else {
          hi = g0;
          lo = max(0, hi - step);
          while (lo > 0 && xs[lo] >= xq) { hi = lo; step <<= 1; lo = max(0, hi - step); }
        }
      }
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (xs[mid] < xq) lo = mid + 1; else hi = mid;
      }
      const int idx = lo < 1 ? 1 : (lo > ms - 1 ? ms - 1 : lo);
      const double xl = xs[idx - 1], xh = xs[idx], yl = ys[idx - 1], yh = ys[idx];
      const double slope = (yh - yl) / (xh - xl);
      tr[g] = slope * (xq - xl) + yl;
    }
    // ---- mask[mask] &= mask1 (:1060-1063) ----
    for (int i = threadIdx.x; i < m; i += blockDim.x)
      if (!mask1[i]) mask[cidx[i]] = 0;
    __syncthreads();
  }
  if (!ok) {
    for (int g = threadIdx.x; g < n; g += blockDim.x) tr[g] = qnan;
    __syncthreads();
  }
  (void)s_val;
  for (int g = threadIdx.x; g < n; g += blockDim.x) {
    const double tv = tr[g];
    flat[o + g] = f[g] / tv;
    if (flat_err) flat_err[o + g] = (flux_err ? flux_err[o + g] : qnan) / tv;
  }
}

// ---- K6 entry -----------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
nanmedian_std_kernel(const double* __restrict__ x, const int64_t* __restrict__ offsets, double* __restrict__ med,
                     double* __restrict__ sd) {
  __shared__ SelSmem sm;
  const int b = blockIdx.x;
  const int64_t o = offsets[b], n = offsets[b + 1] - o;
  const double* xx = x + o;
  const double m = block_nanmedian([&](int64_t i) { return xx[i]; }, n, sm);
  const double s = block_nanstd([&](int64_t i) { return xx[i]; }, n, sm);
  if (threadIdx.x == 0) {
    if (med) med[b] = m;
    if (sd) sd[b] = s;
  }
}

int nanmedian_std(const double* x, const int64_t* h_offsets, int B, double* out_median, double* out_std, int mem,
                  cudaStream_t st) {
  LKB_REQUIRE(x && h_offsets && B > 0, "lkb_nanmedian_std: null/empty argument");
  LKB_TRY(ensure_device());
  const int64_t total = h_offsets[B];
  const double* d_x = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, x, total, &d_x, st));
  int64_t* d_off = nullptr;
  LKB_TRY(ws_get_t<int64_t>(WS_A, B + 1, &d_off));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_off, h_offsets, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  double *d_m = nullptr, *d_s = nullptr;
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0, out_median, B, &d_m));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT1, out_std, B, &d_s));
  nanmedian_std_kernel<<<B, 256, 0, st>>>(d_x, d_off, d_m, d_s);
  LKB_LAUNCH_CHECK();
  LKB_TRY(stage_out_copy<double>(mem, out_median, d_m, B, st));
  LKB_TRY(stage_out_copy<double>(mem, out_std, d_s, B, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

// ---- Savitzky-Golay tables (host, fp64): scipy.signal.savgol_coeffs / _fit_edges_polyfit ----
// Solve the small (p+1)x(p+1) normal equations of the Vandermonde system with scaled abscissae.
static bool solve_dense(std::vector<double>& A, std::vector<double>& Bm, int n, int nrhs) {
  // Gaussian elimination with partial pivoting; A [n][n], Bm [n][nrhs]
  for (int c = 0; c < n; ++c) {
    int piv = c;
    for (int r = c + 1; r < n; ++r)
      if (fabs(A[r * n + c]) > fabs(A[piv * n + c])) piv = r;
    if (A[piv * n + c] == 0.0) return false;
    if (piv != c) {
      for (int k = 0; k < n; ++k) std::swap(A[c * n + k], A[piv * n + k]);
      for (int k = 0; k < nrhs; ++k) std::swap(Bm[c * nrhs + k], Bm[piv * nrhs + k]);
    }
    for (int r = c + 1; r < n; ++r) {
      const double fct = A[r * n + c] / A[c * n + c];
      if (fct == 0.0) continue;
      for (int k = c; k < n; ++k) A[r * n + k] -= fct * A[c * n + k];
      for (int k = 0; k < nrhs; ++k) Bm[r * nrhs + k] -= fct * Bm[c * nrhs + k];
    }
  }
  for (int c = n - 1; c >= 0; --c) {
    for (int k = 0; k < nrhs; ++k) {
      double v = Bm[c * nrhs + k];
      for (int r = c + 1; r < n; ++r) v -= A[c * n + r] * Bm[r * nrhs + k];
      Bm[c * nrhs + k] = v / A[c * n + c];
    }
  }
  return true;
}

// Projection matrix H = V (V^T V)^-1 V^T of the degree-p least-squares fit on w equispaced
// abscissae u = (k - c)/c in [-1, 1].  The columns of V are the Legendre polynomials P_r(u), nearly
// orthogonal on these points, so V^T V stays well conditioned up to polyorder 12 (monomials u^r lose
// ~1e-8 of the taps there).  coeffs[j] = H[center][j] (symmetric FIR); edge[j*half + i] = H[i][j], i < half.
static bool savgol_tables(int w, int p, std::vector<double>& coeffs, std::vector<double>& edge) {
  const int q = p + 1, half = w / 2;
  const double c = 0.5 * (w - 1), sc = c > 0 ? c : 1.0;
  std::vector<double> V((size_t)w * q);
  for (int k = 0; k < w; ++k) {
    const double u = (k - c) / sc;
    double p0 = 1.0, p1 = u;
    for (int r = 0; r < q; ++r) {
      V[(size_t)k * q + r] = p0;
      const double p2 = ((2 * r + 3) * u * p1 - (r + 1) * p0) / (r + 2);     // (r+2) P_{r+2} = (2r+3) u P_{r+1} - (r+1) P_r
      p0 = p1;
      p1 = p2;
    }
  }
  std::vector<double> G((size_t)q * q, 0.0), Vt((size_t)q * w);
  for (int r = 0; r < q; ++r)
    for (int s = 0; s < q; ++s) {
      double acc = 0.0;
      for (int k = 0; k < w; ++k) acc += V[(size_t)k * q + r] * V[(size_t)k * q + s];
      G[r * q + s] = acc;
    }
  for (int r = 0; r < q; ++r)
    for (int k = 0; k < w; ++k) Vt[(size_t)r * w + k] = V[(size_t)k * q + r];
  if (!solve_dense(G, Vt, q, w)) return false;     // Vt := (V^T V)^-1 V^T   [q][w]
  coeffs.assign(w, 0.0);
  edge.assign((size_t)w * (half > 0 ? half : 1), 0.0);
  for (int j = 0; j < w; ++j) {
    double acc = 0.0;
    for (int r = 0; r < q; ++r) acc += V[(size_t)half * q + r] * Vt[(size_t)r * w + j];
    coeffs[j] = acc;
    for (int i = 0; i < half; ++i) {
      double e = 0.0;
      for (int r = 0; r < q; ++r) e += V[(size_t)i * q + r] * Vt[(size_t)r * w + j];
      edge[(size_t)j * half + i] = e;
    }
  }
  return true;
}

// Inverse normal matrix of the degree-p fit on the scaled abscissae u_k = (k - c) / c, c = (w - 1) / 2 (flatten_v2.cuh:
// centre taps c_j = sum_s Ginv[0][s] (j / c)^s, edge polynomials beta = Ginv m).
static bool savgol_ginv(int w, int p, F2Coef& cf) {
  const int q = p + 1;
  if (q > F2_MAXQ) return false;
  const double c = 0.5 * (w - 1), sc = c > 0 ? c : 1.0;
  std::vector<double> G((size_t)q * q, 0.0), I((size_t)q * q, 0.0);
  for (int k = 0; k < w; ++k) {
    const double u = (k - c) / sc;
    double pr = 1.0;
    std::vector<double> pw(q);
    for (int r = 0; r < q; ++r) { pw[r] = pr; pr *= u; }
    for (int r = 0; r < q; ++r)
      for (int s2 = 0; s2 < q; ++s2) G[r * q + s2] += pw[r] * pw[s2];
  }
  for (int r = 0; r < q; ++r) I[r * q + r] = 1.0;
  if (!solve_dense(G, I, q, q)) return false;
  cf.q = q;
  for (int i = 0; i < F2_MAXQ * F2_MAXQ; ++i) cf.Ginv[i] = 0.0;
  for (int r = 0; r < q; ++r)
    for (int s2 = 0; s2 < q; ++s2) cf.Ginv[r * q + s2] = I[r * q + s2];
  cf.A[0] = I[0];
  cf.A[1] = q > 2 ? I[2] / (sc * sc) : 0.0;
  cf.A[2] = q > 4 ? I[4] / (sc * sc * sc * sc) : 0.0;
  return true;
}

int savgol_tables_host(int w, int p, double* coeffs, double* edge) {
  LKB_REQUIRE(w >= 1 && (w & 1), "window_length must be a positive odd integer");
  LKB_REQUIRE(p >= 0 && p < w && p <= 12, "polyorder must be in [0, min(window_length-1, 12)]");
  std::vector<double> c, e;
  if (!savgol_tables(w, p, c, e)) { set_error("singular Savitzky-Golay system"); return LKB_E_SINGULAR; }
  if (coeffs) memcpy(coeffs, c.data(), sizeof(double) * w);
  if (edge && w / 2 > 0) memcpy(edge, e.data(), sizeof(double) * (size_t)w * (w / 2));
  return LKB_OK;
}

struct F2Args {
  const double *t, *f, *fe;
  const uint8_t* ex;
  const int64_t* off;
  double* tro;
  int window_length;
  double break_tolerance;
  int niters;
  double sigma;
  F2Coef cf;
  int tile_out;
  double *flat, *flat_err, *trend;
  int* status;
};

template <int NM, bool DIRECT>
static int launch_flatten2(const F2Args& a, int B, size_t smem, cudaStream_t st) {
  static size_t attr = 0;
  auto* kernel = flatten2_kernel<NM, DIRECT>;
  if (smem > attr) {
    LKB_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = smem;
  }
  kernel<<<B, F2_THREADS, smem, st>>>(a.t, a.f, a.fe, a.ex, a.off, a.tro, a.window_length,
                                      a.break_tolerance, a.niters, a.sigma, a.cf, a.tile_out, a.flat, a.flat_err,
                                      a.trend, a.status);
  return LKB_OK;
}

int flatten(const double* time, const double* flux, const double* flux_err, const uint8_t* exclude_mask,
            const int64_t* h_offsets, int B, int window_length, int polyorder, double break_tolerance, int niters,
            double sigma, double* flat, double* flat_err, double* trend, int mem, cudaStream_t st) {
  LKB_REQUIRE(time && flux && h_offsets && flat && trend && B > 0, "lkb_flatten: null/empty argument");
  LKB_REQUIRE(window_length >= 1 && (window_length & 1), "window_length must be a positive odd integer");
  LKB_REQUIRE(window_length <= 8191, "lkb_flatten: window_length > 8191 unsupported");
  LKB_REQUIRE(niters >= 1, "lkb_flatten: niters must be >= 1");
  if (polyorder >= window_length) polyorder = window_length - 1;     // lightcurve.py:1015-1020
  LKB_REQUIRE(polyorder >= 0 && polyorder <= 12, "lkb_flatten: polyorder outside [0, 12]");
  LKB_TRY(ensure_device());
  const int64_t total = h_offsets[B];
  for (int b = 0; b < B; ++b)
    LKB_REQUIRE(h_offsets[b + 1] - h_offsets[b] < (int64_t)1 << 30, "lkb_flatten: light curve too long");

  std::vector<double> h_c, h_e;
  if (!savgol_tables(window_length, polyorder, h_c, h_e)) {
    set_error("lkb_flatten: singular Savitzky-Golay system");
    return LKB_E_SINGULAR;
  }
  const int half = window_length / 2;

  const double *d_t = nullptr, *d_f = nullptr, *d_fe = nullptr;
  const uint8_t* d_ex = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, time, total, &d_t, st));
  LKB_TRY(stage_in<double>(mem, WS_IN1, flux, total, &d_f, st));
  LKB_TRY(stage_in<double>(mem, WS_IN2, flux_err, total, &d_fe, st));
  LKB_TRY(stage_in<uint8_t>(mem, WS_IN3, exclude_mask, total, &d_ex, st));
  int64_t* d_off = nullptr;
  double *d_c = nullptr, *d_e = nullptr;
  LKB_TRY(ws_get_t<int64_t>(WS_A, B + 1, &d_off));
  LKB_TRY(ws_get_t<double>(WS_B, h_c.size(), &d_c));
  LKB_TRY(ws_get_t<double>(WS_C, h_e.size(), &d_e));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_off, h_offsets, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_c, h_c.data(), sizeof(double) * h_c.size(), cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_e, h_e.data(), sizeof(double) * h_e.size(), cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaStreamSynchronize(st));   // tables are locals
  (void)half;

  double *o_flat = nullptr, *o_fe = nullptr, *o_tr = nullptr;
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0, flat, total, &o_flat));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT1, flat_err, total, &o_fe));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT2, trend, total, &o_tr));

  // ---- v2 kernel (flatten_v2.cuh: bitmask bookkeeping, sliding-moment or direct-tap Savitzky-Golay) whenever the
  // plan allows (flatten_plan.h) ----
  int64_t nmax = 0;
  for (int b = 0; b < B; ++b) nmax = std::max(nmax, h_offsets[b + 1] - h_offsets[b]);
  const FlattenPlan plan = flatten_plan(window_length, polyorder, nmax);
  g_last_flatten_path = LKB_FLATTEN_PATH_V1;
  {
    const int NM = plan.nm, tile_out = plan.tile_out;
    F2Coef cf;
    if (!getenv("LKB_FLATTEN_V1") && plan.route == FLATTEN_V2 && savgol_ginv(window_length, polyorder, cf)) {
      double* tro = nullptr;
      int* d_status = nullptr;
      LKB_TRY(ws_get_t<double>(WS_H, total, &tro));
      LKB_TRY(ws_get_t<int>(WS_N, B, &d_status));
      const size_t smem2 = ((sizeof(F2Smem) + 15) & ~(size_t)15) +
                           sizeof(double) * std::max((size_t)NM * (tile_out + 2 * half + 1), (size_t)(FS_CAP + FS_SAMPLE));
      prof_begin(st);
      const F2Args a{d_t, d_f, d_fe, d_ex, d_off, tro, window_length, break_tolerance, niters, sigma, cf, tile_out,
                     o_flat, o_fe, o_tr, d_status};
      const int rc = NM == 1 ? launch_flatten2<1, false>(a, B, smem2, st)
                     : NM == 3 ? (plan.direct ? launch_flatten2<3, true>(a, B, smem2, st) : launch_flatten2<3, false>(a, B, smem2, st))
                     : (plan.direct ? launch_flatten2<5, true>(a, B, smem2, st) : launch_flatten2<5, false>(a, B, smem2, st));
      LKB_TRY(rc);
      prof_end(st);
      LKB_LAUNCH_CHECK();
      std::vector<int> h_status(B, 0);
      LKB_CUDA_CHECK(cudaMemcpyAsync(h_status.data(), d_status, sizeof(int) * B, cudaMemcpyDeviceToHost, st));
      LKB_CUDA_CHECK(cudaStreamSynchronize(st));
      bool overflow = false;
      for (int b = 0; b < B; ++b) overflow = overflow || h_status[b] == 2;
      if (!overflow) {
        g_last_flatten_path = plan.direct ? LKB_FLATTEN_PATH_V2_DIRECT : LKB_FLATTEN_PATH_V2_MOMENTS;
        LKB_TRY(stage_out_copy<double>(mem, flat, o_flat, total, st));
        LKB_TRY(stage_out_copy<double>(mem, flat_err, o_fe, total, st));
        LKB_TRY(stage_out_copy<double>(mem, trend, o_tr, total, st));
        if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
        return LKB_OK;
      }
      // a light curve with more gap segments than the v2 kernel's shared-memory list: the whole call re-runs below
      g_last_flatten_path = LKB_FLATTEN_PATH_V1_RERUN;
    }
  }

  FlWs ws;
  LKB_TRY(ws_get_t<uint8_t>(WS_D, total, &ws.mask));
  LKB_TRY(ws_get_t<int32_t>(WS_E, total, &ws.cidx));
  LKB_TRY(ws_get_t<double>(WS_F, total, &ws.fc));
  LKB_TRY(ws_get_t<double>(WS_G, total, &ws.tc));
  LKB_TRY(ws_get_t<double>(WS_H, total, &ws.trc));
  LKB_TRY(ws_get_t<uint8_t>(WS_I, total, &ws.mask1));
  LKB_TRY(ws_get_t<int32_t>(WS_J, total, &ws.sidx));
  LKB_TRY(ws_get_t<int32_t>(WS_K, total + B, &ws.cuts));
  LKB_TRY(ws_get_t<double>(WS_L, total, &ws.xs));
  LKB_TRY(ws_get_t<double>(WS_M, total, &ws.ys));

  const size_t smem = sizeof(double) * (((window_length + 3) & ~3) + (size_t)(FL_TI + window_length) * 17 / 16 + 8);
  static size_t attr_smem = 0;
  if (smem > attr_smem) {
    LKB_CUDA_CHECK(cudaFuncSetAttribute(flatten_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_smem = smem;
  }
  prof_begin(st);
  flatten_kernel<<<B, FL_THREADS, smem, st>>>(d_t, d_f, d_fe, d_ex, d_off, ws, window_length, polyorder,
                                            break_tolerance, niters, sigma, d_c, d_e, o_flat, o_fe, o_tr);
  prof_end(st);
  LKB_LAUNCH_CHECK();
  LKB_TRY(stage_out_copy<double>(mem, flat, o_flat, total, st));
  LKB_TRY(stage_out_copy<double>(mem, flat_err, o_fe, total, st));
  LKB_TRY(stage_out_copy<double>(mem, trend, o_tr, total, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

}  // namespace lkb
