// K8: elastic-net coordinate descent, CBVCorrector.correct_elasticnet
//   /root/reference/src/lightkurve/correctors/cbvcorrector.py:358-379
//   sklearn.linear_model.ElasticNet(alpha, l1_ratio, fit_intercept=False).fit(X[mask], y[mask])
// scikit-learn minimises 1/2 ||y - X w||^2 + l1 ||w||_1 + l2/2 ||w||^2 (l1 = alpha l1_ratio n, l2 = alpha (1 - l1_ratio)
// n, n = cadences used) by cyclic coordinate descent and stops when the duality gap is <= tol y.y.  For flux in e-/s that
// stop comes long before the minimiser, so the answer is the iteration's: this kernel reproduces it sweep for sweep
// (oracle/enet.py restates scikit-learn's loop on X; tests/test_enet_emulated.py pins this kernel to it).
//
// Everything the iteration needs is in the Gram matrix of [X | y] over the used cadences, which the K5 first pass
// (rg_rows + the fp64 Gram kernel, regress.cu) builds: G = X^T X, c = X^T y, y.y.  The kernel keeps
//   q = X^T R = c - G w                   (R = y - X w, never formed)
// so a coordinate update is  tmp = q_j + G_jj w_j,  w_j <- soft-threshold,  q -= G[:, j] (w_j_new - w_j_old)  (O(K)),
// and the gap terms are  ||R||^2 = y.y - c.w - w.q,  R.y = y.y - c.w,  X^T R = q.
// Update order, the stopping tests, the three gap forms (A: l1 > 0; B: l1 = 0 < l2; ||X^T R||^2: alpha = 0),
// gap-safe screening (l1 > 0), skipped zero columns and `positive` follow _cd_fast.pyx enet_coordinate_descent.
//
// enet_cd_kernel: one warp per light curve, ENET warps per CTA (fewer when K is large).  The warp's symmetric G
// [K x K] and its vectors live in shared memory (K = 165: 220 KB, one light curve per CTA).  Every lane computes the
// same scalar decisions from the same shared values, so no vote is needed; lane i keeps q[i], q[i + 32], ... up to
// date.  fp64 only, explicit fma() wherever a product is accumulated (the CPU emulator then rounds like the GPU),
// fixed reduction trees, no atomics: results are bitwise reproducible and independent of the rest of the batch.
// No inline PTX: tests/native/cuda_emu.h runs this file on the CPU.
#pragma once
#include "common.cuh"

namespace lkb {

constexpr int ENET_KMAX = 165;                 // = RG_KMAX (the Gram pass's limit)
constexpr int ENET_MAX_WARPS = 8;
constexpr size_t ENET_SMEM_MAX = 227 * 1024;   // opt-in dynamic shared memory per CTA on sm_90

// shared-memory doubles per light curve: G [K*K], q, w, c, diag, xta [K each], active + excluded (2K ints = K doubles)
__host__ __device__ inline size_t enet_slot_doubles(int K) { return (size_t)K * K + 6 * (size_t)K; }

struct EnetGap {
  double gap, dual_norm;
};

// Duality gap of the current (w, q); fills xta = X^T R - l2 w (formulation A) for the screening.  Warp-collective.
__device__ __forceinline__ EnetGap enet_gap(int K, const double* w, const double* q, const double* c, double* xta, double yy,
                                   double l1, double l2, bool positive) {
  const int lane = threadIdx.x & 31;
  double ww = 0.0, cw = 0.0, wq = 0.0, wl1 = 0.0, qq = 0.0;
  double dn = positive ? -__longlong_as_double(0x7ff0000000000000ll) : 0.0;
  for (int i = lane; i < K; i += 32) {
    const double wi = w[i], qi = q[i];
    ww = fma(wi, wi, ww);
    cw = fma(c[i], wi, cw);
    wq = fma(wi, qi, wq);
    wl1 += fabs(wi);
    qq = fma(qi, qi, qq);
    const double x = fma(-l2, wi, qi);
    xta[i] = x;
    dn = positive ? fmax(dn, x) : fmax(dn, fabs(x));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ww += __shfl_xor_sync(0xffffffffu, ww, o);
    cw += __shfl_xor_sync(0xffffffffu, cw, o);
    wq += __shfl_xor_sync(0xffffffffu, wq, o);
    wl1 += __shfl_xor_sync(0xffffffffu, wl1, o);
    qq += __shfl_xor_sync(0xffffffffu, qq, o);
    dn = fmax(dn, __shfl_xor_sync(0xffffffffu, dn, o));
  }
  const double w_l2 = l2 > 0 ? ww : 0.0;
  const double R2 = yy - cw - wq;
  const double Ry = yy - cw;
  EnetGap g;
  if (l1 == 0) {                                       // X^T R = q
    g.dual_norm = qq;
    if (l2 == 0) { g.gap = qq; return g; }             // alpha = 0: first-order condition ||X^T R||^2
    double gap = R2 + 0.5 * l2 * w_l2 - Ry;            // formulation B
    gap += 1 / (2 * l2) * qq;
    g.gap = gap;
    return g;
  }
  const double primal = 0.5 * (R2 + l2 * w_l2) + l1 * wl1;                       // formulation A
  const double scale = dn > l1 ? l1 / dn : 1.0;
  const double dual = -0.5 * (scale * scale) * (R2 + l2 * w_l2) + scale * Ry;
  g.gap = primal - dual;
  g.dual_norm = dn;
  return g;
}

// q_i += G[j, i] * a for all i (warp-collective, then the warp is synchronised)
__device__ __forceinline__ void enet_q_axpy(int K, const double* Gj, double a, double* q) {
  for (int i = threadIdx.x & 31; i < K; i += 32) q[i] = fma(Gj[i], a, q[i]);
  __syncwarp();
}

// Gap-safe screening (arXiv:1802.07481 eq. 11) over the columns not yet excluded, in column order; an excluded
// column's coefficient goes back to zero.  Returns the new number of active columns.
__device__ __forceinline__ int enet_screen(int K, const double* G, const double* d, double* w, double* q, const double* xta,
                                  int* active, int* excluded, EnetGap g, double l1, double l2, bool first) {
  const int lane = threadIdx.x & 31;
  const double thr = sqrt(2 * g.gap) / l1;
  const double den = fmax(l1, g.dual_norm);
  int na = 0;
  for (int j = 0; j < K; ++j) {
    if (first && d[j] == 0) {
      if (lane == 0) { w[j] = 0.0; excluded[j] = 1; }
      continue;
    }
    if (!first && excluded[j]) continue;
    const double dj = (1 - fabs(xta[j] / den)) / sqrt(d[j] + l2);
    if (dj <= thr) {
      if (lane == 0) { active[na] = j; excluded[j] = 0; }
      ++na;
    } else {
      const double wj = w[j];
      __syncwarp();
      if (wj != 0) enet_q_axpy(K, G + (size_t)j * K, wj, q);     // R += w_j X_j
      if (lane == 0) { w[j] = 0.0; excluded[j] = 1; }
    }
  }
  __syncwarp();
  return na;
}

// gram: [B, K+1, K+1], upper triangle (i <= j) of [X | y]^T [X | y]; cnt: cadences used per light curve.
__global__ void __launch_bounds__(32 * ENET_MAX_WARPS, 2)
enet_cd_kernel(const double* __restrict__ gram, const int32_t* __restrict__ cnt, int B, int K, double alpha,
               double l1_ratio, int max_iter, double tol, int positive, double* __restrict__ coeff,
               int32_t* __restrict__ n_iter_out, double* __restrict__ dual_gap_out, uint8_t* __restrict__ converged_out) {
  LKB_DYN_SMEM(double, smem);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.x * (blockDim.x >> 5) + warp;
  if (b >= B) return;                                  // whole warps only: the kernel has no CTA-wide barrier
  const int Ka = K + 1;
  double* G = smem + (size_t)warp * enet_slot_doubles(K);
  double* q = G + (size_t)K * K;
  double* w = q + K;
  double* c = w + K;
  double* d = c + K;
  double* xta = d + K;
  int* active = reinterpret_cast<int*>(xta + K);
  int* excluded = active + K;
  const double* g = gram + (size_t)b * Ka * Ka;
  for (int e = lane; e < K * K; e += 32) {
    const int i = e / K, j = e - i * K;
    G[e] = j >= i ? g[(size_t)i * Ka + j] : g[(size_t)j * Ka + i];
  }
  for (int i = lane; i < K; i += 32) {
    c[i] = g[(size_t)i * Ka + K];
    q[i] = c[i];
    w[i] = 0.0;
    d[i] = g[(size_t)i * Ka + i];
    active[i] = i;
    excluded[i] = 0;
  }
  const double yy = g[(size_t)K * Ka + K];
  __syncwarp();

  const double n = (double)cnt[b];
  const double l1 = alpha * l1_ratio * n, l2 = alpha * (1.0 - l1_ratio) * n;
  const double tol_s = tol * yy;
  const bool pos = positive != 0, screening = l1 != 0;
  EnetGap gp = enet_gap(K, w, q, c, xta, yy, l1, l2, pos);
  __syncwarp();
  int it = 0;
  bool conv = gp.gap <= tol_s;
  if (!conv) {
    int na = K;
    if (screening) na = enet_screen(K, G, d, w, q, xta, active, excluded, gp, l1, l2, true);
    for (it = 0; it < max_iter; ++it) {
      double w_max = 0.0, d_w_max = 0.0;
      for (int f = 0; f < na; ++f) {
        const int j = active[f];
        const double dj = d[j];
        if (dj == 0.0) continue;
        const double wj = w[j];
        const double tmp = fma(wj, dj, q[j]);
        double wn;
        if (pos && tmp < 0) {
          wn = 0.0;
        } else {
          const double sg = tmp == 0 ? 0.0 : (tmp > 0 ? 1.0 : -1.0);
          wn = sg * fmax(fabs(tmp) - l1, 0.0) / (dj + l2);
        }
        if (wn != wj) {
          __syncwarp();                                // every lane has read w[j] and q[j]
          if (lane == 0) w[j] = wn;
          enet_q_axpy(K, G + (size_t)j * K, wj - wn, q);
        }
        d_w_max = fmax(d_w_max, fabs(wn - wj));
        w_max = fmax(w_max, fabs(wn));
      }
      if (w_max == 0.0 || d_w_max / w_max <= tol || it == max_iter - 1) {
        gp = enet_gap(K, w, q, c, xta, yy, l1, l2, pos);
        __syncwarp();
        if (gp.gap <= tol_s) { conv = true; break; }
        if (screening) na = enet_screen(K, G, d, w, q, xta, active, excluded, gp, l1, l2, false);
      }
    }
    if (it == max_iter) it = max_iter - 1;             // the loop ran out: scikit-learn reports max_iter
    ++it;
  }
  for (int i = lane; i < K; i += 32) coeff[(size_t)b * K + i] = w[i];
  if (lane == 0) {
    n_iter_out[b] = it;
    dual_gap_out[b] = gp.gap / n;
    converged_out[b] = conv ? 1 : 0;
  }
}

// Light curves per CTA for K features: as many as fit in shared memory, up to ENET_MAX_WARPS.
inline int enet_warps_per_cta(int K) {
  const size_t per = enet_slot_doubles(K) * sizeof(double);
  int p = (int)(ENET_SMEM_MAX / per);
  return p < 1 ? 1 : (p > ENET_MAX_WARPS ? ENET_MAX_WARPS : p);
}

// Launches enet_cd_kernel on device buffers (gram and cnt as the K5 first pass leaves them).
inline int enet_cd_launch(const double* gram, const int32_t* cnt, int B, int K, double alpha, double l1_ratio,
                          int max_iter, double tol, int positive, double* coeff, int32_t* n_iter, double* dual_gap,
                          uint8_t* converged, cudaStream_t st) {
  const int p = enet_warps_per_cta(K);
  const size_t smem = (size_t)p * enet_slot_doubles(K) * sizeof(double);
  if (smem > ENET_SMEM_MAX) {
    set_error("lkb_elasticnet: K=%d needs %zu bytes of shared memory", K, smem);
    return LKB_E_UNSUPPORTED;
  }
  static size_t attr = 0;
  if (smem > attr) {
    LKB_CUDA_CHECK(cudaFuncSetAttribute(enet_cd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = smem;
  }
  LKB_LAUNCH_SMEM((unsigned)((B + p - 1) / p), 32 * p, smem, st, enet_cd_kernel)(
      gram, cnt, B, K, alpha, l1_ratio, max_iter, tol, positive, coeff, n_iter, dual_gap, converged);
  LKB_LAUNCH_CHECK();
  return LKB_OK;
}

}  // namespace lkb
