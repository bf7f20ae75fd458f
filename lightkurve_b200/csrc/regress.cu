// K5: RegressionCorrector numerics, /root/reference/src/lightkurve/correctors/regressioncorrector.py
//   _fit_coefficients :127-189 (dense branch): A = X^T diag(1/s^2) X + diag(1/prior_sigma^2),
//                                            rhs = X^T (y/s^2) + prior_mu/prior_sigma^2, np.linalg.solve
//   correct() loop     :244-279: niters x { fit on cadence_mask & ~outlier_mask; residuals with the
//                                masked cadences set to NaN; outlier_mask |= sigma_clip(residuals).mask }
//                                then model = X w - median(X w).
// fp64 throughout (the reference is fp64; 7-decimal known answers in
// tests/correctors/test_regressioncorrector.py:13-83).
//
// Kernels:  rg_rows     build the list of cadences entering (iteration 0) or LEAVING (later
//                       iterations: the outlier mask only grows, so A and rhs are DOWNDATED by the
//                       newly clipped rows instead of being rebuilt - N*K^2 work once, not niters times)
//           rg_accum    weighted Gram blocks (64x64 tiles of [X | y]^T W [X | y], upper triangle)
//           rg_solve    add the Gaussian priors, LU with partial pivoting in shared memory (gesv-like)
//           rg_clip     model = X w, residuals, astropy sigma_clip (median / std, <= 5 rounds)
//           rg_final    model - median(model)
//
// K8 (lkb_elasticnet, enet.cuh) reuses rg_rows + the fp64 Gram pass and rg_final: see elasticnet() below.
#include "common.cuh"
#include "enet.cuh"
#include "regress_clip.cuh"
#include "select.cuh"

namespace lkb {

constexpr int RG_BLK = 64;      // Gram tile edge
constexpr int RG_RC = 32;       // cadences per shared-memory chunk
constexpr int RG_KMAX = 165;    // (K+1)^2 doubles must fit in shared memory for the LU

// ---- row lists -------------------------------------------------------------------------------
// first = 1: rows = cadence_mask (& ~outlier, which is empty), used := that.
// first = 0: rows = used & outlier (newly clipped), used := used & ~outlier.
__global__ void __launch_bounds__(256)
rg_rows_kernel(const uint8_t* __restrict__ cadence_mask, const uint8_t* __restrict__ outlier,
               const double* __restrict__ flux_err, int64_t N, int first, RgWs ws) {
  __shared__ int s_wc[8];
  __shared__ int s_base;
  const int b = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint8_t* cm = cadence_mask ? cadence_mask + (int64_t)b * N : nullptr;
  const uint8_t* om = outlier + (int64_t)b * N;
  uint8_t* used = ws.used + (int64_t)b * N;
  int32_t* rows = ws.rows + (int64_t)b * N;
  if (threadIdx.x == 0) s_base = 0;
  __syncthreads();
  for (int64_t c0 = 0; c0 < N; c0 += blockDim.x) {
    const int64_t i = c0 + threadIdx.x;
    bool p = false;
    if (i < N) {
      if (first) {
        p = (cm ? cm[i] != 0 : true) && om[i] == 0;
        used[i] = p ? 1 : 0;
      } else {
        p = used[i] != 0 && om[i] != 0;
        if (p) used[i] = 0;
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, p);
    if (lane == 0) s_wc[warp] = __popc(bal);
    __syncthreads();
    int off = s_base;
    for (int w = 0; w < warp; ++w) off += s_wc[w];
    if (p) {
      const int pos = off + __popc(bal & ((1u << lane) - 1u));
      rows[pos] = (int32_t)i;
      double f = 1.0;
      if (flux_err) f = flux_err[(int64_t)b * N + i];
      ws.wl[(int64_t)b * N + pos] = 1.0 / (f * f);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int w = 0; w < 8; ++w) tot += s_wc[w];
      s_base += tot;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) ws.cnt[b] = s_base;
}

// ---- weighted Gram accumulation -----------------------------------------------------------------
// grid = (n_upper_blocks, B); 128 threads = 8 (i) x 16 (j); thread tile 8 x 4.
// Gathered cadence rows are streamed with cp.async into a double-buffered shared-memory stage
// (chunk c+1 lands while chunk c is multiplied), then weighted in place.
__device__ __forceinline__ void rg_cp8(void* dst_smem, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((uint32_t)__cvta_generic_to_shared(dst_smem)), "l"(src)
               : "memory");
}
struct RgStage {
  double a[RG_RC][RG_BLK];   // [X|y][:, bi block]  (scaled by w after landing)
  double b[RG_RC][RG_BLK];   // [X|y][:, bj block]
  double fe[RG_RC];          // flux_err of the chunk's cadences
  double yv[RG_RC];          // flux of the chunk's cadences (column K)
};

__global__ void __launch_bounds__(128)
rg_accum_kernel(const double* __restrict__ X, int x_batched, const double* __restrict__ y,
                const double* __restrict__ flux_err, int64_t N, int K, int nblk, double sign, RgWs ws) {
  extern __shared__ __align__(16) unsigned char rg_smem[];
  RgStage* st = reinterpret_cast<RgStage*>(rg_smem);
  const int b = blockIdx.y;
  // decode upper-triangular block index
  int bi = 0, rem = blockIdx.x;
  while (rem >= nblk - bi) { rem -= nblk - bi; ++bi; }
  const int bj = bi + rem;
  const bool diag = (bi == bj);
  const int Ka = K + 1;
  const int cnt = ws.cnt[b];
  if (cnt == 0) return;
  const int32_t* rows = ws.rows + (int64_t)b * N;
  const double* yb = y + (int64_t)b * N;
  const double* fe = flux_err ? flux_err + (int64_t)b * N : nullptr;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  double acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;

  auto issue = [&](int c0, int buf) {
    const int nr = min(RG_RC, cnt - c0);
    RgStage& s = st[buf];
    for (int e = threadIdx.x; e < RG_RC * RG_BLK; e += blockDim.x) {
      const int r = e / RG_BLK, c = e % RG_BLK;
      if (r < nr) {
        const int64_t row = rows[c0 + r];
        const double* xr = rg_xrow(X, x_batched, b, N, K, row);
        const int cb = bj * RG_BLK + c;
        if (cb < K) rg_cp8(&s.b[r][c], xr + cb);
        if (!diag) {
          const int ca = bi * RG_BLK + c;
          if (ca < K) rg_cp8(&s.a[r][c], xr + ca);
        }
      }
    }
    if (threadIdx.x < nr) {
      const int64_t row = rows[c0 + threadIdx.x];
      rg_cp8(&s.yv[threadIdx.x], yb + row);
      if (fe) rg_cp8(&s.fe[threadIdx.x], fe + row);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  issue(0, 0);
  int buf = 0;
  for (int c0 = 0; c0 < cnt; c0 += RG_RC, buf ^= 1) {
    const int nr = min(RG_RC, cnt - c0);
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();                     // chunk c0 landed; everybody is done computing on buf^1
    if (c0 + RG_RC < cnt) issue(c0 + RG_RC, buf ^ 1);
    RgStage& s = st[buf];
    // fix-ups (column K = y, zero padding) and the 1/flux_err^2 weighting of the bi tile
    for (int e = threadIdx.x; e < RG_RC * RG_BLK; e += blockDim.x) {
      const int r = e / RG_BLK, c = e % RG_BLK;
      const int cb = bj * RG_BLK + c, ca = bi * RG_BLK + c;
      double vb = 0.0, va = 0.0;
      if (r < nr) {
        const double yy = s.yv[r];
        vb = (cb < K) ? s.b[r][c] : (cb == K ? yy : 0.0);
        va = diag ? vb : ((ca < K) ? s.a[r][c] : (ca == K ? yy : 0.0));
        const double f = fe ? s.fe[r] : 1.0;
        va *= 1.0 / (f * f);
      }
      s.b[r][c] = vb;
      s.a[r][c] = va;
    }
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < RG_RC; ++k) {
      double a[8], bb[4];
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = s.a[k][ty + 8 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) bb[j] = s.b[k][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], bb[j], acc[i][j]);
    }
  }
  double* G = ws.gram + (int64_t)b * Ka * Ka;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int gi = bi * RG_BLK + ty + 8 * i;
    if (gi >= Ka) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gj = bj * RG_BLK + tx + 16 * j;
      if (gj >= Ka) continue;
      G[(int64_t)gi * Ka + gj] += sign * acc[i][j];     // this CTA owns the block: no atomics
    }
  }
}

// ---- weighted Gram accumulation on the FP64 tensor cores -------------------------------------------
// One CTA per light curve; warp w owns the (8 TB)^2 block (bi, bj >= bi) of [X | y]^T W [X | y], i.e. a TB x TB
// grid of m8n8k4 DMMA tiles whose 2 TB operand fragments per k-step are re-used across the TB^2 tiles
// (TB = 4: 15 warps for K = 151, an even 4/4/4/3 split over the four SM sub-partitions).
// Gathered cadence rows land by cp.async in a double-buffered [32 x 164] stage (row stride = 4 mod 16
// doubles: the 16 lanes of a half-warp fragment load hit 16 different bank pairs).
constexpr int RGM_RC = 32;              // cadences per stage (8 k-steps)
constexpr int RGM_LD = 180;             // stage row stride in doubles (>= 8 * 21 tiles, = 4 mod 16)
struct RgmStage {
  double x[RGM_RC][RGM_LD];
  double w[RGM_RC];
};

__device__ __forceinline__ void rg_dmma(double& d0, double& d1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
}

template <int NB5, int TB>
__global__ void __launch_bounds__(32 * NB5 * (NB5 + 1) / 2)
rg_gram_mma_kernel(const double* __restrict__ X, int x_batched, const double* __restrict__ y,
                   int64_t N, int K, double sign, RgWs ws) {
  constexpr int nb5 = NB5;
  extern __shared__ __align__(16) unsigned char rg_smem[];
  RgmStage* st = reinterpret_cast<RgmStage*>(rg_smem);
  const int b = blockIdx.x;
  const int Ka = K + 1;
  // gridDim.y CTAs share a light curve's cadence list (whole stages each); with 2 of them and a zeroed
  // Gram matrix the two atomic adds commute exactly, so the result does not depend on their order
  const int cnt_all = ws.cnt[b];
  const int stages = (cnt_all + RGM_RC - 1) / RGM_RC;
  const int s_lo = (int)((int64_t)stages * blockIdx.y / gridDim.y), s_hi = (int)((int64_t)stages * (blockIdx.y + 1) / gridDim.y);
  const int r_lo = s_lo * RGM_RC;
  const int cnt = min(cnt_all, s_hi * RGM_RC) - r_lo;
  if (cnt <= 0) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // decode this warp's upper-triangular block
  int bi = 0, rem = warp;
  while (rem >= nb5 - bi) { rem -= nb5 - bi; ++bi; }
  const int bj = bi + rem;
  const int32_t* rows = ws.rows + (int64_t)b * N + r_lo;
  const double* wl = ws.wl + (int64_t)b * N + r_lo;
  const double* yb = y + (int64_t)b * N;

  // zero the padding columns once (cp.async only ever writes columns < Ka)
  for (int e = threadIdx.x; e < 2 * RGM_RC * (RGM_LD - Ka); e += blockDim.x) {
    const int s = e / (RGM_RC * (RGM_LD - Ka)), r2 = e % (RGM_RC * (RGM_LD - Ka));
    st[s].x[r2 / (RGM_LD - Ka)][Ka + r2 % (RGM_LD - Ka)] = 0.0;
  }
  auto issue = [&](int c0, int buf) {
    RgmStage& s = st[buf];
    const int nr = min(RGM_RC, cnt - c0);
    for (int e = threadIdx.x; e < RGM_RC * Ka; e += blockDim.x) {
      const int r = e / Ka, c = e - r * Ka;
      const int64_t row = rows[c0 + min(r, nr - 1)];           // tail rows repeat a valid row with weight 0
      const double* src = (c < K) ? rg_xrow(X, x_batched, b, N, K, row) + c : yb + row;
      rg_cp8(&s.x[r][c], src);
    }
    if (threadIdx.x < RGM_RC) {
      const int r = threadIdx.x;
      if (r < nr) rg_cp8(&s.w[r], wl + c0 + r);
      else s.w[r] = 0.0;
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  double acc[TB][TB][2];
#pragma unroll
  for (int i = 0; i < TB; ++i)
#pragma unroll
    for (int j = 0; j < TB; ++j) { acc[i][j][0] = 0.0; acc[i][j][1] = 0.0; }

  issue(0, 0);
  int buf = 0;
  const int kr = lane & 3, kc = lane >> 2;
  for (int c0 = 0; c0 < cnt; c0 += RGM_RC, buf ^= 1) {
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();                     // chunk c0 landed; everybody is done computing on buf^1
    if (c0 + RGM_RC < cnt) issue(c0 + RGM_RC, buf ^ 1);
    RgmStage& s = st[buf];
#pragma unroll 2
    for (int ks = 0; ks < RGM_RC / 4; ++ks) {
      const double* xr = &s.x[ks * 4 + kr][kc];
      const double w = s.w[ks * 4 + kr];
      double a[TB], bb[TB];
#pragma unroll
      for (int i = 0; i < TB; ++i) a[i] = w * xr[min((bi * TB + i) * 8, RGM_LD - 8)];   // (tiles past Ka: discarded)
#pragma unroll
      for (int j = 0; j < TB; ++j) bb[j] = xr[min((bj * TB + j) * 8, RGM_LD - 8)];
#pragma unroll
      for (int i = 0; i < TB; ++i)
#pragma unroll
        for (int j = 0; j < TB; ++j) rg_dmma(acc[i][j][0], acc[i][j][1], a[i], bb[j]);
    }
  }
  double* G = ws.gram + (int64_t)b * Ka * Ka;
#pragma unroll
  for (int i = 0; i < TB; ++i) {
    const int gi = (bi * TB + i) * 8 + (lane >> 2);
    if (gi >= Ka) continue;
#pragma unroll
    for (int j = 0; j < TB; ++j) {
      const int gj = (bj * TB + j) * 8 + 2 * (lane & 3);
      if (gridDim.y == 1) {                   // this warp owns the block
        if (gj < Ka) G[(int64_t)gi * Ka + gj] += sign * acc[i][j][0];
        if (gj + 1 < Ka) G[(int64_t)gi * Ka + gj + 1] += sign * acc[i][j][1];
      } else {
        if (gj < Ka) atomicAdd(&G[(int64_t)gi * Ka + gj], sign * acc[i][j][0]);
        if (gj + 1 < Ka) atomicAdd(&G[(int64_t)gi * Ka + gj + 1], sign * acc[i][j][1]);
      }
    }
  }
}

// ---- solve ------------------------------------------------------------------------------------------
// grad != NULL: iterative-refinement step - solve (A + prior) d = grad - prior (w - mu) for the current w = coeff and
// write w + d (the matrix may be approximate, e.g. the tcgen05 Gram; grad is the exact fp64 gradient of the fit)
__global__ void __launch_bounds__(256)
rg_solve_kernel(int K, const double* __restrict__ prior_mu, const double* __restrict__ prior_sigma, int64_t pstride,
                RgWs ws, double* __restrict__ coeff, int32_t* __restrict__ status, const double* __restrict__ grad,
                double* __restrict__ lu_out, int32_t* __restrict__ piv_out) {
  extern __shared__ __align__(16) double s_m[];        // [K][K+1] augmented
  __shared__ double s_red[8];
  __shared__ int s_redi[8];
  __shared__ int s_piv;
  const int b = blockIdx.x;
  const int Ka = K + 1;
  const double* G = ws.gram + (int64_t)b * Ka * Ka;
  if (prior_sigma) { prior_mu += pstride * b; prior_sigma += pstride * b; }   // pstride: 0 (shared [K]) or K ([B, K])
  // symmetric fill from the upper triangle (only blocks bi <= bj were accumulated, but inside a
  // diagonal block both triangles are present; use i <= j entries everywhere for exact symmetry)
  for (int e = threadIdx.x; e < K * Ka; e += blockDim.x) {
    const int i = e / Ka, j = e % Ka;
    double v = (j >= i) ? G[(int64_t)i * Ka + j] : G[(int64_t)j * Ka + i];
    if (grad && j == K) v = grad[(int64_t)b * K + i];
    if (prior_sigma) {
      const double ps = prior_sigma[i];
      if (j == i) v += 1.0 / (ps * ps);
      if (j == K) v += (grad ? (prior_mu[i] - coeff[(int64_t)b * K + i]) : prior_mu[i]) / (ps * ps);
    }
    s_m[e] = v;
  }
  __syncthreads();
  bool singular = false;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int c = 0; c < K; ++c) {
    // partial pivoting: first row with the largest |value| in column c
    double best = -1.0;
    int bi = c;
    for (int r = c + threadIdx.x; r < K; r += blockDim.x) {
      const double v = fabs(s_m[r * Ka + c]);
      if (v > best) { best = v; bi = r; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (lane == 0) { s_red[warp] = best; s_redi[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      double bb = s_red[0];
      int ii = s_redi[0];
      for (int w = 1; w < nw; ++w)
        if (s_red[w] > bb || (s_red[w] == bb && s_redi[w] < ii)) { bb = s_red[w]; ii = s_redi[w]; }
      s_piv = (bb > 0.0) ? ii : -1;      // exact zero (or NaN) pivot => singular, like LAPACK gesv info > 0
    }
    __syncthreads();
    const int piv = s_piv;
    if (piv < 0) { singular = true; break; }
    if (piv_out && threadIdx.x == 0) piv_out[(int64_t)b * K + c] = piv;
    if (piv != c) {
      for (int k = threadIdx.x; k < Ka; k += blockDim.x) {
        const double tmp = s_m[c * Ka + k];
        s_m[c * Ka + k] = s_m[piv * Ka + k];
        s_m[piv * Ka + k] = tmp;
      }
    }
    __syncthreads();
    const double pv = s_m[c * Ka + c];
    // two rows per warp and trip: their update chains (LDS, FMA, STS) are independent and interleave
    for (int r = c + 1 + 2 * warp; r < K; r += 2 * nw) {
      const bool two = r + 1 < K;
      const double f0 = s_m[r * Ka + c] / pv, f1 = two ? s_m[(r + 1) * Ka + c] / pv : 0.0;
      __syncwarp();
      for (int k = c + 1 + lane; k < Ka; k += 32) {
        const double p = s_m[c * Ka + k];
        const double a0 = s_m[r * Ka + k], a1 = two ? s_m[(r + 1) * Ka + k] : 0.0;
        s_m[r * Ka + k] = fma(-f0, p, a0);
        if (two) s_m[(r + 1) * Ka + k] = fma(-f1, p, a1);
      }
      __syncwarp();
      if (lane == 0) {                               // the multipliers stay in place: s_m = [L \\ U | rhs]
        s_m[r * Ka + c] = f0;
        if (two) s_m[(r + 1) * Ka + c] = f1;
      }
    }
    __syncthreads();
  }
  if (singular) {
    for (int k = threadIdx.x; k < K; k += blockDim.x) coeff[(int64_t)b * K + k] = __longlong_as_double(0x7ff8000000000000ll);
    if (threadIdx.x == 0 && status) status[b] = LKB_E_SINGULAR;
    return;
  }
  if (lu_out)                                          // factors for rg_resolve_kernel (same matrix, another rhs)
    for (int e = threadIdx.x; e < K * K; e += blockDim.x) lu_out[(int64_t)b * K * K + e] = s_m[(e / K) * Ka + (e % K)];
  // back substitution (warp 0)
  if (warp == 0) {
    for (int c = K - 1; c >= 0; --c) {
      double part = 0.0;
      for (int k = c + 1 + lane; k < K; k += 32) part = fma(s_m[c * Ka + k], s_m[k * Ka + K], part);
      part = warp_sum(part);
      if (lane == 0) s_m[c * Ka + K] = (s_m[c * Ka + K] - part) / s_m[c * Ka + c];
      __syncwarp();
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += blockDim.x)
    coeff[(int64_t)b * K + k] = grad ? coeff[(int64_t)b * K + k] + s_m[k * Ka + K] : s_m[k * Ka + K];
  if (threadIdx.x == 0 && status) status[b] = LKB_OK;
}

// Iterative-refinement step with the factors rg_solve_kernel left behind (P (A + prior) = L U, pivots piv):
// d = (A + prior)^-1 [grad - prior (w - mu)], w <- w + d.  Two triangular solves instead of a second elimination
// (the elimination is ~150 dependent block steps per light curve; the substitutions are one warp's dot products).
__global__ void __launch_bounds__(256)
rg_resolve_kernel(int K, const double* __restrict__ prior_mu, const double* __restrict__ prior_sigma, int64_t pstride,
                  const double* __restrict__ lu, const int32_t* __restrict__ piv, double* __restrict__ coeff,
                  const int32_t* __restrict__ status, const double* __restrict__ grad) {
  extern __shared__ __align__(16) double s_m[];        // [K][K] factors, then the right-hand side [K]
  const int b = blockIdx.x;
  if (status && status[b] != LKB_OK) return;           // singular system: the coefficients are already NaN
  if (prior_sigma) { prior_mu += pstride * b; prior_sigma += pstride * b; }
  double* s_r = s_m + (size_t)K * K;
  const double* LU = lu + (int64_t)b * K * K;
  for (int e = threadIdx.x; e < K * K; e += blockDim.x) s_m[e] = LU[e];
  for (int i = threadIdx.x; i < K; i += blockDim.x) {
    double v = grad[(int64_t)b * K + i];
    if (prior_sigma) {
      const double ps = prior_sigma[i];
      v += (prior_mu[i] - coeff[(int64_t)b * K + i]) / (ps * ps);
    }
    s_r[i] = v;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    if (lane == 0) {                                   // the row interchanges, in elimination order
      const int32_t* pv = piv + (int64_t)b * K;
      for (int c = 0; c < K; ++c) {
        const int p = pv[c];
        if (p != c) { const double tmp = s_r[c]; s_r[c] = s_r[p]; s_r[p] = tmp; }
      }
    }
    __syncwarp();
    for (int c = 1; c < K; ++c) {                      // L y = P rhs (unit diagonal)
      double part = 0.0;
      for (int k = lane; k < c; k += 32) part = fma(s_m[c * K + k], s_r[k], part);
      part = warp_sum(part);
      if (lane == 0) s_r[c] -= part;
      __syncwarp();
    }
    for (int c = K - 1; c >= 0; --c) {                 // U d = y
      double part = 0.0;
      for (int k = c + 1 + lane; k < K; k += 32) part = fma(s_m[c * K + k], s_r[k], part);
      part = warp_sum(part);
      if (lane == 0) s_r[c] = (s_r[c] - part) / s_m[c * K + c];
      __syncwarp();
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += blockDim.x) coeff[(int64_t)b * K + k] += s_r[k];
}

// ---- (A + prior)^-1 for propagate_errors (np.linalg.inv at regressioncorrector.py:185) -----------
// Gauss-Jordan with partial pivoting on [M | I] held in an L2-resident global workspace [K][2K].
__global__ void __launch_bounds__(256)
rg_inverse_kernel(int K, const double* __restrict__ prior_sigma, int64_t pstride, RgWs ws, double* __restrict__ work,
                  double* __restrict__ cov, const int32_t* __restrict__ status) {
  __shared__ double s_red[8];
  __shared__ int s_redi[8];
  __shared__ int s_piv;
  const int b = blockIdx.x;
  const int Ka = K + 1, W = 2 * K;
  double* out = cov + (int64_t)b * K * K;
  const double qnan = __longlong_as_double(0x7ff8000000000000ll);
  if (status && status[b] != LKB_OK) {
    for (int e = threadIdx.x; e < K * K; e += blockDim.x) out[e] = qnan;
    return;
  }
  const double* G = ws.gram + (int64_t)b * Ka * Ka;
  if (prior_sigma) prior_sigma += pstride * b;
  double* M = work + (int64_t)b * K * W;
  for (int e = threadIdx.x; e < K * W; e += blockDim.x) {
    const int i = e / W, j = e % W;
    double v;
    if (j < K) {
      v = (j >= i) ? G[(int64_t)i * Ka + j] : G[(int64_t)j * Ka + i];
      if (prior_sigma && j == i) { const double ps = prior_sigma[i]; v += 1.0 / (ps * ps); }
    } else {
      v = (j - K == i) ? 1.0 : 0.0;
    }
    M[e] = v;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  bool singular = false;
  for (int c = 0; c < K; ++c) {
    double best = -1.0;
    int bi = c;
    for (int r = c + threadIdx.x; r < K; r += blockDim.x) {
      const double v = fabs(M[(int64_t)r * W + c]);
      if (v > best) { best = v; bi = r; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    if (lane == 0) { s_red[warp] = best; s_redi[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      double bb = s_red[0];
      int ii = s_redi[0];
      for (int w = 1; w < nw; ++w)
        if (s_red[w] > bb || (s_red[w] == bb && s_redi[w] < ii)) { bb = s_red[w]; ii = s_redi[w]; }
      s_piv = (bb > 0.0) ? ii : -1;
    }
    __syncthreads();
    const int piv = s_piv;
    if (piv < 0) { singular = true; break; }
    if (piv != c)
      for (int k = threadIdx.x; k < W; k += blockDim.x) {
        const double tmp = M[(int64_t)c * W + k];
        M[(int64_t)c * W + k] = M[(int64_t)piv * W + k];
        M[(int64_t)piv * W + k] = tmp;
      }
    __syncthreads();
    const double inv = 1.0 / M[(int64_t)c * W + c];
    __syncthreads();
    for (int k = threadIdx.x; k < W; k += blockDim.x) M[(int64_t)c * W + k] *= inv;
    __syncthreads();
    for (int r = warp; r < K; r += nw) {
      if (r == c) continue;
      const double fct = M[(int64_t)r * W + c];
      __syncwarp();
      if (fct != 0.0)
        for (int k = lane; k < W; k += 32) M[(int64_t)r * W + k] = fma(-fct, M[(int64_t)c * W + k], M[(int64_t)r * W + k]);
      __syncwarp();
    }
    __syncthreads();
  }
  for (int e = threadIdx.x; e < K * K; e += blockDim.x) {
    const int i = e / K, j = e % K;
    out[e] = singular ? qnan : M[(int64_t)i * W + K + j];
  }
}

// ---- model = X w for a whole batch on the FP64 tensor cores (shared design matrix) ------------------
// out[b, n] = sum_k X[n, k] coeff[b, k].  CTA = 64 light curves (their coefficient rows stay in shared
// memory) x a strided set of 32-cadence stages of X (cp.async double buffer); warp w owns the 8-cadence
// row tile (w & 3) and four 8-light-curve column tiles: 1 + 4 fragments per 4 DMMAs.
constexpr int RGE_LC = 64;
struct RgeSmem {
  double w[RGE_LC][RGM_LD];
  double x[2][RGM_RC][RGM_LD];
};

__global__ void __launch_bounds__(256)
rg_model_mma_kernel(const double* __restrict__ X, int64_t N, int K, int B, const double* __restrict__ coeff,
                    double* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char rg_smem[];
  RgeSmem& sm = *reinterpret_cast<RgeSmem*>(rg_smem);
  const int lc0 = blockIdx.y * RGE_LC;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nstage = (int)((N + RGM_RC - 1) / RGM_RC);
  for (int e = threadIdx.x; e < RGE_LC * RGM_LD; e += blockDim.x) {
    const int r = e / RGM_LD, c = e - r * RGM_LD;
    sm.w[r][c] = (c < K && lc0 + r < B) ? coeff[(int64_t)(lc0 + r) * K + c] : 0.0;
  }
  for (int e = threadIdx.x; e < 2 * RGM_RC * (RGM_LD - K); e += blockDim.x) {
    const int sgl = e / (RGM_RC * (RGM_LD - K)), r2 = e % (RGM_RC * (RGM_LD - K));
    sm.x[sgl][r2 / (RGM_LD - K)][K + r2 % (RGM_LD - K)] = 0.0;
  }
  auto issue = [&](int stage, int buf) {
    const int64_t n0 = (int64_t)stage * RGM_RC;
    for (int e = threadIdx.x; e < RGM_RC * K; e += blockDim.x) {
      const int r = e / K, c = e - r * K;
      const int64_t row = min(n0 + r, N - 1);                 // tail rows repeat the last cadence (never stored)
      rg_cp8(&sm.x[buf][r][c], X + row * K + c);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  const int mt = warp & 3, ng = warp >> 2;
  const int kr = lane & 3, kq = lane >> 2;
  const int ksteps = (K + 3) / 4;
  int stage = blockIdx.x, buf = 0;
  if (stage < nstage) issue(stage, 0);
  for (; stage < nstage; stage += gridDim.x, buf ^= 1) {
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    if (stage + (int)gridDim.x < nstage) issue(stage + gridDim.x, buf ^ 1);
    double acc[4][2];
#pragma unroll
    for (int j = 0; j < 4; ++j) { acc[j][0] = 0.0; acc[j][1] = 0.0; }
    const double* xa = &sm.x[buf][mt * 8 + kq][kr];
    const double* wb = &sm.w[ng * 32 + kq][kr];
#pragma unroll 2
    for (int ks = 0; ks < ksteps; ++ks) {
      const double a = xa[ks * 4];
#pragma unroll
      for (int j = 0; j < 4; ++j) rg_dmma(acc[j][0], acc[j][1], a, wb[j * 8 * RGM_LD + ks * 4]);
    }
    const int64_t n = (int64_t)stage * RGM_RC + mt * 8 + kq;
    if (n < N) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int lc = lc0 + ng * 32 + j * 8 + 2 * kr;
        if (lc < B) out[(int64_t)lc * N + n] = acc[j][0];
        if (lc + 1 < B) out[(int64_t)(lc + 1) * N + n] = acc[j][1];
      }
    }
  }
}

__global__ void rg_zero_kernel(double* p, int64_t n, uint8_t* q, int64_t nq) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = 0.0;
  if (q && i < nq) q[i] = 0;
}

// The exact fp64 Gram pass over the listed rows: the FP64 tensor-core kernel when its tiling covers K + 1 columns,
// else the SIMT kernel (LKB_REGRESS_SIMT=1 forces the SIMT kernel, kept for A/B measurements).  `sign` +1 adds the
// rows, -1 removes them; `first` marks the first pass of a call (it may split a light curve over two CTAs).  With
// `exact` the split depends on N alone, never on B, so a light curve's Gram matrix does not depend on the batch.
// Shared by lkb_regress and lkb_elasticnet.
static int rg_gram_pass(const double* d_X, int x_batched, const double* d_y, const double* d_fe, int B, int64_t N,
                        int K, double sign, bool first, bool exact, RgWs ws, cudaStream_t st) {
  const int Ka = K + 1;
  const int ntile = (Ka + 7) / 8;
  const int tb = ntile <= 20 ? 4 : 5;
  const int nb5 = (ntile + tb - 1) / tb;
  static const bool force_simt = getenv("LKB_REGRESS_SIMT") != nullptr;
  const bool use_mma = !force_simt && Ka <= RGM_LD && nb5 <= 5;
  static bool attr = false;
  if (!attr) {
    LKB_CUDA_CHECK(cudaFuncSetAttribute(rg_accum_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)(2 * sizeof(RgStage))));
    const int sm2 = (int)(2 * sizeof(RgmStage));
    LKB_CUDA_CHECK(cudaFuncSetAttribute(rg_gram_mma_kernel<1, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm2));
    LKB_CUDA_CHECK(cudaFuncSetAttribute(rg_gram_mma_kernel<2, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm2));
    LKB_CUDA_CHECK(cudaFuncSetAttribute(rg_gram_mma_kernel<3, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm2));
    LKB_CUDA_CHECK(cudaFuncSetAttribute(rg_gram_mma_kernel<4, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm2));
    LKB_CUDA_CHECK(cudaFuncSetAttribute(rg_gram_mma_kernel<5, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm2));
    LKB_CUDA_CHECK(cudaFuncSetAttribute(rg_gram_mma_kernel<5, 5>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm2));
    attr = true;
  }
  if (use_mma) {
    const size_t sm2 = 2 * sizeof(RgmStage);
    // first pass of a small batch: two CTAs per light curve to fill the SMs (wave quantisation)
    const dim3 g((unsigned)B, (first && (exact || B < 4 * sm_count()) && N >= 4096) ? 2u : 1u);
    const unsigned nt = 32u * nb5 * (nb5 + 1) / 2;
    if (tb == 5) rg_gram_mma_kernel<5, 5><<<g, nt, sm2, st>>>(d_X, x_batched, d_y, N, K, sign, ws);
    else switch (nb5) {
      case 1: rg_gram_mma_kernel<1, 4><<<g, nt, sm2, st>>>(d_X, x_batched, d_y, N, K, sign, ws); break;
      case 2: rg_gram_mma_kernel<2, 4><<<g, nt, sm2, st>>>(d_X, x_batched, d_y, N, K, sign, ws); break;
      case 3: rg_gram_mma_kernel<3, 4><<<g, nt, sm2, st>>>(d_X, x_batched, d_y, N, K, sign, ws); break;
      case 4: rg_gram_mma_kernel<4, 4><<<g, nt, sm2, st>>>(d_X, x_batched, d_y, N, K, sign, ws); break;
      default: rg_gram_mma_kernel<5, 4><<<g, nt, sm2, st>>>(d_X, x_batched, d_y, N, K, sign, ws); break;
    }
  } else {
    const int nblk = (Ka + RG_BLK - 1) / RG_BLK;
    const int nupper = nblk * (nblk + 1) / 2;
    rg_accum_kernel<<<dim3(nupper, B), 128, 2 * sizeof(RgStage), st>>>(d_X, x_batched, d_y, d_fe, N, K, nblk, sign,
                                                                         ws);
  }
  return LKB_OK;
}

bool regress_tc_supported(int B, int64_t N, int K);                                              // regress_tc.cu
int regress_tc_gram(const double* d_X, const double* d_y, const double* d_fe, const uint8_t* d_used, int B, int64_t N,
                    int K, double* d_gram, cudaStream_t st);
int regress_tc_gradient(const double* d_X, const double* d_y, const double* d_fe, const uint8_t* d_used,
                        const double* d_model, int B, int64_t N, int K, double* d_grad, cudaStream_t st);

int regress(const double* X, int x_batched, const double* y, const double* flux_err, const uint8_t* cadence_mask,
            const double* prior_mu, const double* prior_sigma, int B, int64_t N, int K, double clip_sigma, int niters,
            double* coeff, double* model, uint8_t* outlier_mask, int32_t* status_out, double* coeff_cov, int mem,
            cudaStream_t st, int prior_batched, int flags) {
  LKB_REQUIRE(X && y && coeff && model && outlier_mask, "lkb_regress: null argument");
  LKB_REQUIRE(prior_batched == 0 || prior_batched == 1, "lkb_regress_ex: prior_batched must be 0 or 1");
  LKB_REQUIRE((flags & ~LKB_REGRESS_EXACT_INVARIANT) == 0, "lkb_regress_ex: unknown flags");
  const bool exact = (flags & LKB_REGRESS_EXACT_INVARIANT) != 0;
  const int64_t pstride = prior_batched ? K : 0;
  LKB_REQUIRE(B > 0 && B <= 65535 && N > 0 && K > 0 && niters >= 1, "lkb_regress: bad sizes");
  LKB_REQUIRE((prior_mu == nullptr) == (prior_sigma == nullptr), "Please specify both `prior_mu` and `prior_sigma`");
  LKB_REQUIRE(N < ((int64_t)1 << 31), "lkb_regress: N too large");
  if (K > RG_KMAX) { set_error("lkb_regress: K=%d > %d unsupported", K, RG_KMAX); return LKB_E_UNSUPPORTED; }
  LKB_TRY(ensure_device());
  const int Ka = K + 1;
  const size_t BN = (size_t)B * N;

  const double *d_X = nullptr, *d_y = nullptr, *d_fe = nullptr, *d_pm = nullptr, *d_ps = nullptr;
  const uint8_t* d_cm = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, X, (x_batched ? BN : (size_t)N) * K, &d_X, st));
  LKB_TRY(stage_in<double>(mem, WS_IN1, y, BN, &d_y, st));
  LKB_TRY(stage_in<double>(mem, WS_IN2, flux_err, BN, &d_fe, st));
  LKB_TRY(stage_in<uint8_t>(mem, WS_IN3, cadence_mask, BN, &d_cm, st));
  LKB_TRY(stage_in<double>(mem, WS_IN4, prior_mu, (prior_batched ? (size_t)B : 1) * K, &d_pm, st));
  LKB_TRY(stage_in<double>(mem, WS_IN5, prior_sigma, (prior_batched ? (size_t)B : 1) * K, &d_ps, st));

  RgWs ws;
  LKB_TRY(ws_get_t<int32_t>(WS_A, BN, &ws.rows));
  LKB_TRY(ws_get_t<int32_t>(WS_B, B, &ws.cnt));
  LKB_TRY(ws_get_t<uint8_t>(WS_C, BN, &ws.used));
  LKB_TRY(ws_get_t<double>(WS_D, (size_t)B * Ka * Ka, &ws.gram));
  LKB_TRY(ws_get_t<double>(WS_E, BN, &ws.resid));
  LKB_TRY(ws_get_t<double>(WS_H, BN, &ws.wl));

  double *o_c = nullptr, *o_m = nullptr;
  uint8_t* o_om = nullptr;
  int32_t* o_st = nullptr;
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0, coeff, (size_t)B * K, &o_c));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT1, model, BN, &o_m));
  LKB_TRY(stage_out_alloc<uint8_t>(mem, WS_OUT2, outlier_mask, BN, &o_om));
  LKB_TRY(stage_out_alloc<int32_t>(mem, WS_OUT3, status_out, B, &o_st));
  double* o_cov = nullptr;
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT4, coeff_cov, (size_t)B * K * K, &o_cov));
  int32_t* d_status = o_st;
  if (coeff_cov && !d_status) LKB_TRY(ws_get_t<int32_t>(WS_G, B, &d_status));

  {
    const int64_t ng = (int64_t)B * Ka * Ka, nz = ng > (int64_t)BN ? ng : (int64_t)BN;
    rg_zero_kernel<<<(unsigned)((nz + 255) / 256), 256, 0, st>>>(ws.gram, ng, o_om, (int64_t)BN);
    LKB_LAUNCH_CHECK();
  }
  const size_t solve_smem = (size_t)K * Ka * sizeof(double);
  static size_t solve_attr = 0;
  if (solve_smem > solve_attr) {
    LKB_CUDA_CHECK(cudaFuncSetAttribute(rg_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)solve_smem));
    LKB_CUDA_CHECK(cudaFuncSetAttribute(rg_resolve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)solve_smem));
    solve_attr = solve_smem;
  }
  // the first Gram pass of a large shared-design-matrix batch may take the tcgen05 GEMM; every other pass takes the
  // exact fp64 kernels of rg_gram_pass (LKB_REGRESS_SIMT=1: SIMT kernels throughout, kept for A/B measurements).
  // LKB_REGRESS_EXACT_INVARIANT keeps every choice that depends on B or on a shared X out: no tcgen05 Gram, no batched
  // model GEMM (the per-light-curve model of rg_clip / rg_final instead), the Gram split decided by N alone.
  static const bool force_simt = getenv("LKB_REGRESS_SIMT") != nullptr;
  const bool use_tc = !exact && !force_simt && !x_batched && regress_tc_supported(B, N, K);
  // batched model X w as one FP64 tensor-core GEMM when the design matrix is shared by the batch
  const bool gemm_model = !exact && !force_simt && !x_batched && K <= RGM_LD - 1 && B >= 8;
  dim3 gemm_grid(1, (unsigned)((B + RGE_LC - 1) / RGE_LC));
  if (gemm_model) {
    static bool attr = false;
    if (!attr) {
      LKB_CUDA_CHECK(cudaFuncSetAttribute(rg_model_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)sizeof(RgeSmem)));
      attr = true;
    }
    const int nstage = (int)((N + RGM_RC - 1) / RGM_RC);
    int gx = (4 * sm_count() + (int)gemm_grid.y - 1) / (int)gemm_grid.y;
    gemm_grid.x = (unsigned)(gx < 1 ? 1 : (gx > nstage ? nstage : gx));
  }
  const size_t clip_smem = sizeof(double) * (size_t)((K + 1) & ~1) + sizeof(FastSelSmem) +
                           sizeof(double) * (size_t)(FS_CAP + FS_SAMPLE);
  static size_t clip_attr = 0;
  if (clip_smem > clip_attr) {
    LKB_CUDA_CHECK(cudaFuncSetAttribute(rg_clip_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)clip_smem));
    clip_attr = clip_smem;
  }
  for (int it = 0; it < niters; ++it) {
    rg_rows_kernel<<<B, 256, 0, st>>>(d_cm, o_om, d_fe, N, it == 0 ? 1 : 0, ws);
    LKB_LAUNCH_CHECK();
    if (it == 0) prof_begin(st);
    if (it == 0 && use_tc) {
      // first fit of a large shared-design-matrix batch: the Gram matrices as one tcgen05 GEMM (regress_tc.cu)
      LKB_TRY(regress_tc_gram(d_X, d_y, d_fe, ws.used, B, N, K, ws.gram, st));
    } else {
      LKB_TRY(rg_gram_pass(d_X, x_batched, d_y, d_fe, B, N, K, it == 0 ? 1.0 : -1.0, it == 0, exact, ws, st));
    }
    if (it == 0) { prof_end(st); prof_begin(st); }     // second record: everything after the first Gram pass
    LKB_LAUNCH_CHECK();
    double* d_lu = nullptr;
    int32_t* d_piv = nullptr;
    if (use_tc && gemm_model) {                        // the refinement step below reuses the factors
      LKB_TRY(ws_get_t<double>(WS_Y0, (size_t)B * K * K, &d_lu));
      LKB_TRY(ws_get_t<int32_t>(WS_Y1, (size_t)B * K, &d_piv));
    }
    rg_solve_kernel<<<B, 256, solve_smem, st>>>(K, d_pm, d_ps, pstride, ws, o_c, d_status, nullptr, d_lu, d_piv);
    LKB_LAUNCH_CHECK();
    if (gemm_model) {
      rg_model_mma_kernel<<<gemm_grid, 256, sizeof(RgeSmem), st>>>(d_X, N, K, B, o_c, ws.resid);
      LKB_LAUNCH_CHECK();
    }
    if (use_tc && gemm_model) {
      // The tcgen05 Gram matrices carry ~1e-6 relative errors, which a coefficient of order one (the offset of a
      // normalised light curve) turns into ~1e-6 ABSOLUTE errors of the small coefficients.  One step of iterative
      // refinement with the EXACT fp64 gradient X^T W (y - X w) of the cadences in use removes them (the error
      // contracts by ~1e-6 per step): w <- w + (A~ + prior)^-1 [X^T W (y - X w) - prior (w - mu)], then the model again.
      double* d_grad = nullptr;
      LKB_TRY(ws_get_t<double>(WS_X6, (size_t)B * K, &d_grad));
      LKB_TRY(regress_tc_gradient(d_X, d_y, d_fe, ws.used, ws.resid, B, N, K, d_grad, st));
      if (getenv("LKB_REGRESS_REFACTOR"))            // (A/B: eliminate again instead of reusing the factors)
        rg_solve_kernel<<<B, 256, solve_smem, st>>>(K, d_pm, d_ps, pstride, ws, o_c, d_status, d_grad, nullptr, nullptr);
      else
        rg_resolve_kernel<<<B, 256, solve_smem, st>>>(K, d_pm, d_ps, pstride, d_lu, d_piv, o_c, d_status, d_grad);
      LKB_LAUNCH_CHECK();
      rg_model_mma_kernel<<<gemm_grid, 256, sizeof(RgeSmem), st>>>(d_X, N, K, B, o_c, ws.resid);
      LKB_LAUNCH_CHECK();
    }
    rg_clip_kernel<<<B, 512, clip_smem, st>>>(d_X, x_batched, d_y, N, K, o_c, clip_sigma, ws, o_om, gemm_model ? 1 : 0);
    LKB_LAUNCH_CHECK();
  }
  if (gemm_model) {
    rg_model_mma_kernel<<<gemm_grid, 256, sizeof(RgeSmem), st>>>(d_X, N, K, B, o_c, o_m);
    LKB_LAUNCH_CHECK();
  }
  rg_final_kernel<<<B, 512, K * sizeof(double), st>>>(d_X, x_batched, N, K, o_c, o_m, gemm_model ? 1 : 0);
  LKB_LAUNCH_CHECK();
  if (coeff_cov) {
    // covariance of the LAST fit (the Gram matrix in the workspace already excludes every clipped row
    // but the ones found by the final clip, exactly like the reference's last _fit_coefficients call)
    double* d_work = nullptr;
    LKB_TRY(ws_get_t<double>(WS_F, (size_t)B * K * 2 * K, &d_work));
    rg_inverse_kernel<<<B, 256, 0, st>>>(K, d_ps, pstride, ws, d_work, o_cov, d_status);
    LKB_LAUNCH_CHECK();
  }

  if (niters > 0) prof_end(st);
  LKB_TRY(stage_out_copy<double>(mem, coeff, o_c, (size_t)B * K, st));
  LKB_TRY(stage_out_copy<double>(mem, model, o_m, BN, st));
  LKB_TRY(stage_out_copy<uint8_t>(mem, outlier_mask, o_om, BN, st));
  LKB_TRY(stage_out_copy<int32_t>(mem, status_out, o_st, B, st));
  LKB_TRY(stage_out_copy<double>(mem, coeff_cov, o_cov, (size_t)B * K * K, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

// K8: CBVCorrector.correct_elasticnet (cbvcorrector.py:358-379).  The unit-weight Gram matrix [X | y]^T M [X | y] of
// the used cadences (K5's first pass, always the exact fp64 kernels: the ~1e-6 relative error of the tcgen05 Gram
// would move the sweep at which the coordinate descent stops; split over two CTAs by N alone, as under
// LKB_REGRESS_EXACT_INVARIANT), the coordinate descent (enet.cuh), then the model
// X[:, :-1] w[:-1] minus its median over all cadences (rg_final on the coefficients with the last one zeroed).
int elasticnet(const double* X, int x_batched, const double* y, const uint8_t* cadence_mask, int B, int64_t N, int K,
               double alpha, double l1_ratio, int max_iter, double tol, int positive, double* coeff, double* model,
               int32_t* n_iter, double* dual_gap, uint8_t* converged, int mem, cudaStream_t st) {
  LKB_REQUIRE(X && y && coeff && model && n_iter && dual_gap && converged, "lkb_elasticnet: null argument");
  LKB_REQUIRE(B > 0 && B <= 65535 && N > 0 && K > 0, "lkb_elasticnet: bad sizes");
  LKB_REQUIRE(N < ((int64_t)1 << 31), "lkb_elasticnet: N too large");
  if (!(alpha >= 0.0) || !std::isfinite(alpha)) { set_error("lkb_elasticnet: alpha must be >= 0 (got %g)", alpha); return LKB_E_ARG; }
  if (!(l1_ratio >= 0.0 && l1_ratio <= 1.0)) {
    set_error("lkb_elasticnet: l1_ratio must be in [0, 1] (got %g)", l1_ratio);
    return LKB_E_ARG;
  }
  if (max_iter < 1) { set_error("lkb_elasticnet: max_iter must be >= 1 (got %d)", max_iter); return LKB_E_ARG; }
  if (!(tol >= 0.0)) { set_error("lkb_elasticnet: tol must be >= 0 (got %g)", tol); return LKB_E_ARG; }
  if (K > ENET_KMAX) { set_error("lkb_elasticnet: K=%d > %d unsupported", K, ENET_KMAX); return LKB_E_UNSUPPORTED; }
  LKB_TRY(ensure_device());
  const int Ka = K + 1;
  const size_t BN = (size_t)B * N;

  const double *d_X = nullptr, *d_y = nullptr;
  const uint8_t* d_cm = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, X, (x_batched ? BN : (size_t)N) * K, &d_X, st));
  LKB_TRY(stage_in<double>(mem, WS_IN1, y, BN, &d_y, st));
  LKB_TRY(stage_in<uint8_t>(mem, WS_IN3, cadence_mask, BN, &d_cm, st));

  RgWs ws{};
  uint8_t* d_none = nullptr;                           // the (empty) outlier mask rg_rows reads
  double* d_w0 = nullptr;                              // coefficients with the constant's entry zeroed, for the model
  LKB_TRY(ws_get_t<int32_t>(WS_A, BN, &ws.rows));
  LKB_TRY(ws_get_t<int32_t>(WS_B, B, &ws.cnt));
  LKB_TRY(ws_get_t<uint8_t>(WS_C, BN, &ws.used));
  LKB_TRY(ws_get_t<double>(WS_D, (size_t)B * Ka * Ka, &ws.gram));
  LKB_TRY(ws_get_t<double>(WS_H, BN, &ws.wl));
  LKB_TRY(ws_get_t<uint8_t>(WS_E, BN, &d_none));
  LKB_TRY(ws_get_t<double>(WS_F, (size_t)B * K, &d_w0));

  double *o_c = nullptr, *o_m = nullptr, *o_g = nullptr;
  int32_t* o_it = nullptr;
  uint8_t* o_cv = nullptr;
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0, coeff, (size_t)B * K, &o_c));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT1, model, BN, &o_m));
  LKB_TRY(stage_out_alloc<int32_t>(mem, WS_OUT2, n_iter, B, &o_it));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT3, dual_gap, B, &o_g));
  LKB_TRY(stage_out_alloc<uint8_t>(mem, WS_OUT4, converged, B, &o_cv));

  {
    const int64_t ng = (int64_t)B * Ka * Ka, nz = ng > (int64_t)BN ? ng : (int64_t)BN;
    rg_zero_kernel<<<(unsigned)((nz + 255) / 256), 256, 0, st>>>(ws.gram, ng, d_none, (int64_t)BN);
    LKB_LAUNCH_CHECK();
  }
  rg_rows_kernel<<<B, 256, 0, st>>>(d_cm, d_none, nullptr, N, 1, ws);
  LKB_LAUNCH_CHECK();
  {
    // a light curve without a used cadence has no fit (scikit-learn refuses an empty X)
    int32_t* h_cnt = (int32_t*)malloc(sizeof(int32_t) * (size_t)B);
    if (!h_cnt) { set_error("lkb_elasticnet: host allocation failed"); return LKB_E_OOM; }
    cudaError_t e = cudaMemcpyAsync(h_cnt, ws.cnt, sizeof(int32_t) * (size_t)B, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    int empty = -1;
    for (int b = 0; b < B && e == cudaSuccess; ++b)
      if (h_cnt[b] == 0) { empty = b; break; }
    free(h_cnt);
    LKB_CUDA_CHECK(e);
    if (empty >= 0) {
      set_error("lkb_elasticnet: light curve %d has no used cadence", empty);
      return LKB_E_ARG;
    }
  }
  prof_begin(st);
  // exact: the two-CTA split of a light curve depends on N alone, so its Gram matrix (and through the stopping tests
  // its n_iter and coefficients) does not depend on how many light curves share the call
  LKB_TRY(rg_gram_pass(d_X, x_batched, d_y, nullptr, B, N, K, 1.0, true, true, ws, st));
  LKB_LAUNCH_CHECK();
  prof_end(st);
  prof_begin(st);
  LKB_TRY(enet_cd_launch(ws.gram, ws.cnt, B, K, alpha, l1_ratio, max_iter, tol, positive, o_c, o_it, o_g, o_cv, st));
  prof_end(st);
  prof_begin(st);
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_w0, o_c, sizeof(double) * (size_t)B * K, cudaMemcpyDeviceToDevice, st));
  LKB_CUDA_CHECK(cudaMemset2DAsync(d_w0 + (K - 1), sizeof(double) * K, 0, sizeof(double), B, st));
  rg_final_kernel<<<B, 512, K * sizeof(double), st>>>(d_X, x_batched, N, K, d_w0, o_m, 0);
  LKB_LAUNCH_CHECK();
  prof_end(st);

  LKB_TRY(stage_out_copy<double>(mem, coeff, o_c, (size_t)B * K, st));
  LKB_TRY(stage_out_copy<double>(mem, model, o_m, BN, st));
  LKB_TRY(stage_out_copy<int32_t>(mem, n_iter, o_it, B, st));
  LKB_TRY(stage_out_copy<double>(mem, dual_gap, o_g, B, st));
  LKB_TRY(stage_out_copy<uint8_t>(mem, converged, o_cv, B, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

}  // namespace lkb
