// "v2" transform of the NUFFT Lomb-Scargle path (included by ls_nufft.cu; also compiled for the CPU through
// tests/native/cuda_emu.h).  Every light curve is ONE REAL series on the fine grid of M = 2^p cells, transformed as a
// complex series of Mh = M / 2 points  z[n] = g[2n] + i g[2n + 1]:
//     G[k] = E[k] + exp(2 pi i k / M) O[k],   E = (Z[k] + conj Z[Mh - k]) / 2,   O = (Z[k] - conj Z[Mh - k]) / 2i.
// (Round 2, hardware finding: packing TWO light curves into one complex transform leaks the partner's spectral peak
// into a quiet light curve with relative weight ~1e-7 - fp32 rounding of Z at the partner's peak bin - which is
// 2-3x the parity tolerance when the partner is >~ 300x louder; tools/worst_bins_detail.py.  A light curve's own
// transform has no such cross-talk, batches of odd size need no padding, and the result of a light curve no longer
// depends on its neighbour.)
//
// Mh = A * Bc, Bc = 2^V2_PB = 512 fixed, A = 2^pa;  n = n1 Bc + n2,  k = k1 + A k2  (four-step transform):
//   spread : G[lc][c][n1][j]   (c = n2 / TC, j = n2 % TC, TC = 8192 / A columns per CTA), rows n1 < n1max only -
//            the cadences reach just the first df * baseline (20 % at lightkurve's default oversampling) of the grid;
//            kernel weights come from a per-cadence table (built once per call), one thread = one z cell = two fine
//            grid cells of LCS light curves;
//   cols   : one CTA = TC columns of one light curve: length-A transforms over n1 in shared memory (in place, one
//            radix-16 butterfly per thread and pass, twiddles from tables), times exp(2 pi i n2 k1 / Mh), written as
//            T[lc][c][k1][j] - one contiguous 64 KB block per CTA;
//   rows   : one CTA = rows k1 = 1 + 8 g .. 8 (g + 1) and their mirror rows A - k1 of one light curve: length-Bc
//            transforms over n2, then the finish (unpack E / O, deconvolve + tau rotation through one folded table,
//            epilogue) -> power, written in 32-byte runs (8 consecutive k1 at one k2 are 8 consecutive frequency
//            bins); the transform itself never goes back to global memory.  The CTA that would hold row A / 2 twice
//            takes row 0 (which mirrors onto itself) instead.
// All tile geometry is compile-time (template parameters PA and LOGT): every shared-memory offset inside the passes is
// `runtime base + constant`.  A tile is 2^LOGT points, 16 per thread: the float2 kernels take 8192-point tiles (64 KB,
// 512 threads, 2 CTAs per SM); the double2 escalation pass takes 4096-point tiles (64 KB of double2, 256 threads), so
// that it too runs 2 CTAs per SM - at 8192 points its tiles were 128 KB, one CTA per SM, and the column kernel spilled.
#pragma once
#include "nufft_core.h"

namespace lkb {
namespace {

using nufft::V2_PB;
using nufft::V2_THREADS;
using nufft::V2_TILE;
constexpr int V2_LOG_TILE = 13;
static_assert((1 << V2_LOG_TILE) == V2_TILE, "tile size");
constexpr int V2_BC = 1 << V2_PB;
constexpr int V2_R = V2_TILE / (2 * V2_BC);                     // rows per block of the float2 row kernel (8)
constexpr int V2_LSB = V2_BC + V2_BC / 16 + 1;                  // skewed line of Bc points
// real-mode limits: Mh = 2^(p - 1) = A * Bc with 16 <= A <= 8192
constexpr int V2R_P_MIN = V2_PB + 4 + 1, V2R_P_MAX = V2_PB + 13 + 1;

__host__ __device__ constexpr int v2_radix(int plog, int idx) {
  return (idx < plog / 4) ? 16 : ((idx == plog / 4 && (plog % 4)) ? (1 << (plog % 4)) : 0);
}
__host__ __device__ constexpr int v2_log2i(int r) { return r == 16 ? 4 : r == 8 ? 3 : r == 4 ? 2 : r == 2 ? 1 : 0; }
// log2 of the tile of a transform with A = 2^pa: 8192 points in float2; 4096 in double2 (one column of 4096 points at
// A = 4096, so A = 8192 keeps the 8192-point tile and one CTA per SM)
__host__ __device__ constexpr int v2_log_tile(int pa, bool dbl) { return (dbl && pa <= 12) ? 12 : V2_LOG_TILE; }
__device__ __forceinline__ int v2_skew(int a) { return a + (a >> 4); }
// offset of input r of a butterfly (r * nb points further) in a skewed line; exact because the butterfly index is
// either a multiple-of-16 aligned case (nb % 16 == 0) or smaller than nb <= 8
template <int nb>
__host__ __device__ constexpr int v2_in_off(int r) {
  return (nb % 16 == 0) ? r * (nb + nb / 16) : r * nb + ((r * nb) >> 4);
}

// ---- tables -------------------------------------------------------------------------------------------------------
// pass tables of the length-A and the length-Bc transforms, the two-level inter-step table of exp(2 pi i q / Mh)
template <class CT>
__global__ void nufft2_tables_kernel(int pa, int pb, int ph, CT* __restrict__ tw_a, CT* __restrict__ tw_b,
                                     CT* __restrict__ t_hi, CT* __restrict__ t_lo) {
  const int la = nufft::v2_pass_table_len(pa), lb = nufft::v2_pass_table_len(pb), pl = nufft::v2_log2_lo(ph);
  const int nlo = 1 << pl, nhi = 1 << (ph - pl);
  int e = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  int64_t num = 0, den = 1;
  CT* dst = nullptr;
  if (e < la) { nufft::v2_pass_table_entry(pa, e, &num, &den); dst = tw_a + e; }
  else if ((e -= la) < lb) { nufft::v2_pass_table_entry(pb, e, &num, &den); dst = tw_b + e; }
  else if ((e -= lb) < nhi) { num = e; den = nhi; dst = t_hi + e; }
  else if ((e -= nhi) < nlo) { num = e; den = (int64_t)1 << ph; dst = t_lo + e; }
  else return;
  double sn, cs;
  sincospi(2.0 * (double)num / (double)den, &sn, &cs);
  typedef typename nufft::CplxOf<CT>::real RT;
  *dst = nufft::CplxOf<CT>::mk((RT)cs, (RT)sn);
}

// kernel weights of every cadence: Wt[n w + q] = phi((i0_n + q - x_n) / (w / 2)), q = 0 .. w - 1, evaluated in FP64
// from the time stamp itself and rounded once.  (Round 2, hardware finding: with fp32 offsets and expf the weights
// carry ~1e-6 relative errors - a perturbation of the kernel SHAPE that the deconvolution does not undo; it leaked
// strong lines from above the frequency band into the band at 2e-8 of their amplitude, 1.5x the tolerance on light
// curves whose in-band spectrum is 1000x below their variability, and a WIDER kernel made it worse, not better.)
template <class RT>
__global__ void nufft2_weights_kernel(const double* __restrict__ t, int64_t N, double df, int64_t M, int w, double beta,
                                      RT* __restrict__ Wt) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= N * w) return;
  const int64_t n = e / w;
  const int q = (int)(e - n * w);
  const double x = df * t[n] * (double)M + (double)nufft::grid_shift(w);       // as nufft::cad_entry
  const double i0 = ceil(x - 0.5 * (double)w);
  const double z = (i0 + (double)q - x) * (2.0 / (double)w);
  const double s2 = 1.0 - z * z;
  Wt[e] = (s2 > 0.0) ? (RT)exp(beta * (sqrt(s2) - 1.0)) : (RT)0.0;
}

// z index (n = n1 Bc + n2) of position e of the G layout [c][n1][j]
__device__ __forceinline__ int64_t v2_zcell_of(int64_t e, int ptc, int n1max) {
  const int64_t j = e & (((int64_t)1 << ptc) - 1), rest = e >> ptc;
  const int64_t n1 = rest % n1max, c = rest / n1max;
  return (n1 << V2_PB) + (c << ptc) + j;
}

// ---- spread -------------------------------------------------------------------------------------------------------
// G[lc][e] = (cell 2n, cell 2n + 1) of light curves lc0 .. lc0 + LCS - 1; grid (ceil(cells / 256), ceil(B / LCS)).
// y rows [B, ystride] (centred flux); no scaling: a light curve's transform is its own.
template <int LCS>
__global__ void __launch_bounds__(256)
nufft2_spread_kernel(const int32_t* __restrict__ first_ge, const nufft::Cad* __restrict__ cad,
                     const float* __restrict__ Wt, const float* __restrict__ y, int64_t ystride, int B, int w, int p,
                     int ptc, int n1max, float2* __restrict__ G) {
  const int64_t cells = (int64_t)n1max << V2_PB;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= cells) return;
  const int64_t M = (int64_t)1 << p, m = 2 * v2_zcell_of(e, ptc, n1max);
  const int lc0 = (int)blockIdx.y * LCS;
  const float* yr[LCS];
#pragma unroll
  for (int q = 0; q < LCS; ++q) {
    int b = lc0 + q;
    if (b > B - 1) b = B - 1;                      // clamped rows are computed and dropped
    yr[q] = y + (int64_t)b * ystride;
  }
  float a0[LCS], a1[LCS];
#pragma unroll
  for (int q = 0; q < LCS; ++q) { a0[q] = 0.0f; a1[q] = 0.0f; }
  const int64_t L = nufft::table_len(M, w);
  for (int wrap = 0; wrap < 2; ++wrap) {           // wrap = 1: cadences whose support runs past cell M - 1
    const int64_t mm = m + (int64_t)wrap * M;
    if (mm + 1 >= L) break;
    int64_t lo_c = mm - w + 1, hi_c = mm + 2;
    if (lo_c < 0) lo_c = 0;
    if (hi_c > L - 1) hi_c = L - 1;
    const int32_t na = first_ge[lo_c], nb = first_ge[hi_c];          // cadences with mm - w + 1 <= i0 <= mm + 1
    for (int32_t n = na; n < nb; ++n) {
      const int tap = (int)(mm - (int64_t)cad[n].i0);                // in [-1, w - 1]
      const float* wr = Wt + (int64_t)n * w;
      const float w0 = (tap >= 0) ? wr[tap] : 0.0f;                  // weight on cell mm
      const float w1 = (tap + 1 < w) ? wr[tap + 1] : 0.0f;           // weight on cell mm + 1
#pragma unroll
      for (int q = 0; q < LCS; ++q) {
        const float v = yr[q][n];
        a0[q] = fmaf(w0, v, a0[q]);
        a1[q] = fmaf(w1, v, a1[q]);
      }
    }
  }
#pragma unroll
  for (int q = 0; q < LCS; ++q)
    if (lc0 + q < B) G[(int64_t)(lc0 + q) * cells + e] = make_float2(a0[q], a1[q]);
}

// ---- in-place passes over the lines of a tile (compile-time geometry) ---------------------------------------------
// PLOG: log2 of the line length, LS: skewed line stride, IDX / NS: pass number and the product of earlier radices, NT:
// threads of the CTA (16 points each).  nz (first pass only): line positions >= nz hold zeros that were never stored -
// they are not read either
template <int PLOG, int LS, int IDX, int NS, class CT = float2, int NT = V2_THREADS>
__device__ __forceinline__ void v2_pass_t(CT* buf, const CT* __restrict__ tw, int nz = 1 << 30) {
  constexpr int R = v2_radix(PLOG, IDX);
  if constexpr (R != 0) {
    constexpr int LR = v2_log2i(R), NB = 16 / R, PNB = PLOG - LR, nb = 1 << PNB;      // nb butterflies per line
    constexpr bool WIDE = nb > NT;                   // one line, several butterflies of it per thread
    static_assert(WIDE || (NT % nb) == 0, "geometry");
    // per-input offset r * nb in the skewed line: v2_in_off<nb>(r)
    const int t = (int)threadIdx.x;
    CT u[NB][R];
    int base_in[NB];
#pragma unroll
    for (int q = 0; q < NB; ++q) {
      int line, i;
      if constexpr (WIDE) { line = 0; i = t + NT * q; }
      else { line = (t >> PNB) + ((NT * q) >> PNB); i = t & (nb - 1); }
      base_in[q] = line * LS + ((nb % 16 == 0) ? v2_skew(i) : i);
#pragma unroll
      for (int r = 0; r < R; ++r)
        u[q][r] = (IDX > 0 || r * nb < nz) ? buf[base_in[q] + v2_in_off<nb>(r)] : nufft::CplxOf<CT>::mk(0, 0);
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < NB; ++q) {
      int line, i;
      if constexpr (WIDE) { line = 0; i = t + NT * q; }
      else { line = (t >> PNB) + ((NT * q) >> PNB); i = t & (nb - 1); }
      const int k = i & (NS - 1);
      if constexpr (NS > 1) {
#pragma unroll
        for (int r = 1; r < R; ++r) u[q][r] = nufft::cmul(u[q][r], tw[r * NS + k]);
      }
      nufft::SmallDft<R, CT>::run(u[q]);
      const int j = ((i - k) << LR) + k;
      // NS = 1 (then R = 16): skew(16 i + r) = 17 i + r;  NS >= 16: skew(j + r NS) = skew(j) + r NS 17 / 16
      const int base_out = line * LS + ((NS == 1) ? (j + i) : v2_skew(j));
#pragma unroll
      for (int r = 0; r < R; ++r) buf[base_out + ((NS == 1) ? r : r * (NS + NS / 16))] = u[q][r];
    }
    __syncthreads();
    v2_pass_t<PLOG, LS, IDX + 1, NS * R, CT, NT>(buf, tw + ((IDX > 0) ? R * NS : 0));
  }
}

// Number of transforms a launch works on: the grid's y extent, or (escalation pass, sized before the host knows how many
// light curves were listed) the device-side count minus `base`, at most `cap`; blocks stride over them by gridDim.y.
struct V2Count {
  const int* count;     // NULL: gridDim.y transforms
  int base, cap;
};
__device__ __forceinline__ int v2_count(const V2Count nc, int grid_y) {
  if (!nc.count) return grid_y;
  const int n = *nc.count - nc.base;
  return n < 0 ? 0 : (n > nc.cap ? nc.cap : n);
}

// ---- cols ---------------------------------------------------------------------------------------------------------
// grid (Bc / TC, B).  G: pruned fine grids [B][c][n1 < n1max][j]; T: [B][c][k1][j]
// one transform (light curve slot lc): all threads of the CTA
template <int PA, class CT, int LOGT = V2_LOG_TILE>
__device__ __forceinline__ void v2_cols_one(CT* buf, const CT* __restrict__ G, CT* __restrict__ T, int n1max,
                                            const CT* __restrict__ tw_a, const CT* __restrict__ t_hi,
                                            const CT* __restrict__ t_lo, const int64_t lc) {
  constexpr int NT = (1 << LOGT) / 16;
  constexpr int A = 1 << PA, PTC = LOGT - PA, TC = 1 << PTC, LS = A + A / 16 + 1, C = V2_BC / TC;
  // one sweep of the NT threads covers JW columns x RW rows (RW is a multiple of 16: constant skew increments)
  constexpr int JW = TC < NT / 16 ? TC : NT / 16, RW = NT / JW, CG = TC / JW;
  constexpr int LJW = JW == 32 ? 5 : JW == 16 ? 4 : JW == 8 ? 3 : JW == 4 ? 2 : JW == 2 ? 1 : 0;
  static_assert((1 << LJW) == JW && RW % 16 == 0, "geometry");
  const int t = (int)threadIdx.x, c = (int)blockIdx.x;
  const int jl = t & (JW - 1), nl = t >> LJW;
  const int nvalid = n1max << PTC;
  const CT* Gp = G + (lc * C + c) * (int64_t)nvalid;
  const int s_base = jl * LS + v2_skew(nl), g_base = nl * TC + jl;
  // rows the first pass reads: whole input blocks (of A / R1 rows) that contain a row < n1max
  constexpr int NB1 = A / v2_radix(PA, 0);
  const int nz = ((n1max + NB1 - 1) / NB1) * NB1;
#pragma unroll
  for (int u = 0; u < 16; ++u) {
    const int cg = u % CG, nbk = u / CG;                           // column group, row block of this sweep
    if (nbk * RW < nz) {
      const int idx = g_base + nbk * RW * TC + cg * JW;
      buf[s_base + cg * JW * LS + nbk * (RW + RW / 16)] = (idx < nvalid) ? Gp[idx] : nufft::CplxOf<CT>::mk(0, 0);
    }
  }
  __syncthreads();
  v2_pass_t<PA, LS, 0, 1, CT, NT>(buf, tw_a, nz);
  CT* Tp = T + (lc * C + c) * (int64_t)(1 << LOGT);
  const int ph = PA + V2_PB, pl = nufft::v2_log2_lo(ph);
  const unsigned Mmask = (1u << ph) - 1u, lmask = (1u << pl) - 1u;
#pragma unroll
  for (int u = 0; u < 16; ++u) {
    const int cg = u % CG, nbk = u / CG;
    const int k1 = nl + nbk * RW, n2 = c * TC + jl + cg * JW;
    const unsigned q = ((unsigned)n2 * (unsigned)k1) & Mmask;       // n2 k1 < 2^22
    const CT wq = nufft::cmul(t_hi[q >> pl], t_lo[q & lmask]);
    Tp[g_base + nbk * RW * TC + cg * JW] = nufft::cmul(buf[s_base + cg * JW * LS + nbk * (RW + RW / 16)], wq);
  }
}
// grid (Bc / TC, B): one transform per CTA.  (Kept free of any extra kernel parameter: the float2 instantiation sits
// exactly at the 64-register cap of 2 CTAs/SM, and a 16-byte parameter more made ptxas spill 184 bytes.)
template <int PA, class CT = float2>
__global__ void __launch_bounds__(V2_THREADS, sizeof(CT) == 8 ? 2 : 1)
nufft2_cols_kernel(const CT* __restrict__ G, CT* __restrict__ T, int n1max, const CT* __restrict__ tw_a,
                   const CT* __restrict__ t_hi, const CT* __restrict__ t_lo) {
  LKB_DYN_SMEM(CT, buf);
  v2_cols_one<PA, CT>(buf, G, T, n1max, tw_a, t_hi, t_lo, (int64_t)blockIdx.y);
}
// escalation pass (double precision, tiles of 2^v2_log_tile(PA, true) points): blocks stride over a device-side count
// of transforms.  One transform is a call, not inlined into the loop: inlined, ptxas kept the address arithmetic of
// all 16 loads and stores live across iterations and spilled up to 584 bytes at the 128-register cap of 2 CTAs/SM.
template <int PA, int LOGT>
__device__ __noinline__ void v2_cols_list_one(double2* buf, const double2* __restrict__ G, double2* __restrict__ T,
                                              int n1max, const double2* __restrict__ tw_a,
                                              const double2* __restrict__ t_hi, const double2* __restrict__ t_lo,
                                              const int64_t lc) {
  v2_cols_one<PA, double2, LOGT>(buf, G, T, n1max, tw_a, t_hi, t_lo, lc);
}
template <int PA, int LOGT = v2_log_tile(PA, true)>
__global__ void __launch_bounds__((1 << LOGT) / 16, LOGT < V2_LOG_TILE ? 2 : 1)
nufft2_cols_list_kernel(const double2* __restrict__ G, double2* __restrict__ T, int n1max,
                        const double2* __restrict__ tw_a, const double2* __restrict__ t_hi,
                        const double2* __restrict__ t_lo, V2Count nc) {
  LKB_DYN_SMEM(double2, buf);
  const int64_t ntr = v2_count(nc, (int)gridDim.y);
  for (int64_t lc = blockIdx.y; lc < ntr; lc += gridDim.y) {
    __syncthreads();
    v2_cols_list_one<PA, LOGT>(buf, G, T, n1max, tw_a, t_hi, t_lo, lc);
  }
}

// ---- rows + finish -----------------------------------------------------------------------------------------------
// Folded per-frequency table (built once per call, y-independent): with G d = (C + i S) of a light curve at bin j,
//   yc + i ys = E d1 + O d2 - ysum c2,   power = yc^2 wz + ys^2 ww
//   d1 = dec conj(tau),  d2 = exp(2 pi i kk / M) d1,  c2 = (Ctau, Stau),  (wz, ww) = 1 / (2 N CC'), 1 / (2 N SS')
struct V2FTab {
  float4 d;       // d1.x, d1.y, d2.x, d2.y
  float4 c;       // c2.x, c2.y, wz, ww
};
struct V2Finish {
  const V2FTab* ftab;      // [F]
  int64_t k0, F, k_lo;
  const float* ysum;       // [B]
  float Nf;
  int normalization;
  float scale;
  float* power;            // [B, F]
  unsigned* peak;          // [B] or NULL: running maximum of the psd-scaled power of a light curve (float bits)
  const int* lcmap;        // NULL: blockIdx.y is the light curve; else the light curve of transform blockIdx.y
  int log2M;               // (double-precision finish: exp(2 pi i kk / M) is evaluated, not tabulated)
};

__device__ __forceinline__ float v2_normalise(float pw, float Nf, int normalization, float scale) {
  if (normalization == LKB_LS_NORM_PSD_SCALE) return pw * scale;
  if (normalization == LKB_LS_NORM_AMPLITUDE) return sqrtf(pw * (4.0f / Nf));
  return pw;
}
// psd-scaled power (before the normalisation) of one bin from the modes k (g1) and Mh - k (g2) of the packed transform
__device__ __forceinline__ float v2_finish_pw(float2 g1, float2 g2, const V2FTab tb, float ysum, int64_t, int) {
  const float ex = 0.5f * (g1.x + g2.x), ey = 0.5f * (g1.y - g2.y);        // E = (g1 + conj g2) / 2
  const float ox = 0.5f * (g1.y + g2.y), oy = 0.5f * (g2.x - g1.x);        // O = (g1 - conj g2) / 2i
  const float yc = ex * tb.d.x - ey * tb.d.y + ox * tb.d.z - oy * tb.d.w - ysum * tb.c.x;
  const float ys = ex * tb.d.y + ey * tb.d.x + ox * tb.d.w + oy * tb.d.z - ysum * tb.c.y;
  return yc * yc * tb.c.z + ys * ys * tb.c.w;
}
// the same in double precision: G = E + exp(2 pi i kk / M) O first (E and O can be orders of magnitude above G - the
// mirror image of a strong line), then the fp32 table's d1 and window terms
__device__ __forceinline__ float v2_finish_pw(double2 g1, double2 g2, const V2FTab tb, float ysum, int64_t kk, int log2M) {
  const double ex = 0.5 * (g1.x + g2.x), ey = 0.5 * (g1.y - g2.y);
  const double ox = 0.5 * (g1.y + g2.y), oy = 0.5 * (g2.x - g1.x);
  double sw, cw;
  sincospi(ldexp((double)kk, 1 - log2M), &sw, &cw);
  const double gx = ex + cw * ox - sw * oy, gy = ey + cw * oy + sw * ox;
  const double yc = gx * (double)tb.d.x - gy * (double)tb.d.y - (double)ysum * (double)tb.c.x;
  const double ys = gx * (double)tb.d.y + gy * (double)tb.d.x - (double)ysum * (double)tb.c.y;
  return (float)(yc * yc * (double)tb.c.z + ys * ys * (double)tb.c.w);
}

// MODE 1: finish -> power.  MODE 2: the modes k < nk2_keep * A and their mirrors Mh - k go to Zout [B][Mh] in natural
// order (the ragged finish kernel reads them there).  One transform (slot lc; lc_base + lc indexes fa.lcmap).
// Rows per half: R = 2^LOGT / (2 Bc) (8 in float2, 4 in double2); 2 R slots of Bc points fill the tile.
template <int PA, int MODE, class CT, int LOGT = V2_LOG_TILE>
__device__ __forceinline__ void v2_rows_one(CT* buf, const CT* __restrict__ T, const CT* __restrict__ tw_b,
                                            const V2Finish& fa, CT* __restrict__ Zout, int nk2_keep, const int64_t lc,
                                            const int lc_base, const int g) {
  constexpr int NT = (1 << LOGT) / 16, R = (1 << LOGT) / (2 * V2_BC), LR = v2_log2i(R);
  constexpr int A = 1 << PA, PTC = LOGT - PA, TC = 1 << PTC, LS = V2_LSB, Bc = V2_BC;
  static_assert((1 << LR) == R, "geometry");
  const int t = (int)threadIdx.x;
  const bool last = g == (A / (2 * R)) - 1;
  const int64_t Mh = (int64_t)1 << (PA + V2_PB);
  auto slot_k1 = [&](int s) -> int {
    const int h = s >> LR, r = s & (R - 1);
    if (h == 0) return 1 + g * R + r;
    if (last && r == 0) return 0;                    // instead of a second copy of row A / 2
    return A - (g + 1) * R + r;
  };
  const CT* Tp = T + lc * Mh;
#pragma unroll
  for (int u = 0; u < 16; ++u) {
    const int e = t + NT * u;
    const int j = e & (TC - 1), r = (e >> PTC) & (R - 1), h = (e >> (PTC + LR)) & 1, c = e >> (PTC + LR + 1);
    const int s = h * R + r;
    buf[s * LS + v2_skew((c << PTC) + j)] = Tp[(((c << PA) + slot_k1(s)) << PTC) + j];
  }
  __syncthreads();
  v2_pass_t<V2_PB, LS, 0, 1, CT, NT>(buf, tw_b);
  // one slot per thread for all its items: s = t % 2R, k2 = t / 2R + KSTEP u
  constexpr int KSTEP = NT / (2 * R);
  const int s = t & (2 * R - 1), h = s >> LR, r = s & (R - 1), k1 = slot_k1(s);
  if (MODE == 2) {
    const int keep = nk2_keep < Bc / 2 ? nk2_keep : Bc / 2;
    for (int q = t >> (LR + 1); q < 2 * keep; q += KSTEP) {
      const int k2 = q < keep ? q : Bc - 2 * keep + q;          // [0, keep) and [Bc - keep, Bc)
      Zout[lc * Mh + k1 + ((int64_t)k2 << PA)] = buf[s * LS + v2_skew(k2)];
    }
  } else {
  int ps = (1 - h) * R + (R - 1 - r);                              // mode Mh - k: row A - k1, column Bc - 1 - k2
  bool row0 = false;
  if (last && h == 0 && r == R - 1) ps = s;                        // row A / 2 mirrors onto itself
  if (last && h == 1 && r == 0) { ps = s; row0 = true; }           // row 0: column (Bc - k2) mod Bc
  int64_t nK2 = ((fa.k0 + fa.F - 1) >> PA) + 1;
  if (nK2 > Bc) nK2 = Bc;
  const int64_t lcd = fa.lcmap ? (int64_t)fa.lcmap[lc_base + lc] : lc;   // the light curve whose flux this transform holds
  const float ys0 = fa.ysum[lcd];
  float* prow = fa.power + lcd * fa.F;
  const int64_t jbase = (int64_t)k1 - fa.k0;
  float pmax = 0.0f;
  constexpr int UB = 4;                                            // items of a thread: k2 = t / 2R + KSTEP u
  for (int k2b = t >> (LR + 1); k2b < (int)nK2; k2b += KSTEP * UB) {
    V2FTab tb[UB];
    int64_t jj[UB];
    bool valid[UB];
#pragma unroll
    for (int u = 0; u < UB; ++u) {                                 // all table loads of the batch in flight together
      const int k2 = k2b + KSTEP * u;
      jj[u] = jbase + ((int64_t)k2 << PA);
      valid[u] = k2 < (int)nK2 && jj[u] >= fa.k_lo && jj[u] < fa.F;
      if (valid[u]) tb[u] = fa.ftab[jj[u]];
    }
#pragma unroll
    for (int u = 0; u < UB; ++u) {
      if (!valid[u]) continue;
      const int k2 = k2b + KSTEP * u;
      const int pi = row0 ? ((Bc - k2) & (Bc - 1)) : (Bc - 1 - k2);
      const CT g1 = buf[s * LS + v2_skew(k2)], g2 = buf[ps * LS + v2_skew(pi)];
      const float pw = v2_finish_pw(g1, g2, tb[u], ys0, fa.k0 + jj[u], fa.log2M);
      pmax = fmaxf(pmax, pw);
      prow[jj[u]] = v2_normalise(pw, fa.Nf, fa.normalization, fa.scale);
    }
  }
  if (fa.peak) {                                                   // (power >= 0: float bits order as unsigned)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) pmax = fmaxf(pmax, __shfl_xor_sync(0xffffffffu, pmax, o));
    if ((t & 31) == 0 && pmax > 0.0f) atomicMax(fa.peak + lcd, __float_as_uint(pmax));
  }
  }
}

// grid (A / 16, B): one transform per CTA (no extra parameters: see nufft2_cols_kernel).  (Tried: the light curve as
// the FAST block index, so that the CTAs in flight share one 100 KB slice of the finish table - slower: the tile
// reads of many different light curves scatter over DRAM pages, which costs more than the table locality gains.)
template <int PA, int MODE, class CT = float2>
__global__ void __launch_bounds__(V2_THREADS, sizeof(CT) == 8 ? 2 : 1)
nufft2_rows_kernel(const CT* __restrict__ T, const CT* __restrict__ tw_b, V2Finish fa, CT* __restrict__ Zout,
                   int nk2_keep) {
  LKB_DYN_SMEM(CT, buf);
  v2_rows_one<PA, MODE, CT>(buf, T, tw_b, fa, Zout, nk2_keep, (int64_t)blockIdx.y, 0, (int)blockIdx.x);
}
// escalation pass (double precision, finish mode, tiles of 2^v2_log_tile(PA, true) points): blocks stride over a
// device-side count of transforms; transform slot lc holds light curve fa.lcmap[nc.base + lc].  (A call per transform,
// as in nufft2_cols_list_kernel: no spills.)
template <int PA, int LOGT>
__device__ __noinline__ void v2_rows_list_one(double2* buf, const double2* __restrict__ T,
                                              const double2* __restrict__ tw_b, const V2Finish fa, const int64_t lc,
                                              const int lc_base) {
  v2_rows_one<PA, 1, double2, LOGT>(buf, T, tw_b, fa, nullptr, 0, lc, lc_base, (int)blockIdx.x);
}
template <int PA, int LOGT = v2_log_tile(PA, true)>
__global__ void __launch_bounds__((1 << LOGT) / 16, LOGT < V2_LOG_TILE ? 2 : 1)
nufft2_rows_list_kernel(const double2* __restrict__ T, const double2* __restrict__ tw_b, V2Finish fa, V2Count nc) {
  LKB_DYN_SMEM(double2, buf);
  const int64_t ntr = v2_count(nc, (int)gridDim.y);
  for (int64_t lc = blockIdx.y; lc < ntr; lc += gridDim.y) {
    __syncthreads();
    v2_rows_list_one<PA, LOGT>(buf, T, tw_b, fa, lc, nc.base);
  }
}

// ---- precision escalation -------------------------------------------------------------------------------------
// The fp32 transform's rounding noise is proportional to the LARGEST component of a light curve, wherever it lies - for
// instance a strong line above the frequency grid's upper end - while the parity tolerance is relative to the highest
// peak INSIDE the grid.  Measured on config C2 (tools/worst_bins.py): worst bin at 1.09x the tolerance, on light
// curves whose flux excursion is > 1000x their in-band peak amplitude; a generic fp32 NUFFT (pocketfft single precision)
// shows the same noise floor.  So the finish records every light curve's in-band peak, light curves with
//     max |y - mean| > ratio * (in-band peak amplitude)
// are listed, and the listed ones are transformed again in double precision (same kernels, double2 instantiation).
__global__ void nufft2_flag_kernel(const unsigned* __restrict__ peak, const float* __restrict__ absmax, int B, float Nf,
                                   float ratio, int* __restrict__ count, int* __restrict__ list, int* __restrict__ total) {
  const int b = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  bool f = false;
  if (b < B) {
    const float amp = sqrtf(__uint_as_float(peak[b]) * (4.0f / Nf));
    f = absmax[b] > ratio * amp;
  }
  const unsigned bal = __ballot_sync(0xffffffffu, f);
  if (bal) {
    int base = 0;
    if ((threadIdx.x & 31) == 0) {
      base = atomicAdd(count, __popc(bal));
      if (total) atomicAdd(total, __popc(bal));
    }
    base = __shfl_sync(0xffffffffu, base, 0);
    if (f) list[base + __popc(bal & ((1u << (threadIdx.x & 31)) - 1u))] = b;
  }
}

// double-precision fine grids of the listed light curves: G[i][e] for light curve list[nc.base + i], in the layout of
// the double-precision column kernel (ptc = its log2 columns per CTA).  One thread = one z cell of LCS_D listed light
// curves, which share the cell's cadence range and kernel weights (the sums of each light curve run in cadence order,
// as with one light curve per thread); grid (cells / 256, gy), blocks stride over the listed light curves.
constexpr int LCS_D = 4;
__global__ void __launch_bounds__(256)
nufft2_spread_list_kernel(const int32_t* __restrict__ first_ge, const nufft::Cad* __restrict__ cad,
                          const double* __restrict__ Wt, const float* __restrict__ y, int64_t ystride,
                          const int* __restrict__ list, int w, int p, int ptc, int n1max, double2* __restrict__ G,
                          V2Count nc) {
  const int64_t cells = (int64_t)n1max << V2_PB;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= cells) return;
  const int64_t M = (int64_t)1 << p, m = 2 * v2_zcell_of(e, ptc, n1max);
  const int64_t L = nufft::table_len(M, w);
  const int ntr = v2_count(nc, (int)gridDim.y * LCS_D);
  for (int i0 = (int)blockIdx.y * LCS_D; i0 < ntr; i0 += (int)gridDim.y * LCS_D) {
    const float* yr[LCS_D];
#pragma unroll
    for (int q = 0; q < LCS_D; ++q) {
      const int i = (i0 + q < ntr) ? i0 + q : ntr - 1;          // clamped slots are computed and dropped
      yr[q] = y + (int64_t)list[nc.base + i] * ystride;
    }
    double a0[LCS_D], a1[LCS_D];
#pragma unroll
    for (int q = 0; q < LCS_D; ++q) { a0[q] = 0.0; a1[q] = 0.0; }
    for (int wrap = 0; wrap < 2; ++wrap) {
      const int64_t mm = m + (int64_t)wrap * M;
      if (mm + 1 >= L) break;
      int64_t lo_c = mm - w + 1, hi_c = mm + 2;
      if (lo_c < 0) lo_c = 0;
      if (hi_c > L - 1) hi_c = L - 1;
      const int32_t na = first_ge[lo_c], nb = first_ge[hi_c];
      for (int32_t n = na; n < nb; ++n) {
        const int tap = (int)(mm - (int64_t)cad[n].i0);
        const double* wr = Wt + (int64_t)n * w;
        const double w0 = (tap >= 0) ? wr[tap] : 0.0, w1 = (tap + 1 < w) ? wr[tap + 1] : 0.0;
#pragma unroll
        for (int q = 0; q < LCS_D; ++q) {
          const double v = (double)yr[q][n];
          a0[q] = fma(w0, v, a0[q]);
          a1[q] = fma(w1, v, a1[q]);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < LCS_D; ++q)
      if (i0 + q < ntr) G[(int64_t)(i0 + q) * cells + e] = make_double2(a0[q], a1[q]);
  }
}

// ---- launch helpers ------------------------------------------------------------------------------------------------
inline unsigned v2_blocks_for(int64_t n, int per) { return (unsigned)((n + per - 1) / per); }

template <class CT>
struct V2TablesT {
  const CT *tw_a, *tw_b, *t_hi, *t_lo;
};
typedef V2TablesT<float2> V2Tables;
typedef V2TablesT<double2> V2TablesD;
// twiddle tables of the transform of 2^p real cells in workspace slot `slot`
template <class CT>
inline int v2_tables(int p, int slot, cudaStream_t st, V2TablesT<CT>* out) {
  const int ph = p - 1, pa = ph - V2_PB, pl = nufft::v2_log2_lo(ph);
  const int la = nufft::v2_pass_table_len(pa), lb = nufft::v2_pass_table_len(V2_PB), nhi = 1 << (ph - pl), nlo = 1 << pl;
  CT* base = nullptr;
  LKB_TRY(ws_get_t<CT>(slot, (size_t)(la + lb + nhi + nlo + 4), &base));
  CT *tw_a = base, *tw_b = base + la, *t_hi = tw_b + lb, *t_lo = t_hi + nhi;
  LKB_LAUNCH(v2_blocks_for(la + lb + nhi + nlo, 256), 256, st, nufft2_tables_kernel<CT>)(pa, V2_PB, ph, tw_a, tw_b, t_hi, t_lo);
  LKB_LAUNCH_CHECK();
  out->tw_a = tw_a; out->tw_b = tw_b; out->t_hi = t_hi; out->t_lo = t_lo;
  return LKB_OK;
}
// rows n1 of the [A][Bc] grid of z cells that cadences can reach when the last one's support starts at cell i0_last
inline int v2_n1max(int p, int64_t i0_last, int w) {
  const int64_t M = (int64_t)1 << p, A = (M / 2) >> V2_PB;
  const int64_t reach = i0_last + w + 1;                   // fine-grid cells [0, reach) (a support past M wraps to 0)
  if (reach >= M) return (int)A;
  const int64_t n = ((reach + 1) / 2 + V2_BC - 1) >> V2_PB;
  return (int)(n < 1 ? 1 : (n > A ? A : n));
}
inline bool v2_supported(int p) { return p >= V2R_P_MIN && p <= V2R_P_MAX; }

template <int PA, class CT>
int v2_cols_pa(const CT* G, CT* T, int n1max, int B, const V2TablesT<CT>& tb, cudaStream_t st, V2Count nc) {
  constexpr int LOGT = v2_log_tile(PA, sizeof(CT) == 16), A = 1 << PA, TC = (1 << LOGT) / A;
  const size_t smem = (size_t)TC * (A + A / 16 + 1) * sizeof(CT);
  const dim3 grid((unsigned)(V2_BC / TC), (unsigned)B);
  if constexpr (sizeof(CT) == 16) {          // the escalation pass: always with a device-side count
    LKB_CUDA_CHECK(cudaFuncSetAttribute(nufft2_cols_list_kernel<PA>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    LKB_LAUNCH_SMEM(grid, (1 << LOGT) / 16, smem, st, nufft2_cols_list_kernel<PA>)(G, T, n1max, tb.tw_a, tb.t_hi, tb.t_lo, nc);
  } else {
    LKB_CUDA_CHECK(cudaFuncSetAttribute(nufft2_cols_kernel<PA, CT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    LKB_LAUNCH_SMEM(grid, V2_THREADS, smem, st, nufft2_cols_kernel<PA, CT>)(G, T, n1max, tb.tw_a, tb.t_hi, tb.t_lo);
  }
  LKB_LAUNCH_CHECK();
  return LKB_OK;
}
template <int PA, class CT>
int v2_rows_pa(const CT* T, int B, const V2TablesT<CT>& tb, const V2Finish* fa, CT* Zout, int nk2_keep, cudaStream_t st,
               V2Count nc) {
  constexpr int LOGT = v2_log_tile(PA, sizeof(CT) == 16), R = (1 << LOGT) / (2 * V2_BC);
  const size_t smem = (size_t)(2 * R) * V2_LSB * sizeof(CT);
  const dim3 grid((unsigned)((1 << PA) / (2 * R)), (unsigned)B);
  if constexpr (sizeof(CT) == 16) {          // the escalation pass: always with a device-side count, finish mode
    LKB_CUDA_CHECK(cudaFuncSetAttribute(nufft2_rows_list_kernel<PA>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    LKB_LAUNCH_SMEM(grid, (1 << LOGT) / 16, smem, st, nufft2_rows_list_kernel<PA>)(T, tb.tw_b, *fa, nc);
  } else {
    LKB_CUDA_CHECK(cudaFuncSetAttribute(nufft2_rows_kernel<PA, 1, CT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    LKB_CUDA_CHECK(cudaFuncSetAttribute(nufft2_rows_kernel<PA, 2, CT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (fa) LKB_LAUNCH_SMEM(grid, V2_THREADS, smem, st, nufft2_rows_kernel<PA, 1, CT>)(T, tb.tw_b, *fa, nullptr, 0);
    else LKB_LAUNCH_SMEM(grid, V2_THREADS, smem, st, nufft2_rows_kernel<PA, 2, CT>)(T, tb.tw_b, V2Finish(), Zout, nk2_keep);
  }
  LKB_LAUNCH_CHECK();
  return LKB_OK;
}
#define V2_DISPATCH_PA(pa, CALL)                                                                       \
  switch (pa) {                                                                                         \
    case 4: return CALL(4); case 5: return CALL(5); case 6: return CALL(6); case 7: return CALL(7);      \
    case 8: return CALL(8); case 9: return CALL(9); case 10: return CALL(10); case 11: return CALL(11);  \
    case 12: return CALL(12); case 13: return CALL(13);                                                  \
    default: set_error("NUFFT v2: fine grid of 2^%d cells out of range", (pa) + V2_PB + 1); return LKB_E_UNSUPPORTED; \
  }
// G -> T for B transforms of 2^p real cells
template <class CT>
inline int v2_cols(const CT* G, CT* T, int p, int n1max, int B, const V2TablesT<CT>& tb, cudaStream_t st,
                   V2Count nc = V2Count{nullptr, 0, 0}) {
#define V2_CALL(PA) v2_cols_pa<PA, CT>(G, T, n1max, B, tb, st, nc)
  V2_DISPATCH_PA(p - 1 - V2_PB, V2_CALL)
#undef V2_CALL
}
// T -> power (fa != NULL) or -> Zout in natural order, modes k < nk2_keep * A and their mirrors
template <class CT>
inline int v2_rows(const CT* T, int p, int B, const V2TablesT<CT>& tb, const V2Finish* fa, CT* Zout, int nk2_keep,
                   cudaStream_t st, V2Count nc = V2Count{nullptr, 0, 0}) {
#define V2_CALL(PA) v2_rows_pa<PA, CT>(T, B, tb, fa, Zout, nk2_keep, st, nc)
  V2_DISPATCH_PA(p - 1 - V2_PB, V2_CALL)
#undef V2_CALL
}

}  // namespace
}  // namespace lkb
