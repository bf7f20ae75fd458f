// liblkb200 - shared-grid Lomb-Scargle by a type-1 NUFFT (LKB_LS_ALGO_NUFFT; OPT-IN in round 1: written and
// verified on the CPU through tests/native/nufft_host_harness.cpp after the round's GPU budget was spent -
// `auto` never selects it until it has been measured on hardware).
//
// Why: the contraction kernels (ls_tc.cu, ls.cu) do 4 N F flops per light curve; on a REGULAR frequency grid
// the same trig sums are the Fourier coefficients of the (non-uniformly sampled) light curve, which a
// spreading step + one FFT give in N w + 2.5 M log2 M flops (config 2: 5e7 instead of 2.6e10 per light curve),
// within 0.02-0.16 of the parity tolerance in fp32 (tools/nufft_ls_model.py) - more accurate than the
// split-fp16 tensor path (0.47).  The whole batch becomes an HBM sweep: fine grids [B/2, M] complex64.
// This is the algorithm behind the reference's optional ls_method="fastnifty" (nifty-ls / finufft,
// /root/reference/pyproject.toml:48, src/lightkurve/periodogram.py:917-946).
//
// Kernels (all "one thread = one function of nufft_core.h"):
//   nufft_cad_kernel        per cadence: leftmost cell + offset of its kernel support on the M-cell grid
//   nufft_first_ge_kernel   per cell: first cadence whose support starts at or after it (binary search)
//   nufft_spread_kernel     per (cell, pair of light curves): gather of the cadences reaching the cell
//   nufft_fft_pass_kernel   per butterfly: out-of-place Stockham pass of radix 16/8/4/2
//   nufft_deconv_kernel     per mode: 1 / phihat and the grid-shift phase
//   nufft_rot_kernel        per frequency: window terms (tau rotation, 1/CC', 1/SS') from the transform of
//                           a_n = 1 on a grid twice as fine (modes kk and 2 kk)
//   nufft_lowrows_kernel    per (low frequency, light curve): direct fp32/fp64 sums with the cos-1 design matrix
//                           for f * baseline <= LS_LOWF_CYCLES (the rows whose sums cancel)
//   nufft_finish_kernel     per (frequency, pair): unpack the two light curves, deconvolve, epilogue -> power
// HBM traffic at config 2 (B = 1024, M = 2^19): spread 2.1 GB written, 5 passes x 4.3 GB, finish ~1 GB read +
// 0.4 GB written  ~ 25 GB  ~ 4 ms at the measured 6.6 TB/s.  Next steps once measured: fuse the spreading into
// the first pass (80 % of its input is zero for oversample 5), shared-memory passes (2 instead of 5 sweeps).
#include <algorithm>

#include "common.cuh"
#include "ls_common.cuh"
#include "nufft_core.h"
#include "nufft_v2.cuh"

namespace lkb {

using nufft::Cad;

namespace {

constexpr int GL_NQ = 48;
struct GlNodes {
  double x[GL_NQ], w[GL_NQ];
};

__global__ void nufft_cad_kernel(const double* __restrict__ t, int64_t N, double df, int64_t M, int w,
                                 Cad* __restrict__ cad, int* __restrict__ unsorted) {
  const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  cad[n] = nufft::cad_entry(t[n], df, M, w);
  if (n > 0 && t[n] < t[n - 1]) *unsorted = 1;
  if (t[n] < 0.0) *unsorted = 1;
}

__global__ void nufft_first_ge_kernel(const Cad* __restrict__ cad, int64_t N, int64_t L, int32_t* __restrict__ first_ge) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c < L) first_ge[c] = nufft::first_ge_entry(c, cad, N);
}

// Z[pair][m] = sum over cadences of phi * (y[2 pair][n] + i y[2 pair + 1][n])
__global__ void __launch_bounds__(256)
nufft_spread_kernel(const int32_t* __restrict__ first_ge, const Cad* __restrict__ cad, const float* __restrict__ y,
                    int64_t ystride, const float* __restrict__ absmax, int B, int npairs, int w, float beta, int log2M,
                    float2* __restrict__ Z) {
  const int64_t M = (int64_t)1 << log2M;
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= (int64_t)npairs << log2M) return;
  const int64_t pair = gid >> log2M, m = gid & (M - 1);
  const float* y0 = y + (2 * pair) * ystride;
  const float* y1 = (2 * pair + 1 < B) ? y0 + ystride : nullptr;
  const float s0 = absmax ? nufft::pow2_scale(absmax[2 * pair]) : 1.0f;
  const float s1 = (absmax && y1) ? nufft::pow2_scale(absmax[2 * pair + 1]) : 1.0f;
  Z[gid] = nufft::spread_cell(m, first_ge, cad, y0, y1, s0, s1, w, beta, M);
}

template <int R, bool CHAIN>
__global__ void __launch_bounds__(256)
nufft_fft_pass_kernel(const float2* __restrict__ x, float2* __restrict__ y, int64_t Ns, int log2M, int64_t total) {
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= total) return;
  const int64_t M = (int64_t)1 << log2M, per = M / R;
  const int64_t pair = gid / per, i = gid - pair * per;
  nufft::fft_pass_butterfly<R, CHAIN>(x + pair * M, y + pair * M, i, Ns, M);
}

template <bool CHAIN>
void launch_pass(int R, unsigned g, const float2* src, float2* dst, int64_t Ns, int p, int64_t total, cudaStream_t st) {
  if (R == 16) LKB_LAUNCH(g, 256, st, nufft_fft_pass_kernel<16, CHAIN>)(src, dst, Ns, p, total);
  else if (R == 8) LKB_LAUNCH(g, 256, st, nufft_fft_pass_kernel<8, CHAIN>)(src, dst, Ns, p, total);
  else if (R == 4) LKB_LAUNCH(g, 256, st, nufft_fft_pass_kernel<4, CHAIN>)(src, dst, Ns, p, total);
  else LKB_LAUNCH(g, 256, st, nufft_fft_pass_kernel<2, CHAIN>)(src, dst, Ns, p, total);
}

// ---- four-step transform with shared-memory sub-transforms (LKB_NUFFT_FFT=smem): two in-place global sweeps ----
// nufft_core.h "four-step transform".  One CTA = a tile of TC columns (step 1) or TR rows (step 2) of one transform
// in two skewed shared-memory buffers; the radix passes are the same butterflies as the global version.
constexpr int FS_THREADS = 256;
// float2 elements per shared-memory buffer (before skew padding): 4096 -> 2 x 34 KB per CTA, 3 CTAs per SM;
// LKB_NUFFT_TILE overrides (power of two, up to 8192)
inline int64_t fs_tile() {
  int64_t v = 4096;
  if (const char* e = getenv("LKB_NUFFT_TILE")) v = atoll(e);
  if (v < 256) v = 256;
  if (v > 8192) v = 8192;
  int64_t p2 = 256;
  while (p2 * 2 <= v) p2 *= 2;
  return p2;
}

template <bool CHAIN>
__device__ __forceinline__ void smem_line_passes(float2*& src, float2*& dst, int lines, int64_t line_stride, int plog2) {
  const int64_t n = (int64_t)1 << plog2;
  int64_t Ns = 1;
  for (int idx = 0;; ++idx) {
    const int R = nufft::fft_pass_radix(plog2, idx);
    if (R == 0) break;
    const int64_t nb = n / R;
    for (int64_t j = threadIdx.x; j < (int64_t)lines * nb; j += blockDim.x) {
      const int64_t c = j / nb, i = j - c * nb;
      const float2* x = src + c * line_stride;
      float2* y = dst + c * line_stride;
      if (R == 16) nufft::fft_pass_butterfly<16, CHAIN, true>(x, y, i, Ns, n);
      else if (R == 8) nufft::fft_pass_butterfly<8, CHAIN, true>(x, y, i, Ns, n);
      else if (R == 4) nufft::fft_pass_butterfly<4, CHAIN, true>(x, y, i, Ns, n);
      else nufft::fft_pass_butterfly<2, CHAIN, true>(x, y, i, Ns, n);
    }
    __syncthreads();
    Ns *= R;
    float2* tmp = src; src = dst; dst = tmp;
  }
}

// step 1: grid (Bc / TC, npairs)
// what the column kernel needs to compute its input cells itself (FUSED: the spreading never touches global memory)
struct SpreadArgs {
  const int32_t* first_ge;
  const Cad* cad;
  const float* y;
  int64_t ystride;
  const float* absmax;
  int B, w;
  float beta;
};

template <bool CHAIN, bool FUSED>
__global__ void __launch_bounds__(FS_THREADS)
nufft_fft_cols_kernel(float2* __restrict__ Z, int p, int pa, int tc, SpreadArgs sp) {
  LKB_DYN_SMEM(float2, smem);
  const int64_t M = (int64_t)1 << p, A = (int64_t)1 << pa, Bc = M >> pa;
  const int64_t stride = nufft::smem_line(A);
  const int64_t pair = blockIdx.y;
  float2* Zp = Z + pair * M;
  const int64_t c0 = (int64_t)blockIdx.x * tc;
  float2 *src = smem, *dst = smem + (int64_t)tc * stride;
  if (FUSED) {
    const float* y0 = sp.y + (2 * pair) * sp.ystride;
    const float* y1 = (2 * pair + 1 < sp.B) ? y0 + sp.ystride : nullptr;
    const float s0 = nufft::pow2_scale(sp.absmax[2 * pair]);
    const float s1 = y1 ? nufft::pow2_scale(sp.absmax[2 * pair + 1]) : 1.0f;
    for (int64_t idx = threadIdx.x; idx < (int64_t)tc * A; idx += blockDim.x) {
      const int64_t c = idx % tc, n1 = idx / tc;
      src[c * stride + nufft::skew(n1)] =
          nufft::spread_cell(n1 * Bc + c0 + c, sp.first_ge, sp.cad, y0, y1, s0, s1, sp.w, sp.beta, M);
    }
  } else {
    for (int64_t idx = threadIdx.x; idx < (int64_t)tc * A; idx += blockDim.x) {
      const int64_t c = idx % tc, n1 = idx / tc;
      src[c * stride + nufft::skew(n1)] = Zp[n1 * Bc + c0 + c];
    }
  }
  __syncthreads();
  smem_line_passes<CHAIN>(src, dst, tc, stride, pa);
  for (int64_t idx = threadIdx.x; idx < (int64_t)tc * A; idx += blockDim.x) {
    const int64_t c = idx % tc, k1 = idx / tc, n2 = c0 + c;
    Zp[k1 * Bc + n2] = nufft::cmul(src[c * stride + nufft::skew(k1)], nufft::unit_phase(n2 * k1, M));
  }
}

// step 2: grid (A / TR, npairs)
template <bool CHAIN>
__global__ void __launch_bounds__(FS_THREADS)
nufft_fft_rows_kernel(float2* __restrict__ Z, int p, int pa, int tr) {
  LKB_DYN_SMEM(float2, smem);
  const int64_t M = (int64_t)1 << p, Bc = M >> pa;
  const int pb = p - pa;
  const int64_t stride = nufft::smem_line(Bc);
  float2* Zp = Z + (int64_t)blockIdx.y * M + (int64_t)blockIdx.x * tr * Bc;
  float2 *src = smem, *dst = smem + (int64_t)tr * stride;
  for (int64_t idx = threadIdx.x; idx < (int64_t)tr * Bc; idx += blockDim.x) {
    const int64_t r = idx / Bc, n2 = idx - r * Bc;
    src[r * stride + nufft::skew(n2)] = Zp[idx];
  }
  __syncthreads();
  smem_line_passes<CHAIN>(src, dst, tr, stride, pb);
  for (int64_t idx = threadIdx.x; idx < (int64_t)tr * Bc; idx += blockDim.x) {
    const int64_t r = idx / Bc, k2 = idx - r * Bc;
    Zp[idx] = src[r * stride + nufft::skew(k2)];
  }
}

__global__ void nufft_deconv_kernel(int64_t k_first, int64_t count, int64_t M, int w, double beta, GlNodes gl,
                                    float2* __restrict__ dec) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  double re, im;
  nufft::deconv_factor(k_first + k, M, w, beta, gl.x, gl.w, GL_NQ, &re, &im);
  dec[k] = make_float2((float)re, (float)im);
}

// window terms of the rows k >= k_lo from the transform Zw (length M2) of unit strengths: mode kk gives
// (C, S) = sum (cos, sin)(2 pi f t), mode 2 kk gives (C2, S2) = sum (cos, sin)(4 pi f t).
// dec2[j] is the deconvolution factor of mode j (j = 0 .. 2 (k0 + F) - 1).
__global__ void nufft_rot_kernel(const float2* __restrict__ Zw, int64_t M2, const float2* __restrict__ dec2, int64_t k0,
                                 int64_t F, int64_t k_lo, double Nd, float4* __restrict__ rot, float2* __restrict__ rot2) {
  const int64_t k = k_lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= F) return;
  const int64_t kk = k0 + k;
  float2 a, unused;
  nufft::unpack_pair(Zw, kk, M2, dec2[kk], 1.0f, 1.0f, &a, &unused);
  float2 a2;
  nufft::unpack_pair(Zw, 2 * kk, M2, dec2[2 * kk], 1.0f, 1.0f, &a2, &unused);
  LsSums<double> d;
  d.zero();
  d.c = (double)a.x;
  d.s = (double)a.y;
  d.cc = 0.5 * (Nd + (double)a2.x);       // sum cos^2 = (N + sum cos 2wt) / 2
  d.sc = 0.5 * (double)a2.y;              // sum sin cos = sum sin 2wt / 2
  double ct, st, cc, ss;
  ls_rotation(d, Nd, ct, st, cc, ss);
  const double kf = 1.0 / (2.0 * Nd);
  rot[k] = make_float4((float)ct, (float)st, (float)(kf / cc), (float)(kf / ss));
  rot2[k] = make_float2((float)((d.c * ct + d.s * st) / Nd), (float)((d.s * ct - d.c * st) / Nd));
}

// rows with f * baseline <= LS_LOWF_CYCLES: direct sums, one warp per (row, light curve); the design matrix
// holds cos - 1 (ls_common.cuh) and rot / rot2 of these rows come from the fp64 path of ls_window_kernel.
__global__ void __launch_bounds__(128)
nufft_lowrows_kernel(const double* __restrict__ t, int64_t N, const float* __restrict__ yc, int64_t ystride, int B,
                     const double* __restrict__ freq, int64_t F_low, int64_t F, const float4* __restrict__ rot,
                     const float2* __restrict__ rot2, const float* __restrict__ ysum, int normalization, float scale,
                     float* __restrict__ power) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t job = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (job >= F_low * B) return;
  const int64_t b = job / F_low, k = job - b * F_low;
  const double fr = freq[k];
  const float* y = yc + b * ystride;
  double ch = 0.0, sh = 0.0;
  for (int64_t c0 = 0; c0 < N; c0 += 32 * 64) {
    float pc = 0.f, ps = 0.f;
    const int64_t c1 = min(N, c0 + (int64_t)32 * 64);
    for (int64_t i = c0 + lane; i < c1; i += 32) {
      float s, cm1;
      ls_sincos_cycles_low(fr * t[i], s, cm1);
      const float v = y[i];
      pc = fmaf(v, cm1, pc);
      ps = fmaf(v, s, ps);
    }
    ch += (double)pc;
    sh += (double)ps;
  }
  ch = warp_sum(ch);
  sh = warp_sum(sh);
  if (lane == 0)
    power[b * F + k] = ls_epilogue_shared((float)ch, (float)sh, rot[k], rot2[k], ysum[b], (float)N, normalization,
                                          scale, true);
}

__global__ void __launch_bounds__(256)
nufft_finish_kernel(const float2* __restrict__ Z, int log2M, const float2* __restrict__ dec, int64_t k0, int64_t F,
                    int64_t k_lo, const float4* __restrict__ rot, const float2* __restrict__ rot2,
                    const float* __restrict__ ysum, const float* __restrict__ absmax, float Nf, int normalization,
                    float scale, int B, int npairs, int pa, float* __restrict__ power) {
  const int64_t nk = F - k_lo;
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= nk * npairs) return;
  const int64_t pair = gid / nk, k = k_lo + (gid - pair * nk);
  const int64_t M = (int64_t)1 << log2M;
  const int64_t b0 = 2 * pair;
  const float inv0 = 1.0f / nufft::pow2_scale(absmax[b0]);
  const float inv1 = (b0 + 1 < B) ? 1.0f / nufft::pow2_scale(absmax[b0 + 1]) : 1.0f;
  float2 a, b;
  nufft::unpack_pair(Z + pair * M, k0 + k, M, dec[k], inv0, inv1, &a, &b, pa);
  const float4 r = rot[k];
  const float2 r2 = rot2[k];
  power[b0 * F + k] = ls_epilogue_shared(a.x, a.y, r, r2, ysum[b0], Nf, normalization, scale);
  if (b0 + 1 < B) power[(b0 + 1) * F + k] = ls_epilogue_shared(b.x, b.y, r, r2, ysum[b0 + 1], Nf, normalization, scale);
}

// Self-check (LKB_NUFFT_VERIFY=1): 64 warps each pick one (light curve, frequency row >= k_lo) by a hash, recompute
// the two trig sums directly in fp64 and compare them with what the transform delivered; the largest deviation in
// units of 1e-7 * sum |y| goes to *worst (a correct transform stays below ~5, a defect gives >> 100).
__global__ void __launch_bounds__(128)
nufft_verify_kernel(const float2* __restrict__ Z, int log2M, int pa, const float2* __restrict__ dec, int64_t k0, int64_t F,
                    int64_t k_lo, const double* __restrict__ t, int64_t N, const float* __restrict__ yc, int64_t ystride,
                    const float* __restrict__ absmax, const double* __restrict__ freq, int B, float fault,
                    unsigned* __restrict__ worst) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned job = blockIdx.x * (blockDim.x >> 5) + warp;
  unsigned h = job * 2654435761u + 12345u;
  h ^= h >> 15; h *= 2246822519u; h ^= h >> 13;
  const int64_t b = h % (unsigned)B;
  const int64_t k = k_lo + (int64_t)((h >> 8) % (unsigned)(F - k_lo));
  const float* y = yc + b * ystride;
  const double fr = freq[k];
  double c = 0.0, s = 0.0, l1 = 0.0;
  for (int64_t i = lane; i < N; i += 32) {
    double sn, cs;
    ls_sincos_cycles_f64(fr * t[i], sn, cs);
    const double v = (double)y[i];
    c += v * cs;
    s += v * sn;
    l1 += fabs(v);
  }
  c = warp_sum(c);
  s = warp_sum(s);
  l1 = warp_sum(l1);
  if (lane == 0) {
    const int64_t M = (int64_t)1 << log2M, pair = b >> 1;
    const int64_t b0 = 2 * pair;
    const float inv0 = 1.0f / nufft::pow2_scale(absmax[b0]);
    const float inv1 = (b0 + 1 < B) ? 1.0f / nufft::pow2_scale(absmax[b0 + 1]) : 1.0f;
    float2 ha, hb;
    nufft::unpack_pair(Z + pair * M, k0 + k, M, dec[k], inv0, inv1, &ha, &hb, pa);
    const float2 got = (b & 1) ? hb : ha;
    const double dev = fmax(fabs((double)got.x * (double)fault - c), fabs((double)got.y * (double)fault - s));
    const double units = dev / (1e-7 * fmax(l1, 1e-300));
    atomicMax(worst, (unsigned)fmin(units, 4.0e9));
  }
}

// ---- y-independent tables of the v2 path (built in ls_nufft_prepare) ----------------------------------------------
// folded finish table of the rows k >= k_lo (nufft_v2.cuh V2FTab): deconvolution factor x tau rotation, the same
// times exp(2 pi i kk / M), (Ctau, Stau), 1 / (2 N CC'), 1 / (2 N SS')
__global__ void nufft2_ftab_kernel(const float4* __restrict__ rot, const float2* __restrict__ rot2, int64_t k0, int64_t F,
                                   int64_t k_lo, int64_t M, int w, double beta, GlNodes gl, V2FTab* __restrict__ ftab) {
  const int64_t k = k_lo + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= F) return;
  const int64_t kk = k0 + k;
  double dre, dim;
  nufft::deconv_factor(kk, M, w, beta, gl.x, gl.w, GL_NQ, &dre, &dim);
  const float4 r = rot[k];
  const float2 r2 = rot2[k];
  const double ct = (double)r.x, st = (double)r.y;
  const double d1x = dre * ct + dim * st, d1y = dim * ct - dre * st;            // dec * (ct - i st)
  double ws, wc;
  sincospi(2.0 * (double)kk / (double)M, &ws, &wc);
  V2FTab o;
  o.d = make_float4((float)d1x, (float)d1y, (float)(d1x * wc - d1y * ws), (float)(d1x * ws + d1y * wc));
  o.c = make_float4(r2.x, r2.y, r.z, r.w);
  ftab[k] = o;
}

// design matrix of the low rows (f * baseline <= LS_LOWF_CYCLES): D[r][n] = (cos - 1, sin)(2 pi f_r t_n), zero padding
__global__ void nufft2_lowtab_kernel(const double* __restrict__ t, int64_t N, int64_t Npad, const double* __restrict__ freq,
                                     int F_low, float2* __restrict__ D) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (int64_t)F_low * Npad) return;
  const int r = (int)(e / Npad);
  const int64_t n = e - (int64_t)r * Npad;
  float sn = 0.f, cm1 = 0.f;
  if (n < N) ls_sincos_cycles_low(freq[r] * t[n], sn, cm1);
  D[e] = make_float2(cm1, sn);
}

// sums of the low rows: acc[b][r] += sum over this CTA's cadence slice of y_b[n] D[r][n] (fp64 atomics; acc zeroed by
// the caller).  grid (ceil(B / 16), S): one warp = 2 light curves, one CTA = 16 light curves sharing every 256-cadence
// slice of D through shared memory, the cadence range split S ways so that a small batch still fills the SMs (the
// first version walked all cadences in 64 CTAs: 1.9 ms for 11 rows, latency-bound).  Rows in groups of LOWR.
constexpr int LOWR = 12;
__global__ void __launch_bounds__(256, 3)                     // 80 registers, no spills: 3 CTAs per SM
nufft2_lowrows_kernel(const float2* __restrict__ D, int64_t N, int64_t Npad, const float* __restrict__ yc,
                      int64_t ystride, int B, int F_low, int64_t slice, double* __restrict__ acc) {
  __shared__ float2 sD[LOWR][256];
  const int warp = (int)threadIdx.x >> 5, lane = (int)threadIdx.x & 31;
  const int b0 = (int)blockIdx.x * 16 + 2 * warp, b1 = b0 + 1;
  const float* y0 = yc + (int64_t)(b0 < B ? b0 : B - 1) * ystride;
  const float* y1 = yc + (int64_t)(b1 < B ? b1 : B - 1) * ystride;
  const int64_t n_lo = (int64_t)blockIdx.y * slice, n_hi = (n_lo + slice < N) ? n_lo + slice : N;
  for (int r0 = 0; r0 < F_low; r0 += LOWR) {
    const int nr = (F_low - r0 < LOWR) ? F_low - r0 : LOWR;
    float ac0[LOWR], as0[LOWR], ac1[LOWR], as1[LOWR];
#pragma unroll
    for (int r = 0; r < LOWR; ++r) { ac0[r] = as0[r] = ac1[r] = as1[r] = 0.0f; }
    for (int64_t s0 = n_lo; s0 < n_hi; s0 += 256) {               // <= slice / 32 terms per lane in fp32
      // Every load of the step is issued before any arithmetic: the 16 flux values (HBM) and the step's D rows (L2)
      // are in flight together, and the product loop below has no branch to keep the compiler from scheduling so.
      // (With the flux loads inside the product loop behind a per-row `r < nr` test, each of the 8 sub-steps waited
      // for its own HBM round trip: 0.39-0.57 ms at config 2 on an H100 at 700 W, now 0.21 ms.)
      float v0[8], v1[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int64_t n = s0 + lane + 32 * q;
        v0[q] = (n < n_hi) ? y0[n] : 0.0f;
        v1[q] = (n < n_hi) ? y1[n] : 0.0f;
      }
      __syncthreads();
      {
        const int64_t n = s0 + threadIdx.x;
#pragma unroll
        for (int r = 0; r < LOWR; ++r)              // rows past nr are staged as zeros (their sums are not stored)
          sD[r][threadIdx.x] = (r < nr && n < n_hi) ? D[(int64_t)(r0 + r) * Npad + n] : make_float2(0.f, 0.f);
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < 8; ++q) {
#pragma unroll
        for (int r = 0; r < LOWR; ++r) {
          const float2 d = sD[r][lane + 32 * q];
          ac0[r] = fmaf(v0[q], d.x, ac0[r]); as0[r] = fmaf(v0[q], d.y, as0[r]);
          ac1[r] = fmaf(v1[q], d.x, ac1[r]); as1[r] = fmaf(v1[q], d.y, as1[r]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < LOWR; ++r) {
      if (r < nr) {
        const double c0v = warp_sum((double)ac0[r]), s0v = warp_sum((double)as0[r]);
        const double c1v = warp_sum((double)ac1[r]), s1v = warp_sum((double)as1[r]);
        if (lane == 0) {
          if (b0 < B) { atomicAdd(acc + ((int64_t)b0 * F_low + r0 + r) * 2, c0v); atomicAdd(acc + ((int64_t)b0 * F_low + r0 + r) * 2 + 1, s0v); }
          if (b1 < B) { atomicAdd(acc + ((int64_t)b1 * F_low + r0 + r) * 2, c1v); atomicAdd(acc + ((int64_t)b1 * F_low + r0 + r) * 2 + 1, s1v); }
        }
      }
    }
  }
}
// epilogue of the low rows
__global__ void nufft2_lowfinish_kernel(const double* __restrict__ acc, int B, int F_low, int64_t F, int64_t N,
                                        const float4* __restrict__ rot, const float2* __restrict__ rot2,
                                        const float* __restrict__ ysum, int normalization, float scale,
                                        float* __restrict__ power, unsigned* __restrict__ peak) {
  const int e = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (e >= B * F_low) return;
  const int b = e / F_low, k = e - b * F_low;
  const float pw = ls_epilogue_shared((float)acc[2 * (int64_t)e], (float)acc[2 * (int64_t)e + 1], rot[k], rot2[k], ysum[b],
                                      (float)N, LKB_LS_NORM_PSD_RAW, 1.0f, true);
  power[(int64_t)b * F + k] = v2_normalise(pw, (float)N, normalization, scale);
  if (peak && pw > 0.0f) atomicMax(peak + b, __float_as_uint(pw));     // (a handful of rows per light curve)
}

// Escalation pass, low rows: the listed light curves' rows k < F_low once more from direct FP64 sums and the FP64
// floating-mean formula (ls_common.cuh: ls_power_from_sums).  The sines and cosines of a (row, cadence chunk) are
// evaluated once and reused for every listed light curve.  grid (F_low, ceil(N / 2048)), 256 threads.
//   accW [F_low][4]      : sum s, c, c^2, s c                 (y-independent)
//   accY [cap][F_low][2] : sum y s, sum y c                   (slot i = light curve list[base + i])
//   accS [cap]           : sum y
constexpr int LOWX_PER = 8;                               // cadences per thread
constexpr int LOWX_LC = 4;                                // listed light curves per step
__global__ void __launch_bounds__(256)
nufft2_lowacc_kernel(const int* __restrict__ list, V2Count nc, const double* __restrict__ t, int64_t N,
                     const float* __restrict__ yc, int64_t ystride, const double* __restrict__ freq, int F_low,
                     double* __restrict__ accW, double* __restrict__ accY, double* __restrict__ accS) {
  const int ntr = v2_count(nc, 0);
  if (ntr <= 0) return;
  const int k = (int)blockIdx.x, lane = threadIdx.x & 31;
  const int64_t n0 = (int64_t)blockIdx.y * (256 * LOWX_PER) + threadIdx.x;
  const double fr = freq[k];
  double sn[LOWX_PER], cs[LOWX_PER];
  double ws = 0.0, wc = 0.0, wcc = 0.0, wsc = 0.0;
#pragma unroll
  for (int q = 0; q < LOWX_PER; ++q) {
    const int64_t n = n0 + (int64_t)q * 256;
    sn[q] = 0.0; cs[q] = 0.0;
    if (n < N) {
      ls_sincos_cycles_f64(fr * t[n], sn[q], cs[q]);
      ws += sn[q]; wc += cs[q]; wcc += cs[q] * cs[q]; wsc += sn[q] * cs[q];
    }
  }
  ws = warp_sum(ws); wc = warp_sum(wc); wcc = warp_sum(wcc); wsc = warp_sum(wsc);
  if (lane == 0) {
    atomicAdd(accW + 4 * k + 0, ws); atomicAdd(accW + 4 * k + 1, wc);
    atomicAdd(accW + 4 * k + 2, wcc); atomicAdd(accW + 4 * k + 3, wsc);
  }
  // LOWX_LC listed light curves per step, all their flux loads issued before any sum (one light curve per step waited
  // for one HBM round trip per listed light curve: 0.056 ms for 31 of them at config 2 on an H100)
  for (int i0 = 0; i0 < ntr; i0 += LOWX_LC) {
    float v[LOWX_LC][LOWX_PER];
#pragma unroll
    for (int j = 0; j < LOWX_LC; ++j) {
      const float* y = yc + (int64_t)list[nc.base + ((i0 + j < ntr) ? i0 + j : ntr - 1)] * ystride;
#pragma unroll
      for (int q = 0; q < LOWX_PER; ++q) {
        const int64_t n = n0 + (int64_t)q * 256;
        v[j][q] = (n < N) ? y[n] : 0.0f;
      }
    }
#pragma unroll
    for (int j = 0; j < LOWX_LC; ++j) {
      const int i = i0 + j;
      if (i >= ntr) break;                                 // (the same for the whole block)
      double sh = 0.0, ch = 0.0, sy = 0.0;
#pragma unroll
      for (int q = 0; q < LOWX_PER; ++q) {
        const double vq = (double)v[j][q];
        sh = fma(vq, sn[q], sh);
        ch = fma(vq, cs[q], ch);
        sy += vq;
      }
      sh = warp_sum(sh); ch = warp_sum(ch);
      if (k == 0) sy = warp_sum(sy);
      if (lane == 0) {
        atomicAdd(accY + ((int64_t)i * F_low + k) * 2 + 0, sh);
        atomicAdd(accY + ((int64_t)i * F_low + k) * 2 + 1, ch);
        if (k == 0) atomicAdd(accS + i, sy);
      }
    }
  }
}
__global__ void nufft2_lowexact_finish_kernel(const int* __restrict__ list, V2Count nc, const double* __restrict__ accW,
                                              const double* __restrict__ accY, const double* __restrict__ accS,
                                              int F_low, int64_t F, int64_t N, int normalization, float scale,
                                              float* __restrict__ power) {
  const int ntr = v2_count(nc, 0);
  const int e = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (e >= ntr * F_low) return;
  const int i = e / F_low, k = e - i * F_low;
  LsSums<double> d;
  d.sh = accY[2 * (int64_t)e]; d.ch = accY[2 * (int64_t)e + 1];
  d.s = accW[4 * k]; d.c = accW[4 * k + 1]; d.cc = accW[4 * k + 2]; d.sc = accW[4 * k + 3];
  power[(int64_t)list[nc.base + i] * F + k] =
      ls_normalize(ls_power_from_sums(d, (double)N, accS[i]), (double)N, normalization, (double)scale);
}

// Self-check of the v2 path: Zn [nv][Mh] holds the transforms of the first nv light curves in natural order (modes
// below nk2_keep * A and their mirrors); same sampling and units as nufft_verify_kernel.
__global__ void __launch_bounds__(128)
nufft2_verify_kernel(const float2* __restrict__ Zn, int p, const float2* __restrict__ dec, int64_t k0, int64_t F,
                     int64_t k_lo, const double* __restrict__ t, int64_t N, const float* __restrict__ yc, int64_t ystride,
                     const double* __restrict__ freq, int nv, float fault, unsigned* __restrict__ worst) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned job = blockIdx.x * (blockDim.x >> 5) + warp;
  unsigned h = job * 2654435761u + 12345u;
  h ^= h >> 15; h *= 2246822519u; h ^= h >> 13;
  const int64_t b = h % (unsigned)nv;
  const int64_t k = k_lo + (int64_t)((h >> 8) % (unsigned)(F - k_lo));
  const float* y = yc + b * ystride;
  const double fr = freq[k];
  double c = 0.0, s = 0.0, l1 = 0.0;
  for (int64_t i = lane; i < N; i += 32) {
    double sn, cs;
    ls_sincos_cycles_f64(fr * t[i], sn, cs);
    const double v = (double)y[i];
    c += v * cs;
    s += v * sn;
    l1 += fabs(v);
  }
  c = warp_sum(c);
  s = warp_sum(s);
  l1 = warp_sum(l1);
  if (lane == 0) {
    const int64_t M = (int64_t)1 << p, Mh = M >> 1, kk = k0 + k;
    const float2 g1 = Zn[b * Mh + kk], g2 = Zn[b * Mh + ((Mh - kk) & (Mh - 1))];
    const float2 E = make_float2(0.5f * (g1.x + g2.x), 0.5f * (g1.y - g2.y));
    const float2 O = make_float2(0.5f * (g1.y + g2.y), 0.5f * (g2.x - g1.x));
    double wsn, wcs;
    sincospi(2.0 * (double)kk / (double)M, &wsn, &wcs);
    const float2 G = make_float2(E.x + (float)wcs * O.x - (float)wsn * O.y, E.y + (float)wcs * O.y + (float)wsn * O.x);
    const float2 got = nufft::cmul(G, dec[k]);
    const double dev = fmax(fabs((double)got.x * (double)fault - c), fabs((double)got.y * (double)fault - s));
    const double units = dev / (1e-7 * fmax(l1, 1e-300));
    atomicMax(worst, (unsigned)fmin(units, 4.0e9));
  }
}

__global__ void nufft_fill_kernel(float* __restrict__ p, int64_t n, float v) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

inline unsigned blocks_for(int64_t n, int per) { return (unsigned)((n + per - 1) / per); }

// all FFT passes of `npairs` length-2^p transforms; *result points at the buffer holding the output
int fft_passes(float2* a, float2* b, int p, int npairs, cudaStream_t st, float2** result) {
  const int64_t M = (int64_t)1 << p;
  float2 *src = a, *dst = b;
  int64_t Ns = 1;
  const char* ce = getenv("LKB_NUFFT_TWIDDLE_CHAIN");
  const bool chain = ce && atoi(ce) != 0;
  for (int idx = 0;; ++idx) {
    const int R = nufft::fft_pass_radix(p, idx);
    if (R == 0) break;
    const int64_t total = (int64_t)npairs * (M / R);
    const unsigned g = blocks_for(total, 256);
    // LKB_NUFFT_TWIDDLE_CHAIN=1: one sincospif per butterfly + product tree (fewer instructions, 2.5x the rounding
    // error of the transform; off by default until the passes have been profiled)
    if (chain) launch_pass<true>(R, g, src, dst, Ns, p, total, st);
    else launch_pass<false>(R, g, src, dst, Ns, p, total, st);
    LKB_LAUNCH_CHECK();
    Ns *= R;
    float2* tmp = src; src = dst; dst = tmp;
  }
  *result = src;
  return LKB_OK;
}

// LKB_NUFFT_FFT: "smem" = four-step transform in shared memory, "fused" = the same with the spreading done inside
// the column kernel's load phase (the fine grids are written once, already half transformed)
// "v2" (nufft_v2.cuh; default where the fine grid allows it, 2^14 .. 2^23 cells) = one real transform per light
// curve, pruned + tiled, table twiddles, finish fused into the row kernel; "global" = the pair-packed round-1 form
// with one global sweep per radix pass (also the window terms' transform of the shared-grid plan; the single-term flux
// transforms take it only on request, single_term_log2 below).
int fft_mode(int p = 0) {
  const char* e = getenv("LKB_NUFFT_FFT");
  if (e && strcmp(e, "smem") == 0) return 1;
  if (e && strcmp(e, "fused") == 0) return 2;
  if (e && strcmp(e, "global") == 0) return 0;
  return v2_supported(p) ? 3 : 0;
}

// in-place four-step transform of `npairs` length-2^p arrays; result in the [A][Bc] layout (pa returned).
// sp != NULL: the input is not read from Z but spread on the fly from the light curves described by *sp.
template <bool CHAIN>
int fft_fourstep_t(float2* Z, int p, int npairs, cudaStream_t st, int* pa_out, const SpreadArgs* sp) {
  const int pa = nufft::fourstep_pa(p), pb = p - pa;
  const int64_t A = (int64_t)1 << pa, Bc = (int64_t)1 << pb;
  const int tc = (int)std::max<int64_t>(1, std::min<int64_t>(Bc, fs_tile() / A));
  const int tr = (int)std::max<int64_t>(1, std::min<int64_t>(A, fs_tile() / Bc));
  const size_t smem_c = 2 * (size_t)tc * nufft::smem_line(A) * sizeof(float2);
  const size_t smem_r = 2 * (size_t)tr * nufft::smem_line(Bc) * sizeof(float2);
  LKB_CUDA_CHECK(cudaFuncSetAttribute(nufft_fft_cols_kernel<CHAIN, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_c));
  LKB_CUDA_CHECK(cudaFuncSetAttribute(nufft_fft_cols_kernel<CHAIN, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_c));
  LKB_CUDA_CHECK(cudaFuncSetAttribute(nufft_fft_rows_kernel<CHAIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_r));
  const dim3 gc((unsigned)(Bc / tc), (unsigned)npairs);
  if (sp) LKB_LAUNCH_SMEM(gc, FS_THREADS, smem_c, st, nufft_fft_cols_kernel<CHAIN, true>)(Z, p, pa, tc, *sp);
  else LKB_LAUNCH_SMEM(gc, FS_THREADS, smem_c, st, nufft_fft_cols_kernel<CHAIN, false>)(Z, p, pa, tc, SpreadArgs());
  LKB_LAUNCH_CHECK();
  LKB_LAUNCH_SMEM(dim3((unsigned)(A / tr), (unsigned)npairs), FS_THREADS, smem_r, st, nufft_fft_rows_kernel<CHAIN>)(Z, p, pa, tr);
  LKB_LAUNCH_CHECK();
  *pa_out = pa;
  return LKB_OK;
}
int fft_fourstep(float2* Z, int p, int npairs, cudaStream_t st, int* pa_out, const SpreadArgs* sp) {
  const char* ce = getenv("LKB_NUFFT_TWIDDLE_CHAIN");
  return (ce && atoi(ce) != 0) ? fft_fourstep_t<true>(Z, p, npairs, st, pa_out, sp)
                               : fft_fourstep_t<false>(Z, p, npairs, st, pa_out, sp);
}

// Fine-grid size and kernel: upsampling factor >= 2, "exponential of semicircle" kernel of 10 cells, beta = 2.30 w.
//  * Width 8 (round 2's first half) let the aliasing images of a strong line ABOVE the frequency grid (a near-regular
//    cadence repeats the spectrum every 1 / dt) back into the band at 2.5e-8 of its amplitude - 1.5x the tolerance on
//    light curves whose in-band spectrum is 1000x below their variability; width 10 puts it at 3e-10
//    (tools/worst_bins.py, DESIGN.md section 2).
//  * A smaller grid with a wider kernel (upsampling 1.25 .. 2: config 2 would transform 2^18 instead of 2^19 cells
//    with a 14-cell kernel, FP64 model error 2e-12) was tried because the transform is 70 % of the step: in FP32 it is
//    NOT usable here - the deconvolution 1 / phihat(k) grows steeply towards the band edge at low upsampling and
//    amplifies the grid's rounding noise 10x (emulated config-2 light curve: rms error 0.14 of the tolerance instead
//    of 0.015, worst bin 3.3x instead of 1.08x).  LKB_NUFFT_SIGMA=1.25 selects it for experiments; the default is 2.
double upsampling_min() {
  double s = 2.0;
  if (const char* e = getenv("LKB_NUFFT_SIGMA")) s = atof(e);
  return s < 1.25 ? 1.25 : (s > 2.0 ? 2.0 : s);
}
int fine_log2(int64_t kmax_plus_1) { return nufft::fine_grid_log2(kmax_plus_1, upsampling_min()); }
// Flux grid of the single-term transforms (shared and ragged): at least 2^V2R_P_MIN cells, so that every grid takes the
// v2 transform - one real transform per light curve, whose result does not depend on its neighbours in the batch.
// Below 2^14 cells the round-1 form packed two light curves into one complex transform, and the fp32 rounding of a
// loud light curve's peak leaked into its quiet partner (DESIGN.md section 2).  Only the grid grows: sigma =
// min(2, grid_sigma) stays 2, so the kernel width and shape stay those of the smallest grid.  LKB_NUFFT_FFT =
// global / smem / fused asks for the round-1 transforms and keeps their grid size.
bool round1_requested() {
  const char* e = getenv("LKB_NUFFT_FFT");
  return e && (strcmp(e, "global") == 0 || strcmp(e, "smem") == 0 || strcmp(e, "fused") == 0);
}
int single_term_log2(int64_t kmax_plus_1) {
  const int p = fine_log2(kmax_plus_1);
  return round1_requested() ? p : std::max(p, V2R_P_MIN);
}
int kernel_width(double sigma) {
  int w = nufft::es_width(sigma);
  if (const char* e = getenv("LKB_NUFFT_W")) w = atoi(e);
  if (w < 4) w = 4;
  if (w > 16) w = 16;
  return w & ~1;                                  // even widths only
}

// precision escalation threshold (nufft_v2.cuh): max |y - mean| over the in-band peak amplitude; <= 0 turns it off
float escalate_ratio() {
  if (const char* e = getenv("LKB_NUFFT_ESCALATE")) return (float)atof(e);
  return 250.0f;
}

}  // namespace

// Regular grid f_k = (k0 + k) df with integer k0 >= 0, df * baseline <= 1, fine grids that fit 2^24 cells.
bool ls_nufft_supported(int64_t F, bool regular, double grid_f0, double grid_df, double t_last) {
  if (!regular || F < 2 || !(grid_df > 0.0) || !(grid_f0 >= 0.0)) return false;
  const double q = grid_f0 / grid_df, k0 = rint(q);
  if (fabs(q - k0) > 1e-9 * fmax(1.0, q) || k0 > 1.0e7) return false;
  if (!(grid_df * t_last <= 1.0 + 1e-9)) return false;      // oversample 1: df * baseline = 1 up to rounding
  const int64_t kmax = (int64_t)k0 + F;
  return fine_log2(2 * kmax) <= 24;
}

// ---- shared-grid path in two steps: ls_nufft_prepare (tables + window terms, once per call) and ls_nufft_run (spread
// + FFT + finish for a block of light curves; callable per chunk of a pipelined host-mode call, `ws_alt` = 1 selects a
// second set of fine-grid buffers so that two chunks can be in flight on two streams) ----
struct NufftPlan {
  int w, p;
  float beta;
  int64_t k0, M;
  const Cad* cad;
  const int32_t* fge;
  const float2* dec;
  int n1max;            // v2: rows of the [A][Bc] grid of z cells the cadences reach
  V2Tables tb;          // v2: twiddle tables (valid when fft_mode(p) == 3)
  const float* Wt;      // v2: kernel weights [N, w]
  const double* Wtd;    // v2: the same in double precision (escalation pass)
  int* esc_total;       // v2: device counter of escalated light curves since ls_nufft_begin_call
  V2TablesD tbd;        // v2: double-precision twiddle tables (escalation pass)
  const V2FTab* ftab;   // v2: folded finish table [F] (rows >= F_low)
  const float2* lowD;   // v2: design matrix of the low rows [F_low, Npad]
  int64_t Npad;
};
static NufftPlan g_plan;
// transform and grid sizes of the most recent NUFFT call: {1 = v2 / 0 = round-1 pair-packed, p, p2} (diagnostic)
static int g_last_plan[3] = {-1, 0, 0};
static void record_plan(bool v2, int p, int p2) {
  g_last_plan[0] = v2 ? 1 : 0;
  g_last_plan[1] = p;
  g_last_plan[2] = p2;
}
void ls_nufft_last_plan(int* out) {
  for (int i = 0; i < 3; ++i) out[i] = g_last_plan[i];
}

// light curves that took the double-precision pass since the last ls_nufft_begin_call (diagnostic; synchronises)
void ls_nufft_begin_call(cudaStream_t st) {
  if (g_plan.esc_total) cudaMemsetAsync(g_plan.esc_total, 0, sizeof(int), st);
}
int ls_nufft_last_escalated() {
  if (!g_plan.esc_total) return 0;
  int h = 0;
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  if (cudaMemcpy(&h, g_plan.esc_total, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  return h;
}


// d_t: times shifted to t[0] = 0 (ascending - checked here).  d_rot / d_rot2 rows [0, F_low) are already filled by
// ls_window_kernel (fp64 path); the rows >= F_low are filled here from one transform of unit strengths.
int ls_nufft_prepare(const double* d_t, int64_t N, int64_t F, double grid_f0, double grid_df, float4* d_rot,
                     float2* d_rot2, int64_t F_low, cudaStream_t st, const double* d_freq, int64_t Npad) {
  const int64_t k0 = (int64_t)rint(grid_f0 / grid_df);
  // p2: the window terms' grid (one transform of unit strengths, y-independent)
  const int p = single_term_log2(k0 + F), p2 = fine_log2(2 * (k0 + F));
  const double sigma = fmin(2.0, nufft::grid_sigma(p, k0 + F));   // (the validated rule: beta = 2.30 w from sigma = 2 on)
  const int w = kernel_width(sigma);
  const float beta = (float)nufft::es_beta(w, sigma);
  const int64_t M = (int64_t)1 << p, M2 = (int64_t)1 << p2;
  GlNodes gl;
  nufft::gauss_legendre(GL_NQ, gl.x, gl.w);

  Cad *cad = nullptr, *cad2 = nullptr;
  int32_t *fge = nullptr, *fge2 = nullptr;
  float2 *dec = nullptr, *dec2 = nullptr, *Zw = nullptr;
  float* ones = nullptr;
  int* flag = nullptr;
  const int64_t L = nufft::table_len(M, w), L2 = nufft::table_len(M2, w);
  LKB_TRY(ws_get_t<Cad>(WS_A, N, &cad));
  LKB_TRY(ws_get_t<int32_t>(WS_B, L, &fge));
  LKB_TRY(ws_get_t<float2>(WS_C, F, &dec));
  LKB_TRY(ws_get_t<Cad>(WS_J, N, &cad2));
  LKB_TRY(ws_get_t<int32_t>(WS_O, L2, &fge2));
  LKB_TRY(ws_get_t<float2>(WS_P, 2 * M2, &Zw));
  LKB_TRY(ws_get_t<float2>(WS_IN3, 2 * (k0 + F), &dec2));
  LKB_TRY(ws_get_t<float>(WS_IN4, N, &ones));
  LKB_TRY(ws_get_t<int>(WS_IN5, 1, &flag));

  // ---- tables of the two fine grids, sortedness check ----
  LKB_CUDA_CHECK(cudaMemsetAsync(flag, 0, sizeof(int), st));
  LKB_LAUNCH(blocks_for(N, 256), 256, st, nufft_cad_kernel)(d_t, N, grid_df, M, w, cad, flag);
  LKB_LAUNCH_CHECK();
  LKB_LAUNCH(blocks_for(N, 256), 256, st, nufft_cad_kernel)(d_t, N, grid_df, M2, w, cad2, flag);
  LKB_LAUNCH_CHECK();
  int h_flag = 0;
  Cad h_last;
  LKB_CUDA_CHECK(cudaMemcpyAsync(&h_flag, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
  LKB_CUDA_CHECK(cudaMemcpyAsync(&h_last, cad + (N - 1), sizeof(Cad), cudaMemcpyDeviceToHost, st));
  LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  if (h_flag) {
    set_error("lkb_ls_power_shared: the NUFFT path needs ascending times");
    return LKB_E_UNSUPPORTED;
  }
  g_plan.n1max = 0;
  g_plan.Wt = nullptr;
  g_plan.Wtd = nullptr;
  g_plan.esc_total = nullptr;
  g_plan.ftab = nullptr;
  g_plan.lowD = nullptr;
  g_plan.Npad = Npad;
  const bool v2 = fft_mode(p) == 3 && d_freq != nullptr;
  if (v2) {
    g_plan.n1max = v2_n1max(p, (int64_t)h_last.i0, w);
    LKB_TRY(v2_tables(p, WS_IN6, st, &g_plan.tb));
    float* Wt = nullptr;
    LKB_TRY(ws_get_t<float>(WS_X0, (size_t)N * w, &Wt));
    LKB_LAUNCH(blocks_for(N * w, 256), 256, st, nufft2_weights_kernel<float>)(d_t, N, grid_df, M, w, (double)beta, Wt);
    LKB_LAUNCH_CHECK();
    g_plan.Wt = Wt;
    double* Wtd = nullptr;
    LKB_TRY(ws_get_t<double>(WS_Y0, (size_t)N * w + 2, &Wtd));
    g_plan.esc_total = reinterpret_cast<int*>(Wtd + (size_t)N * w);
    LKB_CUDA_CHECK(cudaMemsetAsync(g_plan.esc_total, 0, sizeof(int), st));
    LKB_LAUNCH(blocks_for(N * w, 256), 256, st, nufft2_weights_kernel<double>)(d_t, N, grid_df, M, w, (double)beta, Wtd);
    LKB_LAUNCH_CHECK();
    g_plan.Wtd = Wtd;
    LKB_TRY(v2_tables(p, WS_Y1, st, &g_plan.tbd));
    if (F_low > 0) {
      float2* lowD = nullptr;
      LKB_TRY(ws_get_t<float2>(WS_X2, (size_t)F_low * Npad, &lowD));
      LKB_LAUNCH(blocks_for(F_low * Npad, 256), 256, st, nufft2_lowtab_kernel)(d_t, N, Npad, d_freq, (int)F_low, lowD);
      LKB_LAUNCH_CHECK();
      g_plan.lowD = lowD;
    }
  }
  LKB_LAUNCH(blocks_for(L, 256), 256, st, nufft_first_ge_kernel)(cad, N, L, fge);
  LKB_LAUNCH_CHECK();
  LKB_LAUNCH(blocks_for(L2, 256), 256, st, nufft_first_ge_kernel)(cad2, N, L2, fge2);
  LKB_LAUNCH_CHECK();
  LKB_LAUNCH(blocks_for(F, 128), 128, st, nufft_deconv_kernel)(k0, F, M, w, (double)beta, gl, dec);
  LKB_LAUNCH_CHECK();
  LKB_LAUNCH(blocks_for(2 * (k0 + F), 128), 128, st, nufft_deconv_kernel)(0, 2 * (k0 + F), M2, w, (double)beta, gl, dec2);
  LKB_LAUNCH_CHECK();

  // ---- window terms of the rows >= F_low: one transform of unit strengths on the 2x finer grid ----
  if (F_low < F) {
    LKB_LAUNCH(blocks_for(N, 256), 256, st, nufft_fill_kernel)(ones, N, 1.0f);
    LKB_LAUNCH_CHECK();
    LKB_LAUNCH(blocks_for(M2, 256), 256, st, nufft_spread_kernel)(fge2, cad2, ones, 0, nullptr, 1, 1, w, beta, p2, Zw);
    LKB_LAUNCH_CHECK();
    float2* Zw_out = nullptr;
    LKB_TRY(fft_passes(Zw, Zw + M2, p2, 1, st, &Zw_out));
    LKB_LAUNCH(blocks_for(F - F_low, 128), 128, st, nufft_rot_kernel)(Zw_out, M2, dec2, k0, F, F_low, (double)N, d_rot, d_rot2);
    LKB_LAUNCH_CHECK();
    if (v2) {
      V2FTab* ftab = nullptr;
      LKB_TRY(ws_get_t<V2FTab>(WS_X1, (size_t)F, &ftab));
      LKB_LAUNCH(blocks_for(F - F_low, 128), 128, st, nufft2_ftab_kernel)(d_rot, d_rot2, k0, F, F_low, M, w, (double)beta, gl,
                                                                       ftab);
      LKB_LAUNCH_CHECK();
      g_plan.ftab = ftab;
    }
  }
  g_plan.w = w;
  g_plan.p = p;
  g_plan.beta = beta;
  g_plan.k0 = k0;
  g_plan.M = M;
  g_plan.cad = cad;
  g_plan.fge = fge;
  g_plan.dec = dec;
  record_plan(v2, p, p2);
  return LKB_OK;
}

// d_yc: centred flux rows [B, ystride] fp32 of THIS block of light curves (with their d_ysumf / d_absmax / d_pow
// rows); d_t / d_freq / d_rot / d_rot2 as in ls_nufft_prepare, which must have run on an earlier point of the stream
// order.  prof: record the library's profiling events around the batch kernels.
int ls_nufft_run(const double* d_t, int64_t N, const float* d_yc, int64_t ystride, const float* d_ysumf,
                 const float* d_absmax, int B, const double* d_freq, int64_t F, const float4* d_rot,
                 const float2* d_rot2, int64_t F_low, int normalization, double norm_scale, float* d_pow,
                 cudaStream_t st, int ws_alt, bool prof) {
  const NufftPlan pl = g_plan;
  const int w = pl.w, p = pl.p;
  const float beta = pl.beta;
  const int64_t k0 = pl.k0, M = pl.M;
  const int npairs = (B + 1) / 2;
  const int mode = (pl.Wt != nullptr) ? 3 : fft_mode(p) == 3 ? 0 : fft_mode(p);
  const char* ve = getenv("LKB_NUFFT_VERIFY");
  const bool verify = ve && atoi(ve) != 0 && F_low < F;
  if (mode == 3) {
    // ---- v2: one real transform per light curve (nufft_v2.cuh): spread -> column transforms -> row transforms + finish
    const int64_t Mh = M >> 1;
    const size_t cells = (size_t)pl.n1max << V2_PB;
    float2 *T = nullptr, *G = nullptr;
    LKB_TRY(ws_get_t<float2>(ws_alt ? WS_OUT4 : WS_H, (size_t)B * Mh, &T));
    LKB_TRY(ws_get_t<float2>(ws_alt ? WS_OUT5 : WS_I, std::max((size_t)B * cells, verify ? (size_t)4 * Mh : (size_t)0), &G));
    unsigned* d_worst = nullptr;
    if (verify) LKB_TRY(ws_get_t<unsigned>(ws_alt ? WS_OUT7 : WS_OUT6, 1, &d_worst));
    const int ptc = V2_LOG_TILE - (p - 1 - V2_PB);
    if (prof) prof_begin(st);
    constexpr int LCS = 8;
    LKB_LAUNCH(dim3(blocks_for((int64_t)cells, 256), (unsigned)((B + LCS - 1) / LCS)), 256, st, nufft2_spread_kernel<LCS>)(
        pl.fge, pl.cad, pl.Wt, d_yc, ystride, B, w, p, ptc, pl.n1max, G);
    LKB_LAUNCH_CHECK();
    LKB_TRY(v2_cols(G, T, p, pl.n1max, B, pl.tb, st));
    // in-band peak of every light curve (psd-scaled power, float bits), filled by the two finish kernels
    const float esc_ratio = escalate_ratio();
    unsigned* d_peak = nullptr;
    int* d_list = nullptr;                                       // [0] = count, [1 ..] = listed light curves
    if (esc_ratio > 0.0f && F_low < F) {
      LKB_TRY(ws_get_t<unsigned>(ws_alt ? WS_Y3 : WS_Y2, (size_t)2 * B + 1, &d_peak));      // peak [B] | count | list [B]
      d_list = reinterpret_cast<int*>(d_peak + B);
      LKB_CUDA_CHECK(cudaMemsetAsync(d_peak, 0, sizeof(unsigned) * ((size_t)B + 1), st));
    }
    V2Finish fa;
    fa.ftab = pl.ftab; fa.k0 = k0; fa.F = F; fa.k_lo = F_low; fa.ysum = d_ysumf; fa.Nf = (float)N;
    fa.normalization = normalization; fa.scale = (float)norm_scale; fa.power = d_pow;
    fa.peak = d_peak; fa.lcmap = nullptr; fa.log2M = p;
    if (F_low < F) LKB_TRY(v2_rows(T, p, B, pl.tb, &fa, (float2*)nullptr, 0, st));
    if (F_low > 0) {
      double* acc = nullptr;
      LKB_TRY(ws_get_t<double>(ws_alt ? WS_X4 : WS_X3, (size_t)B * F_low * 2, &acc));
      LKB_CUDA_CHECK(cudaMemsetAsync(acc, 0, sizeof(double) * (size_t)B * F_low * 2, st));
      const int groups = (B + 15) / 16;
      // cadence slices of a FIXED length: the partition of a light curve's sums must not depend on the batch size, or
      // its low rows would change in the last bit with the chunk of the host-mode pipeline it happens to land in
      // (bitwise permutation invariance is asserted at full size)
      const int64_t slice = 2048;
      LKB_LAUNCH(dim3((unsigned)groups, (unsigned)((N + slice - 1) / slice)), 256, st, nufft2_lowrows_kernel)(
          pl.lowD, N, pl.Npad, d_yc, ystride, B, (int)F_low, slice, acc);
      LKB_LAUNCH_CHECK();
      LKB_LAUNCH(blocks_for((int64_t)B * F_low, 256), 256, st, nufft2_lowfinish_kernel)(
          acc, B, (int)F_low, F, N, d_rot, d_rot2, d_ysumf, normalization, (float)norm_scale, d_pow, d_peak);
      LKB_LAUNCH_CHECK();
    }
    // ---- precision escalation (nufft_v2.cuh): light curves whose flux excursion dwarfs their in-band peak are
    // transformed again in double precision.  No host round trip: the launches are sized for `cap` light curves per
    // round and read the device-side count (blocks stride over the listed light curves; rounds past the count exit).
    if (d_peak) {
      LKB_LAUNCH(blocks_for(B, 256), 256, st, nufft2_flag_kernel)(d_peak, d_absmax, B, (float)N, esc_ratio, d_list, d_list + 1,
                                                                pl.esc_total);
      LKB_LAUNCH_CHECK();
      // one round for batches up to 1024 light curves (double-precision buffers for all of them: 5 GB at config 2,
      // from the grow-only pool); larger batches go round by round
      int cap_max = 1024;
      if (const char* e = getenv("LKB_NUFFT_ESCALATE_CAP")) cap_max = std::max(1, atoi(e));     // (tests: several rounds)
      const int cap = std::min(B, cap_max), gy = std::min(cap, 32);
      const size_t lowlen = F_low > 0 ? (size_t)F_low * 4 + (size_t)cap * F_low * 2 + cap : 0;
      double *Gbuf = nullptr;
      double2* Td = nullptr;
      LKB_TRY(ws_get_t<double>(ws_alt ? WS_Y6 : WS_Y4, 2 * (size_t)cap * cells + lowlen, &Gbuf));
      LKB_TRY(ws_get_t<double2>(ws_alt ? WS_Y7 : WS_Y5, (size_t)cap * Mh, &Td));
      double2* Gd = reinterpret_cast<double2*>(Gbuf);
      double* accW = Gbuf + 2 * (size_t)cap * cells;
      double* accY = accW + (size_t)F_low * 4;
      double* accS = accY + (size_t)cap * F_low * 2;
      const int* lst = d_list + 1;
      const int ptc_d = v2_log_tile(p - 1 - V2_PB, true) - (p - 1 - V2_PB);      // the double-precision tile's columns
      for (int base = 0; base < B; base += cap) {
        const V2Count nc = {d_list, base, cap};
        LKB_LAUNCH(dim3(blocks_for((int64_t)cells, 256), (unsigned)((gy + LCS_D - 1) / LCS_D)), 256, st,
                   nufft2_spread_list_kernel)(pl.fge, pl.cad, pl.Wtd, d_yc, ystride, lst, w, p, ptc_d, pl.n1max, Gd, nc);
        LKB_LAUNCH_CHECK();
        LKB_TRY(v2_cols(Gd, Td, p, pl.n1max, gy, pl.tbd, st, nc));
        V2Finish fd = fa;
        fd.peak = nullptr;
        fd.lcmap = lst;
        LKB_TRY(v2_rows(Td, p, gy, pl.tbd, &fd, (double2*)nullptr, 0, st, nc));
        if (F_low > 0) {
          LKB_CUDA_CHECK(cudaMemsetAsync(accW, 0, sizeof(double) * lowlen, st));
          LKB_LAUNCH(dim3((unsigned)F_low, blocks_for(N, 256 * LOWX_PER)), 256, st, nufft2_lowacc_kernel)(
              lst, nc, d_t, N, d_yc, ystride, d_freq, (int)F_low, accW, accY, accS);
          LKB_LAUNCH_CHECK();
          LKB_LAUNCH(blocks_for((int64_t)cap * F_low, 256), 256, st, nufft2_lowexact_finish_kernel)(
              lst, nc, accW, accY, accS, (int)F_low, F, N, normalization, (float)norm_scale, d_pow);
          LKB_LAUNCH_CHECK();
        }
      }
    }
    if (prof) prof_end(st);
    if (verify) {            // the first light curves' transforms once more, written out this time (G is free again)
      const int nv = std::min(B, 4);
      const int nk2 = (int)((k0 + F) >> (p - 1 - V2_PB)) + 1;
      LKB_TRY(v2_rows(T, p, nv, pl.tb, (const V2Finish*)nullptr, G, nk2, st));
      const char* fe = getenv("LKB_NUFFT_INJECT_FAULT");
      LKB_CUDA_CHECK(cudaMemsetAsync(d_worst, 0, sizeof(unsigned), st));
      LKB_LAUNCH(16, 128, st, nufft2_verify_kernel)(G, p, pl.dec, k0, F, F_low, d_t, N, d_yc, ystride, d_freq, nv,
                                                  fe ? (float)atof(fe) : 1.0f, d_worst);
      LKB_LAUNCH_CHECK();
      unsigned h_worst = 0;
      LKB_CUDA_CHECK(cudaMemcpyAsync(&h_worst, d_worst, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
      LKB_CUDA_CHECK(cudaStreamSynchronize(st));
      if (h_worst > 100u) {
        set_error("NUFFT self-check failed: transform deviates from the direct sums by %u x 1e-7 sum|y|", h_worst);
        return LKB_E_VERIFY;
      }
    }
    return LKB_OK;
  }
  float2 *Za = nullptr, *Zb = nullptr;
  LKB_TRY(ws_get_t<float2>(ws_alt ? WS_OUT4 : WS_H, (size_t)npairs * M, &Za));
  LKB_TRY(ws_get_t<float2>(ws_alt ? WS_OUT5 : WS_I, (size_t)npairs * M, &Zb));
  unsigned* d_worst = nullptr;
  if (verify) LKB_TRY(ws_get_t<unsigned>(ws_alt ? WS_OUT7 : WS_OUT6, 1, &d_worst));

  // ---- the batch: spread, FFT, finish - optionally in groups of light-curve pairs small enough for the fine grids
  // of a group (two buffers) to stay in the 50 MB L2 across the passes (LKB_NUFFT_GROUP_MB, default 0 = one group;
  // to be tuned on hardware: more launches against HBM sweeps turned into L2 sweeps) ----
  int group = npairs;
  if (const char* e = getenv("LKB_NUFFT_GROUP_MB")) {
    const double mb = atof(e);
    if (mb > 0.0) {
      const double per_pair = 2.0 * (double)M * sizeof(float2) / 1048576.0;
      group = (int)fmax(1.0, floor(mb / per_pair));
      if (group > npairs) group = npairs;
    }
  }
  if (prof) prof_begin(st);
  for (int g0 = 0; g0 < npairs; g0 += group) {
    const int np_g = std::min(group, npairs - g0);
    const int B_g = std::min(B - 2 * g0, 2 * np_g);              // light curves in this group
    float2* Za_g = Za + (size_t)g0 * M;
    float2* Zb_g = Zb + (size_t)g0 * M;
    if (mode != 2) {
      LKB_LAUNCH(blocks_for((int64_t)np_g * M, 256), 256, st, nufft_spread_kernel)(
          pl.fge, pl.cad, d_yc + (size_t)2 * g0 * ystride, ystride, d_absmax + 2 * g0, B_g, np_g, w, beta, p, Za_g);
      LKB_LAUNCH_CHECK();
    }
    float2* Zout = nullptr;
    int pa = 0;                                               // 0: natural order, else the four-step layout
    if (mode == 2) {
      SpreadArgs sp;
      sp.first_ge = pl.fge;
      sp.cad = pl.cad;
      sp.y = d_yc + (size_t)2 * g0 * ystride;
      sp.ystride = ystride;
      sp.absmax = d_absmax + 2 * g0;
      sp.B = B_g;
      sp.w = w;
      sp.beta = beta;
      LKB_TRY(fft_fourstep(Za_g, p, np_g, st, &pa, &sp));
      Zout = Za_g;
    } else if (mode == 1) {
      LKB_TRY(fft_fourstep(Za_g, p, np_g, st, &pa, nullptr));
      Zout = Za_g;
    } else {
      LKB_TRY(fft_passes(Za_g, Zb_g, p, np_g, st, &Zout));
    }
    if (F_low < F) {
      LKB_LAUNCH(blocks_for((F - F_low) * np_g, 256), 256, st, nufft_finish_kernel)(
          Zout, p, pl.dec, k0, F, F_low, d_rot, d_rot2, d_ysumf + 2 * g0, d_absmax + 2 * g0, (float)N, normalization,
          (float)norm_scale, B_g, np_g, pa, d_pow + (size_t)2 * g0 * F);
      LKB_LAUNCH_CHECK();
      if (verify && g0 == 0) {            // self-check on the first group (one small kernel + one read-back)
        const char* fe = getenv("LKB_NUFFT_INJECT_FAULT");       // test hook: pretend the transform is off by x
        LKB_CUDA_CHECK(cudaMemsetAsync(d_worst, 0, sizeof(unsigned), st));
        LKB_LAUNCH(16, 128, st, nufft_verify_kernel)(Zout, p, pa, pl.dec, k0, F, F_low, d_t, N, d_yc, ystride, d_absmax,
                                                   d_freq, B_g, fe ? (float)atof(fe) : 1.0f, d_worst);
        LKB_LAUNCH_CHECK();
        unsigned h_worst = 0;
        LKB_CUDA_CHECK(cudaMemcpyAsync(&h_worst, d_worst, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
        LKB_CUDA_CHECK(cudaStreamSynchronize(st));
        if (h_worst > 100u) {
          set_error("NUFFT self-check failed: transform deviates from the direct sums by %u x 1e-7 sum|y|", h_worst);
          return LKB_E_VERIFY;
        }
      }
    }
  }
  if (prof) prof_end(st);
  if (F_low > 0) {
    LKB_LAUNCH(blocks_for(F_low * B, 4), 128, st, nufft_lowrows_kernel)(d_t, N, d_yc, ystride, B, d_freq, F_low, F, d_rot,
                                                                   d_rot2, d_ysumf, normalization, (float)norm_scale,
                                                                   d_pow);
    LKB_LAUNCH_CHECK();
  }
  return LKB_OK;
}



// one-shot form (the whole batch on one stream)
int ls_nufft_launch(const double* d_t, int64_t N, const float* d_yc, int64_t ystride, const float* d_ysumf,
                    const float* d_absmax, int B, const double* d_freq, int64_t F, double grid_f0, double grid_df,
                    float4* d_rot, float2* d_rot2, int64_t F_low, int normalization, double norm_scale, float* d_pow,
                    cudaStream_t st) {
  LKB_TRY(ls_nufft_prepare(d_t, N, F, grid_f0, grid_df, d_rot, d_rot2, F_low, st, d_freq, ystride));
  return ls_nufft_run(d_t, N, d_yc, ystride, d_ysumf, d_absmax, B, d_freq, F, d_rot, d_rot2, F_low, normalization,
                      norm_scale, d_pow, st, 0, true);
}

// =====================================================================================================
// Ragged batches (K1 shapes: every light curve has its own times; one shared regular frequency grid).
// Opt-in through LKB_LS_RAGGED_NUFFT=1 (round 1: CPU-verified arithmetic, CUDA glue not yet run on hardware).
// Same pipeline, with per-light-curve cadence tables in the padded CSR layout of the K1 prologue, cell ranges by
// binary search (nufft::spread_cell_search), and the window terms of each light curve taken from a second
// transform of unit strengths (pairs packed the same way) inside the finish kernel - no rot arrays.
// =====================================================================================================
namespace {

__global__ void nufft_cad_ragged_kernel(const double* __restrict__ t, const int64_t* __restrict__ off,
                                        const int64_t* __restrict__ poff, const double* __restrict__ span, double df,
                                        int64_t M, int64_t M2, int w, Cad* __restrict__ cad, Cad* __restrict__ cad2,
                                        int* __restrict__ bad) {
  const int b = blockIdx.y;
  const int64_t n = off[b + 1] - off[b], po = poff[b];
  if (blockIdx.x == 0 && threadIdx.x == 0 && !(df * span[b] <= 1.0 + 1e-9)) *bad = 1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double ti = t[po + i];
    cad[po + i] = nufft::cad_entry(ti, df, M, w);
    cad2[po + i] = nufft::cad_entry(ti, df, M2, w);
    if (ti < 0.0 || (i > 0 && ti < t[po + i - 1])) *bad = 1;
  }
}

__global__ void __launch_bounds__(256)
nufft_absmax_ragged_kernel(const float* __restrict__ y, const int64_t* __restrict__ off, const int64_t* __restrict__ poff,
                           float* __restrict__ absmax) {
  __shared__ float s_max[8];
  const int b = blockIdx.x;
  const int64_t n = off[b + 1] - off[b], po = poff[b];
  float mx = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) mx = fmaxf(mx, fabsf(y[po + i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = 0.f;
    for (int wv = 0; wv < (int)(blockDim.x >> 5); ++wv) m = fmaxf(m, s_max[wv]);
    absmax[b] = m;
  }
}

// Z[pair][m] for the flux (y != NULL, scaled) or for unit strengths (y == NULL)
__global__ void __launch_bounds__(256)
nufft_spread_ragged_kernel(const Cad* __restrict__ cad, const float* __restrict__ y, const int64_t* __restrict__ off,
                           const int64_t* __restrict__ poff, const float* __restrict__ absmax, int B, int npairs, int w,
                           float beta, int log2M, float2* __restrict__ Z) {
  const int64_t M = (int64_t)1 << log2M;
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= (int64_t)npairs << log2M) return;
  const int64_t pair = gid >> log2M, m = gid & (M - 1);
  const int64_t b0 = 2 * pair, b1 = b0 + 1;
  float2 v = make_float2(0.f, 0.f);
  {
    const int64_t po = poff[b0], n = off[b0 + 1] - off[b0];
    v.x = nufft::spread_cell_search(m, cad + po, n, y ? y + po : nullptr, y ? nufft::pow2_scale(absmax[b0]) : 1.0f, w,
                                    beta, M);
  }
  if (b1 < B) {
    const int64_t po = poff[b1], n = off[b1 + 1] - off[b1];
    v.y = nufft::spread_cell_search(m, cad + po, n, y ? y + po : nullptr, y ? nufft::pow2_scale(absmax[b1]) : 1.0f, w,
                                    beta, M);
  }
  Z[gid] = v;
}

// v2 (one real transform per light curve): G[lc][e] = (cell 2n, cell 2n + 1) in the column kernel's layout, rows
// n1 < n1max only; y == NULL: unit strengths (window terms)
__global__ void __launch_bounds__(256)
nufft2_spread_ragged_kernel(const Cad* __restrict__ cad, const float* __restrict__ y, const int64_t* __restrict__ off,
                            const int64_t* __restrict__ poff, int w, float beta, int p, int ptc, int n1max,
                            float2* __restrict__ G, const double* __restrict__ t, double df) {
  const int64_t cells = (int64_t)n1max << V2_PB;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= cells) return;
  const int64_t M = (int64_t)1 << p, m = 2 * v2_zcell_of(e, ptc, n1max);
  const int64_t lc = blockIdx.y, po = poff[lc], n = off[lc + 1] - off[lc];
  float2 v;
  if (t) {                       // kernel weights in FP64 from the time stamps (nufft_core.h: spread_cell_search_acc)
    const double dfM = df * (double)M;
    v.x = nufft::spread_cell_search_acc(m, cad + po, t + po, n, y ? y + po : nullptr, w, (double)beta, dfM, M);
    v.y = nufft::spread_cell_search_acc(m + 1, cad + po, t + po, n, y ? y + po : nullptr, w, (double)beta, dfM, M);
  } else {
    v.x = nufft::spread_cell_search(m, cad + po, n, y ? y + po : nullptr, 1.0f, w, beta, M);
    v.y = nufft::spread_cell_search(m + 1, cad + po, n, y ? y + po : nullptr, 1.0f, w, beta, M);
  }
  G[lc * cells + e] = v;
}

// mode kk of ONE real series from its half-length transform Zn (natural order, length Mh = M / 2)
__device__ __forceinline__ float2 v2_unpack_real(const float2* __restrict__ Zn, int64_t kk, int64_t M) {
  const int64_t Mh = M >> 1;
  const float2 g1 = Zn[kk], g2 = Zn[(Mh - kk) & (Mh - 1)];
  const float2 E = make_float2(0.5f * (g1.x + g2.x), 0.5f * (g1.y - g2.y));
  const float2 O = make_float2(0.5f * (g1.y + g2.y), 0.5f * (g2.x - g1.x));
  double wsn, wcs;
  sincospi(2.0 * (double)kk / (double)M, &wsn, &wcs);
  const float wc = (float)wcs, ws = (float)wsn;
  return make_float2(E.x + wc * O.x - ws * O.y, E.y + wc * O.y + ws * O.x);
}

__device__ __forceinline__ float ragged_power(float2 hs, float2 win1, float2 win2, double Nd, double ysum,
                                              int normalization, double scale) {
  LsSums<double> d;
  d.zero();
  d.ch = (double)hs.x;
  d.sh = (double)hs.y;
  d.c = (double)win1.x;
  d.s = (double)win1.y;
  d.cc = 0.5 * (Nd + (double)win2.x);
  d.sc = 0.5 * (double)win2.y;
  return ls_normalize(ls_power_from_sums(d, Nd, ysum), Nd, normalization, scale);
}

// power[b, k] for the rows that are not "low" for light curve b
__global__ void __launch_bounds__(256)
nufft_finish_ragged_kernel(const float2* __restrict__ Z, int log2M, const float2* __restrict__ Zw, int log2M2,
                           const float2* __restrict__ dec, const float2* __restrict__ dec2, int64_t k0, int64_t F,
                           double f0, double df, const int64_t* __restrict__ off, const double* __restrict__ span,
                           const double* __restrict__ ysum, const float* __restrict__ absmax, int normalization,
                           const double* __restrict__ norm_scale, int B, int npairs, int pa, int pa2,
                           float* __restrict__ power) {
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= F * npairs) return;
  const int64_t pair = gid / F, k = gid - pair * F;
  const int64_t M = (int64_t)1 << log2M, M2 = (int64_t)1 << log2M2, kk = k0 + k;
  const int64_t b0 = 2 * pair, b1 = b0 + 1;
  const bool has1 = b1 < B;
  const float inv0 = 1.0f / nufft::pow2_scale(absmax[b0]);
  const float inv1 = has1 ? 1.0f / nufft::pow2_scale(absmax[b1]) : 1.0f;
  float2 ha, hb, w1a, w1b, w2a, w2b;
  nufft::unpack_pair(Z + pair * M, kk, M, dec[k], inv0, inv1, &ha, &hb, pa);
  nufft::unpack_pair(Zw + pair * M2, kk, M2, dec2[kk], 1.0f, 1.0f, &w1a, &w1b, pa2);
  nufft::unpack_pair(Zw + pair * M2, 2 * kk, M2, dec2[2 * kk], 1.0f, 1.0f, &w2a, &w2b, pa2);
  const double fr = f0 + (double)k * df;
  if (fr * span[b0] > LS_LOWF_CYCLES) {
    const double Nd = (double)(off[b0 + 1] - off[b0]);
    power[b0 * F + k] = ragged_power(ha, w1a, w2a, Nd, ysum[b0], normalization, norm_scale ? norm_scale[b0] : 1.0);
  }
  if (has1 && fr * span[b1] > LS_LOWF_CYCLES) {
    const double Nd = (double)(off[b1 + 1] - off[b1]);
    power[b1 * F + k] = ragged_power(hb, w1b, w2b, Nd, ysum[b1], normalization, norm_scale ? norm_scale[b1] : 1.0);
  }
}

// v2: power[b, k] from the per-light-curve transforms Zn [B][M / 2] (flux) and Zwn [B][M2 / 2] (unit strengths on the
// 2x finer grid), both in natural order
__global__ void __launch_bounds__(256)
nufft2_finish_ragged_kernel(const float2* __restrict__ Zn, int p, const float2* __restrict__ Zwn, int p2,
                            const float2* __restrict__ dec, const float2* __restrict__ dec2, int64_t k0, int64_t F,
                            double f0, double df, const int64_t* __restrict__ off, const double* __restrict__ span,
                            const double* __restrict__ ysum, int normalization, const double* __restrict__ norm_scale,
                            int B, float* __restrict__ power) {
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= F * B) return;
  const int64_t b = gid / F, k = gid - b * F;
  const double fr = f0 + (double)k * df;
  if (!(fr * span[b] > LS_LOWF_CYCLES)) return;
  const int64_t M = (int64_t)1 << p, M2 = (int64_t)1 << p2, kk = k0 + k;
  const float2 hs = nufft::cmul(v2_unpack_real(Zn + b * (M >> 1), kk, M), dec[k]);
  const float2 w1 = nufft::cmul(v2_unpack_real(Zwn + b * (M2 >> 1), kk, M2), dec2[kk]);
  const float2 w2 = nufft::cmul(v2_unpack_real(Zwn + b * (M2 >> 1), 2 * kk, M2), dec2[2 * kk]);
  const double Nd = (double)(off[b + 1] - off[b]);
  power[b * F + k] = ragged_power(hs, w1, w2, Nd, ysum[b], normalization, norm_scale ? norm_scale[b] : 1.0);
}

// rows with f * baseline_b <= LS_LOWF_CYCLES: direct fp64 sums, one warp per (row, light curve)
__global__ void __launch_bounds__(128)
nufft_lowrows_ragged_kernel(const double* __restrict__ t, const float* __restrict__ y, const int64_t* __restrict__ off,
                            const int64_t* __restrict__ poff, const double* __restrict__ span,
                            const double* __restrict__ ysum, double f0, double df, int64_t F_low_max, int64_t F,
                            int normalization, const double* __restrict__ norm_scale, int B, float* __restrict__ power) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t job = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (job >= F_low_max * B) return;
  const int64_t b = job / F_low_max, k = job - b * F_low_max;
  const double fr = f0 + (double)k * df;
  if (k >= F || fr * span[b] > LS_LOWF_CYCLES) return;
  const int64_t n = off[b + 1] - off[b], po = poff[b];
  if (n <= 0) return;
  LsSums<double> d;
  d.zero();
  for (int64_t i = lane; i < n; i += 32) {
    double s, c;
    ls_sincos_cycles_f64(fr * t[po + i], s, c);
    d.add((double)y[po + i], s, c);
  }
  d.warp_reduce();
  if (lane == 0)
    power[b * F + k] = ls_normalize(ls_power_from_sums(d, (double)n, ysum[b]), (double)n, normalization,
                                    norm_scale ? norm_scale[b] : 1.0);
}

// Multi-term periodogram (nterms = NT), power[b, k] for the rows that are not "low" for light curve b.  Harmonic j of
// f_k = (k0 + k) df is mode j kk of the same transforms: modes j kk (j <= NT) of the flux transform Zn [B][M / 2] give
// YC_j, YS_j, modes j kk (j <= 2 NT) of the unit-strength transform Zwn [B][M2 / 2] give C_j, S_j.  dec / dec2 hold the
// deconvolution factor of every mode index [0, NT (k0 + F)) / [0, 2 NT (k0 + F)).
// A bin where some harmonic's window sum is nearly coherent, |C_j + i S_j| >= LS_CHI2_COHERENT N, is a low row in
// disguise: j f sits near a multiple of the sampling rate of a near-regular cadence (a TESS 2-min light curve: 720 / d,
// which the harmonics of a grid up to the Nyquist frequency reach), the normal matrix cancels like that of
// f * baseline <= 2, and the fp32 sums miss the tolerance there (emulated 2-min light curves: up to 300x within one bin
// of 720 / d).  Such bins take the direct fp64 sums, in this thread.  Irregular cadences reach the limit only by chance,
// with probability ~exp(-N / 16) per harmonic and bin: never at N >= 300, a fifth of the bins or more at N ~ 40.
constexpr double LS_CHI2_COHERENT = 0.25;
// Paths of the multi-term NUFFT periodogram.  LKB_CHI2_OBSERVE(path) marks where one is taken; it expands to nothing
// here, and tests/native/nufft_chi2_emu_driver.cpp, which runs this file on the CPU, defines it to count, so that each
// emulated case can assert that it reached the paths it was written for.  Counted per (light curve, bin) for the
// first two and per group of light curves for the last.
enum Chi2Path {
  CHI2_PATH_COHERENT = 0,   // nufft2_finish_chi2_ragged_kernel: a nearly coherent window sum, bin recomputed in fp64
  CHI2_PATH_LOW_ROW,        // nufft_lowrows_chi2_ragged_kernel: f * baseline <= LS_LOWF_CYCLES, direct fp64 sums
  CHI2_PATH_GROUP,          // ls_nufft_ragged_v2: one group of light curves through the fine-grid buffers
  CHI2_PATH_COUNT
};
#ifndef LKB_CHI2_OBSERVE
#define LKB_CHI2_OBSERVE(path) ((void)0)
#endif
template <int NT>
__global__ void __launch_bounds__(256)
nufft2_finish_chi2_ragged_kernel(const float2* __restrict__ Zn, int p, const float2* __restrict__ Zwn, int p2,
                                 const float2* __restrict__ dec, const float2* __restrict__ dec2, int64_t k0, int64_t F,
                                 double f0, double df, const int64_t* __restrict__ off, const int64_t* __restrict__ poff,
                                 const double* __restrict__ t, const float* __restrict__ y,
                                 const double* __restrict__ span, const double* __restrict__ ysum, int normalization,
                                 const double* __restrict__ norm_scale, int B, float* __restrict__ power) {
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= F * B) return;
  const int64_t b = gid / F, k = gid - b * F;
  const double fr = f0 + (double)k * df;
  if (!(fr * span[b] > LS_LOWF_CYCLES)) return;
  const int64_t M = (int64_t)1 << p, M2 = (int64_t)1 << p2, kk = k0 + k;
  const float2* zw = Zwn + b * (M2 >> 1);
  const float2* zy = Zn + b * (M >> 1);
  Chi2Sums<NT> d;
#pragma unroll
  for (int j = 0; j < 2 * NT; ++j) {
    const int64_t m = (j + 1) * kk;
    const float2 a = nufft::cmul(v2_unpack_real(zw, m, M2), dec2[m]);
    d.C[j] = (double)a.x;
    d.S[j] = (double)a.y;
  }
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    const int64_t m = (j + 1) * kk;
    const float2 h = nufft::cmul(v2_unpack_real(zy, m, M), dec[m]);
    d.YC[j] = (double)h.x;
    d.YS[j] = (double)h.y;
  }
  const int64_t n = off[b + 1] - off[b];
  const double Nd = (double)n;
  bool coherent = false;
#pragma unroll
  for (int j = 0; j < 2 * NT; ++j) coherent |= d.C[j] * d.C[j] + d.S[j] * d.S[j] >= LS_CHI2_COHERENT * LS_CHI2_COHERENT * Nd * Nd;
  if (coherent) {
    LKB_CHI2_OBSERVE(CHI2_PATH_COHERENT);
    d.zero();
    for (int64_t i = 0; i < n; ++i) chi2_add<NT>(d, (double)y[poff[b] + i], fr * t[poff[b] + i]);
  }
  double pw;
  chi2_solve<NT>(d, Nd, ysum[b], pw, nullptr);
  power[b * F + k] = ls_normalize(pw, Nd, normalization, norm_scale ? norm_scale[b] : 1.0);
}

// the rows with f * baseline_b <= LS_LOWF_CYCLES of the multi-term periodogram: direct fp64 sums (the accumulation of
// ls.cu's ls_chi2_kernel), one warp per (row, light curve)
template <int NT>
__global__ void __launch_bounds__(128)
nufft_lowrows_chi2_ragged_kernel(const double* __restrict__ t, const float* __restrict__ y,
                                 const int64_t* __restrict__ off, const int64_t* __restrict__ poff,
                                 const double* __restrict__ span, const double* __restrict__ ysum, double f0, double df,
                                 int64_t F_low_max, int64_t F, int normalization, const double* __restrict__ norm_scale,
                                 int B, float* __restrict__ power) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t job = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (job >= F_low_max * B) return;
  const int64_t b = job / F_low_max, k = job - b * F_low_max;
  const double fr = f0 + (double)k * df;
  if (k >= F || fr * span[b] > LS_LOWF_CYCLES) return;
  const int64_t n = off[b + 1] - off[b], po = poff[b];
  if (n <= 0) return;
  Chi2Sums<NT> d;
  d.zero();
  for (int64_t i = lane; i < n; i += 32) chi2_add<NT>(d, (double)y[po + i], fr * t[po + i]);
  chi2_warp_reduce<NT>(d);
  if (lane == 0) {
    LKB_CHI2_OBSERVE(CHI2_PATH_LOW_ROW);
    double pw;
    chi2_solve<NT>(d, (double)n, ysum[b], pw, nullptr);
    power[b * F + k] = ls_normalize(pw, (double)n, normalization, norm_scale ? norm_scale[b] : 1.0);
  }
}

}  // namespace

namespace {
// Ragged batch through the v2 transform: every light curve is one real series on the flux grid (2^p cells) and one on
// the window grid (2^p2 cells, unit strengths); groups of light curves share the buffers when the fine grids of the
// whole batch exceed cap_mb.  nterms = 0: the single-term periodogram (window modes kk, 2 kk; flux mode kk);
// nterms = n in [1, 4]: the multi-term one (window modes j kk, j <= 2n; flux modes j kk, j <= n).
int ls_nufft_ragged_v2(const double* d_t, const float* d_y, const int64_t* d_off, const int64_t* d_po, int B,
                       int64_t ptotal, int64_t nmax, const double* d_span, const double* h_span, const double* d_ysum,
                       int64_t F, double f0, double df, int64_t k0, int p, int p2, int w, float beta, double cap_mb,
                       int normalization, const double* d_ns, float* d_pow, cudaStream_t st, int nterms) {
  const int64_t M = (int64_t)1 << p, M2 = (int64_t)1 << p2, Mh = M >> 1, Mh2 = M2 >> 1;
  double span_max = 0.0;
  for (int b = 0; b < B; ++b) span_max = fmax(span_max, h_span[b]);
  const int n1max = v2_n1max(p, (int64_t)nufft::cad_entry(span_max, df, M, w).i0, w);
  const int n1max2 = v2_n1max(p2, (int64_t)nufft::cad_entry(span_max, df, M2, w).i0, w);
  const size_t cells = (size_t)n1max << V2_PB, cells2 = (size_t)n1max2 << V2_PB;
  const double per_lc_mb = (2.0 * (double)Mh + 2.0 * (double)Mh2 + (double)std::max(cells, cells2)) * sizeof(float2) / 1048576.0;
  int group = (int)fmax(1.0, floor(cap_mb / per_lc_mb));
  if (group > B) group = B;
  GlNodes gl;
  nufft::gauss_legendre(GL_NQ, gl.x, gl.w);
  V2Tables tb, tb2;
  LKB_TRY(v2_tables(p, WS_IN7, st, &tb));
  LKB_TRY(v2_tables(p2, WS_OUT1, st, &tb2));
  Cad *cad = nullptr, *cad2 = nullptr;
  float2 *dec = nullptr, *dec2 = nullptr, *T = nullptr, *Zn = nullptr, *Tw = nullptr, *Zwn = nullptr, *G = nullptr;
  int* flag = nullptr;
  LKB_TRY(ws_get_t<Cad>(WS_K, ptotal + 4, &cad));
  LKB_TRY(ws_get_t<Cad>(WS_L, ptotal + 4, &cad2));
  LKB_TRY(ws_get_t<float2>(WS_N, (size_t)group * Mh, &T));
  LKB_TRY(ws_get_t<float2>(WS_O, (size_t)group * Mh, &Zn));
  LKB_TRY(ws_get_t<float2>(WS_P, (size_t)group * Mh2, &Tw));
  LKB_TRY(ws_get_t<float2>(WS_OUT3, (size_t)group * Mh2, &Zwn));
  LKB_TRY(ws_get_t<float2>(WS_OUT2, (size_t)group * std::max(cells, cells2), &G));
  // flux modes below kmax, window modes below 2 kmax; the single-term finish indexes dec by row k, the multi-term one
  // by mode index
  const int64_t kmax = (int64_t)std::max(nterms, 1) * (k0 + F);
  const int64_t dec_first = nterms ? 0 : k0, dec_len = nterms ? kmax : F;
  LKB_TRY(ws_get_t<float2>(WS_IN4, dec_len, &dec));
  LKB_TRY(ws_get_t<float2>(WS_IN5, 2 * kmax, &dec2));
  LKB_TRY(ws_get_t<int>(WS_IN6, 1, &flag));

  LKB_CUDA_CHECK(cudaMemsetAsync(flag, 0, sizeof(int), st));
  {
    const unsigned gx = (unsigned)std::min<int64_t>(64, (nmax + 255) / 256);
    LKB_LAUNCH(dim3(gx ? gx : 1, (unsigned)B), 256, st, nufft_cad_ragged_kernel)(d_t, d_off, d_po, d_span, df, M, M2, w, cad,
                                                                          cad2, flag);
    LKB_LAUNCH_CHECK();
  }
  int h_flag = 0;
  LKB_CUDA_CHECK(cudaMemcpyAsync(&h_flag, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
  LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  if (h_flag) { set_error("NUFFT (ragged): a light curve has unsorted times"); return LKB_E_UNSUPPORTED; }
  LKB_LAUNCH(blocks_for(dec_len, 128), 128, st, nufft_deconv_kernel)(dec_first, dec_len, M, w, (double)beta, gl, dec);
  LKB_LAUNCH_CHECK();
  LKB_LAUNCH(blocks_for(2 * kmax, 128), 128, st, nufft_deconv_kernel)(0, 2 * kmax, M2, w, (double)beta, gl, dec2);
  LKB_LAUNCH_CHECK();

  // kernel weights in FP64 from the time stamps (default; LKB_NUFFT_RAGGED_W32=1: the fp32 form, for A/B timing)
  const double* t_acc = getenv("LKB_NUFFT_RAGGED_W32") ? nullptr : d_t;
  const int ptc = V2_LOG_TILE - (p - 1 - V2_PB), ptc2 = V2_LOG_TILE - (p2 - 1 - V2_PB);
  const int nk2 = (int)(kmax >> (p - 1 - V2_PB)) + 1, nk2w = (int)((2 * kmax) >> (p2 - 1 - V2_PB)) + 1;
  prof_begin(st);
  for (int b0 = 0; b0 < B; b0 += group) {
    LKB_CHI2_OBSERVE(CHI2_PATH_GROUP);
    const int Bg = std::min(group, B - b0);
    const int64_t *off_g = d_off + b0, *po_g = d_po + b0;
    double span_min = 1e300;
    for (int b = b0; b < b0 + Bg; ++b) span_min = fmin(span_min, h_span[b]);
    const double nlow = floor((LS_LOWF_CYCLES / span_min - f0) / df) + 2.0;
    const int64_t F_low_max = nlow < 0.0 ? 0 : (nlow > (double)F ? F : (int64_t)nlow);
    // window terms: unit strengths on the 2x finer grid (modes kk and 2 kk), then the flux
    LKB_LAUNCH(dim3(blocks_for((int64_t)cells2, 256), (unsigned)Bg), 256, st, nufft2_spread_ragged_kernel)(
        cad2, nullptr, off_g, po_g, w, beta, p2, ptc2, n1max2, G, t_acc, df);
    LKB_LAUNCH_CHECK();
    LKB_TRY(v2_cols(G, Tw, p2, n1max2, Bg, tb2, st));
    LKB_TRY(v2_rows(Tw, p2, Bg, tb2, nullptr, Zwn, nk2w, st));
    LKB_LAUNCH(dim3(blocks_for((int64_t)cells, 256), (unsigned)Bg), 256, st, nufft2_spread_ragged_kernel)(
        cad, d_y, off_g, po_g, w, beta, p, ptc, n1max, G, t_acc, df);
    LKB_LAUNCH_CHECK();
    LKB_TRY(v2_cols(G, T, p, n1max, Bg, tb, st));
    LKB_TRY(v2_rows(T, p, Bg, tb, nullptr, Zn, nk2, st));
    const double* ns_g = d_ns ? d_ns + b0 : nullptr;
    float* pow_g = d_pow + (size_t)b0 * F;
#define LKB_CHI2_FINISH(NT)                                                                                            \
  LKB_LAUNCH(blocks_for(F * Bg, 256), 256, st, nufft2_finish_chi2_ragged_kernel<NT>)(                                  \
      Zn, p, Zwn, p2, dec, dec2, k0, F, f0, df, off_g, po_g, d_t, d_y, d_span + b0, d_ysum + b0, normalization, ns_g, \
      Bg, pow_g)
#define LKB_CHI2_LOW(NT)                                                                                               \
  LKB_LAUNCH(blocks_for(F_low_max * Bg, 4), 128, st, nufft_lowrows_chi2_ragged_kernel<NT>)(                            \
      d_t, d_y, off_g, po_g, d_span + b0, d_ysum + b0, f0, df, F_low_max, F, normalization, ns_g, Bg, pow_g)
    switch (nterms) {
      case 0:
        LKB_LAUNCH(blocks_for(F * Bg, 256), 256, st, nufft2_finish_ragged_kernel)(
            Zn, p, Zwn, p2, dec, dec2, k0, F, f0, df, off_g, d_span + b0, d_ysum + b0, normalization, ns_g, Bg, pow_g);
        break;
      case 1: LKB_CHI2_FINISH(1); break;
      case 2: LKB_CHI2_FINISH(2); break;
      case 3: LKB_CHI2_FINISH(3); break;
      default: LKB_CHI2_FINISH(4); break;
    }
    LKB_LAUNCH_CHECK();
    if (F_low_max > 0) {
      switch (nterms) {
        case 0:
          LKB_LAUNCH(blocks_for(F_low_max * Bg, 4), 128, st, nufft_lowrows_ragged_kernel)(
              d_t, d_y, off_g, po_g, d_span + b0, d_ysum + b0, f0, df, F_low_max, F, normalization, ns_g, Bg, pow_g);
          break;
        case 1: LKB_CHI2_LOW(1); break;
        case 2: LKB_CHI2_LOW(2); break;
        case 3: LKB_CHI2_LOW(3); break;
        default: LKB_CHI2_LOW(4); break;
      }
      LKB_LAUNCH_CHECK();
    }
#undef LKB_CHI2_FINISH
#undef LKB_CHI2_LOW
  }
  prof_end(st);
  return LKB_OK;
}

// f_k = (k0 + k) df with integer k0, and 0 < df * baseline <= 1 for every light curve
int ragged_grid_check(int B, const double* h_span, double f0, double df, int64_t* k0) {
  const double q = f0 / df, k0d = rint(q);
  if (!(df > 0.0) || !(f0 >= 0.0) || fabs(q - k0d) > 1e-9 * fmax(1.0, q) || k0d > 1.0e7) {
    set_error("NUFFT (ragged): the grid is not f_k = (k0 + k) df with integer k0");
    return LKB_E_UNSUPPORTED;
  }
  for (int b = 0; b < B; ++b) {
    if (!(h_span[b] > 0.0) || !(df * h_span[b] <= 1.0 + 1e-9)) {
      set_error("NUFFT (ragged): a light curve has zero baseline or df * baseline > 1");
      return LKB_E_UNSUPPORTED;
    }
  }
  *k0 = (int64_t)k0d;
  return LKB_OK;
}

// fine-grid budget of a ragged call: LKB_NUFFT_RAGGED_MB (default 16384)
double ragged_cap_mb() {
  double cap_mb = 16384.0;
  if (const char* e = getenv("LKB_NUFFT_RAGGED_MB")) { const double v = atof(e); if (v > 0.0) cap_mb = v; }
  return cap_mb;
}
}  // namespace

bool ls_nufft_ragged_enabled() {               // `auto` of the ragged entry may use this path (default: yes)
  const char* e = getenv("LKB_LS_RAGGED_NUFFT");
  return !e || atoi(e) != 0;
}

// One shared regular grid f_k = f0 + k df (k0 = f0 / df integer), light curves in the K1 prologue's layout
// (d_t / d_y padded CSR with offsets d_po; d_off the unpadded offsets; d_span, d_ysum per light curve).
// h_span: host copy of d_span.  Returns LKB_E_UNSUPPORTED when a light curve is not eligible (unsorted times,
// df * baseline > 1): the caller then runs the direct kernel.
// The fine grids of all light curves need 24 (M + 2 M2) bytes per pair; batches whose grids exceed
// LKB_NUFFT_RAGGED_MB (default 16384) are processed in groups of pairs through the same buffers.
int ls_nufft_ragged_launch(const double* d_t, const float* d_y, const int64_t* d_off, const int64_t* d_po,
                           const int64_t* h_off, int B, int64_t ptotal, int64_t nmax, const double* d_span,
                           const double* h_span, const double* d_ysum, int64_t F, double f0, double df,
                           int normalization, const double* d_ns, float* d_pow, cudaStream_t st) {
  (void)h_off;
  int64_t k0 = 0;
  LKB_TRY(ragged_grid_check(B, h_span, f0, df, &k0));
  // flux grid 2^p, window grid 2^p2 = 2^(p + 1).  Both must be in the v2 range: above it (2^20 < k0 + F) the call is
  // refused and `auto` runs the direct kernel, rather than pair-packing the window grid (LKB_NUFFT_FFT = global /
  // smem / fused: the round-1 transforms up to 2^24 cells)
  const bool round1 = round1_requested();
  const int p = single_term_log2(k0 + F), p2 = round1 ? fine_log2(2 * (k0 + F)) : p + 1;
  if (p2 > 24) { set_error("NUFFT (ragged): fine grid larger than 2^24 cells"); return LKB_E_UNSUPPORTED; }
  if (!round1 && !(v2_supported(p) && v2_supported(p2))) {
    set_error("NUFFT (ragged): fine grids of 2^%d / 2^%d cells are outside the v2 transform's range", p, p2);
    return LKB_E_UNSUPPORTED;
  }
  const double sigma = fmin(2.0, nufft::grid_sigma(p, k0 + F));   // (the validated rule: beta = 2.30 w from sigma = 2 on)
  const int w = kernel_width(sigma);
  const float beta = (float)nufft::es_beta(w, sigma);
  const int64_t M = (int64_t)1 << p, M2 = (int64_t)1 << p2;
  const int npairs_all = (B + 1) / 2;
  const double cap_mb = ragged_cap_mb();
  const double per_pair_mb = (2.0 * (double)M + 2.0 * (double)M2) * sizeof(float2) / 1048576.0;
  int group = (int)fmax(1.0, floor(cap_mb / per_pair_mb));
  if (group > npairs_all) group = npairs_all;
  GlNodes gl;
  nufft::gauss_legendre(GL_NQ, gl.x, gl.w);

  // v2 (one real transform per light curve, nufft_v2.cuh) when both fine grids are in range
  if (fft_mode(p) == 3 && fft_mode(p2) == 3) {
    record_plan(true, p, p2);
    return ls_nufft_ragged_v2(d_t, d_y, d_off, d_po, B, ptotal, nmax, d_span, h_span, d_ysum, F, f0, df, k0, p, p2, w, beta,
                              cap_mb, normalization, d_ns, d_pow, st, 0);
  }
  record_plan(false, p, p2);

  Cad *cad = nullptr, *cad2 = nullptr;
  float2 *dec = nullptr, *dec2 = nullptr, *Za = nullptr, *Zb = nullptr, *Zw = nullptr;
  float* absmax = nullptr;
  int* flag = nullptr;
  LKB_TRY(ws_get_t<Cad>(WS_K, ptotal + 4, &cad));
  LKB_TRY(ws_get_t<Cad>(WS_L, ptotal + 4, &cad2));
  LKB_TRY(ws_get_t<float>(WS_M, B, &absmax));
  LKB_TRY(ws_get_t<float2>(WS_N, (size_t)group * M, &Za));
  LKB_TRY(ws_get_t<float2>(WS_O, (size_t)group * M, &Zb));
  LKB_TRY(ws_get_t<float2>(WS_P, (size_t)2 * group * M2, &Zw));
  LKB_TRY(ws_get_t<float2>(WS_IN4, F, &dec));
  LKB_TRY(ws_get_t<float2>(WS_IN5, 2 * (k0 + F), &dec2));
  LKB_TRY(ws_get_t<int>(WS_IN6, 1, &flag));

  LKB_CUDA_CHECK(cudaMemsetAsync(flag, 0, sizeof(int), st));
  {
    const unsigned gx = (unsigned)std::min<int64_t>(64, (nmax + 255) / 256);
    LKB_LAUNCH(dim3(gx ? gx : 1, (unsigned)B), 256, st, nufft_cad_ragged_kernel)(d_t, d_off, d_po, d_span, df, M, M2, w, cad,
                                                                          cad2, flag);
    LKB_LAUNCH_CHECK();
  }
  int h_flag = 0;
  LKB_CUDA_CHECK(cudaMemcpyAsync(&h_flag, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
  LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  if (h_flag) { set_error("NUFFT (ragged): a light curve has unsorted times"); return LKB_E_UNSUPPORTED; }
  LKB_LAUNCH(B, 256, st, nufft_absmax_ragged_kernel)(d_y, d_off, d_po, absmax);
  LKB_LAUNCH_CHECK();
  LKB_LAUNCH(blocks_for(F, 128), 128, st, nufft_deconv_kernel)(k0, F, M, w, (double)beta, gl, dec);
  LKB_LAUNCH_CHECK();
  LKB_LAUNCH(blocks_for(2 * (k0 + F), 128), 128, st, nufft_deconv_kernel)(0, 2 * (k0 + F), M2, w, (double)beta, gl, dec2);
  LKB_LAUNCH_CHECK();

  prof_begin(st);
  for (int g0 = 0; g0 < npairs_all; g0 += group) {
    const int npairs = std::min(group, npairs_all - g0);
    const int b0 = 2 * g0, Bg = std::min(B - b0, 2 * npairs);
    const int64_t *off_g = d_off + b0, *po_g = d_po + b0;
    const float* amax_g = absmax + b0;
    // rows k with (f0 + k df) * span_b <= LS_LOWF_CYCLES for at least one light curve of the group
    double span_min = 1e300;
    for (int b = b0; b < b0 + Bg; ++b) span_min = fmin(span_min, h_span[b]);
    const double nlow = floor((LS_LOWF_CYCLES / span_min - f0) / df) + 2.0;
    const int64_t F_low_max = nlow < 0.0 ? 0 : (nlow > (double)F ? F : (int64_t)nlow);
    float2* Zw_out = nullptr;
    float2* Zout = nullptr;
    int pa = 0, pa2 = 0;                       // LKB_NUFFT_FFT=smem|fused: four-step transforms (in place)
    {
    // window terms: unit strengths on the 2x finer grid
    LKB_LAUNCH(blocks_for((int64_t)npairs * M2, 256), 256, st, nufft_spread_ragged_kernel)(cad2, nullptr, off_g, po_g, amax_g,
                                                                                    Bg, npairs, w, beta, p2, Zw);
    LKB_LAUNCH_CHECK();
    if (fft_mode() != 0) {
      LKB_TRY(fft_fourstep(Zw, p2, npairs, st, &pa2, nullptr));
      Zw_out = Zw;
    } else {
      LKB_TRY(fft_passes(Zw, Zw + (size_t)npairs * M2, p2, npairs, st, &Zw_out));
    }
    // flux
    LKB_LAUNCH(blocks_for((int64_t)npairs * M, 256), 256, st, nufft_spread_ragged_kernel)(cad, d_y, off_g, po_g, amax_g, Bg,
                                                                                   npairs, w, beta, p, Za);
    LKB_LAUNCH_CHECK();
    if (fft_mode() != 0) {
      LKB_TRY(fft_fourstep(Za, p, npairs, st, &pa, nullptr));
      Zout = Za;
    } else {
      LKB_TRY(fft_passes(Za, Zb, p, npairs, st, &Zout));
    }
    }
    LKB_LAUNCH(blocks_for(F * npairs, 256), 256, st, nufft_finish_ragged_kernel)(
        Zout, p, Zw_out, p2, dec, dec2, k0, F, f0, df, off_g, d_span + b0, d_ysum + b0, amax_g, normalization,
        d_ns ? d_ns + b0 : nullptr, Bg, npairs, pa, pa2, d_pow + (size_t)b0 * F);
    LKB_LAUNCH_CHECK();
    if (F_low_max > 0) {
      LKB_LAUNCH(blocks_for(F_low_max * Bg, 4), 128, st, nufft_lowrows_ragged_kernel)(
          d_t, d_y, off_g, po_g, d_span + b0, d_ysum + b0, f0, df, F_low_max, F, normalization,
          d_ns ? d_ns + b0 : nullptr, Bg, d_pow + (size_t)b0 * F);
      LKB_LAUNCH_CHECK();
    }
  }
  prof_end(st);
  return LKB_OK;
}

// Multi-term ("chi2", nterms in [1, 4]) periodogram of a ragged batch on one shared grid f_k = (k0 + k) df through the
// v2 transforms: same inputs as ls_nufft_ragged_launch.  Harmonic j of every row is a mode of the same two transforms,
// so the flux grid is sized for modes up to nterms (k0 + F) and the unit-strength grid for modes up to
// 2 nterms (k0 + F); each row then solves its (2 nterms + 1)^2 normal equations in fp64.  Returns LKB_E_UNSUPPORTED
// (the caller runs the direct kernel) when a light curve is not eligible (unsorted times, df * baseline > 1) or either
// fine grid is outside the v2 range [2^14, 2^23].
int ls_nufft_chi2_ragged_launch(const double* d_t, const float* d_y, const int64_t* d_off, const int64_t* d_po,
                                const int64_t* h_off, int B, int64_t ptotal, int64_t nmax, const double* d_span,
                                const double* h_span, const double* d_ysum, int64_t F, double f0, double df,
                                int normalization, const double* d_ns, float* d_pow, cudaStream_t st, int nterms) {
  (void)h_off;
  if (nterms < 1 || nterms > 4) { set_error("NUFFT (ragged chi2): nterms must be in [1, 4]"); return LKB_E_ARG; }
  int64_t k0 = 0;
  LKB_TRY(ragged_grid_check(B, h_span, f0, df, &k0));
  const int64_t kmax = (int64_t)nterms * (k0 + F);
  // both grids at least 2^V2R_P_MIN cells, as for the single-term transforms (single_term_log2): a small grid takes the
  // v2 transform instead of being refused; sigma = min(2, grid_sigma) keeps the kernel width and shape
  const int p = std::max(fine_log2(kmax), V2R_P_MIN), p2 = std::max(fine_log2(2 * kmax), V2R_P_MIN);
  if (p2 > V2R_P_MAX || fft_mode(p) != 3 || fft_mode(p2) != 3) {
    set_error("NUFFT (ragged chi2): fine grids of 2^%d / 2^%d cells are outside the v2 transform's range", p, p2);
    return LKB_E_UNSUPPORTED;
  }
  const double sigma = fmin(2.0, nufft::grid_sigma(p, kmax));
  const int w = kernel_width(sigma);
  const float beta = (float)nufft::es_beta(w, sigma);
  record_plan(true, p, p2);
  return ls_nufft_ragged_v2(d_t, d_y, d_off, d_po, B, ptotal, nmax, d_span, h_span, d_ysum, F, f0, df, k0, p, p2, w, beta,
                            ragged_cap_mb(), normalization, d_ns, d_pow, st, nterms);
}

}  // namespace lkb
