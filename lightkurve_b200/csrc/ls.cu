// Lomb-Scargle kernels (generalised floating-mean periodogram, Zechmeister & Kuerster 2009),
// the arithmetic lightkurve obtains from astropy at
//   /root/reference/src/lightkurve/periodogram.py:961-964  (LombScargle(...).power)
// followed by lightkurve's own rescale at :969-975 (fused here as the epilogue).
//
//   K1  ls_direct_kernel      ragged batch: one warp per group of LS_FPW frequency bins, the
//                             light curve's (time, flux) tiles staged into shared memory by the
//                             TMA engine (cp.async.bulk + mbarrier), fp64 phase reduction,
//                             MUFU sin/cos, fp32 lane partials flushed to fp64 per tile,
//                             warp-shuffle reduction, fp64 epilogue.
//   K2a ls_window_kernel      shared cadence grid: the y-independent sums (S, C, CC, SC) -> the
//                             rotation tau and 1/CC', 1/SS' once per frequency.
//   K2b ls_shared_simt_kernel shared cadence grid, CUDA-core contraction: sin/cos design-matrix
//                             tiles synthesised on the fly in shared memory and contracted with
//                             a [cadence x light-curve] flux tile (register-tiled fp32 FMA).
//   (K2c, the tcgen05 contraction, lives in ls_tc.cu.)
#include "common.cuh"
#include "ptx.cuh"
#include "ls_common.cuh"
#include <stdlib.h>
#include <stdint.h>
#include <type_traits>
#include <vector>

namespace lkb {

// ls_nufft.cu: the opt-in NUFFT path for ragged batches (LKB_LS_RAGGED_NUFFT=1)
bool ls_nufft_ragged_enabled();
int ls_nufft_ragged_launch(const double* d_t, const float* d_y, const int64_t* d_off, const int64_t* d_po,
                           const int64_t* h_off, int B, int64_t ptotal, int64_t nmax, const double* d_span,
                           const double* h_span, const double* d_ysum, int64_t F, double f0, double df,
                           int normalization, const double* d_ns, float* d_pow, cudaStream_t st);
int ls_nufft_chi2_ragged_launch(const double* d_t, const float* d_y, const int64_t* d_off, const int64_t* d_po,
                                const int64_t* h_off, int B, int64_t ptotal, int64_t nmax, const double* d_span,
                                const double* h_span, const double* d_ysum, int64_t F, double f0, double df,
                                int normalization, const double* d_ns, float* d_pow, cudaStream_t st, int nterms);

// `auto` of the multi-term periodogram takes the NUFFT path from this much work on (sum over the light curves of
// cadences x frequency bins).  Measured crossover on an H100 (tools/bench_chi2.py, DESIGN.md section 4 K1c): at 2e7 the
// direct kernel is faster for nterms 1-3 and as fast at 4; at 8e7 the NUFFT path is faster for every nterms.
constexpr double LS_CHI2_NUFFT_MIN_WORK = 5e7;

// Is fq[0 .. Fb) the regular grid f0 + k df (f0 >= 0, df > 0, every bin within 1e-6 df)?
static bool regular_grid(const double* fq, int64_t Fb, double* f0, double* df) {
  if (Fb < 2 || Fb >= ((int64_t)1 << 31)) return false;
  *f0 = fq[0];
  *df = fq[1] - fq[0];
  if (!(*f0 >= 0.0) || !(*df > 0.0)) return false;
  for (int64_t k = 0; k < Fb; ++k)
    if (fabs(fq[k] - (*f0 + (double)k * *df)) > 1e-6 * *df) return false;
  return true;
}

// Per-cadence entry of a regular-grid light curve (ragged path): fixed-point phases of the grid origin and of one
// grid step, plus the fp32 rotation by one step - the bins after a warp's first are obtained by rotating (cos, sin)
// (4 FMA-pipe ops) instead of two more MUFU evaluations.
struct __align__(8) LsTabEntry {
  unsigned long long a, b;      // frac(f0 t) 2^64, frac(df t) 2^64
  float cb, sb;                 // cos / sin of 2 pi frac(df t)
};
static_assert(sizeof(LsTabEntry) == 24, "LsTabEntry must be 24 bytes");



// =====================================================================================
// Prologue: centre the flux the way astropy does (y - dot(w, y), w = 1/N), shift time to
// the light curve's first cadence (power is shift-invariant; the shift keeps f*t small),
// convert flux to fp32, and lay each light curve out at a 16-byte aligned offset so that
// the TMA bulk copies in K1 are legal.
// =====================================================================================
template <typename TY>
__global__ void __launch_bounds__(256)
ls_prep_ragged_kernel(const double* __restrict__ t, const TY* __restrict__ y,
                      const int64_t* __restrict__ offsets, const int64_t* __restrict__ poffsets,
                      double* __restrict__ t_out, float* __restrict__ y_out, double* __restrict__ tspan,
                      const double* __restrict__ grid_f0, const double* __restrict__ grid_df,
                      LsTabEntry* __restrict__ tab_out, double* __restrict__ ysum,
                      double* __restrict__ y_out64 = nullptr) {
  __shared__ double red[33];
  __shared__ int s_const;
  __shared__ double s_span[8];
  const int b = blockIdx.x;
  const int64_t o = offsets[b], n = offsets[b + 1] - o, po = poffsets[b], np_ = poffsets[b + 1] - po;
  if (n <= 0) return;
  double acc = 0.0;
  if (threadIdx.x == 0) s_const = 1;
  __syncthreads();
  const double y0 = (double)y[o];
  int is_const = 1;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    double v = (double)y[o + i];
    acc += v;
    if (v != y0) is_const = 0;
  }
  if (!is_const) s_const = 0;
  const double mean = block_sum(acc, red) / (double)n;
  const bool cst = s_const != 0;
  const double t0 = t[o];
  double span = 0.0, resid = 0.0;
  for (int64_t i = threadIdx.x; i < np_; i += blockDim.x) {
    LsTabEntry e;
    e.a = 0ull; e.b = 0ull; e.cb = 1.0f; e.sb = 0.0f;
    if (i < n) {
      const double tr = t[o + i] - t0;
      span = fmax(span, fabs(tr));
      t_out[po + i] = tr;
      const double yd = cst ? 0.0 : ((double)y[o + i] - mean);
      const float yv = (float)yd;
      if (y_out64) {              // chi2 / model path keeps the centred flux in fp64
        y_out64[po + i] = yd;
        resid += yd;
      } else {
        y_out[po + i] = yv;
        resid += (double)yv;
      }
      if (tab_out) {      // fixed-point phase table of this light curve's regular grid (ls_common.cuh)
        const double x = grid_f0[b] * tr, z = grid_df[b] * tr;
        e.a = __double2ull_rd((x - floor(x)) * 18446744073709551616.0);
        e.b = __double2ull_rd((z - floor(z)) * 18446744073709551616.0);
        double sb, cb;
        sincospi(2.0 * (z - rint(z)), &sb, &cb);
        e.cb = (float)cb;
        e.sb = (float)sb;
      }
    } else {
      t_out[po + i] = 0.0;
      if (y_out64) y_out64[po + i] = 0.0;
      else y_out[po + i] = 0.0f;
    }
    if (tab_out) tab_out[po + i] = e;
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) span = fmax(span, __shfl_xor_sync(0xffffffffu, span, s));
  if ((threadIdx.x & 31) == 0) s_span[threadIdx.x >> 5] = span;
  __syncthreads();
  if (threadIdx.x == 0) {
    double m = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) m = fmax(m, s_span[w]);
    tspan[b] = m;
  }
  const double rs = block_sum(resid, red);
  if (threadIdx.x == 0) ysum[b] = rs;
}

// Same for a [B, N] matrix sharing one time grid: writes Yc [B, Npad] fp32, zero padded.
template <typename TY>
__global__ void __launch_bounds__(256)
ls_prep_shared_kernel(const TY* __restrict__ y, int64_t N, int64_t Npad, float* __restrict__ y_out,
                      float* __restrict__ y_absmax, float* __restrict__ ysum) {
  __shared__ double red[33];
  __shared__ int s_const;
  __shared__ float s_max[8];
  const int b = blockIdx.x;
  const TY* yr = y + (int64_t)b * N;
  float* yo = y_out + (int64_t)b * Npad;
  if (threadIdx.x == 0) s_const = 1;
  __syncthreads();
  const double y0 = (double)yr[0];
  double acc = 0.0;
  int is_const = 1;
  for (int64_t i = threadIdx.x; i < N; i += blockDim.x) {
    double v = (double)yr[i];
    acc += v;
    if (v != y0) is_const = 0;
  }
  if (!is_const) s_const = 0;
  const double mean = block_sum(acc, red) / (double)N;
  const bool cst = s_const != 0;
  float mx = 0.f;
  double resid = 0.0;
  for (int64_t i = threadIdx.x; i < Npad; i += blockDim.x) {
    float v = (i < N && !cst) ? (float)((double)yr[i] - mean) : 0.0f;
    yo[i] = v;
    resid += (double)v;
    mx = fmaxf(mx, fabsf(v));
  }
  const double rs = block_sum(resid, red);
  if (threadIdx.x == 0 && ysum) ysum[b] = (float)rs;
  if (y_absmax) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
      float m = 0.f;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) m = fmaxf(m, s_max[w]);
      y_absmax[b] = m;
    }
  }
}

// t_out[i] = t[i] - t[0] for i < N, 0 for the padding cadences [N, Npad)
// also raises *unsorted (nullable) when the times are not ascending (the NUFFT path needs sorted times) and adds an
// order-sensitive 64-bit checksum of the time stamps to *hash (nullable): the key of the cached plan
__global__ void ls_shift_time_kernel(const double* __restrict__ t, int64_t N, int64_t Npad, double* __restrict__ t_out,
                                     int* __restrict__ unsorted, unsigned long long* __restrict__ hash) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < Npad) t_out[i] = (i < N) ? (t[i] - t[0]) : 0.0;
  if (unsorted && i > 0 && i < N && t[i] < t[i - 1]) *unsorted = 1;
  if (hash) {
    unsigned long long h = 0ull;
    if (i < N) {
      h = (unsigned long long)__double_as_longlong(t[i]) + 0x9E3779B97F4A7C15ull * (unsigned long long)(i + 1);
      h ^= h >> 30; h *= 0xBF58476D1CE4E5B9ull; h ^= h >> 27; h *= 0x94D049BB133111EBull; h ^= h >> 31;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) h += __shfl_xor_sync(0xffffffffu, h, o);
    if ((threadIdx.x & 31) == 0 && h) atomicAdd(hash, h);
  }
}

// =====================================================================================
// K1: direct sums, ragged batch.
// grid = (ceil(Fmax / LS_FPB), B), block = LS_WARPS*32.
// =====================================================================================
constexpr int LS_WARPS = 8;
constexpr int LS_FPW = 4;                       // frequency bins per warp
constexpr int LS_FPB = LS_WARPS * LS_FPW;       // frequency bins per block

// REGULAR = every frequency grid is f0 + k df: phases come from the fixed-point table (16 B per
// cadence, no fp64 on the hot loop); otherwise fp64 phase = f * t (8 B per cadence).
template <bool REGULAR>
__global__ void __launch_bounds__(LS_WARPS * 32)
ls_direct_kernel(const double* __restrict__ tws, const LsTabEntry* __restrict__ tabws, const float* __restrict__ yws,
                 const int64_t* __restrict__ offsets, const int64_t* __restrict__ poffsets,
                 const double* __restrict__ freq, const int64_t* __restrict__ freq_offsets, int64_t F_shared,
                 const double* __restrict__ tspan, const double* __restrict__ ysum, int normalization,
                 const double* __restrict__ norm_scale, float* __restrict__ power) {
  constexpr int TN = REGULAR ? 768 : 1536;      // cadences per shared-memory tile (<= 42 KB static smem)
  using Elem = typename std::conditional<REGULAR, LsTabEntry, double>::type;
  __shared__ __align__(16) Elem s_t[2][TN];
  __shared__ __align__(16) float s_y[2][TN];
  __shared__ __align__(8) uint64_t s_bar[2];

  const int b = blockIdx.y;
  const int64_t n = offsets[b + 1] - offsets[b];
  const int64_t po = poffsets[b], np_ = poffsets[b + 1] - po;
  const int64_t fo = freq_offsets ? freq_offsets[b] : 0;
  const int64_t F = freq_offsets ? (freq_offsets[b + 1] - fo) : F_shared;
  const int64_t po_out = freq_offsets ? fo : (int64_t)b * F_shared;
  const int64_t f_blk = (int64_t)blockIdx.x * LS_FPB;
  if (f_blk >= F) return;
  if (n <= 0) {      // empty light curve: numpy semantics of an empty mean -> NaN everywhere
    for (int64_t f = f_blk + threadIdx.x; f < min(F, f_blk + (int64_t)LS_FPB); f += blockDim.x)
      power[po_out + f] = __int_as_float(0x7fc00000);
    return;
  }

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t f_base = f_blk + warp * LS_FPW;

  double fr[LS_FPW];
  double fmin_abs = 1e300;
#pragma unroll
  for (int j = 0; j < LS_FPW; ++j) {
    fr[j] = (f_base + j < F) ? freq[fo + f_base + j] : 0.0;
    if (f_base + j < F) fmin_abs = fmin(fmin_abs, fabs(fr[j]));
  }
  // low-frequency group (see ls_common.cuh): full fp64 evaluation, warp-uniform choice
  const bool lowf = fmin_abs * tspan[b] <= LS_LOWF_CYCLES;

  if (threadIdx.x == 0) {
    ptx::mbar_init(&s_bar[0], 1);
    ptx::mbar_init(&s_bar[1], 1);
    ptx::mbar_fence_init();
  }
  __syncthreads();

  const Elem* src = REGULAR ? reinterpret_cast<const Elem*>(tabws) : reinterpret_cast<const Elem*>(tws);
  const int ntiles = (int)((np_ + TN - 1) / TN);
  auto issue = [&](int tile) {
    const int buf = tile & 1;
    const int64_t c0 = (int64_t)tile * TN;
    const uint32_t cnt = (uint32_t)min((int64_t)TN, np_ - c0);   // multiple of 4
    ptx::mbar_arrive_expect_tx(&s_bar[buf], cnt * (uint32_t)(sizeof(Elem) + 4));
    ptx::bulk_g2s(&s_t[buf][0], src + po + c0, cnt * (uint32_t)sizeof(Elem), &s_bar[buf]);
    ptx::bulk_g2s(&s_y[buf][0], yws + po + c0, cnt * 4u, &s_bar[buf]);
  };
  if (threadIdx.x == 0) issue(0);

  LsSums<double> dsum[LS_FPW];
#pragma unroll
  for (int j = 0; j < LS_FPW; ++j) dsum[j].zero();

  for (int tile = 0; tile < ntiles; ++tile) {
    const int buf = tile & 1;
    if (threadIdx.x == 0 && tile + 1 < ntiles) {
      ptx::fence_proxy_async_smem();
      issue(tile + 1);
    }
    ptx::mbar_wait(&s_bar[buf], (tile >> 1) & 1);

    const int64_t c0 = (int64_t)tile * TN;
    const int cnt = (int)min((int64_t)TN, n - c0);   // true (unpadded) cadences in this tile
    if (lowf) {
      for (int i = lane; i < cnt; i += 32) {
        const double tt = tws[po + c0 + i];          // rare path: read the times straight from L2
        const double yy = (double)s_y[buf][i];
#pragma unroll
        for (int j = 0; j < LS_FPW; ++j) {
          double s, c;
          ls_sincos_cycles_f64(fr[j] * tt, s, c);
          dsum[j].add(yy, s, c);
        }
      }
    } else {
      LsSums<float> fs[LS_FPW];
#pragma unroll
      for (int j = 0; j < LS_FPW; ++j) fs[j].zero();
      for (int i = lane; i < cnt; i += 32) {
        const float yy = s_y[buf][i];
        if constexpr (REGULAR) {
          const LsTabEntry e = s_t[buf][i];
          const uint32_t ph = (uint32_t)((e.a + (unsigned long long)f_base * e.b) >> 32);   // exact for bin f_base
          float s, c;
          ls_sincos_fixed32(ph, s, c);
          fs[0].add(yy, s, c);
#pragma unroll
          for (int j = 1; j < LS_FPW; ++j) {              // next bins: rotate by one grid step
            const float s2 = fmaf(s, e.cb, c * e.sb), c2 = fmaf(c, e.cb, -s * e.sb);
            s = s2;
            c = c2;
            fs[j].add(yy, s, c);
          }
        } else {
          const double tt = s_t[buf][i];
#pragma unroll
          for (int j = 0; j < LS_FPW; ++j) {
            float s, c;
            ls_sincos_cycles(fr[j] * tt, s, c);
            fs[j].add(yy, s, c);
          }
        }
      }
#pragma unroll
      for (int j = 0; j < LS_FPW; ++j) dsum[j].accumulate(fs[j]);
    }
    __syncthreads();   // everyone done with `buf` before it is refilled
  }

#pragma unroll
  for (int j = 0; j < LS_FPW; ++j) {
    dsum[j].warp_reduce();
    if (lane == 0 && f_base + j < F) {
      const double p = ls_power_from_sums(dsum[j], (double)n, ysum[b]);
      power[po_out + f_base + j] = ls_normalize(p, (double)n, normalization, norm_scale ? norm_scale[b] : 1.0);
    }
  }
}

// =====================================================================================
// K2a: per-frequency window terms on the shared grid.
// One warp per frequency; rot[f] = {cos tau, sin tau, 1/(2 N CC'), 1/(2 N SS')}.
// =====================================================================================
template <bool REGULAR>
__global__ void __launch_bounds__(128)
ls_window_kernel(const double* __restrict__ t, const ulonglong2* __restrict__ tab, int64_t N,
                 const double* __restrict__ freq, int64_t F, float4* __restrict__ rot, float2* __restrict__ rot2) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t f = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
  if (f >= F) return;
  const double fr = freq[f];
  const unsigned long long kf = (unsigned long long)f;
  LsSums<double> d;
  d.zero();
  const bool lowf = fabs(fr) * fabs(t[N - 1]) <= LS_LOWF_CYCLES;     // t is shifted to t[0] = 0 and sorted
  if (lowf) {
    for (int64_t i = lane; i < N; i += 32) {
      double s, c;
      ls_sincos_cycles_f64(fr * t[i], s, c);
      d.add(0.0, s, c);
    }
  } else
  for (int64_t c0 = 0; c0 < N; c0 += 32 * 64) {
    LsSums<float> fs;
    fs.zero();
    const int64_t c1 = min(N, c0 + 32 * 64);
    for (int64_t i = c0 + lane; i < c1; i += 32) {
      float s, c;
      if (REGULAR) {
        const ulonglong2 e = tab[i];
        ls_sincos_fixed(e.x + kf * e.y, s, c);
      } else {
        ls_sincos_cycles(fr * t[i], s, c);
      }
      fs.add(0.f, s, c);
    }
    d.accumulate(fs);
  }
  d.warp_reduce();
  if (lane == 0) {
    double ct, st, cc, ss;
    ls_rotation(d, (double)N, ct, st, cc, ss);
    const double k = 1.0 / (2.0 * (double)N);
    rot[f] = make_float4((float)ct, (float)st, (float)(k / cc), (float)(k / ss));
    rot2[f] = make_float2((float)((d.c * ct + d.s * st) / (double)N), (float)((d.s * ct - d.c * st) / (double)N));
  }
}

// =====================================================================================
// K2b: CUDA-core contraction on the shared grid.
//   Sh[f,b] = sum_n sin(2 pi f t_n) y_b[n],  Ch likewise;  epilogue -> power[b, f].
// Block tile 128 frequencies x 128 light curves, k-tile 16 cadences, 256 threads,
// 8x8x{cos,sin} register tile per thread, double-buffered shared memory.
// =====================================================================================
constexpr int SG_BM = 128, SG_BN = 128, SG_BK = 16, SG_LDY = SG_BN + 4;
struct SgStage {
  float ac[SG_BK][SG_BM];
  float as[SG_BK][SG_BM];
  float y[SG_BK][SG_LDY];
};

__global__ void __launch_bounds__(256)
ls_shared_simt_kernel(const double* __restrict__ t, int64_t N, int64_t Npad, const float* __restrict__ yc, int B,
                      const double* __restrict__ freq, int64_t F, const float4* __restrict__ rot,
                      const float2* __restrict__ rot2, const float* __restrict__ ysum, double lowf_max,
                      int normalization, double norm_scale, float* __restrict__ power) {
  extern __shared__ __align__(16) unsigned char sg_smem[];
  SgStage* st = reinterpret_cast<SgStage*>(sg_smem);

  const int tid = threadIdx.x;
  const int64_t f0 = (int64_t)blockIdx.x * SG_BM;
  const int b0 = blockIdx.y * SG_BN;
  const int tx = tid & 15, ty = tid >> 4;

  // design-matrix role: one frequency per thread, 8 cadences of each k-tile
  const int gf = tid & (SG_BM - 1), gk0 = (tid >> 7) * 8;
  const double my_f = (f0 + gf < F) ? freq[f0 + gf] : 0.0;
  const bool my_low = fabs(my_f) <= lowf_max;
  // flux-tile role: two float4 per thread
  const int yr0 = tid >> 2, yq = tid & 3;            // rows yr0 and yr0+64, k-quad yq

  float acc_c[8][8], acc_s[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) { acc_c[i][j] = 0.f; acc_s[i][j] = 0.f; }

  float gc[8], gs[8];
  float4 yv[2];
  const int nkt = (int)(Npad / SG_BK);

  auto gen = [&](int kt) {
    const int64_t n0 = (int64_t)kt * SG_BK + gk0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int64_t nn = n0 + i;
      const double tt = (nn < N) ? t[nn] : 0.0;
      if (my_low) ls_sincos_cycles_low(my_f * tt, gs[i], gc[i]);
      else ls_sincos_cycles(my_f * tt, gs[i], gc[i]);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int bb = b0 + yr0 + 64 * r;
      yv[r] = (bb < B) ? *reinterpret_cast<const float4*>(yc + (int64_t)bb * Npad + (int64_t)kt * SG_BK + yq * 4)
                       : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto put = [&](int s) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      st[s].ac[gk0 + i][gf] = gc[i];
      st[s].as[gk0 + i][gf] = gs[i];
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int row = yr0 + 64 * r;
      st[s].y[yq * 4 + 0][row] = yv[r].x;
      st[s].y[yq * 4 + 1][row] = yv[r].y;
      st[s].y[yq * 4 + 2][row] = yv[r].z;
      st[s].y[yq * 4 + 3][row] = yv[r].w;
    }
  };

  gen(0);
  put(0);
  __syncthreads();
  for (int kt = 0; kt < nkt; ++kt) {
    const int cur = kt & 1;
    if (kt + 1 < nkt) gen(kt + 1);
#pragma unroll
    for (int k = 0; k < SG_BK; ++k) {
      float a_c[8], a_s[8], yy[8];
      *reinterpret_cast<float4*>(&a_c[0]) = *reinterpret_cast<const float4*>(&st[cur].ac[k][tx * 4]);
      *reinterpret_cast<float4*>(&a_c[4]) = *reinterpret_cast<const float4*>(&st[cur].ac[k][64 + tx * 4]);
      *reinterpret_cast<float4*>(&a_s[0]) = *reinterpret_cast<const float4*>(&st[cur].as[k][tx * 4]);
      *reinterpret_cast<float4*>(&a_s[4]) = *reinterpret_cast<const float4*>(&st[cur].as[k][64 + tx * 4]);
      *reinterpret_cast<float4*>(&yy[0]) = *reinterpret_cast<const float4*>(&st[cur].y[k][ty * 4]);
      *reinterpret_cast<float4*>(&yy[4]) = *reinterpret_cast<const float4*>(&st[cur].y[k][64 + ty * 4]);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          acc_c[i][j] = fmaf(a_c[i], yy[j], acc_c[i][j]);
          acc_s[i][j] = fmaf(a_s[i], yy[j], acc_s[i][j]);
        }
    }
    if (kt + 1 < nkt) put(cur ^ 1);
    __syncthreads();
  }

  // epilogue: rotate by tau, divide by CC'/SS', lightkurve normalisation
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t f = f0 + (i < 4 ? tx * 4 + i : 64 + tx * 4 + (i - 4));
    if (f >= F) continue;
    const float4 r = rot[f];
    const float2 r2 = rot2[f];
    const bool low = fabs(freq[f]) <= lowf_max;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int bb = b0 + (j < 4 ? ty * 4 + j : 64 + ty * 4 + (j - 4));
      if (bb >= B) continue;
      power[(int64_t)bb * F + f] =
          ls_epilogue_shared(acc_c[i][j], acc_s[i][j], r, r2, ysum[bb], (float)N, normalization, (float)norm_scale,
                             low);
    }
  }
}

// =====================================================================================
// K1n: multi-term ("chi2") periodogram - astropy lombscargle_chi2 / fastchi2 as lightkurve calls it for
// nterms > 1 (/root/reference/src/lightkurve/periodogram.py:948-964):
//   P = 0.5 * XTy^T (XTX)^-1 XTy,  X = [1, sin(w t), cos(w t), ..., sin(n w t), cos(n w t)].
// Same staging as K1; per frequency the warp accumulates the harmonic trig sums S_j, C_j (j <= 2n,
// they give XTX through product-to-sum identities) and YS_j, YC_j (j <= n); the harmonics come
// from the angle-addition recurrence, the (2n+1)x(2n+1) solve runs in fp64 on lane 0.
// Optionally returns the fitted parameters theta (LombScargle.model, periodogram.py:1010).
// =====================================================================================
template <int NT>
__global__ void __launch_bounds__(LS_WARPS * 32)
ls_chi2_kernel(const double* __restrict__ tws, const double* __restrict__ yws, const int64_t* __restrict__ offsets,
               const int64_t* __restrict__ poffsets, const double* __restrict__ freq,
               const int64_t* __restrict__ freq_offsets, int64_t F_shared, const double* __restrict__ ysum,
               int normalization, const double* __restrict__ norm_scale, float* __restrict__ power,
               double* __restrict__ theta_out) {
  constexpr int TN = 1024;
  __shared__ __align__(16) double s_t[2][TN];
  __shared__ __align__(16) double s_y[2][TN];
  __shared__ __align__(8) uint64_t s_bar[2];

  const int b = blockIdx.y;
  const int64_t n = offsets[b + 1] - offsets[b];
  const int64_t po = poffsets[b], np_ = poffsets[b + 1] - po;
  const int64_t fo = freq_offsets ? freq_offsets[b] : 0;
  const int64_t F = freq_offsets ? (freq_offsets[b + 1] - fo) : F_shared;
  const int64_t po_out = freq_offsets ? fo : (int64_t)b * F_shared;
  const int64_t f_blk = (int64_t)blockIdx.x * LS_WARPS;           // one frequency per warp
  if (f_blk >= F) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t fi = f_blk + warp;
  const bool f_ok = fi < F;
  if (n <= 0) {
    if (f_ok && lane == 0) power[po_out + fi] = __int_as_float(0x7fc00000);
    return;
  }
  const double fr = f_ok ? freq[fo + fi] : 0.0;

  if (threadIdx.x == 0) {
    ptx::mbar_init(&s_bar[0], 1);
    ptx::mbar_init(&s_bar[1], 1);
    ptx::mbar_fence_init();
  }
  __syncthreads();
  const int ntiles = (int)((np_ + TN - 1) / TN);
  auto issue = [&](int tile) {
    const int buf = tile & 1;
    const int64_t c0 = (int64_t)tile * TN;
    const uint32_t cnt = (uint32_t)min((int64_t)TN, np_ - c0);
    ptx::mbar_arrive_expect_tx(&s_bar[buf], cnt * 16u);
    ptx::bulk_g2s(&s_t[buf][0], tws + po + c0, cnt * 8u, &s_bar[buf]);
    ptx::bulk_g2s(&s_y[buf][0], yws + po + c0, cnt * 8u, &s_bar[buf]);
  };
  if (threadIdx.x == 0) issue(0);

  Chi2Sums<NT> d;
  d.zero();
  for (int tile = 0; tile < ntiles; ++tile) {
    const int buf = tile & 1;
    if (threadIdx.x == 0 && tile + 1 < ntiles) {
      ptx::fence_proxy_async_smem();
      issue(tile + 1);
    }
    ptx::mbar_wait(&s_bar[buf], (tile >> 1) & 1);
    const int64_t c0 = (int64_t)tile * TN;
    const int cnt = (int)min((int64_t)TN, n - c0);
    // fp64 throughout: this path is not the throughput path, and the normal equations of a
    // multi-harmonic fit are far less forgiving than the single-term closed form
    for (int i = lane; i < cnt; i += 32) {
      chi2_add<NT>(d, s_y[buf][i], fr * s_t[buf][i]);
    }
    __syncthreads();
  }
  chi2_warp_reduce<NT>(d);
  if (lane == 0 && f_ok) {
    double p;
    chi2_solve<NT>(d, (double)n, ysum[b], p, theta_out ? theta_out + (po_out + fi) * (2 * NT + 1) : nullptr);
    power[po_out + fi] = ls_normalize(p, (double)n, normalization, norm_scale ? norm_scale[b] : 1.0);
  }
}

// =====================================================================================
// Host launchers
// =====================================================================================
int ls_power_ragged(const double* t, const void* y, int y_dtype, const int64_t* h_offsets, int B,
                    const double* freq, const int64_t* h_freq_offsets, int64_t F, int normalization,
                    const double* norm_scale, float* power, int mem, cudaStream_t st, int algo) {
  LKB_REQUIRE(B > 0 && t && y && h_offsets && freq && power, "lkb_ls_power: null argument");
  LKB_REQUIRE(algo == LKB_LS_ALGO_AUTO || algo == LKB_LS_ALGO_SIMT || algo == LKB_LS_ALGO_NUFFT,
              "lkb_ls_power: algo must be AUTO, SIMT (direct sums) or NUFFT");
  LKB_REQUIRE(y_dtype == LKB_DTYPE_F32 || y_dtype == LKB_DTYPE_F64, "lkb_ls_power: bad y_dtype");
  LKB_REQUIRE(normalization >= 0 && normalization <= 2, "lkb_ls_power: bad normalization");
  LKB_REQUIRE(normalization != LKB_LS_NORM_PSD_SCALE || norm_scale, "lkb_ls_power: norm_scale required");
  LKB_TRY(ensure_device());
  const int64_t total = h_offsets[B];
  // padded offsets (16-byte alignment of every light curve for the TMA bulk copies)
  int64_t* h_po = (int64_t*)malloc(sizeof(int64_t) * (B + 1));
  if (!h_po) { set_error("host malloc failed"); return LKB_E_OOM; }
  h_po[0] = 0;
  int64_t Fmax = F, Ftot = 0;
  for (int b = 0; b < B; ++b) {
    const int64_t n = h_offsets[b + 1] - h_offsets[b];
    if (n < 0) { free(h_po); set_error("lkb_ls_power: offsets not monotone"); return LKB_E_ARG; }
    h_po[b + 1] = h_po[b] + ((n + 3) / 4) * 4;
  }
  if (h_freq_offsets) {
    Fmax = 0;
    for (int b = 0; b < B; ++b) Fmax = max(Fmax, h_freq_offsets[b + 1] - h_freq_offsets[b]);
    Ftot = h_freq_offsets[B];
  } else {
    Ftot = F;
  }
  const int64_t ptotal = h_po[B];
  const size_t ysz = (y_dtype == LKB_DTYPE_F32) ? 4 : 8;

  int64_t *d_off = nullptr, *d_po = nullptr, *d_fo = nullptr;
  int s = ws_get_t<int64_t>(WS_A, B + 1, &d_off);
  if (s == LKB_OK) s = ws_get_t<int64_t>(WS_B, B + 1, &d_po);
  if (s == LKB_OK && h_freq_offsets) s = ws_get_t<int64_t>(WS_C, B + 1, &d_fo);
  double* d_t = nullptr;
  float* d_y = nullptr;
  if (s == LKB_OK) s = ws_get_t<double>(WS_D, ptotal + 4, &d_t);
  if (s == LKB_OK) s = ws_get_t<float>(WS_E, ptotal + 4, &d_y);
  double *d_span = nullptr, *d_ysum = nullptr;
  if (s == LKB_OK) s = ws_get_t<double>(WS_F, B, &d_span);
  if (s == LKB_OK) s = ws_get_t<double>(WS_J, B, &d_ysum);
  // Regular frequency grids?  Decided on the host from `freq` (device-mode callers: one small read-back of the
  // grid - it is what makes the fixed-point phases and the NUFFT path available to device-resident batches).
  bool regular = !getenv("LKB_LS_FORCE_FP64_PHASE");
  std::vector<double> h_f0(B, 0.0), h_df(B, 0.0), h_freq_copy;
  const double* freq_h = freq;
  if (regular && mem == LKB_MEM_DEVICE) {
    h_freq_copy.resize((size_t)Ftot);
    cudaError_t ce = cudaMemcpyAsync(h_freq_copy.data(), freq, sizeof(double) * (size_t)Ftot, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    if (ce != cudaSuccess) { free(h_po); set_error("frequency read-back failed: %s", cudaGetErrorString(ce)); return LKB_E_CUDA; }
    freq_h = h_freq_copy.data();
  }
  if (regular) {
    for (int b = 0; b < B && regular; ++b) {
      const int64_t fo = h_freq_offsets ? h_freq_offsets[b] : 0;
      const int64_t Fb = h_freq_offsets ? h_freq_offsets[b + 1] - fo : F;
      regular = regular_grid(freq_h + fo, Fb, &h_f0[b], &h_df[b]);
      if (regular && !h_freq_offsets) {          // one shared grid: same (f0, df) for every light curve
        for (int bb = 1; bb < B; ++bb) { h_f0[bb] = h_f0[0]; h_df[bb] = h_df[0]; }
        break;
      }
    }
  }
  double *d_gf0 = nullptr, *d_gdf = nullptr;
  LsTabEntry* d_tab = nullptr;
  if (s == LKB_OK && regular) {
    s = ws_get_t<double>(WS_G, B, &d_gf0);
    if (s == LKB_OK) s = ws_get_t<double>(WS_H, B, &d_gdf);
    if (s == LKB_OK) s = ws_get_t<LsTabEntry>(WS_I, ptotal + 4, &d_tab);
  }
  if (s != LKB_OK) { free(h_po); return s; }
  cudaError_t e = cudaMemcpyAsync(d_off, h_offsets, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_po, h_po, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess && h_freq_offsets)
    e = cudaMemcpyAsync(d_fo, h_freq_offsets, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess && regular) e = cudaMemcpyAsync(d_gf0, h_f0.data(), sizeof(double) * B, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess && regular) e = cudaMemcpyAsync(d_gdf, h_df.data(), sizeof(double) * B, cudaMemcpyHostToDevice, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);   // h_po is freed below
  free(h_po);
  if (e != cudaSuccess) { set_error("offset upload failed: %s", cudaGetErrorString(e)); return LKB_E_CUDA; }

  const double* dt_in = nullptr;
  const void* dy_in = nullptr;
  const double *d_freq = nullptr, *d_ns = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, t, total, &dt_in, st));
  {
    const unsigned char* tmp = nullptr;
    LKB_TRY(stage_in<unsigned char>(mem, WS_IN1, (const unsigned char*)y, total * ysz, &tmp, st));
    dy_in = tmp;
  }
  LKB_TRY(stage_in<double>(mem, WS_IN2, freq, Ftot, &d_freq, st));
  LKB_TRY(stage_in<double>(mem, WS_IN3, norm_scale, B, &d_ns, st));
  const int64_t out_count = h_freq_offsets ? Ftot : (int64_t)B * F;
  float* d_pow = nullptr;
  LKB_TRY(stage_out_alloc<float>(mem, WS_OUT0, power, out_count, &d_pow));

  if (y_dtype == LKB_DTYPE_F32)
    ls_prep_ragged_kernel<float><<<B, 256, 0, st>>>(dt_in, (const float*)dy_in, d_off, d_po, d_t, d_y, d_span, d_gf0,
                                                    d_gdf, d_tab, d_ysum);
  else
    ls_prep_ragged_kernel<double><<<B, 256, 0, st>>>(dt_in, (const double*)dy_in, d_off, d_po, d_t, d_y, d_span, d_gf0,
                                                     d_gdf, d_tab, d_ysum);
  LKB_LAUNCH_CHECK();

  dim3 grid((unsigned)((Fmax + LS_FPB - 1) / LS_FPB), (unsigned)B);
  LKB_REQUIRE(B <= 65535, "lkb_ls_power: B > 65535 per call (split the batch)");
  // NUFFT path of ls_nufft.cu (one shared regular grid f_k = (k0 + k) df): what `auto` picks when the job is large
  // enough for its launches to pay (config 5's share: ~100x fewer operations than the direct sums); light curves
  // that do not qualify (empty / tiny, unsorted times, df * baseline > 1) send the whole call to the direct kernel
  // under `auto`, and fail an explicit NUFFT request.  LKB_LS_RAGGED_NUFFT=0 keeps `auto` on the direct kernel.
  const bool want_nufft = algo == LKB_LS_ALGO_NUFFT ||
                          (algo == LKB_LS_ALGO_AUTO && ls_nufft_ragged_enabled() && (double)total * (double)F >= 2.5e7);
  if (algo == LKB_LS_ALGO_NUFFT && !(regular && !h_freq_offsets)) {
    set_error("lkb_ls_power: the NUFFT path needs host-visible, regular, shared frequencies");
    return LKB_E_UNSUPPORTED;
  }
  if (want_nufft && regular && !h_freq_offsets) {
    int64_t nmax = 0, nmin = INT64_MAX;
    for (int b = 0; b < B; ++b) {
      const int64_t n = h_offsets[b + 1] - h_offsets[b];
      nmax = n > nmax ? n : nmax;
      nmin = n < nmin ? n : nmin;
    }
    int rc = LKB_E_UNSUPPORTED;
    if (nmin >= 8) {
      std::vector<double> h_span(B);
      LKB_CUDA_CHECK(cudaMemcpyAsync(h_span.data(), d_span, sizeof(double) * B, cudaMemcpyDeviceToHost, st));
      LKB_CUDA_CHECK(cudaStreamSynchronize(st));
      rc = ls_nufft_ragged_launch(d_t, d_y, d_off, d_po, h_offsets, B, ptotal, nmax, d_span, h_span.data(), d_ysum, F,
                                  h_f0[0], h_df[0], normalization, d_ns, d_pow, st);
      if (rc == LKB_OK) {
        g_last_ls_algo = LKB_LS_ALGO_NUFFT;
        LKB_TRY(stage_out_copy<float>(mem, power, d_pow, out_count, st));
        if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
        return LKB_OK;
      }
    } else {
      set_error("lkb_ls_power: the NUFFT path needs at least 8 cadences per light curve");
    }
    if (rc != LKB_E_UNSUPPORTED || algo == LKB_LS_ALGO_NUFFT) return rc;
  }
  g_last_ls_algo = LKB_LS_ALGO_SIMT;
  prof_begin(st);
  if (regular)
    ls_direct_kernel<true><<<grid, LS_WARPS * 32, 0, st>>>(d_t, d_tab, d_y, d_off, d_po, d_freq, d_fo, F, d_span,
                                                           d_ysum, normalization, d_ns, d_pow);
  else
    ls_direct_kernel<false><<<grid, LS_WARPS * 32, 0, st>>>(d_t, d_tab, d_y, d_off, d_po, d_freq, d_fo, F, d_span,
                                                            d_ysum, normalization, d_ns, d_pow);
  prof_end(st);
  LKB_LAUNCH_CHECK();
  LKB_TRY(stage_out_copy<float>(mem, power, d_pow, out_count, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

int ls_power_chi2(const double* t, const void* y, int y_dtype, const int64_t* h_offsets, int B, const double* freq,
                  const int64_t* h_freq_offsets, int64_t F, int nterms, int normalization, const double* norm_scale,
                  float* power, double* theta, int mem, cudaStream_t st, int algo) {
  LKB_REQUIRE(B > 0 && B <= 65535 && t && y && h_offsets && freq && power, "lkb_ls_power_chi2: null/bad argument");
  LKB_REQUIRE(algo == LKB_LS_ALGO_AUTO || algo == LKB_LS_ALGO_SIMT || algo == LKB_LS_ALGO_NUFFT,
              "lkb_ls_power_chi2: algo must be AUTO, SIMT (direct sums) or NUFFT");
  LKB_REQUIRE(y_dtype == LKB_DTYPE_F32 || y_dtype == LKB_DTYPE_F64, "lkb_ls_power_chi2: bad y_dtype");
  LKB_REQUIRE(nterms >= 1 && nterms <= 4, "lkb_ls_power_chi2: nterms must be in [1, 4]");
  LKB_REQUIRE(normalization >= 0 && normalization <= 2, "lkb_ls_power_chi2: bad normalization");
  LKB_REQUIRE(normalization != LKB_LS_NORM_PSD_SCALE || norm_scale, "lkb_ls_power_chi2: norm_scale required");
  LKB_TRY(ensure_device());
  const int64_t total = h_offsets[B];
  std::vector<int64_t> h_po(B + 1, 0);
  for (int b = 0; b < B; ++b) {
    const int64_t n = h_offsets[b + 1] - h_offsets[b];
    LKB_REQUIRE(n >= 0, "lkb_ls_power_chi2: offsets not monotone");
    h_po[b + 1] = h_po[b] + ((n + 3) / 4) * 4;
  }
  int64_t Fmax = F, Ftot = F;
  if (h_freq_offsets) {
    Fmax = 0;
    for (int b = 0; b < B; ++b) Fmax = max(Fmax, h_freq_offsets[b + 1] - h_freq_offsets[b]);
    Ftot = h_freq_offsets[B];
  }
  const int64_t ptotal = h_po[B];
  const size_t ysz = (y_dtype == LKB_DTYPE_F32) ? 4 : 8;
  const int M = 2 * nterms + 1;
  int64_t *d_off = nullptr, *d_po = nullptr, *d_fo = nullptr;
  double *d_t = nullptr, *d_span = nullptr, *d_ysum = nullptr;
  double* d_y = nullptr;
  LKB_TRY(ws_get_t<int64_t>(WS_A, B + 1, &d_off));
  LKB_TRY(ws_get_t<int64_t>(WS_B, B + 1, &d_po));
  if (h_freq_offsets) LKB_TRY(ws_get_t<int64_t>(WS_C, B + 1, &d_fo));
  LKB_TRY(ws_get_t<double>(WS_D, ptotal + 4, &d_t));
  LKB_TRY(ws_get_t<double>(WS_E, ptotal + 4, &d_y));
  LKB_TRY(ws_get_t<double>(WS_F, B, &d_span));
  LKB_TRY(ws_get_t<double>(WS_J, B, &d_ysum));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_off, h_offsets, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_po, h_po.data(), sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  if (h_freq_offsets)
    LKB_CUDA_CHECK(cudaMemcpyAsync(d_fo, h_freq_offsets, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  const double *dt_in = nullptr, *d_freq = nullptr, *d_ns = nullptr;
  const void* dy_in = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, t, total, &dt_in, st));
  {
    const unsigned char* tmp = nullptr;
    LKB_TRY(stage_in<unsigned char>(mem, WS_IN1, (const unsigned char*)y, total * ysz, &tmp, st));
    dy_in = tmp;
  }
  LKB_TRY(stage_in<double>(mem, WS_IN2, freq, Ftot, &d_freq, st));
  LKB_TRY(stage_in<double>(mem, WS_IN3, norm_scale, B, &d_ns, st));
  const int64_t out_count = h_freq_offsets ? Ftot : (int64_t)B * F;
  float* d_pow = nullptr;
  double* d_theta = nullptr;
  LKB_TRY(stage_out_alloc<float>(mem, WS_OUT0, power, out_count, &d_pow));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT1, theta, out_count * M, &d_theta));

  // NUFFT path of ls_nufft.cu (one shared regular grid f_k = (k0 + k) df, no theta): what `auto` picks when the job is
  // large enough to pay for its transforms; light curves that do not qualify (fewer than 8 cadences, unsorted times,
  // df * baseline > 1, fine grids outside the v2 range) send the whole call to the direct kernel under `auto` and fail
  // an explicit NUFFT request.  LKB_LS_RAGGED_NUFFT=0 keeps `auto` on the direct kernel.
  if (algo == LKB_LS_ALGO_NUFFT ||
      (algo == LKB_LS_ALGO_AUTO && ls_nufft_ragged_enabled() && (double)total * (double)F >= LS_CHI2_NUFFT_MIN_WORK)) {
    int64_t nmax = 0, nmin = INT64_MAX;
    for (int b = 0; b < B; ++b) {
      const int64_t n = h_offsets[b + 1] - h_offsets[b];
      nmax = n > nmax ? n : nmax;
      nmin = n < nmin ? n : nmin;
    }
    double f0 = 0.0, df = 0.0;
    bool eligible = !h_freq_offsets && !theta && nmin >= 8;
    if (eligible) {
      std::vector<double> h_freq_copy;
      const double* freq_h = freq;
      if (mem == LKB_MEM_DEVICE) {
        h_freq_copy.resize((size_t)F);
        LKB_CUDA_CHECK(cudaMemcpyAsync(h_freq_copy.data(), freq, sizeof(double) * (size_t)F, cudaMemcpyDeviceToHost, st));
        LKB_CUDA_CHECK(cudaStreamSynchronize(st));
        freq_h = h_freq_copy.data();
      }
      eligible = regular_grid(freq_h, F, &f0, &df);
    }
    int rc = LKB_E_UNSUPPORTED;
    if (eligible) {
      // the transforms take the centred flux in fp32, as in ls_power_ragged (ysum: sum of the fp32 values)
      float* d_yf = nullptr;
      LKB_TRY(ws_get_t<float>(WS_E, ptotal + 4, &d_yf));
      if (y_dtype == LKB_DTYPE_F32)
        ls_prep_ragged_kernel<float><<<B, 256, 0, st>>>(dt_in, (const float*)dy_in, d_off, d_po, d_t, d_yf, d_span,
                                                        nullptr, nullptr, nullptr, d_ysum);
      else
        ls_prep_ragged_kernel<double><<<B, 256, 0, st>>>(dt_in, (const double*)dy_in, d_off, d_po, d_t, d_yf, d_span,
                                                         nullptr, nullptr, nullptr, d_ysum);
      LKB_LAUNCH_CHECK();
      std::vector<double> h_span(B);
      LKB_CUDA_CHECK(cudaMemcpyAsync(h_span.data(), d_span, sizeof(double) * B, cudaMemcpyDeviceToHost, st));
      LKB_CUDA_CHECK(cudaStreamSynchronize(st));
      rc = ls_nufft_chi2_ragged_launch(d_t, d_yf, d_off, d_po, h_offsets, B, ptotal, nmax, d_span, h_span.data(), d_ysum,
                                       F, f0, df, normalization, d_ns, d_pow, st, nterms);
      if (rc == LKB_OK) {
        g_last_ls_algo = LKB_LS_ALGO_NUFFT;
        LKB_TRY(stage_out_copy<float>(mem, power, d_pow, out_count, st));
        if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
        return LKB_OK;
      }
    } else {
      set_error("lkb_ls_power_chi2: the NUFFT path needs one host-visible, regular, shared frequency grid, no theta "
                "and at least 8 cadences per light curve");
    }
    if (rc != LKB_E_UNSUPPORTED || algo == LKB_LS_ALGO_NUFFT) return rc;
  }
  g_last_ls_algo = LKB_LS_ALGO_SIMT;
  if (y_dtype == LKB_DTYPE_F32)
    ls_prep_ragged_kernel<float><<<B, 256, 0, st>>>(dt_in, (const float*)dy_in, d_off, d_po, d_t, nullptr, d_span,
                                                    nullptr, nullptr, nullptr, d_ysum, d_y);
  else
    ls_prep_ragged_kernel<double><<<B, 256, 0, st>>>(dt_in, (const double*)dy_in, d_off, d_po, d_t, nullptr, d_span,
                                                     nullptr, nullptr, nullptr, d_ysum, d_y);
  LKB_LAUNCH_CHECK();
  dim3 grid((unsigned)((Fmax + LS_WARPS - 1) / LS_WARPS), (unsigned)B);
  prof_begin(st);
  switch (nterms) {
    case 1: ls_chi2_kernel<1><<<grid, LS_WARPS * 32, 0, st>>>(d_t, d_y, d_off, d_po, d_freq, d_fo, F, d_ysum, normalization, d_ns, d_pow, d_theta); break;
    case 2: ls_chi2_kernel<2><<<grid, LS_WARPS * 32, 0, st>>>(d_t, d_y, d_off, d_po, d_freq, d_fo, F, d_ysum, normalization, d_ns, d_pow, d_theta); break;
    case 3: ls_chi2_kernel<3><<<grid, LS_WARPS * 32, 0, st>>>(d_t, d_y, d_off, d_po, d_freq, d_fo, F, d_ysum, normalization, d_ns, d_pow, d_theta); break;
    default: ls_chi2_kernel<4><<<grid, LS_WARPS * 32, 0, st>>>(d_t, d_y, d_off, d_po, d_freq, d_fo, F, d_ysum, normalization, d_ns, d_pow, d_theta); break;
  }
  prof_end(st);
  LKB_LAUNCH_CHECK();
  LKB_TRY(stage_out_copy<float>(mem, power, d_pow, out_count, st));
  LKB_TRY(stage_out_copy<double>(mem, theta, d_theta, out_count * M, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

int ls_tc_launch(const double* d_t, const ulonglong2* d_tab, int64_t N, int64_t Npad, const float* d_yc,
                 const float* d_absmax, int B, const double* d_freq, int64_t F, float4* d_rot, float2* d_rot2,
                 double lowf_max, double grid_f0, double grid_df, int normalization,
                 double norm_scale, float* d_pow, cudaStream_t st, cudaEvent_t rot_ready, int ws_alt = 0);   // ls_tc.cu
bool ls_tc_supported(int B, int64_t N, int64_t F);
bool ls_nufft_supported(int64_t F, bool regular, double grid_f0, double grid_df, double t_last);              // ls_nufft.cu
int ls_nufft_prepare(const double* d_t, int64_t N, int64_t F, double grid_f0, double grid_df, float4* d_rot,
                     float2* d_rot2, int64_t F_low, cudaStream_t st, const double* d_freq, int64_t Npad);
int ls_nufft_run(const double* d_t, int64_t N, const float* d_yc, int64_t ystride, const float* d_ysumf,
                 const float* d_absmax, int B, const double* d_freq, int64_t F, const float4* d_rot,
                 const float2* d_rot2, int64_t F_low, int normalization, double norm_scale, float* d_pow,
                 cudaStream_t st, int ws_alt, bool prof);
int ls_nufft_launch(const double* d_t, int64_t N, const float* d_yc, int64_t ystride, const float* d_ysumf,
                    const float* d_absmax, int B,
                    const double* d_freq, int64_t F, double grid_f0, double grid_df, float4* d_rot, float2* d_rot2,
                    int64_t F_low, int normalization, double norm_scale, float* d_pow, cudaStream_t st);

int ls_power_shared(const double* t, const void* y, int y_dtype, int B, int64_t N, const double* freq, int64_t F,
                    int normalization, const double* norm_scale, float* power, int mem, cudaStream_t st,
                    int algo) {
  LKB_REQUIRE(B > 0 && N > 0 && F > 0 && t && y && freq && power, "lkb_ls_power_shared: null/empty argument");
  LKB_REQUIRE(y_dtype == LKB_DTYPE_F32 || y_dtype == LKB_DTYPE_F64, "lkb_ls_power_shared: bad y_dtype");
  LKB_REQUIRE(normalization >= 0 && normalization <= 2, "lkb_ls_power_shared: bad normalization");
  LKB_REQUIRE(normalization != LKB_LS_NORM_PSD_SCALE || norm_scale, "lkb_ls_power_shared: norm_scale required");
  LKB_REQUIRE(algo >= 0 && algo <= 3, "lkb_ls_power_shared: bad algo");
  LKB_TRY(ensure_device());
  const int64_t Npad = ((N + 63) / 64) * 64;
  const size_t ysz = (y_dtype == LKB_DTYPE_F32) ? 4 : 8;

  const double *dt_in = nullptr, *d_freq = nullptr;
  const void* dy_in = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, t, N, &dt_in, st));
  LKB_TRY(stage_in<double>(mem, WS_IN2, freq, F, &d_freq, st));
  double ns = 1.0;
  if (norm_scale) {
    if (mem == LKB_MEM_HOST) ns = *norm_scale;
    else LKB_CUDA_CHECK(cudaMemcpyAsync(&ns, norm_scale, sizeof(double), cudaMemcpyDeviceToHost, st));
    if (mem == LKB_MEM_DEVICE) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  }
  double* d_t = nullptr;
  LKB_TRY(ws_get_t<double>(WS_D, Npad, &d_t));
  // One small device->host read-back per call: grid regularity, f0, f1, the baseline t[N-1] and whether the times
  // ascend.  Regular frequency grid (f_k = f0 + k df)?  Then phases are generated in 64-bit fixed point from a
  // per-cadence table {frac(f0 t_n), frac(df t_n)} instead of an fp64 multiply/round/convert chain - and the
  // NUFFT path becomes eligible.
  ulonglong2* d_tab = nullptr;
  double h_meta[6] = {1.0, 0.0, 0.0, 0.0, 0.0, 0.0};  // {regularity deviation, f0, f1, t_last, unsorted (int bits), t checksum}
  {
    double* d_meta = nullptr;
    LKB_TRY(ws_get_t<double>(WS_K, 6, &d_meta));
    LKB_CUDA_CHECK(cudaMemsetAsync(d_meta, 0, 6 * sizeof(double), st));
    ls_shift_time_kernel<<<(unsigned)((Npad + 255) / 256), 256, 0, st>>>(dt_in, N, Npad, d_t,
                                                                         reinterpret_cast<int*>(d_meta + 4),
                                                                         reinterpret_cast<unsigned long long*>(d_meta + 5));
    LKB_LAUNCH_CHECK();
    ls_grid_regularity_kernel<<<64, 256, 0, st>>>(d_freq, F, reinterpret_cast<float*>(d_meta));
    LKB_LAUNCH_CHECK();
    ls_meta_kernel<<<1, 1, 0, st>>>(d_freq, F, d_t, N, d_meta);
    LKB_LAUNCH_CHECK();
    LKB_CUDA_CHECK(cudaMemcpyAsync(h_meta, d_meta, 6 * sizeof(double), cudaMemcpyDeviceToHost, st));
    LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  }
  int h_unsorted = 0;
  memcpy(&h_unsorted, &h_meta[4], sizeof(int));
  unsigned long long h_thash = 0;
  memcpy(&h_thash, &h_meta[5], sizeof(h_thash));
  const double grid_f0 = h_meta[1], grid_df = h_meta[2] - h_meta[1];
  const bool regular = F >= 2 && F < ((int64_t)1 << 31) && !getenv("LKB_LS_FORCE_FP64_PHASE") &&
                       h_meta[0] <= 1e-6 && grid_f0 >= 0.0 && grid_df > 0.0;
  // frequencies with f * baseline <= LS_LOWF_CYCLES are "low rows" (ls_common.cuh)
  const double lowf_max = (h_meta[3] > 0.0) ? LS_LOWF_CYCLES / h_meta[3] : 0.0;
  // Which kernel family.  NUFFT (ls_nufft.cu: spread + FFT, an HBM sweep) is what `auto` picks whenever the grid
  // allows it (regular, integer f0 / df, df * baseline <= 1, ascending times) and the job is large enough for its
  // ~15 launches to pay (config 2: an HBM sweep against the O(N F) tensor-core contraction, and closer
  // to the fp64 sums - tests/test_gpu_fullsize.py::test_config2_worst_bins).  LKB_LS_AUTO_NO_NUFFT=1 restores the
  // round-1 choice (tcgen05 / SIMT contraction).  The contraction kernels remain the path for irregular grids.
  const bool nufft_ok = ls_nufft_supported(F, regular, grid_f0, grid_df, h_meta[3]) && !h_unsorted;
  const bool use_nufft = algo == LKB_LS_ALGO_NUFFT ||
                         (algo == LKB_LS_ALGO_AUTO && nufft_ok && !getenv("LKB_LS_AUTO_NO_NUFFT") &&
                          (double)B * (double)N * (double)F >= 2.5e7);
  if (use_nufft && !nufft_ok) {
    set_error(h_unsorted ? "lkb_ls_power_shared: the NUFFT path needs ascending times"
                         : "lkb_ls_power_shared: the NUFFT path needs a regular grid f_k = (k0 + k) df with integer k0 "
                           "and df * baseline <= 1");
    return LKB_E_UNSUPPORTED;
  }
  g_last_ls_algo = use_nufft ? LKB_LS_ALGO_NUFFT : LKB_LS_ALGO_SIMT;
  const bool use_tc = !use_nufft && ((algo == LKB_LS_ALGO_TCGEN05) || (algo == LKB_LS_ALGO_AUTO && ls_tc_supported(B, N, F)));
  if (algo == LKB_LS_ALGO_TCGEN05 && !ls_tc_supported(B, N, F)) {
    set_error("lkb_ls_power_shared: tcgen05 path unsupported for this shape");
    return LKB_E_UNSUPPORTED;
  }
  if (use_tc) g_last_ls_algo = LKB_LS_ALGO_TCGEN05;
  // Host-mode calls on the tensor / NUFFT paths are pipelined over chunks of light curves: the flux rows of chunk
  // c + 1 go up and the power rows of chunk c - 1 come down (two copy streams) while chunk c is computed.  Fully
  // asynchronous when the caller's buffers are page-locked; with pageable numpy memory the copies still work,
  // they just overlap less.
  constexpr int PIPE_CHUNK = 256;                    // one light-curve tile of the tensor kernel
  const bool pipelined = mem == LKB_MEM_HOST && B > PIPE_CHUNK && !getenv("LKB_LS_NO_PIPELINE") && (use_tc || use_nufft);
  unsigned char* d_ystage = nullptr;
  if (pipelined) {
    LKB_TRY(ws_get_t<unsigned char>(WS_IN1, (size_t)B * N * ysz, &d_ystage));
    dy_in = d_ystage;
  } else {
    const unsigned char* tmp = nullptr;
    LKB_TRY(stage_in<unsigned char>(mem, WS_IN1, (const unsigned char*)y, (size_t)B * N * ysz, &tmp, st));
    dy_in = tmp;
  }
  float* d_pow = nullptr;
  LKB_TRY(stage_out_alloc<float>(mem, WS_OUT0, power, (size_t)B * F, &d_pow));

  float *d_yc = nullptr, *d_absmax = nullptr;
  float4* d_rot = nullptr;
  LKB_TRY(ws_get_t<float>(WS_E, (size_t)B * Npad, &d_yc));
  LKB_TRY(ws_get_t<float4>(WS_F, F, &d_rot));
  LKB_TRY(ws_get_t<float>(WS_G, B, &d_absmax));
  float2* d_rot2 = nullptr;
  float* d_ysumf = nullptr;
  LKB_TRY(ws_get_t<float2>(WS_M, F, &d_rot2));
  LKB_TRY(ws_get_t<float>(WS_N, B, &d_ysumf));

  auto prep_rows = [&](int b_lo, int nb) {
    if (y_dtype == LKB_DTYPE_F32)
      ls_prep_shared_kernel<float><<<nb, 256, 0, st>>>((const float*)dy_in + (size_t)b_lo * N, N, Npad,
                                                       d_yc + (size_t)b_lo * Npad, d_absmax + b_lo, d_ysumf + b_lo);
    else
      ls_prep_shared_kernel<double><<<nb, 256, 0, st>>>((const double*)dy_in + (size_t)b_lo * N, N, Npad,
                                                        d_yc + (size_t)b_lo * Npad, d_absmax + b_lo, d_ysumf + b_lo);
  };
  if (!pipelined) {
    prep_rows(0, B);
    LKB_LAUNCH_CHECK();
  }
  // ---- y-independent part: phase table, window terms (tau rotation, CC', SS'), NUFFT tables.  It is CACHED: a call
  // with the same time stamps (count, checksum, baseline), the same regular grid and the same kernel family as the
  // previous library call finds everything still in its workspace slots (g_epoch: no other entry point ran in
  // between) and goes straight to the light curves - repeated calls on one grid (chunks of a collection, the ranks'
  // pieces of a sharded batch, bench steps) pay for the tables once.  LKB_LS_NO_PLAN_CACHE=1 disables it.
  struct SharedPlanKey {
    bool valid;
    int64_t epoch, N, F, F_win;
    double f0, f1, t_last, dev;
    unsigned long long thash;
    int family;
  };
  static SharedPlanKey g_key = {false, 0, 0, 0, 0, 0.0, 0.0, 0.0, 0.0, 0ull, 0};
  cudaStream_t aux;
  cudaEvent_t ev_fork, ev_join;
  LKB_TRY(aux_stream_get(&aux, &ev_fork, &ev_join));
  if (!getenv("LKB_LS_OVERLAP_WINDOW")) aux = st;
  int64_t F_win = F;
  if (use_nufft) {     // only the low rows need the fp64 window path; the rest comes from the kernels
    const double nlow = floor((lowf_max - grid_f0) / grid_df) + 2.0;
    F_win = (nlow < 0.0) ? 0 : (nlow > (double)F ? F : (int64_t)nlow);
  }
  const int family = use_nufft ? LKB_LS_ALGO_NUFFT : use_tc ? LKB_LS_ALGO_TCGEN05 : LKB_LS_ALGO_SIMT;
  const bool plan_hit = g_key.valid && g_key.epoch + 1 == g_epoch && g_key.N == N && g_key.F == F && g_key.F_win == F_win &&
                        g_key.f0 == h_meta[1] && g_key.f1 == h_meta[2] && g_key.t_last == h_meta[3] &&
                        g_key.dev == h_meta[0] && g_key.thash == h_thash && g_key.family == family &&
                        !getenv("LKB_LS_NO_PLAN_CACHE");
  if (regular && !use_nufft) LKB_TRY(ws_get_t<ulonglong2>(WS_L, Npad, &d_tab));
  LKB_CUDA_CHECK(cudaEventRecord(ev_fork, st));
  LKB_CUDA_CHECK(cudaStreamWaitEvent(aux, ev_fork, 0));
  if (!plan_hit) {
    g_key.valid = false;
    if (d_tab) {
      ls_phase_table_kernel<<<(unsigned)((Npad + 255) / 256), 256, 0, st>>>(d_t, N, Npad, grid_f0, grid_df, d_tab);
      LKB_LAUNCH_CHECK();
      LKB_CUDA_CHECK(cudaEventRecord(ev_fork, st));
      LKB_CUDA_CHECK(cudaStreamWaitEvent(aux, ev_fork, 0));
    }
    // The window terms depend only on (t, freq).  They CAN run on the library's side stream, co-resident
    // with the contraction kernel (LKB_LS_OVERLAP_WINDOW=1), where their MUFU work competes with the contraction's
    // own for issue slots and for the power budget; by default they run in order on the caller's stream.
    if (F_win > 0) {
      if (d_tab) ls_window_kernel<true><<<(unsigned)((F_win + 3) / 4), 128, 0, aux>>>(d_t, d_tab, N, d_freq, F_win, d_rot, d_rot2);
      else ls_window_kernel<false><<<(unsigned)((F_win + 3) / 4), 128, 0, aux>>>(d_t, d_tab, N, d_freq, F_win, d_rot, d_rot2);
      LKB_LAUNCH_CHECK();
    }
  }
  LKB_CUDA_CHECK(cudaEventRecord(ev_join, aux));
  if (use_nufft && !plan_hit) {     // tables and window terms of the rows above the low ones, on `st`
    LKB_CUDA_CHECK(cudaStreamWaitEvent(st, ev_join, 0));
    LKB_TRY(ls_nufft_prepare(d_t, N, F, grid_f0, grid_df, d_rot, d_rot2, F_win, st, d_freq, Npad));
  }
  if (use_nufft) ls_nufft_begin_call(st);
  if (!plan_hit) {
    g_key.valid = true;
    g_key.N = N; g_key.F = F; g_key.F_win = F_win; g_key.f0 = h_meta[1]; g_key.f1 = h_meta[2]; g_key.t_last = h_meta[3];
    g_key.dev = h_meta[0]; g_key.thash = h_thash; g_key.family = family;
  }
  g_key.epoch = g_epoch;

  if ((use_tc || use_nufft) && pipelined) {
    cudaStream_t s_h2d, s_d2h;
    cudaEvent_t* ev;
    int nev;
    LKB_TRY(pipe_streams_get(&s_h2d, &s_d2h, &ev, &nev));
    // chunk boundaries: the tensor path in tiles of PIPE_CHUNK light curves; the NUFFT path ramps up (64, 64, 128, then
    // PIPE_CHUNK) - its kernels are short, so the time before the first power rows can start down the link (upload of
    // chunk 0 + its kernels) is what the end-to-end step adds to the 7.5 ms the download takes by itself
    int c_lo[520];
    int nchunk = 0;
    {
      static const int ramp[3] = {64, 64, 128};
      int b0 = 0;
      while (b0 < B && nchunk < 518) {
        const int sz = (use_nufft && nchunk < 3 && !getenv("LKB_LS_NO_RAMP")) ? ramp[nchunk] : PIPE_CHUNK;
        c_lo[nchunk++] = b0;
        b0 += sz;
      }
      c_lo[nchunk] = B;
    }
    // chunks alternate between two compute streams (and two workspace sets): the last, partly filled wave of one
    // chunk's tensor kernel overlaps the first wave of the next chunk
    cudaStream_t cs[2] = {st, st};
    {
      cudaStream_t a2; cudaEvent_t f2, j2;
      LKB_TRY(aux_stream_get(&a2, &f2, &j2));
      if (!getenv("LKB_LS_ONE_COMPUTE_STREAM")) cs[1] = a2;
    }
    // nothing may start before the earlier work on `st` (prologue kernels, window terms) is done
    LKB_CUDA_CHECK(cudaEventRecord(ev[0], st));
    LKB_CUDA_CHECK(cudaStreamWaitEvent(s_h2d, ev[0], 0));
    LKB_CUDA_CHECK(cudaStreamWaitEvent(s_d2h, ev[0], 0));
    if (cs[1] != st) LKB_CUDA_CHECK(cudaStreamWaitEvent(cs[1], ev[0], 0));
    for (int c = 0; c < nchunk; ++c) {
      const int b_lo = c_lo[c], nb = c_lo[c + 1] - b_lo;
      cudaStream_t sc = cs[c & 1];
      cudaEvent_t e_in = ev[1 + (2 * c) % (nev - 1)], e_out = ev[1 + (2 * c + 1) % (nev - 1)];
      LKB_CUDA_CHECK(cudaMemcpyAsync(d_ystage + (size_t)b_lo * N * ysz, (const unsigned char*)y + (size_t)b_lo * N * ysz,
                                     (size_t)nb * N * ysz, cudaMemcpyHostToDevice, s_h2d));
      LKB_CUDA_CHECK(cudaEventRecord(e_in, s_h2d));
      LKB_CUDA_CHECK(cudaStreamWaitEvent(sc, e_in, 0));
      if (y_dtype == LKB_DTYPE_F32)
        ls_prep_shared_kernel<float><<<nb, 256, 0, sc>>>((const float*)dy_in + (size_t)b_lo * N, N, Npad,
                                                         d_yc + (size_t)b_lo * Npad, d_absmax + b_lo, d_ysumf + b_lo);
      else
        ls_prep_shared_kernel<double><<<nb, 256, 0, sc>>>((const double*)dy_in + (size_t)b_lo * N, N, Npad,
                                                          d_yc + (size_t)b_lo * Npad, d_absmax + b_lo, d_ysumf + b_lo);
      LKB_LAUNCH_CHECK();
      if (use_nufft)
        LKB_TRY(ls_nufft_run(d_t, N, d_yc + (size_t)b_lo * Npad, Npad, d_ysumf + b_lo, d_absmax + b_lo, nb, d_freq, F,
                             d_rot, d_rot2, F_win, normalization, ns, d_pow + (size_t)b_lo * F, sc, (sc != st) ? 1 : 0,
                             true));
      else
      LKB_TRY(ls_tc_launch(d_t, d_tab, N, Npad, d_yc + (size_t)b_lo * Npad, d_absmax + b_lo, nb, d_freq, F, d_rot, d_rot2,
                           lowf_max, grid_f0, grid_df, normalization, ns, d_pow + (size_t)b_lo * F, sc, ev_join,
                           (sc != st) ? 1 : 0));
      LKB_CUDA_CHECK(cudaEventRecord(e_out, sc));
      // The power rows of chunk c - 1 go down only now, AFTER chunk c has been enqueued (s_d2h has waited for chunk
      // c - 1 only): into pageable memory (a plain numpy array) cudaMemcpyAsync blocks the host until the copy is
      // done, and issued right after its own chunk it would keep chunk c + 1 from being enqueued - no overlap at all
      // (ADVICE.md, round 1).  One chunk late, the blocking copy runs while the next chunk computes; page-locked
      // destinations are asynchronous either way.
      if (c > 0) {
        const int p_lo = c_lo[c - 1], p_nb = c_lo[c] - p_lo;
        LKB_CUDA_CHECK(cudaMemcpyAsync(power + (size_t)p_lo * F, d_pow + (size_t)p_lo * F, (size_t)p_nb * F * sizeof(float),
                                       cudaMemcpyDeviceToHost, s_d2h));
      }
      LKB_CUDA_CHECK(cudaStreamWaitEvent(s_d2h, e_out, 0));
    }
    {
      const int p_lo = c_lo[nchunk - 1], p_nb = B - p_lo;
      LKB_CUDA_CHECK(cudaMemcpyAsync(power + (size_t)p_lo * F, d_pow + (size_t)p_lo * F, (size_t)p_nb * F * sizeof(float),
                                     cudaMemcpyDeviceToHost, s_d2h));
    }
    if (cs[1] != st) LKB_CUDA_CHECK(cudaStreamSynchronize(cs[1]));
    LKB_CUDA_CHECK(cudaStreamSynchronize(s_d2h));
    LKB_CUDA_CHECK(cudaStreamSynchronize(st));
    return LKB_OK;
  }
  if (use_nufft) {
    LKB_CUDA_CHECK(cudaStreamWaitEvent(st, ev_join, 0));
    LKB_TRY(ls_nufft_run(d_t, N, d_yc, Npad, d_ysumf, d_absmax, B, d_freq, F, d_rot, d_rot2, F_win, normalization, ns, d_pow,
                         st, 0, true));
  } else if (use_tc) {
    LKB_TRY(ls_tc_launch(d_t, d_tab, N, Npad, d_yc, d_absmax, B, d_freq, F, d_rot, d_rot2, lowf_max, grid_f0, grid_df, normalization, ns, d_pow, st, ev_join));
  } else {
    static bool attr_set = false;
    if (!attr_set) {
      LKB_CUDA_CHECK(cudaFuncSetAttribute(ls_shared_simt_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          (int)(2 * sizeof(SgStage))));
      attr_set = true;
    }
    dim3 grid((unsigned)((F + SG_BM - 1) / SG_BM), (unsigned)((B + SG_BN - 1) / SG_BN));
    LKB_CUDA_CHECK(cudaStreamWaitEvent(st, ev_join, 0));
    prof_begin(st);
    ls_shared_simt_kernel<<<grid, 256, 2 * sizeof(SgStage), st>>>(d_t, N, Npad, d_yc, B, d_freq, F, d_rot,
                                                                 d_rot2, d_ysumf, lowf_max, normalization, ns, d_pow);
    prof_end(st);
    LKB_LAUNCH_CHECK();
  }
  LKB_TRY(stage_out_copy<float>(mem, power, d_pow, (size_t)B * F, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

}  // namespace lkb
