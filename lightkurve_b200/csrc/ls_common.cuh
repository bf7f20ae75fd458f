// Device math shared by the Lomb-Scargle kernels.
// Math: astropy lombscargle_slow (fit_mean=True, center_data=True, dy=1 => w = 1/N,
// normalization="psd"), restated in oracle/ls.py:ls_slow_psd.
#pragma once
#include "common.cuh"

namespace lkb {

// sin/cos of 2*pi*phase where `phase` is in CYCLES and may be large: reduce in fp64
// (H1 of SURVEY.md: fp32 omega*t loses the phase at Kepler baselines), evaluate in fp32
// on the MUFU pipe.
__device__ __forceinline__ void ls_sincos_cycles(double phase, float& s, float& c) {
  const double magic = 6755399441055744.0;   // 1.5 * 2^52: round-to-nearest-integer trick
  const double r = __dadd_rn(phase, magic);
  const double frac = __dsub_rn(phase, __dsub_rn(r, magic));   // in [-0.5, 0.5]
  const float x = (float)frac * 6.283185307179586f;
  s = __sinf(x);
  c = __cosf(x);
}
// Low-frequency rows of the shared-grid contractions (f * baseline <= LS_LOWF_CYCLES): the design
// matrix carries cos - 1 = -2 sin^2(phase / 2) instead of cos.  sum y (cos - 1) is a sum of SMALL
// well-conditioned terms (sum y cos would be ~sum y + a tiny signal, amplifying fp32 / tensor-core
// accumulation error by 1 / (f T)^2); the epilogue adds sum y back.  `x` = phase in cycles, [-0.5, 0.5].
__device__ __forceinline__ float ls_cos_minus1(float x) {
  const float h = __sinf(3.14159265358979f * x);
  return -2.0f * h * h;
}
__device__ __forceinline__ void ls_sincos_cycles_low(double phase, float& s, float& cm1) {
  const double magic = 6755399441055744.0;
  const double r = __dadd_rn(phase, magic);
  const float x = (float)__dsub_rn(phase, __dsub_rn(r, magic));
  s = __sinf(x * 6.283185307179586f);
  cm1 = ls_cos_minus1(x);
}

// Full-fp64 unit for the LOW-FREQUENCY bins (f * baseline <~ 2 cycles): there cos(wt) barely
// varies, CC' = E[c'^2] - E[c']^2 cancels to ~1e-3..1e-7 of its terms and fp32 sums (or MUFU
// sin/cos) would leave a 1e-4..1e-2 relative error in the power.  Only a handful of bins per
// light curve take this path (the lightkurve default grid starts at f * baseline = 0.2).
constexpr double LS_LOWF_CYCLES = 2.0;
__device__ __forceinline__ void ls_sincos_cycles_f64(double phase, double& s, double& c) {
  sincospi(2.0 * (phase - rint(phase)), &s, &c);
}

// sin/cos of a fixed-point phase given by its top 32 bits (cycles * 2^32): the top 23 bits become
// the mantissa of a float in [1, 2), one FFMA maps it to radians in [0, 2 pi)  (3 integer/FMA ops,
// no fp64, no conversion instruction; quantisation 2^-23 cycle = 7.5e-7 rad, below the MUFU error).
__device__ __forceinline__ void ls_sincos_fixed32(uint32_t ph, float& s, float& c) {
  const float m = __uint_as_float((ph >> 9) | 0x3f800000u);
  const float r = fmaf(m, 6.283185307179586f, -6.283185307179586f);
  s = __sinf(r);
  c = __cosf(r);
}
__device__ __forceinline__ void ls_sincos_fixed(unsigned long long ph, float& s, float& c) {
  ls_sincos_fixed32((uint32_t)(ph >> 32), s, c);
}
__device__ __forceinline__ void ls_sincos_fixed_low(unsigned long long ph, float& s, float& cm1) {
  const float x = __uint_as_float(((uint32_t)(ph >> 32) >> 9) | 0x3f800000u) - 1.0f;   // [0, 1) cycles
  const float xc = x - (x >= 0.5f ? 1.0f : 0.0f);                                     // [-0.5, 0.5)
  s = __sinf(xc * 6.283185307179586f);
  cm1 = ls_cos_minus1(xc);
}

// Regular frequency grids f_k = f0 + k df (the lightkurve default, and what astropy's "fast"
// method requires): phase(k, n) = frac(f0 t_n) + k frac(df t_n) is evaluated in 64-bit FIXED POINT
// (cycles * 2^64, wrap-around = mod 1 for free) - exact integer arithmetic instead of an fp64
// multiply / round / subtract / convert chain per design-matrix element.  This kernel builds the
// per-cadence table {a_n, b_n}; padding cadences get 0.
static __global__ void ls_phase_table_kernel(const double* __restrict__ t, int64_t N, int64_t Npad, double f0, double df,
                                      ulonglong2* __restrict__ tab) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Npad) return;
  ulonglong2 v = make_ulonglong2(0ull, 0ull);
  if (i < N) {
    const double x = f0 * t[i], y = df * t[i];
    const double fx = x - floor(x), fy = y - floor(y);
    v.x = __double2ull_rd(fx * 18446744073709551616.0);
    v.y = __double2ull_rd(fy * 18446744073709551616.0);
  }
  tab[i] = v;
}

// max_k |freq[k] - (f0 + k df)| / |df| (0 for a perfectly regular grid)
static __global__ void ls_grid_regularity_kernel(const double* __restrict__ freq, int64_t F, float* __restrict__ out) {
  if (F < 2) return;
  const double f0 = freq[0], df = freq[1] - freq[0];
  float worst = 0.f;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < F; k += (int64_t)gridDim.x * blockDim.x) {
    const double dev = fabs(freq[k] - (f0 + (double)k * df)) / fabs(df);
    worst = fmaxf(worst, (float)dev);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) worst = fmaxf(worst, __shfl_xor_sync(0xffffffffu, worst, o));
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(out), __float_as_int(worst));   // worst >= 0
}

// meta[0] (written as float bits by the regularity kernel, 0 when F < 2) -> double; meta[1..3] = f0, f1, t_last
static __global__ void ls_meta_kernel(const double* __restrict__ freq, int64_t F, const double* __restrict__ t,
                                      int64_t N, double* __restrict__ meta) {
  const float dev = *reinterpret_cast<const float*>(meta);
  meta[0] = (F >= 2) ? (double)dev : 1.0;
  meta[1] = freq[0];
  meta[2] = (F >= 2) ? freq[1] : freq[0];
  meta[3] = fabs(t[N - 1]);
}

template <typename T>
struct LsSums {
  T sh, ch, s, c, cc, sc;
  __device__ __forceinline__ void zero() { sh = ch = s = c = cc = sc = (T)0; }
  __device__ __forceinline__ void add(T y, T sn, T cs) {
    sh += y * sn;
    ch += y * cs;
    s += sn;
    c += cs;
    cc += cs * cs;
    sc += sn * cs;
  }
  template <typename U>
  __device__ __forceinline__ void accumulate(const LsSums<U>& o) {
    sh += (T)o.sh; ch += (T)o.ch; s += (T)o.s; c += (T)o.c; cc += (T)o.cc; sc += (T)o.sc;
  }
  __device__ __forceinline__ void warp_reduce() {
    sh = warp_sum(sh); ch = warp_sum(ch); s = warp_sum(s); c = warp_sum(c); cc = warp_sum(cc); sc = warp_sum(sc);
  }
};

// tau rotation and the floating-mean corrected CC', SS' (weights w = 1/N).
__device__ __forceinline__ void ls_rotation(const LsSums<double>& d, double N, double& ct, double& st,
                                            double& ccp, double& ssp) {
  const double Sb = d.s / N, Cb = d.c / N, CCb = d.cc / N, SCb = d.sc / N, SSb = 1.0 - CCb;
  const double S2 = 2.0 * SCb - 2.0 * Sb * Cb;
  const double C2 = (2.0 * CCb - 1.0) - (Cb * Cb - Sb * Sb);
  const double ta = 0.5 * atan2(S2, C2);
  sincos(ta, &st, &ct);
  const double Ctau = Cb * ct + Sb * st, Stau = Sb * ct - Cb * st;
  ccp = CCb * ct * ct + 2.0 * SCb * ct * st + SSb * st * st - Ctau * Ctau;
  ssp = SSb * ct * ct - 2.0 * SCb * ct * st + CCb * st * st - Stau * Stau;
}

// astropy normalization="psd": 0.5 * N * (YC^2/CC + YS^2/SS).  `ysum` = sum of the (centred, then
// fp32-rounded) flux actually fed to the sums: YC = sum(w y c') - Y sum(w c') with Y = ysum / N
// (astropy keeps this term; it only matters when c' is nearly constant, i.e. f * baseline << 1).
__device__ __forceinline__ double ls_power_from_sums(const LsSums<double>& d, double N, double ysum) {
  double ct, st, ccp, ssp;
  ls_rotation(d, N, ct, st, ccp, ssp);
  const double Y = ysum / N;
  const double Ctau = (d.c * ct + d.s * st) / N, Stau = (d.s * ct - d.c * st) / N;
  const double YC = (d.ch * ct + d.sh * st) / N - Y * Ctau, YS = (d.sh * ct - d.ch * st) / N - Y * Stau;
  return 0.5 * N * (YC * YC / ccp + YS * YS / ssp);
}

// lightkurve rescale, periodogram.py:969-975
__device__ __forceinline__ float ls_normalize(double p_raw, double N, int normalization, double scale) {
  if (normalization == LKB_LS_NORM_PSD_SCALE) return (float)(p_raw * scale);
  if (normalization == LKB_LS_NORM_AMPLITUDE) return (float)(sqrt(p_raw) * sqrt(4.0 / N));
  return (float)p_raw;
}

// shared-grid epilogue: rot = {cos tau, sin tau, 1/(2 N CC'), 1/(2 N SS')}, rot2 = {Ctau, Stau}
// (= sum(w c'), sum(w s')), ysum = sum of the light curve's effective centred flux.
__device__ __forceinline__ float ls_epilogue_shared(float ch, float sh, const float4 rot, const float2 rot2,
                                                    float ysum, float N, int normalization, float scale,
                                                    bool low_row = false) {
  if (low_row) ch += ysum;      // the design matrix held cos - 1 for this frequency (see ls_cos_minus1)
  const float yc = ch * rot.x + sh * rot.y - ysum * rot2.x, ys = sh * rot.x - ch * rot.y - ysum * rot2.y;
  const float p = yc * yc * rot.z + ys * ys * rot.w;
  if (normalization == LKB_LS_NORM_PSD_SCALE) return p * scale;
  if (normalization == LKB_LS_NORM_AMPLITUDE) return sqrtf(p * (4.0f / N));
  return p;
}

// Multi-term ("chi2") periodogram, shared by the direct kernel (ls.cu: ls_chi2_kernel) and the NUFFT path's low rows
// (ls_nufft.cu): the harmonic trig sums S_j, C_j (j <= 2n) and YS_j, YC_j (j <= n) of one frequency, and the fp64
// solve of the (2n+1)x(2n+1) normal equations they give.
template <int NT>
struct Chi2Sums {
  double S[2 * NT], C[2 * NT], YS[NT], YC[NT];
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int j = 0; j < 2 * NT; ++j) { S[j] = 0.0; C[j] = 0.0; }
#pragma unroll
    for (int j = 0; j < NT; ++j) { YS[j] = 0.0; YC[j] = 0.0; }
  }
};

template <int NT>
__device__ void chi2_solve(const Chi2Sums<NT>& d, double N, double ysum, double& power, double* theta) {
  constexpr int M = 2 * NT + 1;
  double A[M][M + 1];
  auto Cd = [&](int m) { return m == 0 ? N : d.C[m - 1]; };
  auto Sd = [&](int m) { return m == 0 ? 0.0 : (m > 0 ? d.S[m - 1] : -d.S[-m - 1]); };
  A[0][0] = N;
  A[0][M] = ysum;
  for (int i = 1; i <= NT; ++i) {
    const int si = 2 * i - 1, ci = 2 * i;
    A[0][si] = A[si][0] = d.S[i - 1];
    A[0][ci] = A[ci][0] = d.C[i - 1];
    A[si][M] = d.YS[i - 1];
    A[ci][M] = d.YC[i - 1];
    for (int j = 1; j <= NT; ++j) {
      const int sj = 2 * j - 1, cj = 2 * j;
      const int dm = i > j ? i - j : j - i;
      A[si][sj] = 0.5 * (Cd(dm) - Cd(i + j));
      A[ci][cj] = 0.5 * (Cd(dm) + Cd(i + j));
      A[si][cj] = 0.5 * (Sd(i + j) + Sd(i - j));
      A[cj][si] = A[si][cj];
    }
  }
  double rhs[M];
  for (int i = 0; i < M; ++i) rhs[i] = A[i][M];
  bool ok = true;
  for (int c = 0; c < M && ok; ++c) {
    int piv = c;
    for (int r = c + 1; r < M; ++r)
      if (fabs(A[r][c]) > fabs(A[piv][c])) piv = r;
    if (!(fabs(A[piv][c]) > 0.0)) { ok = false; break; }
    if (piv != c)
      for (int k = 0; k <= M; ++k) { const double tmp = A[c][k]; A[c][k] = A[piv][k]; A[piv][k] = tmp; }
    for (int r = c + 1; r < M; ++r) {
      const double fct = A[r][c] / A[c][c];
      for (int k = c; k <= M; ++k) A[r][k] -= fct * A[c][k];
    }
  }
  double th[M];
  const double qnan = __longlong_as_double(0x7ff8000000000000ll);
  if (ok) {
    for (int c = M - 1; c >= 0; --c) {
      double v = A[c][M];
      for (int k = c + 1; k < M; ++k) v -= A[c][k] * th[k];
      th[c] = v / A[c][c];
    }
    double acc = 0.0;
    for (int i = 0; i < M; ++i) acc += rhs[i] * th[i];
    power = 0.5 * acc;
  } else {
    power = qnan;
    for (int i = 0; i < M; ++i) th[i] = qnan;
  }
  if (theta)
    for (int i = 0; i < M; ++i) theta[i] = th[i];
}

template <int NT>
__device__ __forceinline__ void chi2_warp_reduce(Chi2Sums<NT>& d) {
#pragma unroll
  for (int j = 0; j < 2 * NT; ++j) { d.S[j] = warp_sum(d.S[j]); d.C[j] = warp_sum(d.C[j]); }
#pragma unroll
  for (int j = 0; j < NT; ++j) { d.YS[j] = warp_sum(d.YS[j]); d.YC[j] = warp_sum(d.YC[j]); }
}

// one cadence of the sums: flux yy at phase `phase` (cycles); harmonics from the angle-addition recurrence
template <int NT>
__device__ __forceinline__ void chi2_add(Chi2Sums<NT>& d, double yy, double phase) {
  double s1, c1;
  ls_sincos_cycles_f64(phase, s1, c1);
  double sj = s1, cj = c1;
#pragma unroll
  for (int j = 0; j < 2 * NT; ++j) {
    d.S[j] += sj;
    d.C[j] += cj;
    if (j < NT) { d.YS[j] = fma(yy, sj, d.YS[j]); d.YC[j] = fma(yy, cj, d.YC[j]); }
    const double sn = fma(sj, c1, cj * s1), cn = fma(cj, c1, -sj * s1);
    sj = sn;
    cj = cn;
  }
}

}  // namespace lkb
