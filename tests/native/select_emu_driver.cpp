// Runs the K6 order-statistic primitives (lightkurve_b200/csrc/select.cuh) on the CPU through tests/native/cuda_emu.h
// (TEST INFRASTRUCTURE).  Built by tests/test_select_emulated.py.
#include "cuda_emu.h"

#include "../../lightkurve_b200/csrc/select.cuh"

namespace lkb {
int64_t g_launches = 0;
int g_last_ls_algo = -1;
int64_t g_epoch = 0;
void set_error(const char*, ...) {}
}  // namespace lkb

namespace {

// per-segment outputs; seen/obs_bad are per element (CSR like the input)
struct SelOut {
  double *med, *sd, *obs_lo, *br_lo, *br_hi;
  int *observed, *resets, *br_valid, *seen;
  long long *gets, *obs_calls, *obs_bad;
};

// mode 0: block_nanmedian; 1: block_nanmedian_fast without a bracket; 2: block_nanmedian_fast with the caller's
// bracket (br_in_*).  pass_m: hand the number of non-NaN values to the fast variant (m_known) instead of -1.
// Every mode then runs block_nanstd on the same segment.
__global__ void select_kernel(const double* x, const int64_t* off, int mode, int pass_m, const double* br_in_lo,
                              const double* br_in_hi, const int* br_in_valid, SelOut o) {
  __shared__ lkb::SelSmem sm;
  __shared__ lkb::FastSelSmem fs;
  __shared__ double cand[lkb::FS_CAP + lkb::FS_SAMPLE];
  __shared__ lkb::FastBracket br;
  const int b = blockIdx.x;
  const double* xx = x + off[b];
  const int64_t n = off[b + 1] - off[b];
  int* seen = o.seen + off[b];
  long long gets = 0, calls = 0, bad = 0, mcnt = 0;
  int resets = 0;
  double my_lo = __longlong_as_double(0x7ff8000000000000ll);
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) mcnt += (xx[i] == xx[i]) ? 1 : 0;
  const long long m = lkb::block_sum_ll(mcnt, sm.redll);
  if (threadIdx.x == 0) {
    fs.cand = cand;
    br.lo = br_in_lo[b];
    br.hi = br_in_hi[b];
    br.valid = br_in_valid[b] != 0;
  }
  __syncthreads();
  auto get = [&](int64_t i) { gets++; return xx[i]; };
  auto obs = [&](int64_t i, double v, double lo, bool valid) {
    if (!valid) return;
    calls++;
    seen[i]++;
    my_lo = lo;
    if (__double_as_longlong(v) != __double_as_longlong(xx[i])) bad++;
  };
  auto reset = [&]() {
    resets++;
    calls = 0;
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) seen[i] = 0;
  };
  bool observed = false;
  double med;
  if (mode == 0)
    med = lkb::block_nanmedian(get, n, sm);
  else
    med = lkb::block_nanmedian_fast(get, n, sm, fs, pass_m ? m : -1, obs, &observed, mode == 2 ? &br : nullptr, reset);
  const double sd = lkb::block_nanstd([&](int64_t i) { return xx[i]; }, n, sm);
  const long long t_gets = lkb::block_sum_ll(gets, sm.redll), t_calls = lkb::block_sum_ll(calls, sm.redll);
  const long long t_bad = lkb::block_sum_ll(bad, sm.redll);
  if (threadIdx.x == 0) {
    o.med[b] = med;
    o.sd[b] = sd;
    o.observed[b] = observed ? 1 : 0;
    o.resets[b] = resets;
    o.gets[b] = t_gets;
    o.obs_calls[b] = t_calls;
    o.obs_bad[b] = t_bad;
    o.obs_lo[b] = my_lo;
    o.br_lo[b] = br.lo;
    o.br_hi[b] = br.hi;
    o.br_valid[b] = br.valid ? 1 : 0;
  }
}

}  // namespace

extern "C" {

int emu_select(const double* x, const int64_t* off, int B, int threads, int mode, int pass_m, const double* br_in_lo,
               const double* br_in_hi, const int* br_in_valid, double* med, double* sd, int* observed, int* resets,
               long long* gets, long long* obs_calls, long long* obs_bad, double* obs_lo, double* br_lo, double* br_hi,
               int* br_valid, int* seen) {
  SelOut o{med, sd, obs_lo, br_lo, br_hi, observed, resets, br_valid, seen, gets, obs_calls, obs_bad};
  LKB_LAUNCH(B, threads, 0, select_kernel)(x, off, mode, pass_m, br_in_lo, br_in_hi, br_in_valid, o);
  return 0;
}

}  // extern "C"
