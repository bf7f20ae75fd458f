// Entries of K11 (lkb_sigma_clip) and K4 + K11 + K12 (lkb_cdpp); the kernel is in clip.cuh.  Compiled with
// -fmad=false: the clip bounds are numpy's c - (s * sigma), rounded twice, so a value on a bound is judged the same.
#include "clip.cuh"

namespace lkb {

int flatten(const double*, const double*, const double*, const uint8_t*, const int64_t*, int, int, int, double, int,
            double, double*, double*, double*, int, cudaStream_t);

static int check_offsets(const int64_t* h_off, int B, const char* who) {
  if (h_off[0] != 0) { set_error("%s: offsets[0] must be 0", who); return LKB_E_ARG; }
  for (int b = 0; b < B; ++b)
    if (h_off[b + 1] < h_off[b] || h_off[b + 1] - h_off[b] >= ((int64_t)1 << 31)) {
      set_error("%s: light curve %d has a negative or too large length", who, b);
      return LKB_E_ARG;
    }
  return LKB_OK;
}

// Launches clip_cdpp_kernel on B light curves; a.x, a.work (when some light curve streams) and the outputs are device
// pointers, h_off the host offsets.
static int clip_launch(ClipArgs a, const int64_t* h_off, int B, cudaStream_t st) {
  const ClipPlan p = clip_plan(h_off, B, CL_RES_CAP);
  a.res_cap = p.res_cap;
  a.cand = p.cand;
  int64_t* d_off = nullptr;
  LKB_TRY(ws_get_t<int64_t>(WS_X3, B + 1, &d_off));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_off, h_off, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  a.off = d_off;
  static size_t attr = 0;
  if (p.smem > attr) {
    LKB_CUDA_CHECK(cudaFuncSetAttribute(clip_cdpp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
    attr = p.smem;
  }
  prof_begin(st);
  clip_cdpp_kernel<<<B, CL_THREADS, p.smem, st>>>(a);
  prof_end(st);
  LKB_LAUNCH_CHECK();
  return LKB_OK;
}

int sigma_clip(const double* x, const int64_t* h_off, int B, double sigma_lower, double sigma_upper, int maxiters,
               uint8_t* mask_out, double* center_out, double* std_out, int64_t* n_kept_out, int mem, cudaStream_t st) {
  LKB_REQUIRE(x && h_off && B > 0, "lkb_sigma_clip: null/empty argument");
  LKB_TRY(check_offsets(h_off, B, "lkb_sigma_clip"));
  LKB_TRY(ensure_device());
  const int64_t total = h_off[B];
  ClipArgs a{};
  const double* d_x = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, x, total, &d_x, st));
  a.x = d_x;
  if (clip_plan(h_off, B, CL_RES_CAP).streams) {
    if (mem == LKB_MEM_HOST) a.work = const_cast<double*>(d_x);       // the staged copy is ours: clip it in place
    else LKB_TRY(ws_get_t<double>(WS_X2, total, &a.work));
  }
  a.sigma_lower = sigma_lower;
  a.sigma_upper = sigma_upper;
  a.maxiters = maxiters;
  LKB_TRY(stage_out_alloc<uint8_t>(mem, WS_OUT0, mask_out, total, &a.mask));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT1, center_out, B, &a.center));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT2, std_out, B, &a.sd));
  LKB_TRY(stage_out_alloc<int64_t>(mem, WS_OUT3, n_kept_out, B, &a.n_kept));
  LKB_TRY(clip_launch(a, h_off, B, st));
  LKB_TRY(stage_out_copy<uint8_t>(mem, mask_out, a.mask, total, st));
  LKB_TRY(stage_out_copy<double>(mem, center_out, a.center, B, st));
  LKB_TRY(stage_out_copy<double>(mem, std_out, a.sd, B, st));
  LKB_TRY(stage_out_copy<int64_t>(mem, n_kept_out, a.n_kept, B, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

int cdpp(const double* time, const double* flux, const int64_t* h_off, int B, const int32_t* durations, int D,
         int savgol_window, int savgol_polyorder, double sigma, double* cdpp_out, int mem, cudaStream_t st) {
  LKB_REQUIRE(time && flux && h_off && durations && cdpp_out && B > 0 && D > 0, "lkb_cdpp: null/empty argument");
  for (int d = 0; d < D; ++d) LKB_REQUIRE(durations[d] >= 1, "lkb_cdpp: transit durations must be >= 1 cadence");
  LKB_TRY(check_offsets(h_off, B, "lkb_cdpp"));
  if (savgol_polyorder >= savgol_window) savgol_polyorder = savgol_window - 1;     // as flatten clamps it
  LKB_TRY(ensure_device());
  const int64_t total = h_off[B];
  const double *d_t = nullptr, *d_f = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, time, total, &d_t, st));
  LKB_TRY(stage_in<double>(mem, WS_IN1, flux, total, &d_f, st));
  double *d_flat = nullptr, *d_trend = nullptr;
  LKB_TRY(ws_get_t<double>(WS_X0, total, &d_flat));
  LKB_TRY(ws_get_t<double>(WS_X1, total, &d_trend));
  // estimate_cdpp's flatten: break_tolerance 5, niters 3, sigma 3, no mask; its output stays on the device
  LKB_TRY(flatten(d_t, d_f, nullptr, nullptr, h_off, B, savgol_window, savgol_polyorder, 5.0, 3, 3.0, d_flat, nullptr,
                  d_trend, LKB_MEM_DEVICE, st));
  ClipArgs a{};
  a.x = d_flat;
  a.work = d_flat;                                               // the flattened flux is ours: clip it in place
  a.sigma_lower = sigma;
  a.sigma_upper = sigma;
  a.maxiters = 5;                                                // remove_outliers' default
  int32_t* d_dur = nullptr;
  LKB_TRY(ws_get_t<int32_t>(WS_X4, D, &d_dur));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_dur, durations, sizeof(int32_t) * D, cudaMemcpyHostToDevice, st));
  a.dur = d_dur;
  a.D = D;
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0, cdpp_out, (size_t)B * D, &a.cdpp));
  LKB_TRY(clip_launch(a, h_off, B, st));
  LKB_TRY(stage_out_copy<double>(mem, cdpp_out, a.cdpp, (size_t)B * D, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

}  // namespace lkb
