// Entries of K15 (lkb_fill_gaps_plan, lkb_fill_gaps); the kernels are in gapfill.cuh.  Compiled with -fmad=false so
// that 1.2 * dt, mean + std * z and the interpolation of flux_err round like numpy's separate operations.
#include <vector>

#include "gapfill.cuh"

namespace lkb {

int nanmedian_std(const double*, const int64_t*, int, double*, double*, int, cudaStream_t);

static int gf_check_offsets(const int64_t* h_off, int B, const char* what) {
  LKB_REQUIRE(h_off[0] == 0, "lkb_fill_gaps: offsets[0] must be 0");
  for (int b = 0; b < B; ++b) {
    const int64_t n = h_off[b + 1] - h_off[b];
    if (n < 0) {
      set_error("%s: light curve %d has a negative length", what, b);
      return LKB_E_ARG;
    }
  }
  return LKB_OK;
}

int normalize_compact(const double* t, const double* flux, const double* flux_err, const int64_t* h_off, int B,
                      const double* median, int64_t* h_noff, int32_t* bad_out, double* t_out, double* flux_out,
                      double* err_out, double* ends_out, int mem, cudaStream_t st) {
  LKB_REQUIRE(t && flux && flux_err && h_off && median && h_noff && bad_out && t_out && flux_out && err_out &&
              ends_out, "lkb_normalize_compact: null argument");
  LKB_REQUIRE(B > 0 && B <= 2147483647, "lkb_normalize_compact: bad B");
  LKB_TRY(gf_check_offsets(h_off, B, "lkb_normalize_compact"));
  LKB_TRY(ensure_device());
  const int64_t total = h_off[B];
  NormArgs a{};
  LKB_TRY(stage_in<double>(mem, WS_IN0, t, total, &a.t, st));
  LKB_TRY(stage_in<double>(mem, WS_IN1, flux, total, &a.y, st));
  LKB_TRY(stage_in<double>(mem, WS_IN2, flux_err, total, &a.e, st));
  LKB_TRY(stage_in<double>(mem, WS_IN3, median, B, &a.med, st));
  int64_t* d_csr = nullptr;
  LKB_TRY(ws_get_t<int64_t>(WS_Y0, 3 * ((size_t)B + 1), &d_csr));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_csr, h_off, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  a.off = d_csr;
  a.count = d_csr + B + 1;
  int32_t* d_bad = nullptr;
  LKB_TRY(ws_get_t<int32_t>(WS_Y1, B, &d_bad));
  a.bad = d_bad;
  normalize_compact_kernel<<<B, GF_THREADS, 0, st>>>(a);
  LKB_LAUNCH_CHECK();
  std::vector<int64_t> count(B);
  LKB_CUDA_CHECK(cudaMemcpyAsync(count.data(), a.count, sizeof(int64_t) * B, cudaMemcpyDeviceToHost, st));
  LKB_CUDA_CHECK(cudaMemcpyAsync(bad_out, d_bad, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, st));
  LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  h_noff[0] = 0;
  for (int b = 0; b < B; ++b) h_noff[b + 1] = h_noff[b] + count[b];
  const int64_t kept = h_noff[B];
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_csr + 2 * ((size_t)B + 1), h_noff, sizeof(int64_t) * (B + 1),
                                 cudaMemcpyHostToDevice, st));
  a.noff = d_csr + 2 * ((size_t)B + 1);
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0, t_out, kept, &a.t_out));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT1, flux_out, kept, &a.y_out));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT2, err_out, kept, &a.e_out));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT3, ends_out, 2 * (size_t)B, &a.ends));
  prof_begin(st);
  normalize_compact_kernel<<<B, GF_THREADS, 0, st>>>(a);
  prof_end(st);
  LKB_LAUNCH_CHECK();
  LKB_TRY(stage_out_copy<double>(mem, t_out, a.t_out, kept, st));
  LKB_TRY(stage_out_copy<double>(mem, flux_out, a.y_out, kept, st));
  LKB_TRY(stage_out_copy<double>(mem, err_out, a.e_out, kept, st));
  LKB_TRY(stage_out_copy<double>(mem, ends_out, a.ends, 2 * (size_t)B, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

int fill_gaps_plan(const double* t, const double* flux, const int64_t* h_off, int B, double* dt_out,
                   double* mean_out, int64_t* n_ins_out, int32_t* flags_out, int mem, cudaStream_t st) {
  LKB_REQUIRE(t && flux && h_off && dt_out && mean_out && n_ins_out && flags_out, "lkb_fill_gaps_plan: null argument");
  LKB_REQUIRE(B > 0 && B <= 2147483647, "lkb_fill_gaps_plan: bad B");
  LKB_TRY(gf_check_offsets(h_off, B, "lkb_fill_gaps_plan"));
  LKB_TRY(ensure_device());
  const int64_t total = h_off[B];
  std::vector<int64_t> h_doff(B + 1);
  h_doff[0] = 0;
  for (int b = 0; b < B; ++b) {
    const int64_t n = h_off[b + 1] - h_off[b];
    h_doff[b + 1] = h_doff[b] + (n > 1 ? n - 1 : 0);
  }
  const double *d_t = nullptr, *d_y = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, t, total, &d_t, st));
  LKB_TRY(stage_in<double>(mem, WS_IN1, flux, total, &d_y, st));
  int64_t* d_csr = nullptr;
  LKB_TRY(ws_get_t<int64_t>(WS_Y0, 2 * ((size_t)B + 1), &d_csr));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_csr, h_off, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_csr + B + 1, h_doff.data(), sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  double* d_steps = nullptr;
  LKB_TRY(ws_get_t<double>(WS_Y1, h_doff[B] ? (size_t)h_doff[B] : 1, &d_steps));
  double *d_dt = nullptr, *d_mean = nullptr;
  int64_t* d_ins = nullptr;
  int32_t* d_flags = nullptr;
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0, dt_out, B, &d_dt));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT1, mean_out, B, &d_mean));
  LKB_TRY(stage_out_alloc<int64_t>(mem, WS_OUT2, n_ins_out, B, &d_ins));
  LKB_TRY(stage_out_alloc<int32_t>(mem, WS_OUT3, flags_out, B, &d_flags));
  prof_begin(st);
  gap_steps_kernel<<<B, GF_THREADS, 0, st>>>(d_t, d_csr, d_csr + B + 1, d_steps, d_flags);
  LKB_LAUNCH_CHECK();
  // the median step: K6 on the device (a light curve without steps gets NaN)
  LKB_TRY(nanmedian_std(d_steps, h_doff.data(), B, d_dt, nullptr, LKB_MEM_DEVICE, st));
  gap_plan_kernel<<<B, GF_THREADS, 0, st>>>(d_t, d_y, d_csr, d_dt, d_ins, d_mean, d_flags);
  prof_end(st);
  LKB_LAUNCH_CHECK();
  LKB_TRY(stage_out_copy<double>(mem, dt_out, d_dt, B, st));
  LKB_TRY(stage_out_copy<double>(mem, mean_out, d_mean, B, st));
  LKB_TRY(stage_out_copy<int64_t>(mem, n_ins_out, d_ins, B, st));
  LKB_TRY(stage_out_copy<int32_t>(mem, flags_out, d_flags, B, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

int fill_gaps(const double* t, const double* flux, const double* flux_err, const int64_t* h_off, int B,
              const double* dt, const double* mean, const double* std, const double* z, const int64_t* h_noff,
              double* t_out, double* flux_out, double* err_out, int mem, cudaStream_t st) {
  LKB_REQUIRE(t && flux && flux_err && h_off && dt && mean && std && h_noff && t_out && flux_out && err_out,
              "lkb_fill_gaps: null argument");
  LKB_REQUIRE(B > 0 && B <= 2147483647, "lkb_fill_gaps: bad B");
  LKB_TRY(gf_check_offsets(h_off, B, "lkb_fill_gaps"));
  LKB_REQUIRE(h_noff[0] == 0, "lkb_fill_gaps: out_offsets[0] must be 0");
  for (int b = 0; b < B; ++b)
    if (h_noff[b + 1] - h_noff[b] < h_off[b + 1] - h_off[b]) {
      set_error("lkb_fill_gaps: light curve %d has fewer output than input cadences", b);
      return LKB_E_ARG;
    }
  const int64_t total = h_off[B], ntotal = h_noff[B], nz = ntotal - total;
  LKB_REQUIRE(nz == 0 || z, "lkb_fill_gaps: z is required when cadences are inserted");
  LKB_TRY(ensure_device());
  FillArgs a{};
  LKB_TRY(stage_in<double>(mem, WS_IN0, t, total, &a.t, st));
  LKB_TRY(stage_in<double>(mem, WS_IN1, flux, total, &a.y, st));
  LKB_TRY(stage_in<double>(mem, WS_IN2, flux_err, total, &a.e, st));
  LKB_TRY(stage_in<double>(mem, WS_IN3, dt, B, &a.dt, st));
  LKB_TRY(stage_in<double>(mem, WS_IN4, mean, B, &a.mean, st));
  LKB_TRY(stage_in<double>(mem, WS_IN5, std, B, &a.std, st));
  LKB_TRY(stage_in<double>(mem, WS_IN6, nz ? z : nullptr, nz, &a.z, st));
  int64_t* d_csr = nullptr;
  LKB_TRY(ws_get_t<int64_t>(WS_Y0, 2 * ((size_t)B + 1), &d_csr));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_csr, h_off, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_csr + B + 1, h_noff, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  a.off = d_csr;
  a.noff = d_csr + B + 1;
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0, t_out, ntotal, &a.t_out));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT1, flux_out, ntotal, &a.y_out));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT2, err_out, ntotal, &a.e_out));
  prof_begin(st);
  gap_fill_kernel<<<B, GF_THREADS, 0, st>>>(a);
  prof_end(st);
  LKB_LAUNCH_CHECK();
  LKB_TRY(stage_out_copy<double>(mem, t_out, a.t_out, ntotal, st));
  LKB_TRY(stage_out_copy<double>(mem, flux_out, a.y_out, ntotal, st));
  LKB_TRY(stage_out_copy<double>(mem, err_out, a.e_out, ntotal, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

}  // namespace lkb
