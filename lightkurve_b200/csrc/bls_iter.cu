// Entries of K14 (lkb_bls_best, lkb_transit_compact); the kernels are in bls_iter.cuh.  Compiled with -fmad=false like
// the other kernels that must round as numpy does (the mean of the two box levels, the time steps).
#include <vector>

#include "bls_iter.cuh"

namespace lkb {

int bls_best(const double* power, const double* depth, const double* depth_err, const double* duration,
             const double* transit_time, const double* depth_snr, const double* period, const int64_t* h_pofs, int B,
             int64_t P, double* period_out, double* duration_out, double* transit_time_out, double* depth_out,
             double* depth_err_out, double* depth_snr_out, double* power_out, int64_t* index_out, int mem,
             cudaStream_t st) {
  LKB_REQUIRE(power && depth && depth_err && duration && transit_time && depth_snr && period,
              "lkb_bls_best: null input");
  LKB_REQUIRE(period_out && duration_out && transit_time_out && depth_out && depth_err_out && depth_snr_out &&
              power_out && index_out, "lkb_bls_best: null output");
  LKB_REQUIRE(B > 0 && B <= 65535 && P > 0, "lkb_bls_best: bad sizes");
  if (h_pofs) {
    LKB_REQUIRE(h_pofs[0] == 0 && h_pofs[B] == P, "lkb_bls_best: period_offsets[0] must be 0 and period_offsets[B] == P");
    for (int b = 0; b < B; ++b)
      if (h_pofs[b + 1] <= h_pofs[b]) {
        set_error("lkb_bls_best: light curve %d has an empty or negative period segment", b);
        return LKB_E_ARG;
      }
  }
  LKB_TRY(ensure_device());
  const int64_t total = h_pofs ? P : (int64_t)B * P;
  BestArgs a{};
  LKB_TRY(stage_in<double>(mem, WS_IN0, power, total, &a.power, st));
  LKB_TRY(stage_in<double>(mem, WS_IN1, depth, total, &a.depth, st));
  LKB_TRY(stage_in<double>(mem, WS_IN2, depth_err, total, &a.depth_err, st));
  LKB_TRY(stage_in<double>(mem, WS_IN3, duration, total, &a.duration, st));
  LKB_TRY(stage_in<double>(mem, WS_IN4, transit_time, total, &a.transit_time, st));
  LKB_TRY(stage_in<double>(mem, WS_IN5, depth_snr, total, &a.depth_snr, st));
  LKB_TRY(stage_in<double>(mem, WS_IN6, period, P, &a.period, st));
  a.pofs = nullptr;
  if (h_pofs) {
    int64_t* d = nullptr;
    LKB_TRY(ws_get_t<int64_t>(WS_X0, (size_t)B + 1, &d));
    LKB_CUDA_CHECK(cudaMemcpyAsync(d, h_pofs, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
    a.pofs = d;
  }
  a.P = P;
  double* outs[7] = {period_out, duration_out, transit_time_out, depth_out, depth_err_out, depth_snr_out, power_out};
  double* d_outs[7];
  for (int k = 0; k < 7; ++k) LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0 + k, outs[k], B, &d_outs[k]));
  a.period_out = d_outs[0];
  a.duration_out = d_outs[1];
  a.transit_time_out = d_outs[2];
  a.depth_out = d_outs[3];
  a.depth_err_out = d_outs[4];
  a.depth_snr_out = d_outs[5];
  a.power_out = d_outs[6];
  LKB_TRY(stage_out_alloc<int64_t>(mem, WS_X1, index_out, B, &a.index_out));
  prof_begin(st);
  bls_best_kernel<<<B, BI_THREADS, 0, st>>>(a);
  prof_end(st);
  LKB_LAUNCH_CHECK();
  for (int k = 0; k < 7; ++k) LKB_TRY(stage_out_copy<double>(mem, outs[k], d_outs[k], B, st));
  LKB_TRY(stage_out_copy<int64_t>(mem, index_out, a.index_out, B, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

int transit_compact(const double* t, const double* y, const double* dy, const int32_t* idx, const int64_t* h_off,
                    int B, const uint8_t* in_transit, const double* stats, int round, const int64_t* h_orig_off,
                    int8_t* masked_in, double* t_out, double* y_out, double* dy_out, double* w_out, int32_t* idx_out,
                    int64_t* h_noff, int64_t* h_doff, double* tinfo, uint8_t* dy_finite, double* dt, int mem,
                    cudaStream_t st) {
  LKB_REQUIRE(t && y && dy && idx && h_off && in_transit && stats && h_orig_off && masked_in,
              "lkb_transit_compact: null input");
  LKB_REQUIRE(t_out && y_out && dy_out && w_out && idx_out && h_noff && h_doff && tinfo && dy_finite && dt,
              "lkb_transit_compact: null output");
  LKB_REQUIRE(B > 0 && round >= 0 && round <= 127, "lkb_transit_compact: bad sizes or round");
  LKB_REQUIRE(h_off[0] == 0 && h_orig_off[0] == 0, "lkb_transit_compact: offsets[0] must be 0");
  for (int b = 0; b < B; ++b) {
    const int64_t n = h_off[b + 1] - h_off[b];
    if (n < 0 || n > h_orig_off[b + 1] - h_orig_off[b] || n >= ((int64_t)1 << 31)) {
      set_error("lkb_transit_compact: light curve %d has %lld cadences, its original light curve %lld", b,
                (long long)n, (long long)(h_orig_off[b + 1] - h_orig_off[b]));
      return LKB_E_ARG;
    }
  }
  LKB_TRY(ensure_device());
  const int64_t total = h_off[B], orig_total = h_orig_off[B];
  CompactArgs a{};
  LKB_TRY(stage_in<double>(mem, WS_IN0, t, total, &a.t, st));
  LKB_TRY(stage_in<double>(mem, WS_IN1, y, total, &a.y, st));
  LKB_TRY(stage_in<double>(mem, WS_IN2, dy, total, &a.dy, st));
  LKB_TRY(stage_in<int32_t>(mem, WS_IN3, idx, total, &a.idx, st));
  LKB_TRY(stage_in<uint8_t>(mem, WS_IN4, in_transit, total, &a.in_transit, st));
  const double* d_stats = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN5, stats, (size_t)B * BI_STAT_COLS, &d_stats, st));
  // CSRs on the device: offsets, survivors, steps, original light curves
  int64_t* d_csr = nullptr;
  LKB_TRY(ws_get_t<int64_t>(WS_X0, 4 * ((size_t)B + 1), &d_csr));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_csr, h_off, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_csr + 3 * ((size_t)B + 1), h_orig_off, sizeof(int64_t) * (B + 1),
                                 cudaMemcpyHostToDevice, st));
  int32_t* d_flags = nullptr;
  int64_t* d_count = nullptr;
  LKB_TRY(ws_get_t<int32_t>(WS_X1, B, &d_flags));
  LKB_TRY(ws_get_t<int64_t>(WS_X2, B, &d_count));
  transit_count_kernel<<<(B + BI_THREADS - 1) / BI_THREADS, BI_THREADS, 0, st>>>(d_csr, B, d_stats, d_flags,
                                                                                  d_count);
  LKB_LAUNCH_CHECK();
  std::vector<int64_t> count(B);
  LKB_CUDA_CHECK(cudaMemcpyAsync(count.data(), d_count, sizeof(int64_t) * B, cudaMemcpyDeviceToHost, st));
  LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  h_noff[0] = h_doff[0] = 0;
  for (int b = 0; b < B; ++b) {
    h_noff[b + 1] = h_noff[b] + count[b];
    h_doff[b + 1] = h_doff[b] + (count[b] > 1 ? count[b] - 1 : 0);
  }
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_csr + ((size_t)B + 1), h_noff, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice,
                                 st));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_csr + 2 * ((size_t)B + 1), h_doff, sizeof(int64_t) * (B + 1),
                                 cudaMemcpyHostToDevice, st));
  a.off = d_csr;
  a.noff = d_csr + ((size_t)B + 1);
  a.doff = d_csr + 2 * ((size_t)B + 1);
  a.orig_off = d_csr + 3 * ((size_t)B + 1);
  a.flags = d_flags;
  a.round = round;
  const int64_t kept = h_noff[B], steps = h_doff[B];
  if (mem == LKB_MEM_HOST) {                       // masked_in is read and written
    int8_t* d = nullptr;
    LKB_TRY(ws_get_t<int8_t>(WS_OUT0, orig_total ? (size_t)orig_total : 1, &d));
    if (orig_total) LKB_CUDA_CHECK(cudaMemcpyAsync(d, masked_in, (size_t)orig_total, cudaMemcpyHostToDevice, st));
    a.masked_in = d;
  } else {
    a.masked_in = masked_in;
  }
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT1, t_out, kept, &a.t_out));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT2, y_out, kept, &a.y_out));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT3, dy_out, kept, &a.dy_out));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT4, w_out, kept, &a.w_out));
  LKB_TRY(stage_out_alloc<int32_t>(mem, WS_OUT5, idx_out, kept, &a.idx_out));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT6, tinfo, 3 * (size_t)B, &a.tinfo));
  LKB_TRY(stage_out_alloc<uint8_t>(mem, WS_OUT7, dy_finite, B, &a.dy_finite));
  LKB_TRY(stage_out_alloc<double>(mem, WS_X3, dt, steps, &a.dt));
  prof_begin(st);
  transit_compact_kernel<<<B, BI_THREADS, 0, st>>>(a);
  prof_end(st);
  LKB_LAUNCH_CHECK();
  LKB_TRY(stage_out_copy<int8_t>(mem, masked_in, a.masked_in, orig_total, st));
  LKB_TRY(stage_out_copy<double>(mem, t_out, a.t_out, kept, st));
  LKB_TRY(stage_out_copy<double>(mem, y_out, a.y_out, kept, st));
  LKB_TRY(stage_out_copy<double>(mem, dy_out, a.dy_out, kept, st));
  LKB_TRY(stage_out_copy<double>(mem, w_out, a.w_out, kept, st));
  LKB_TRY(stage_out_copy<int32_t>(mem, idx_out, a.idx_out, kept, st));
  LKB_TRY(stage_out_copy<double>(mem, tinfo, a.tinfo, 3 * (size_t)B, st));
  LKB_TRY(stage_out_copy<uint8_t>(mem, dy_finite, a.dy_finite, B, st));
  LKB_TRY(stage_out_copy<double>(mem, dt, a.dt, steps, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

}  // namespace lkb
