// Runs K14 (lightkurve_b200/csrc/bls_iter.cuh: bls_best_kernel, transit_count_kernel, transit_compact_kernel) on the
// CPU through tests/native/cuda_emu.h (TEST INFRASTRUCTURE).  Built with -ffp-contract=off, as bls_iter.cu is built
// with -fmad=false, by tests/test_bls_iter_emulated.py.
#include "cuda_emu.h"

#include <vector>

#include "../../lightkurve_b200/csrc/bls_iter.cuh"

namespace lkb {
int64_t g_launches = 0;
int g_last_ls_algo = -1;
int64_t g_epoch = 0;
void set_error(const char*, ...) {}
}  // namespace lkb

extern "C" {

// One bls_best launch; pofs NULL: shared grid of P periods.  out [7 B]: period, duration, transit_time, depth,
// depth_err, depth_snr, power.
void emu_bls_best(const double* const* k3, const double* period, const int64_t* pofs, int B, int64_t P, double* out,
                  int64_t* index) {
  lkb::BestArgs a{};
  a.power = k3[0];
  a.depth = k3[1];
  a.depth_err = k3[2];
  a.duration = k3[3];
  a.transit_time = k3[4];
  a.depth_snr = k3[5];
  a.period = period;
  a.pofs = pofs;
  a.P = P;
  double* o[7];
  for (int k = 0; k < 7; ++k) o[k] = out + (size_t)k * B;
  a.period_out = o[0];
  a.duration_out = o[1];
  a.transit_time_out = o[2];
  a.depth_out = o[3];
  a.depth_err_out = o[4];
  a.depth_snr_out = o[5];
  a.power_out = o[6];
  a.index_out = index;
  LKB_LAUNCH(B, lkb::BI_THREADS, 0, lkb::bls_best_kernel)(a);
}

// The count and compaction launches of lkb_transit_compact, with the host step between them.  noff, doff: [B + 1] out.
void emu_transit_compact(const double* t, const double* y, const double* dy, const int32_t* idx, const int64_t* off,
                         int B, const uint8_t* in_transit, const double* stats, int round, const int64_t* orig_off,
                         int8_t* masked_in, double* t_out, double* y_out, double* dy_out, double* w_out,
                         int32_t* idx_out, int64_t* noff, int64_t* doff, double* tinfo, uint8_t* dy_finite,
                         double* dt) {
  std::vector<int32_t> flags(B);
  std::vector<int64_t> count(B);
  LKB_LAUNCH((B + lkb::BI_THREADS - 1) / lkb::BI_THREADS, lkb::BI_THREADS, 0, lkb::transit_count_kernel)(
      off, B, stats, flags.data(), count.data());
  noff[0] = doff[0] = 0;
  for (int b = 0; b < B; ++b) {
    noff[b + 1] = noff[b] + count[b];
    doff[b + 1] = doff[b] + (count[b] > 1 ? count[b] - 1 : 0);
  }
  lkb::CompactArgs a{};
  a.t = t;
  a.y = y;
  a.dy = dy;
  a.idx = idx;
  a.off = off;
  a.in_transit = in_transit;
  a.flags = flags.data();
  a.noff = noff;
  a.doff = doff;
  a.orig_off = orig_off;
  a.round = round;
  a.masked_in = masked_in;
  a.t_out = t_out;
  a.y_out = y_out;
  a.dy_out = dy_out;
  a.w_out = w_out;
  a.idx_out = idx_out;
  a.tinfo = tinfo;
  a.dy_finite = dy_finite;
  a.dt = dt;
  LKB_LAUNCH(B, lkb::BI_THREADS, 0, lkb::transit_compact_kernel)(a);
}

}  // extern "C"
