// Runs the K10 BLS vetting kernel (lightkurve_b200/csrc/bls_stats.cuh) on the CPU through tests/native/cuda_emu.h
// (TEST INFRASTRUCTURE).  Built by tests/test_bls_stats_emulated.py.
#include "cuda_emu.h"

#include <stdarg.h>
#include <stdio.h>

#include "../../lightkurve_b200/csrc/bls_stats.cuh"

namespace lkb {
int64_t g_launches = 0;
int g_last_ls_algo = -1;
int64_t g_epoch = 0;
static char g_err[512];
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace lkb

extern "C" {

const char* emu_last_error() { return lkb::g_err; }

// bls_stats_launch on host buffers (offsets and transit_offsets [B + 1])
int emu_bls_stats(const double* t, const double* y, const double* dy, const int64_t* offsets, int B,
                  const double* period, const double* duration, const double* transit_time,
                  const int64_t* transit_offsets, double* stats, int64_t* transit_first, int32_t* transit_n,
                  int32_t* per_transit_count, double* per_transit_ll, uint8_t* in_transit, int32_t* status) {
  return lkb::bls_stats_launch(t, y, dy, offsets, B, period, duration, transit_time, transit_offsets, stats,
                               transit_first, transit_n, per_transit_count, per_transit_ll, in_transit, status,
                               nullptr);
}

}  // extern "C"
