// Runs the K8 elastic-net coordinate-descent kernel (lightkurve_b200/csrc/enet.cuh) on the CPU through
// tests/native/cuda_emu.h (TEST INFRASTRUCTURE).  Built by tests/test_enet_emulated.py.
#include "cuda_emu.h"

#include <stdarg.h>
#include <stdio.h>

#include "../../lightkurve_b200/csrc/enet.cuh"

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
int emu_warps_per_cta(int K) { return lkb::enet_warps_per_cta(K); }

// enet_cd_launch on host buffers: gram [B, K+1, K+1] (upper triangle used), cnt [B]
int emu_enet_cd(const double* gram, const int32_t* cnt, int B, int K, double alpha, double l1_ratio, int max_iter,
                double tol, int positive, double* coeff, int32_t* n_iter, double* dual_gap, uint8_t* converged) {
  return lkb::enet_cd_launch(gram, cnt, B, K, alpha, l1_ratio, max_iter, tol, positive, coeff, n_iter, dual_gap,
                             converged, nullptr);
}

}  // extern "C"
