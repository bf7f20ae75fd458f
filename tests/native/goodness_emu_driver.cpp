// Runs the K9 goodness-metric kernels (lightkurve_b200/csrc/goodness.cuh) on the CPU through tests/native/cuda_emu.h
// (TEST INFRASTRUCTURE).  Built by tests/test_goodness_emulated.py.
#include "cuda_emu.h"

#include <stdarg.h>
#include <stdio.h>

#include <vector>

#include "../../lightkurve_b200/csrc/goodness.cuh"

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

// gm_underfit_launch on host buffers
int emu_underfit(const double* pool, int P, const double* target, int B, int64_t G, const int64_t* nb_off,
                 const int32_t* nb_idx, double* metric, int32_t* n_used, double* c3_mean) {
  const int64_t W = lkb::gm_words(G);
  std::vector<uint32_t> pb((size_t)P * W), tb((size_t)B * W);
  return lkb::gm_underfit_launch(pool, P, target, B, G, nb_off, nb_idx, nb_off, pb.data(), tb.data(), metric, n_used,
                                 c3_mean, nullptr);
}

// gm_overfit_launch on host buffers (offsets [B + 1] required)
int emu_overfit(const float* corrected, const float* original, const float* noise, const int64_t* offsets, int B,
                int S, int32_t* n_positive, double* sum_positive, double* noise_mean) {
  return lkb::gm_overfit_launch(corrected, original, noise, offsets, B, S, n_positive, sum_positive, noise_mean,
                                nullptr);
}

}  // extern "C"
