// Runs the K5 sigma clip and final model (lightkurve_b200/csrc/regress_clip.cuh: rg_clip_kernel, rg_final_kernel) on
// the CPU through tests/native/cuda_emu.h (TEST INFRASTRUCTURE).  Built by tests/test_regress_clip_emulated.py.
#include "cuda_emu.h"

#include <vector>

#include "../../lightkurve_b200/csrc/regress_clip.cuh"

namespace lkb {
int64_t g_launches = 0;
int g_last_ls_algo = -1;
int64_t g_epoch = 0;
void set_error(const char*, ...) {}
}  // namespace lkb

extern "C" {

// One clip of B light curves, then the final model, as regress() launches them (512 threads, the same dynamic shared
// memory).  used [B, N]: the cadences inside the fit.  model_ready = 1: the kernels take X w from xw [B, N] (regress()
// has it from rg_model_mma_kernel); 0: they compute it from X (shared [N, K] or, x_batched, [B, N, K]) and coeff.
// outlier [B, N] starts zeroed, as in regress().
int emu_clip_final(const double* X, int x_batched, const double* y, const uint8_t* used, int B, int64_t N, int K,
                   const double* coeff, double clip_sigma, int model_ready, const double* xw, uint8_t* outlier,
                   double* model) {
  std::vector<double> resid((size_t)B * N, 0.0);
  std::vector<uint8_t> used_ws(used, used + (size_t)B * N);
  lkb::RgWs ws{};
  ws.used = used_ws.data();
  ws.resid = resid.data();
  if (model_ready) {
    memcpy(resid.data(), xw, sizeof(double) * (size_t)B * N);
    memcpy(model, xw, sizeof(double) * (size_t)B * N);
  }
  memset(outlier, 0, (size_t)B * N);
  const size_t clip_smem = sizeof(double) * (size_t)((K + 1) & ~1) + sizeof(lkb::FastSelSmem) +
                           sizeof(double) * (size_t)(lkb::FS_CAP + lkb::FS_SAMPLE);
  LKB_LAUNCH_SMEM(B, 512, clip_smem, 0, lkb::rg_clip_kernel)(X, x_batched, y, N, K, coeff, clip_sigma, ws, outlier,
                                                             model_ready);
  LKB_LAUNCH_SMEM(B, 512, K * sizeof(double), 0, lkb::rg_final_kernel)(X, x_batched, N, K, coeff, model, model_ready);
  return 0;
}

}  // extern "C"
