// Runs K15 (lightkurve_b200/csrc/gapfill.cuh: gap_steps_kernel, gap_plan_kernel, gap_fill_kernel) on the CPU through
// tests/native/cuda_emu.h (TEST INFRASTRUCTURE).  Built with -ffp-contract=off, as gapfill.cu is built with
// -fmad=false, by tests/test_gapfill_emulated.py.  The median step (K6 on the GPU) is given by the caller.
#include "cuda_emu.h"

#include <vector>

#include "../../lightkurve_b200/csrc/gapfill.cuh"

namespace lkb {
int64_t g_launches = 0;
int g_last_ls_algo = -1;
int64_t g_epoch = 0;
void set_error(const char*, ...) {}
}  // namespace lkb

extern "C" {

// steps [doff[B]], flags [B]
void emu_gap_steps(const double* t, const int64_t* off, const int64_t* doff, int B, double* steps, int32_t* flags) {
  LKB_LAUNCH(B, lkb::GF_THREADS, 0, lkb::gap_steps_kernel)(t, off, doff, steps, flags);
}

void emu_gap_plan(const double* t, const double* y, const int64_t* off, int B, const double* dt, int64_t* n_ins,
                  double* mean, int32_t* flags) {
  LKB_LAUNCH(B, lkb::GF_THREADS, 0, lkb::gap_plan_kernel)(t, y, off, dt, n_ins, mean, flags);
}

void emu_gap_fill(const double* t, const double* y, const double* e, const int64_t* off, const int64_t* noff, int B,
                  const double* dt, const double* mean, const double* std, const double* z, double* t_out,
                  double* y_out, double* e_out) {
  lkb::FillArgs a{};
  a.t = t;
  a.y = y;
  a.e = e;
  a.off = off;
  a.noff = noff;
  a.dt = dt;
  a.mean = mean;
  a.std = std;
  a.z = z;
  a.t_out = t_out;
  a.y_out = y_out;
  a.e_out = e_out;
  LKB_LAUNCH(B, lkb::GF_THREADS, 0, lkb::gap_fill_kernel)(a);
}

}  // extern "C"
