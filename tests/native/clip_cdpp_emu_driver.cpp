// Runs K11/K12 (lightkurve_b200/csrc/clip.cuh: clip_cdpp_kernel) on the CPU through tests/native/cuda_emu.h
// (TEST INFRASTRUCTURE).  Built with -ffp-contract=off, as clip.cu is built with -fmad=false, by
// tests/test_clip_cdpp_emulated.py.
#include "cuda_emu.h"

#include <vector>

#include "../../lightkurve_b200/csrc/clip.cuh"

namespace lkb {
int64_t g_launches = 0;
int g_last_ls_algo = -1;
int64_t g_epoch = 0;
void set_error(const char*, ...) {}
}  // namespace lkb

extern "C" {

// One launch on B light curves, planned as clip.cu plans it, except that light curves longer than `res_cap` (the
// library's is CL_RES_CAP) work in global memory.  dur == NULL: the clip only.  Returns 1 when some light curve
// streamed, 0 when none did.
int emu_clip_cdpp(const double* x, const int64_t* off, int B, double sigma_lower, double sigma_upper, int maxiters,
                  uint8_t* mask, double* center, double* sd, int64_t* n_kept, const int32_t* dur, int D, double* cdpp,
                  int64_t res_cap) {
  const lkb::ClipPlan p = lkb::clip_plan(off, B, res_cap < 0 ? lkb::CL_RES_CAP : res_cap);
  std::vector<double> work(p.streams ? (size_t)off[B] : 0);
  lkb::ClipArgs a{};
  a.x = x;
  a.off = off;
  a.work = work.data();
  a.sigma_lower = sigma_lower;
  a.sigma_upper = sigma_upper;
  a.maxiters = maxiters;
  a.res_cap = p.res_cap;
  a.cand = p.cand;
  a.mask = mask;
  a.center = center;
  a.sd = sd;
  a.n_kept = n_kept;
  a.dur = dur;
  a.D = D;
  a.cdpp = cdpp;
  LKB_LAUNCH_SMEM(B, lkb::CL_THREADS, p.smem, 0, lkb::clip_cdpp_kernel)(a);
  return p.streams ? 1 : 0;
}

int emu_cl_res_cap(void) { return lkb::CL_RES_CAP; }

}  // extern "C"
