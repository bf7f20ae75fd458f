// Runs K13 (lightkurve_b200/csrc/foldbin.cuh: fold_kernel, bin_kernel) on the CPU through tests/native/cuda_emu.h
// (TEST INFRASTRUCTURE).  Built with -ffp-contract=off, as foldbin.cu is built with -fmad=false, by
// tests/test_fold_bin_emulated.py.
#include "cuda_emu.h"

#include <vector>

#include "../../lightkurve_b200/csrc/foldbin.cuh"

namespace lkb {
int64_t g_launches = 0;
int g_last_ls_algo = -1;
int64_t g_epoch = 0;
void set_error(const char*, ...) {}
}  // namespace lkb

extern "C" {

// One fold launch on B light curves, planned as foldbin.cu plans it, except that light curves longer than `res_cap`
// (< 0: the library's FB_FOLD_CAP) sort in global memory.  par: [4 B] t0, shift, period, wrap.  Returns 1 when some
// light curve sorted in global memory.
int emu_fold(const double* t, const int64_t* off, int B, const double* par, int normalize, double* phase,
             int32_t* perm, int64_t res_cap) {
  std::vector<int64_t> woff(B);
  const lkb::FbPlan p = lkb::fb_plan(off, B, res_cap < 0 ? lkb::FB_FOLD_CAP : res_cap, lkb::FB_FOLD_BPC, woff.data());
  std::vector<uint64_t> work(3 * (size_t)p.work_cadences + 1);
  lkb::FoldArgs a{};
  a.t = t;
  a.off = off;
  a.par = par;
  a.normalize = normalize;
  a.phase = phase;
  a.perm = perm;
  a.work = work.data();
  a.woff = woff.data();
  a.res_cap = p.res_cap;
  LKB_LAUNCH_SMEM(B, lkb::FB_THREADS, p.smem, 0, lkb::fold_kernel)(a);
  return p.work_cadences > 0 ? 1 : 0;
}

// One bin launch; edges as times (starts, ends) or as indices (sidx, eidx).  status [B] gets each light curve's
// FbStatus.  Returns 1 when some light curve sorted in global memory.
int emu_bin(const double* t, const double* f, const double* fe, const int64_t* off, int B, const int64_t* boff,
            const double* starts, const double* ends, const int32_t* sidx, const int32_t* eidx, int agg,
            double* centre, double* flux, double* err, int32_t* count, int32_t* status, int64_t res_cap) {
  std::vector<int64_t> woff(B);
  const lkb::FbPlan p = lkb::fb_plan(off, B, res_cap < 0 ? lkb::FB_BIN_CAP : res_cap, lkb::FB_BIN_BPC, woff.data());
  std::vector<uint64_t> work(4 * (size_t)p.work_cadences + 1);
  std::vector<int32_t> blo((size_t)boff[B] + 1);
  lkb::BinArgs a{};
  a.t = t;
  a.f = f;
  a.fe = fe;
  a.off = off;
  a.boff = boff;
  a.starts = starts;
  a.ends = ends;
  a.sidx = sidx;
  a.eidx = eidx;
  a.agg = agg;
  a.centre = centre;
  a.flux = flux;
  a.err = err;
  a.count = count;
  a.blo = blo.data();
  a.status = status;
  a.work = work.data();
  a.woff = woff.data();
  a.res_cap = p.res_cap;
  LKB_LAUNCH_SMEM(B, lkb::FB_THREADS, p.smem, 0, lkb::bin_kernel)(a);
  return p.work_cadences > 0 ? 1 : 0;
}

int emu_fold_cap(void) { return (int)lkb::FB_FOLD_CAP; }
int emu_bin_cap(void) { return (int)lkb::FB_BIN_CAP; }

}  // extern "C"
