// Runs the K4 v2 kernel (lightkurve_b200/csrc/flatten_v2.cuh) on the CPU through tests/native/cuda_emu.h
// (TEST INFRASTRUCTURE).  Built by tests/test_flatten_emulated.py.
#include "cuda_emu.h"

#include <stdarg.h>
#include <stdio.h>

#include <algorithm>
#include <vector>

#include "../../lightkurve_b200/csrc/flatten_v2.cuh"
#include "../../lightkurve_b200/csrc/flatten_plan.h"

namespace lkb {
int64_t g_launches = 0;
int g_last_ls_algo = -1;
int64_t g_epoch = 0;
void set_error(const char*, ...) {}
}  // namespace lkb

extern "C" {
// The plan flatten.cu makes for these shapes (flatten_plan.h): returns the route, writes the tile and the tap mode.
int emu_flatten_plan(int window, int polyorder, int64_t nmax, int* tile_out, int* direct) {
  const lkb::FlattenPlan pl = lkb::flatten_plan(window, polyorder, nmax);
  *tile_out = pl.tile_out;
  *direct = pl.direct ? 1 : 0;
  return pl.route;
}

// one call = flatten of B light curves (CSR offsets); cf_* as computed by the test from numpy (Ginv [q*q], A[3]);
// the tile and the tap mode are flatten.cu's plan unless tile_out > 0 overrides the tile
int emu_flatten2(const double* t, const double* f, const double* fe, const unsigned char* ex, const int64_t* off, int B,
                 int window, int polyorder, double break_tol, int niters, double sigma, const double* A, const double* Ginv,
                 int tile_out, double* flat, double* flat_err, double* trend, int* status) {
  int64_t nmax = 0;
  for (int b = 0; b < B; ++b) nmax = std::max(nmax, off[b + 1] - off[b]);
  const lkb::FlattenPlan pl = lkb::flatten_plan(window, polyorder, nmax);
  if (tile_out <= 0) tile_out = pl.tile_out;
  lkb::F2Coef cf;
  cf.q = polyorder + 1;
  for (int i = 0; i < 3; ++i) cf.A[i] = A[i];
  for (int i = 0; i < lkb::F2_MAXQ * lkb::F2_MAXQ; ++i) cf.Ginv[i] = 0.0;
  for (int i = 0; i < cf.q * cf.q; ++i) cf.Ginv[i] = Ginv[i];
  const int NM = pl.nm;
  const int half = window / 2;
  const size_t smem = ((sizeof(lkb::F2Smem) + 15) & ~(size_t)15) +
                      sizeof(double) * std::max((size_t)NM * (tile_out + 2 * half + 1), (size_t)(lkb::FS_CAP + lkb::FS_SAMPLE));
  std::vector<double> tro((size_t)off[B] + 1, 0.0);
#define EMU_F2(NM_, DIRECT_)                                                                                       \
  LKB_LAUNCH_SMEM(B, lkb::F2_THREADS, smem, 0, lkb::flatten2_kernel<NM_, DIRECT_>)(t, f, fe, ex, off, tro.data(), window, \
                                                                                break_tol, niters, sigma, cf, tile_out, \
                                                                                flat, flat_err, trend, status)
  if (NM == 1) EMU_F2(1, false);
  else if (NM == 3 && pl.direct) EMU_F2(3, true);
  else if (NM == 3) EMU_F2(3, false);
  else if (pl.direct) EMU_F2(5, true);
  else EMU_F2(5, false);
#undef EMU_F2
  return 0;
}
}
