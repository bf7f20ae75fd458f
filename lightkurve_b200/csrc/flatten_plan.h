// K4 path and tile planning, host only (no CUDA): flatten.cu picks its kernel here, and
// tests/native/flatten_emu_driver.cpp runs the v2 kernel with the same plan on the CPU.
//
// v2 (flatten_v2.cuh) filters the interior of a segment tile by tile: a tile holds tile_out outputs and the
// 2 * half inputs around them in NM shared-memory arrays (NM = 1, 3 or 5 for polyorder 0-1, 2-3, 4-5).  Each
// output is either
//   * a difference of prefix sums of (q - qc)^s x_q, s < NM, re-centred on the output by binomial expansion
//     ("moments", O(1) per output).  The prefix sums round like eps * T (T = tile_out + 2 * half inputs); the
//     re-centring multiplies that by (T / 2 half)^(NM - 1) against the size of the centred sum, so the relative
//     error of an output is about eps * T * (T / 2 half)^(NM - 1);
//   * or the dot product of the 2 * half + 1 centre taps with the inputs ("direct", O(window) per output, no
//     cancellation),
// whichever keeps that bound within F2_MOMENT_TOL.  NM = 1 (a plain windowed sum) always takes moments.
// v1 (flatten.cu's FIR kernel) runs when v2 cannot: polyorder > 5, a tile of fewer than 128 outputs (long windows),
// or a light curve longer than F2_MAXN cadences (then the whole batch runs on v1).
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>

namespace lkb {

constexpr int F2_MAXN = 131072;                 // cadences per light curve the v2 bitmask holds
constexpr double F2_MOMENT_TOL = 2e-10;         // largest predicted relative error of a moment-based output

// why a call runs on v1 (FLATTEN_V1_*), or FLATTEN_V2
enum FlattenRoute { FLATTEN_V2 = 0, FLATTEN_V1_POLYORDER = 1, FLATTEN_V1_TILE = 2, FLATTEN_V1_LENGTH = 3 };

struct FlattenPlan {
  int route;      // FlattenRoute
  int nm;         // prefix-sum arrays of the v2 kernel (shared memory: nm * (tile_out + 2 * half + 1) doubles)
  int tile_out;   // outputs per v2 tile
  bool direct;    // v2 interior by direct taps instead of moments
};

// Relative rounding error predicted for a moment-based output (see above).
inline double flatten_moment_error(int nm, int tile_out, int half) {
  const double eps = 2.220446049250313e-16, T = (double)tile_out + 2.0 * half;
  return nm == 1 ? eps * T : eps * T * std::pow(T / (2.0 * half), nm - 1);
}

// window_length odd in [1, 8191], polyorder in [0, min(window_length - 1, 12)], nmax = longest light curve.
inline FlattenPlan flatten_plan(int window_length, int polyorder, int64_t nmax) {
  const int half = window_length / 2;
  FlattenPlan pl;
  pl.nm = polyorder <= 1 ? 1 : polyorder <= 3 ? 3 : 5;
  // shared memory: nm arrays of tile_out + 2 half + 1 doubles within 64 KiB
  pl.tile_out = std::min(2048, std::min(65536 / (8 * pl.nm) - 2 * half - 1, 4094 - 2 * half));
  // fourth-order moments: short tiles keep (T / 2 half)^4 small
  if (pl.nm == 5) pl.tile_out = std::min(pl.tile_out, std::max(128, 10 * half));
  pl.route = polyorder > 5 ? FLATTEN_V1_POLYORDER
             : pl.tile_out < 128 ? FLATTEN_V1_TILE
             : nmax > F2_MAXN ? FLATTEN_V1_LENGTH
             : FLATTEN_V2;
  pl.direct = pl.nm > 1 && flatten_moment_error(pl.nm, pl.tile_out, half) > F2_MOMENT_TOL;
  return pl;
}

}  // namespace lkb
