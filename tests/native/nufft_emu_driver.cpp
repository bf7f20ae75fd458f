// Runs lightkurve_b200/csrc/ls_nufft.cu - the WHOLE translation unit: kernels, launch shapes, workspace use,
// orchestration - on the CPU through tests/native/cuda_emu.h (TEST INFRASTRUCTURE).  Built by
// tests/test_nufft_emulated.py:  g++ -std=c++17 -O1 -pthread -I/usr/local/cuda/include -shared -fPIC ...
#include "cuda_emu.h"

#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <map>

#include "../../lightkurve_b200/csrc/ls_nufft.cu"

// ---- the pieces of api.cu the translation unit links against ----
namespace lkb {
int64_t g_launches = 0;
static char g_err[512];
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
static std::map<int, std::pair<void*, size_t>> g_ws;
int ws_get(int slot, size_t bytes, void** out) {
  auto& e = g_ws[slot];
  if (e.second != bytes) {             // exact size, no slack: an out-of-bounds access is visible to ASan
    free(e.first);
    e.first = calloc(bytes ? bytes : 1, 1);
    e.second = bytes;
  }
  *out = e.first;
  return LKB_OK;
}
int ensure_device() { return LKB_OK; }
void prof_begin(cudaStream_t) {}
void prof_end(cudaStream_t) {}
}  // namespace lkb

extern "C" {

const char* emu_last_error() { return lkb::g_err; }
int emu_last_escalated() { return lkb::ls_nufft_last_escalated(); }
void emu_last_nufft_plan(int* out3) { lkb::ls_nufft_last_plan(out3); }

// diagnostic: copy of a workspace slot as the last call left it (returns the slot's size in bytes)
int64_t emu_ws_read(int slot, void* dst, int64_t bytes) {
  auto it = lkb::g_ws.find(slot);
  if (it == lkb::g_ws.end()) return -1;
  if (dst && bytes > 0) memcpy(dst, it->second.first, (size_t)std::min<int64_t>(bytes, (int64_t)it->second.second));
  return (int64_t)it->second.second;
}

// shared cadence grid: t_rel [N] (ascending, t_rel[0] = 0), yc [B, ystride] centred fp32, ysum/absmax [B],
// rot/rot2 [F] (rows < F_low pre-filled by the caller), power [B, F] out
int emu_nufft_shared(const double* t_rel, int64_t N, const float* yc, int64_t ystride, const float* ysum,
                     const float* absmax, int B, const double* freq, int64_t F, double f0, double df, float* rot,
                     float* rot2, int64_t F_low, int normalization, double norm_scale, float* power) {
  return lkb::ls_nufft_launch(t_rel, N, yc, ystride, ysum, absmax, B, freq, F, f0, df, reinterpret_cast<float4*>(rot),
                              reinterpret_cast<float2*>(rot2), F_low, normalization, norm_scale, power, nullptr);
}

// the chunked form used by the pipelined host-mode loop: prepare once, then run blocks of light curves
int emu_nufft_shared_chunked(const double* t_rel, int64_t N, const float* yc, int64_t ystride, const float* ysum,
                             const float* absmax, int B, const double* freq, int64_t F, double f0, double df,
                             float* rot, float* rot2, int64_t F_low, int normalization, double norm_scale,
                             float* power, int chunk) {
  int rc = lkb::ls_nufft_prepare(t_rel, N, F, f0, df, reinterpret_cast<float4*>(rot), reinterpret_cast<float2*>(rot2),
                                 F_low, nullptr, freq, ystride);
  for (int b0 = 0, c = 0; rc == LKB_OK && b0 < B; b0 += chunk, ++c) {
    const int nb = std::min(chunk, B - b0);
    rc = lkb::ls_nufft_run(t_rel, N, yc + (size_t)b0 * ystride, ystride, ysum + b0, absmax + b0, nb, freq, F,
                           reinterpret_cast<const float4*>(rot), reinterpret_cast<const float2*>(rot2), F_low,
                           normalization, norm_scale, power + (size_t)b0 * F, nullptr, c & 1, true);
  }
  return rc;
}

// ragged batch in the K1 prologue's layout (padded CSR): t/y [ptotal], off/poff [B+1], span/ysum [B]
int emu_nufft_ragged(const double* t, const float* y, const int64_t* off, const int64_t* poff, int B, int64_t ptotal,
                     int64_t nmax, const double* span, const double* ysum, int64_t F, double f0, double df,
                     int normalization, const double* norm_scale, float* power) {
  return lkb::ls_nufft_ragged_launch(t, y, off, poff, off, B, ptotal, nmax, span, span, ysum, F, f0, df, normalization,
                                     norm_scale, power, nullptr);
}

}  // extern "C"
