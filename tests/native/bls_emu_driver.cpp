// Runs lightkurve_b200/csrc/bls.cu - the WHOLE translation unit: prologue, lookup tables, launch planning, both
// search paths and both histogram placements - on the CPU through tests/native/cuda_emu.h (TEST INFRASTRUCTURE).
// Built by tests/test_bls_emulated.py with -ffp-contract=off: the library compiles bls.cu with -fmad=false, and its
// bit-exact claims (bin indices, the C code's objective arithmetic) depend on no a*b+c being contracted.
#include "cuda_emu.h"

#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <map>

// which kernel paths the calls since the last emu_bls_reset_paths() took (LKB_BLS_OBSERVE in bls.cu)
static std::atomic<long long> g_bls_paths[16];
static inline void lkb_emu_bls_observe(int path) { g_bls_paths[path].fetch_add(1, std::memory_order_relaxed); }
#define LKB_BLS_OBSERVE(path) lkb_emu_bls_observe(path)

// boundary-path table budget (entries per table group), settable so that small inputs form several groups
static int64_t g_table_budget = (int64_t)1 << 28;
#define BLS_TABLE_BUDGET g_table_budget

#include "../../lightkurve_b200/csrc/bls.cu"

// ---- the pieces of api.cu the translation unit links against ----
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
int big_copy_h2d(void* dst, const void* src, size_t bytes, cudaStream_t) { memcpy(dst, src, bytes); return LKB_OK; }
int big_copy_d2h(void* dst, const void* src, size_t bytes, cudaStream_t) { memcpy(dst, src, bytes); return LKB_OK; }
}  // namespace lkb

extern "C" {

const char* emu_last_error() { return lkb::g_err; }

int emu_bls_path_count() { return lkb::BLS_PATH_COUNT; }
void emu_bls_paths(long long* out) {
  for (int i = 0; i < lkb::BLS_PATH_COUNT; ++i) out[i] = g_bls_paths[i].load();
}
void emu_bls_reset_paths() {
  for (auto& c : g_bls_paths) c.store(0);
}
void emu_bls_set_table_budget(int64_t entries) { g_table_budget = entries; }
int64_t emu_launches() { return lkb::g_launches; }

// lkb_bls_power_ex on host buffers (period_offsets == nullptr: one grid shared by all light curves)
int emu_bls_power(const double* t, const double* y, const double* dy, const int64_t* offsets, int B,
                  const double* period, const int64_t* period_offsets, int64_t P, const double* duration, int D,
                  int oversample, int objective, double* power, double* depth, double* depth_err,
                  double* duration_out, double* transit_time, double* depth_snr, double* log_likelihood,
                  int32_t* best_bins) {
  return lkb::bls_power(t, y, dy, offsets, B, period, period_offsets, P, duration, D, oversample, objective, power,
                        depth, depth_err, duration_out, transit_time, depth_snr, log_likelihood, best_bins,
                        LKB_MEM_HOST, nullptr);
}

int emu_bls_bin_index(const double* t_rel, int64_t N, double min_t, double period, double bin_duration,
                      int32_t* ind) {
  return lkb::bls_bin_index(t_rel, N, min_t, period, bin_duration, ind, LKB_MEM_HOST, nullptr);
}

}  // extern "C"
