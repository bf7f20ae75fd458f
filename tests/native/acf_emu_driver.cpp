// Runs the K7 windowed-autocorrelation kernels and their launcher (lightkurve_b200/csrc/acf.cuh) on the CPU through
// tests/native/cuda_emu.h (TEST INFRASTRUCTURE).  Built by tests/test_acf_emulated.py.
#include "cuda_emu.h"

#include <stdarg.h>
#include <stdio.h>

#include <map>

#include "../../lightkurve_b200/csrc/acf.cuh"

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
int big_copy_h2d(void* d, const void* s, size_t n, cudaStream_t) { memcpy(d, s, n); return LKB_OK; }
int big_copy_d2h(void* d, const void* s, size_t n, cudaStream_t) { memcpy(d, s, n); return LKB_OK; }
}  // namespace lkb

extern "C" {

const char* emu_last_error() { return lkb::g_err; }
int64_t emu_launches() { return lkb::g_launches; }

// the lkb_acf_windows contract; `mem` 0 stages through the (emulated) workspace, 1 passes the pointers through
int emu_acf_windows(const double* x, const int64_t* x_offsets, int B, const int64_t* win_offsets,
                    const int64_t* win_start, const int64_t* win_len, double* metric, double* acf, int mem) {
  return lkb::acf_windows_launch(x, x_offsets, B, win_offsets, win_start, win_len, metric, acf, mem, nullptr);
}

}  // extern "C"
