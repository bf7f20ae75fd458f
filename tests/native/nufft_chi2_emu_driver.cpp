// The multi-term (nterms 1..4) NUFFT Lomb-Scargle path of lightkurve_b200/csrc/ls_nufft.cu on the CPU through
// tests/native/cuda_emu.h (TEST INFRASTRUCTURE): the single-term driver (its workspace / error stubs and wrappers) plus
// one wrapper around ls_nufft_chi2_ragged_launch.  Built by tests/test_nufft_chi2_emulated.py.
#include "nufft_emu_driver.cpp"

extern "C" {

// ragged batch in the K1 prologue's layout (padded CSR): t/y [ptotal], off/poff [B+1], span/ysum [B]; power [B, F]
int emu_nufft_chi2_ragged(const double* t, const float* y, const int64_t* off, const int64_t* poff, int B,
                          int64_t ptotal, int64_t nmax, const double* span, const double* ysum, int64_t F, double f0,
                          double df, int normalization, const double* norm_scale, float* power, int nterms) {
  return lkb::ls_nufft_chi2_ragged_launch(t, y, off, poff, off, B, ptotal, nmax, span, span, ysum, F, f0, df,
                                          normalization, norm_scale, power, nullptr, nterms);
}

}  // extern "C"
