// Entries of K13 (lkb_fold, lkb_bin); the kernels are in foldbin.cuh.  Compiled with -fmad=false: the phase, the bin
// edges read from the time-sorted cadences and the bin centres round as numpy's separate operations do.
#include <vector>

#include "foldbin.cuh"

namespace lkb {

static int fb_check_offsets(const int64_t* h_off, int B, const char* who) {
  if (h_off[0] != 0) { set_error("%s: offsets[0] must be 0", who); return LKB_E_ARG; }
  for (int b = 0; b < B; ++b)
    if (h_off[b + 1] < h_off[b] || h_off[b + 1] - h_off[b] >= ((int64_t)1 << 31)) {
      set_error("%s: light curve %d has a negative or too large length", who, b);
      return LKB_E_ARG;
    }
  return LKB_OK;
}

// Device copies of the CSR offsets and the workspace offsets, and the global sort buffers of a launch.
static int fb_stage_plan(const int64_t* h_off, int B, const std::vector<int64_t>& woff, int64_t work_u64,
                         const int64_t** d_off, const int64_t** d_woff, uint64_t** d_work, cudaStream_t st) {
  int64_t* o = nullptr;
  LKB_TRY(ws_get_t<int64_t>(WS_X0, 2 * (size_t)B + 1, &o));
  LKB_CUDA_CHECK(cudaMemcpyAsync(o, h_off, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  LKB_CUDA_CHECK(cudaMemcpyAsync(o + B + 1, woff.data(), sizeof(int64_t) * B, cudaMemcpyHostToDevice, st));
  *d_off = o;
  *d_woff = o + B + 1;
  *d_work = nullptr;
  if (work_u64) LKB_TRY(ws_get_t<uint64_t>(WS_X1, (size_t)work_u64, d_work));
  return LKB_OK;
}

int fold(const double* t, const int64_t* h_off, int B, const double* t0, const double* shift, const double* period,
         const double* wrap, int normalize, double* phase_out, int32_t* perm_out, int mem, cudaStream_t st) {
  LKB_REQUIRE(t && h_off && t0 && shift && period && wrap && phase_out && perm_out && B > 0,
              "lkb_fold: null/empty argument");
  LKB_TRY(fb_check_offsets(h_off, B, "lkb_fold"));
  for (int b = 0; b < B; ++b)
    if (!(period[b] > 0.0)) { set_error("lkb_fold: light curve %d has a non-positive period", b); return LKB_E_ARG; }
  LKB_TRY(ensure_device());
  const int64_t total = h_off[B];
  std::vector<int64_t> woff(B);
  const FbPlan p = fb_plan(h_off, B, FB_FOLD_CAP, FB_FOLD_BPC, woff.data());
  std::vector<double> par(4 * (size_t)B);
  for (int b = 0; b < B; ++b) {
    par[4 * b] = t0[b];
    par[4 * b + 1] = shift[b];
    par[4 * b + 2] = period[b];
    par[4 * b + 3] = wrap[b];
  }
  FoldArgs a{};
  LKB_TRY(fb_stage_plan(h_off, B, woff, 3 * p.work_cadences, &a.off, &a.woff, &a.work, st));
  double* d_par = nullptr;
  LKB_TRY(ws_get_t<double>(WS_X2, par.size(), &d_par));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_par, par.data(), sizeof(double) * par.size(), cudaMemcpyHostToDevice, st));
  a.par = d_par;
  LKB_TRY(stage_in<double>(mem, WS_IN0, t, total, &a.t, st));
  a.normalize = normalize ? 1 : 0;
  a.res_cap = p.res_cap;
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0, phase_out, total, &a.phase));
  LKB_TRY(stage_out_alloc<int32_t>(mem, WS_OUT1, perm_out, total, &a.perm));
  static size_t attr = 0;
  if (p.smem > attr) {
    LKB_CUDA_CHECK(cudaFuncSetAttribute(fold_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
    attr = p.smem;
  }
  prof_begin(st);
  fold_kernel<<<B, FB_THREADS, p.smem, st>>>(a);
  prof_end(st);
  LKB_LAUNCH_CHECK();
  LKB_TRY(stage_out_copy<double>(mem, phase_out, a.phase, total, st));
  LKB_TRY(stage_out_copy<int32_t>(mem, perm_out, a.perm, total, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

int bin(const double* t, const double* f, const double* fe, const int64_t* h_off, int B, const int64_t* h_boff,
        const double* starts, const double* ends, const int32_t* sidx, const int32_t* eidx, int agg,
        double* centre_out, double* flux_out, double* err_out, int32_t* count_out, int mem, cudaStream_t st) {
  LKB_REQUIRE(t && f && h_off && h_boff && centre_out && flux_out && err_out && count_out && B > 0,
              "lkb_bin: null/empty argument");
  LKB_REQUIRE((starts && ends && !sidx && !eidx) || (!starts && !ends && sidx && eidx),
              "lkb_bin: give the bin edges either as times (starts, ends) or as indices (sidx, eidx)");
  LKB_REQUIRE(agg == LKB_BIN_NANMEAN || agg == LKB_BIN_NANMEDIAN, "lkb_bin: unknown aggregate");
  LKB_TRY(fb_check_offsets(h_off, B, "lkb_bin"));
  if (h_boff[0] != 0) { set_error("lkb_bin: bin_offsets[0] must be 0"); return LKB_E_ARG; }
  for (int b = 0; b < B; ++b)
    if (h_boff[b + 1] < h_boff[b] || h_boff[b + 1] - h_boff[b] >= ((int64_t)1 << 31)) {
      set_error("lkb_bin: light curve %d has a negative or too large number of bins", b);
      return LKB_E_ARG;
    }
  LKB_TRY(ensure_device());
  const int64_t total = h_off[B], nbins = h_boff[B];
  std::vector<int64_t> woff(B);
  const FbPlan p = fb_plan(h_off, B, FB_BIN_CAP, FB_BIN_BPC, woff.data());
  BinArgs a{};
  LKB_TRY(fb_stage_plan(h_off, B, woff, 4 * p.work_cadences, &a.off, &a.woff, &a.work, st));
  int64_t* d_boff = nullptr;
  LKB_TRY(ws_get_t<int64_t>(WS_X2, B + 1, &d_boff));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_boff, h_boff, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  a.boff = d_boff;
  LKB_TRY(stage_in<double>(mem, WS_IN0, t, total, &a.t, st));
  LKB_TRY(stage_in<double>(mem, WS_IN1, f, total, &a.f, st));
  LKB_TRY(stage_in<double>(mem, WS_IN2, fe, total, &a.fe, st));
  LKB_TRY(stage_in<double>(mem, WS_IN3, starts, nbins, &a.starts, st));
  LKB_TRY(stage_in<double>(mem, WS_IN4, ends, nbins, &a.ends, st));
  LKB_TRY(stage_in<int32_t>(mem, WS_IN5, sidx, nbins, &a.sidx, st));
  LKB_TRY(stage_in<int32_t>(mem, WS_IN6, eidx, nbins, &a.eidx, st));
  a.agg = agg == LKB_BIN_NANMEDIAN ? FB_NANMEDIAN : FB_NANMEAN;
  a.res_cap = p.res_cap;
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0, centre_out, nbins, &a.centre));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT1, flux_out, nbins, &a.flux));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT2, err_out, nbins, &a.err));
  LKB_TRY(stage_out_alloc<int32_t>(mem, WS_OUT3, count_out, nbins, &a.count));
  LKB_TRY(ws_get_t<int32_t>(WS_X3, nbins ? (size_t)nbins : 1, &a.blo));
  LKB_TRY(ws_get_t<int32_t>(WS_X4, B, &a.status));
  static size_t attr = 0;
  if (p.smem > attr) {
    LKB_CUDA_CHECK(cudaFuncSetAttribute(bin_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
    attr = p.smem;
  }
  prof_begin(st);
  bin_kernel<<<B, FB_THREADS, p.smem, st>>>(a);
  prof_end(st);
  LKB_LAUNCH_CHECK();
  std::vector<int32_t> status(B);
  LKB_CUDA_CHECK(cudaMemcpyAsync(status.data(), a.status, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, st));
  LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  for (int b = 0; b < B; ++b) {
    if (status[b] == FB_BAD_INDEX) {
      set_error("lkb_bin: light curve %d has a bin edge index outside its %lld cadences", b,
                (long long)(h_off[b + 1] - h_off[b]));
      return LKB_E_ARG;
    }
    if (status[b] == FB_BAD_STARTS) {
      set_error("lkb_bin: the bin starts of light curve %d do not ascend", b);
      return LKB_E_ARG;
    }
  }
  LKB_TRY(stage_out_copy<double>(mem, centre_out, a.centre, nbins, st));
  LKB_TRY(stage_out_copy<double>(mem, flux_out, a.flux, nbins, st));
  LKB_TRY(stage_out_copy<double>(mem, err_out, a.err, nbins, st));
  LKB_TRY(stage_out_copy<int32_t>(mem, count_out, a.count, nbins, st));
  if (mem == LKB_MEM_HOST) LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

}  // namespace lkb
