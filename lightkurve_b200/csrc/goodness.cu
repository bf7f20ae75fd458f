// K9 C entries: lkb_underfit_metric and lkb_overfit_terms (kernels in goodness.cuh).
#include "goodness.cuh"

#include <vector>

namespace lkb {

int underfit_metric(const double* pool, int P, const double* target, int B, int64_t G, const int64_t* h_nb_off,
                    const int32_t* h_nb_idx, double* metric, int32_t* n_used, double* c3_mean, int mem,
                    cudaStream_t st) {
  LKB_REQUIRE(pool && target && h_nb_off && h_nb_idx && metric, "lkb_underfit_metric: null argument");
  LKB_REQUIRE(P > 0 && P <= 65535 && B > 0 && B <= 65535 && G > 0, "lkb_underfit_metric: bad sizes");
  LKB_REQUIRE(h_nb_off[0] == 0, "lkb_underfit_metric: nb_offsets[0] must be 0");
  for (int b = 0; b < B; ++b)
    if (h_nb_off[b + 1] < h_nb_off[b]) {
      set_error("lkb_underfit_metric: nb_offsets not monotone at target %d", b);
      return LKB_E_ARG;
    }
  const int64_t nnb = h_nb_off[B];
  for (int64_t k = 0; k < nnb; ++k)
    if (h_nb_idx[k] < 0 || h_nb_idx[k] >= P) {
      set_error("lkb_underfit_metric: neighbour index %d outside the pool of %d", h_nb_idx[k], P);
      return LKB_E_ARG;
    }
  LKB_TRY(ensure_device());
  const int64_t W = gm_words(G);
  const double *d_pool = nullptr, *d_t = nullptr;
  LKB_TRY(stage_in<double>(mem, WS_IN0, pool, (size_t)P * G, &d_pool, st));
  LKB_TRY(stage_in<double>(mem, WS_IN1, target, (size_t)B * G, &d_t, st));
  int64_t* d_off = nullptr;
  int32_t* d_idx = nullptr;
  uint32_t *d_pb = nullptr, *d_tb = nullptr;
  LKB_TRY(ws_get_t<int64_t>(WS_A, (size_t)B + 1, &d_off));
  LKB_TRY(ws_get_t<int32_t>(WS_B, nnb ? (size_t)nnb : 1, &d_idx));
  LKB_TRY(ws_get_t<uint32_t>(WS_C, (size_t)P * W, &d_pb));
  LKB_TRY(ws_get_t<uint32_t>(WS_D, (size_t)B * W, &d_tb));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_off, h_nb_off, sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  if (nnb) LKB_CUDA_CHECK(cudaMemcpyAsync(d_idx, h_nb_idx, sizeof(int32_t) * nnb, cudaMemcpyHostToDevice, st));
  double *o_m = nullptr, *o_c3 = nullptr;
  int32_t* o_n = nullptr;
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT0, metric, B, &o_m));
  LKB_TRY(stage_out_alloc<int32_t>(mem, WS_OUT1, n_used, B, &o_n));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT2, c3_mean, B, &o_c3));
  prof_begin(st);
  LKB_TRY(gm_underfit_launch(d_pool, P, d_t, B, G, d_off, d_idx, h_nb_off, d_pb, d_tb, o_m, o_n, o_c3, st));
  prof_end(st);
  LKB_TRY(stage_out_copy<double>(mem, metric, o_m, B, st));
  LKB_TRY(stage_out_copy<int32_t>(mem, n_used, o_n, B, st));
  LKB_TRY(stage_out_copy<double>(mem, c3_mean, o_c3, B, st));
  // the host offset / index arrays are read by the copies above: wait for them before returning (device mode too)
  LKB_CUDA_CHECK(cudaStreamSynchronize(st));
  return LKB_OK;
}

int overfit_terms(const float* corrected, const float* original, const float* noise, const int64_t* h_offsets, int B,
                  int64_t F, int S, int32_t* n_positive, double* sum_positive, double* noise_mean, int mem,
                  cudaStream_t st) {
  LKB_REQUIRE(corrected && original && n_positive && sum_positive, "lkb_overfit_terms: null argument");
  LKB_REQUIRE(B > 0 && B <= 2147483647 && S >= 0 && S < 65535, "lkb_overfit_terms: bad sizes");
  LKB_REQUIRE(S == 0 || (noise && noise_mean), "lkb_overfit_terms: noise rows need `noise` and `noise_mean`");
  std::vector<int64_t> off((size_t)B + 1);
  if (h_offsets) {
    LKB_REQUIRE(h_offsets[0] == 0, "lkb_overfit_terms: offsets[0] must be 0");
    for (int b = 0; b <= B; ++b) {
      if (b && h_offsets[b] < h_offsets[b - 1]) {
        set_error("lkb_overfit_terms: offsets not monotone at light curve %d", b - 1);
        return LKB_E_ARG;
      }
      off[b] = h_offsets[b];
    }
  } else {
    LKB_REQUIRE(F > 0, "lkb_overfit_terms: F must be > 0 without offsets");
    for (int b = 0; b <= B; ++b) off[b] = (int64_t)b * F;
  }
  const int64_t tot = off[B];
  LKB_TRY(ensure_device());
  const float *d_c = nullptr, *d_o = nullptr, *d_n = nullptr;
  LKB_TRY(stage_in<float>(mem, WS_IN0, corrected, (size_t)tot, &d_c, st));
  LKB_TRY(stage_in<float>(mem, WS_IN1, original, (size_t)tot, &d_o, st));
  LKB_TRY(stage_in<float>(mem, WS_IN2, S ? noise : nullptr, (size_t)tot * S, &d_n, st));
  int64_t* d_off = nullptr;
  LKB_TRY(ws_get_t<int64_t>(WS_A, (size_t)B + 1, &d_off));
  LKB_CUDA_CHECK(cudaMemcpyAsync(d_off, off.data(), sizeof(int64_t) * (B + 1), cudaMemcpyHostToDevice, st));
  int32_t* o_np = nullptr;
  double *o_sp = nullptr, *o_nm = nullptr;
  LKB_TRY(stage_out_alloc<int32_t>(mem, WS_OUT0, n_positive, B, &o_np));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT1, sum_positive, B, &o_sp));
  LKB_TRY(stage_out_alloc<double>(mem, WS_OUT2, S ? noise_mean : nullptr, (size_t)B * S, &o_nm));
  prof_begin(st);
  LKB_TRY(gm_overfit_launch(d_c, d_o, d_n, d_off, B, S, o_np, o_sp, o_nm, st));
  prof_end(st);
  LKB_TRY(stage_out_copy<int32_t>(mem, n_positive, o_np, B, st));
  LKB_TRY(stage_out_copy<double>(mem, sum_positive, o_sp, B, st));
  LKB_TRY(stage_out_copy<double>(mem, S ? noise_mean : nullptr, o_nm, (size_t)B * S, st));
  LKB_CUDA_CHECK(cudaStreamSynchronize(st));               // `off` lives on this stack frame
  return LKB_OK;
}

}  // namespace lkb
