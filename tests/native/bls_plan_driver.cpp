// C entry points over the K3 launch planner (lightkurve_b200/csrc/bls_plan.h, host-only code) for
// tests/test_bls_plan.py.  Built with g++ by the test; no CUDA involved.
#include "../../lightkurve_b200/csrc/bls_plan.h"

#include <cstring>

using namespace lkb;

static BlsPlan g_plan;
static char g_err[256];

extern "C" {

const char* emu_last_error() { return g_err; }

// Plans light curves [0, B) in one table group.  pofs == NULL: shared grid of P periods.  Returns 0, or -5 on refusal.
int emu_bls_plan(const double* per, const int64_t* pofs, int64_t P, int B, double bin_duration, int oversample,
                 int ghist_bins, int64_t hist_cap, int64_t* n_cta, int64_t* n_launch, int64_t* ghist_bytes) {
  BlsPlanLimits lim;
  lim.ghist_bins = ghist_bins;
  if (hist_cap > 0) lim.hist_cap = (size_t)hist_cap;
  g_plan = BlsPlan();
  g_err[0] = 0;
  if (!bls_plan(per, pofs, P, 0, B, bin_duration, oversample, lim, g_plan, g_err, sizeof g_err)) return -5;
  *n_cta = (int64_t)g_plan.cta.size();
  *n_launch = (int64_t)g_plan.launch.size();
  *ghist_bytes = (int64_t)g_plan.ghist_bytes;
  return 0;
}

// cta: [n_cta, 3] (p, b, n); launch: [n_launch, 6] (cta_begin, cta_end, W, stride, ghist, smem)
void emu_bls_plan_get(int64_t* cta, int64_t* launch) {
  for (size_t i = 0; i < g_plan.cta.size(); ++i) {
    cta[3 * i] = g_plan.cta[i].p;
    cta[3 * i + 1] = g_plan.cta[i].b;
    cta[3 * i + 2] = g_plan.cta[i].n;
  }
  for (size_t i = 0; i < g_plan.launch.size(); ++i) {
    const BlsLaunch& l = g_plan.launch[i];
    int64_t* o = launch + 6 * i;
    o[0] = l.cta_begin; o[1] = l.cta_end; o[2] = l.W; o[3] = l.stride; o[4] = l.ghist; o[5] = (int64_t)l.smem;
  }
}

// groups: [B, 3] (b0, b1, table) of which the first return-value rows are set; to: [B + 1]
int emu_bls_table_groups(const int64_t* n, const double* x_max, int B, double inv_delta, int enabled, int shared,
                         int64_t budget, int64_t* groups, int64_t* to) {
  std::vector<int64_t> h_to;
  const std::vector<BlsTableGroup> g = bls_table_groups(n, x_max, B, inv_delta, enabled != 0, shared != 0, budget, h_to);
  for (size_t i = 0; i < g.size(); ++i) {
    groups[3 * i] = g[i].b0;
    groups[3 * i + 1] = g[i].b1;
    groups[3 * i + 2] = g[i].table ? 1 : 0;
  }
  memcpy(to, h_to.data(), sizeof(int64_t) * (B + 1));
  return (int)g.size();
}

}
