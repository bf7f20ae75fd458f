// K3 launch planning, host only (no CUDA): bls.cu plans its search launches here, and
// tests/native/bls_plan_driver.cpp compiles the same code with g++ to test the planner's invariants.
//
// A trial period is one warp; a CTA is W warps on consecutive periods of one light curve.  Each light
// curve's grid is cut into chunks whose bin counts nb = ceil(period / bin_duration) + oversample stay
// within nb_max <= nb_min + nb_min / 4 + 64, so that the warps of a chunk share one histogram stride.
// The chunking, W and the histogram placement of a chunk depend on that light curve's grid alone, so
// every CTA covers exactly the periods a one-light-curve call would give it.  The boundary-path choice
// is CTA-uniform, so this is what keeps a batched result bitwise equal to the one-light-curve result.
//
// Shared grid (pofs == nullptr): one launch per chunk over all light curves (grid order: light curve
// major, CTA minor), global-histogram chunks split into groups of whole light curves by the workspace cap.
// Per-light-curve grids: chunks of all light curves that share (W, placement, stride bucket) form one
// launch; the stride bucket is bls_stride_bucket() for shared-memory histograms (dynamic shared memory
// sized for the bucket's largest stride) and a single bucket per W for global histograms (their stride
// only spaces the workspace slots).  Global-histogram launches are split into groups of CTAs whose slots
// fit the workspace cap.  So the launch count depends on the grids' bin-count range, not on the batch size,
// except where the global-histogram workspace of the batch exceeds the cap.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <map>
#include <tuple>
#include <vector>

namespace lkb {

constexpr int BLS_WARPS = 8;
constexpr int BLS_TILE = 1024;

// One CTA of the search: periods p .. p + n - 1 (indices into the period array) of light curve b.
struct BlsCta {
  int32_t p;
  uint16_t b;
  uint16_t n;
};

struct BlsLaunch {
  int64_t cta_begin, cta_end;   // range of BlsPlan::cta
  int W;                        // warps (periods) per CTA
  int stride;                   // histogram stride in double2 entries
  int ghist;                    // 1: histograms in the global workspace, 0: in shared memory
  size_t smem;                  // dynamic shared memory per CTA
};

struct BlsPlanLimits {
  size_t smem_cap = 200 * 1024;              // largest CTA that keeps its histograms in shared memory
  size_t smem_sm = 227 * 1024;               // shared memory per SM (occupancy rule)
  int ghist_bins = -1;                       // >= 0: global histograms for strides above this (LKB_BLS_GHIST_BINS)
  size_t hist_cap = (size_t)12 << 30;        // global-histogram workspace cap in bytes (LKB_BLS_HIST_CAP_MB)
};

struct BlsPlan {
  std::vector<BlsCta> cta;
  std::vector<BlsLaunch> launch;
  size_t ghist_bytes = 0;                    // global-histogram workspace the largest launch needs
};

// One chunk of one grid: periods [p0, p1) of the period array.
struct BlsChunk {
  int64_t p0, p1;
  int nb_max, stride, W, ghist;
  size_t smem, hist_bytes;
};

inline size_t bls_fixed_smem() { return (size_t)(3 * BLS_TILE + 2 + 2 * BLS_WARPS * 32) * sizeof(double); }

// Chunks of the grid per[p_begin .. p_end).
inline void bls_chunks(const double* per, int64_t p_begin, int64_t p_end, double bin_duration, int oversample,
                       const BlsPlanLimits& lim, std::vector<BlsChunk>& out) {
  const size_t fixed_smem = bls_fixed_smem();
  int64_t p0 = p_begin;
  while (p0 < p_end) {
    int nb_min = (int)std::ceil(per[p0] / bin_duration) + oversample, nb_max = nb_min;
    int64_t p1 = p0 + 1;
    while (p1 < p_end) {
      const int nb = (int)std::ceil(per[p1] / bin_duration) + oversample;
      const int lo = nb < nb_min ? nb : nb_min, hi = nb > nb_max ? nb : nb_max;
      if (hi > lo + lo / 4 + 64) break;
      nb_min = lo; nb_max = hi;
      ++p1;
    }
    BlsChunk c;
    c.p0 = p0;
    c.p1 = p1;
    c.nb_max = nb_max;
    c.stride = ((nb_max + 1 + 3) / 4) * 4;
    // warps (= periods) per CTA: as many as fit with their private histograms in shared memory
    int W = BLS_WARPS;
    while (W > 1 && fixed_smem + (size_t)W * 2 * c.stride * sizeof(double) > lim.smem_cap) W >>= 1;
    size_t smem = fixed_smem + (size_t)W * 2 * c.stride * sizeof(double);
    // Occupancy beats locality here (measured: 108 -> 84 ms on the config-3 probe): once the shared-memory
    // histograms would leave fewer than 4 CTAs (32 warps) per SM, keep them in the L2-resident workspace.
    if (lim.ghist_bins >= 0 ? c.stride > lim.ghist_bins : 4 * (smem + 1024) > lim.smem_sm) smem = lim.smem_cap + 1;
    c.ghist = smem > lim.smem_cap;
    if (c.ghist) {
      W = BLS_WARPS;
      smem = fixed_smem;
    }
    c.W = W;
    c.smem = smem;
    c.hist_bytes = (size_t)W * 2 * c.stride * sizeof(double);
    out.push_back(c);
    p0 = p1;
  }
}

// Stride bucket of a shared-memory chunk: bucket k holds strides in (u_(k-1), u_k], u_0 = 64, u_(k+1) = round4(1.25 u_k).
inline int bls_stride_bucket(int stride) {
  int k = 0;
  for (int64_t u = 64; stride > u; u = ((u + u / 4) + 3) / 4 * 4) ++k;
  return k;
}

// A chunk whose global histograms would not fit the workspace cap for ONE light curve is refused, as a
// one-light-curve call refuses it.
inline bool bls_chunk_fits(const BlsChunk& c, const BlsPlanLimits& lim, char* err, size_t errlen) {
  if (!c.ghist) return true;
  const size_t gx = (size_t)((c.p1 - c.p0 + c.W - 1) / c.W);
  const size_t per_lc = gx * c.hist_bytes;
  if (per_lc <= lim.hist_cap) return true;
  if (err) snprintf(err, errlen, "lkb_bls_power: %d bins per period needs %zu bytes of histogram workspace per light curve",
                    c.nb_max, per_lc);
  return false;
}

// Plans the search of light curves [b0, b1).  pofs == nullptr: every light curve searches per[0 .. P);
// else light curve b searches per[pofs[b] .. pofs[b + 1]).  Appends to `plan`; false (and `err`) on refusal.
inline bool bls_plan(const double* per, const int64_t* pofs, int64_t P, int b0, int b1, double bin_duration,
                     int oversample, const BlsPlanLimits& lim, BlsPlan& plan, char* err, size_t errlen) {
  std::vector<BlsChunk> chunks;
  if (pofs == nullptr) {
    bls_chunks(per, 0, P, bin_duration, oversample, lim, chunks);
    size_t n_cta = plan.cta.size();
    for (const BlsChunk& c : chunks) n_cta += (size_t)(b1 - b0) * (size_t)((c.p1 - c.p0 + c.W - 1) / c.W);
    plan.cta.reserve(n_cta);
    for (const BlsChunk& c : chunks) {
      if (!bls_chunk_fits(c, lim, err, errlen)) return false;
      const int64_t gx = (c.p1 - c.p0 + c.W - 1) / c.W;
      int b_group = b1 - b0;
      if (c.ghist)
        b_group = (int)std::min<size_t>((size_t)(b1 - b0), std::max<size_t>(1, lim.hist_cap / ((size_t)gx * c.hist_bytes)));
      for (int bb = b0; bb < b1; bb += b_group) {
        const int be = std::min(b1, bb + b_group);
        BlsLaunch l;
        l.cta_begin = (int64_t)plan.cta.size();
        for (int b = bb; b < be; ++b)
          for (int64_t x = 0; x < gx; ++x) {
            const int64_t p = c.p0 + x * c.W;
            plan.cta.push_back(BlsCta{(int32_t)p, (uint16_t)b, (uint16_t)std::min<int64_t>(c.W, c.p1 - p)});
          }
        l.cta_end = (int64_t)plan.cta.size();
        l.W = c.W;
        l.stride = c.stride;
        l.ghist = c.ghist;
        l.smem = c.smem;
        if (c.ghist) plan.ghist_bytes = std::max(plan.ghist_bytes, (size_t)(l.cta_end - l.cta_begin) * c.hist_bytes);
        plan.launch.push_back(l);
      }
    }
    return true;
  }
  struct Bucket {
    std::vector<BlsCta> cta;
    int stride = 0;
    size_t smem = 0;
  };
  std::map<std::tuple<int, int, int>, Bucket> buckets;      // (placement, W, stride bucket)
  for (int b = b0; b < b1; ++b) {
    chunks.clear();
    bls_chunks(per, pofs[b], pofs[b + 1], bin_duration, oversample, lim, chunks);
    for (const BlsChunk& c : chunks) {
      if (!bls_chunk_fits(c, lim, err, errlen)) return false;
      Bucket& k = buckets[std::make_tuple(c.ghist, c.W, c.ghist ? 0 : bls_stride_bucket(c.stride))];
      for (int64_t p = c.p0; p < c.p1; p += c.W)
        k.cta.push_back(BlsCta{(int32_t)p, (uint16_t)b, (uint16_t)std::min<int64_t>(c.W, c.p1 - p)});
      k.stride = std::max(k.stride, c.stride);
      k.smem = std::max(k.smem, c.smem);
    }
  }
  for (auto& kv : buckets) {
    const int ghist = std::get<0>(kv.first), W = std::get<1>(kv.first);
    Bucket& k = kv.second;
    const size_t per_cta = (size_t)W * 2 * k.stride * sizeof(double);
    const int64_t n = (int64_t)k.cta.size();
    const int64_t group = ghist ? (int64_t)std::max<size_t>(1, lim.hist_cap / per_cta) : n;
    for (int64_t c0 = 0; c0 < n; c0 += group) {
      const int64_t c1 = std::min(n, c0 + group);
      BlsLaunch l;
      l.cta_begin = (int64_t)plan.cta.size();
      plan.cta.insert(plan.cta.end(), k.cta.begin() + c0, k.cta.begin() + c1);
      l.cta_end = (int64_t)plan.cta.size();
      l.W = W;
      l.stride = k.stride;
      l.ghist = ghist;
      l.smem = k.smem;
      if (ghist) plan.ghist_bytes = std::max(plan.ghist_bytes, (size_t)(c1 - c0) * per_cta);
      plan.launch.push_back(l);
    }
  }
  return true;
}

// Boundary-path lookup tables: light curve b gets nT = x_max / delta + 3 entries ("first cadence at or after
// j * delta"), to[b] .. to[b + 1] of a cumulative table index.  Light curves are processed in groups
// [b0, b1), each with its tables in one workspace of at most `budget` entries; a group without a table
// (table == false) runs the cadence path only.
struct BlsTableGroup {
  int b0, b1;
  bool table;
};

constexpr double BLS_TABLE_MAX_CELLS = 6.0e7;
// (a test build may define a small budget to get several table groups from small inputs)
#ifndef BLS_TABLE_BUDGET
#define BLS_TABLE_BUDGET ((int64_t)1 << 28)
#endif

// shared == true: the batch-wide rule of the shared-grid entry (one group; no table for any light curve when
// one of them exceeds BLS_TABLE_MAX_CELLS or the batch exceeds the budget).  shared == false: groups of
// consecutive light curves whose tables fit the budget, so that each light curve gets a table exactly when a
// one-light-curve call would give it one; a light curve that cannot have one forms a group of its own.
inline std::vector<BlsTableGroup> bls_table_groups(const int64_t* n, const double* x_max, int B, double inv_delta,
                                                   bool enabled, bool shared, int64_t budget, std::vector<int64_t>& to) {
  to.assign((size_t)B + 1, 0);
  std::vector<BlsTableGroup> groups;
  if (shared || !enabled) {
    bool ok = enabled;
    for (int b = 0; b < B && ok; ++b) {
      int64_t nT = 0;
      if (n[b] > 0) {
        const double cells = x_max[b] * inv_delta;
        if (!(cells >= 0.0) || cells > BLS_TABLE_MAX_CELLS) { ok = false; break; }
        nT = (int64_t)cells + 3;
      }
      to[b + 1] = to[b] + nT;
    }
    if (!ok) std::fill(to.begin(), to.end(), 0);
    groups.push_back(BlsTableGroup{0, B, ok && to[B] > 0 && to[B] <= budget});
    return groups;
  }
  int g0 = 0;
  for (int b = 0; b < B; ++b) {
    int64_t nT = 0;
    bool cannot = false;
    if (n[b] > 0) {
      const double cells = x_max[b] * inv_delta;
      if (!(cells >= 0.0) || cells > BLS_TABLE_MAX_CELLS) cannot = true;
      else nT = (int64_t)cells + 3;
    }
    if (cannot) {
      if (b > g0) groups.push_back(BlsTableGroup{g0, b, to[b] > to[g0]});
      groups.push_back(BlsTableGroup{b, b + 1, false});
      to[b + 1] = to[b];
      g0 = b + 1;
      continue;
    }
    if (b > g0 && to[b] - to[g0] + nT > budget) {
      groups.push_back(BlsTableGroup{g0, b, to[b] > to[g0]});
      g0 = b;
    }
    to[b + 1] = to[b] + nT;
  }
  if (B > g0) groups.push_back(BlsTableGroup{g0, B, to[B] > to[g0]});
  return groups;
}

}  // namespace lkb
