"""Iterative transit search (LightCurveCollection.find_transit_candidates, n_candidates=3) on config-5-like light curves
with up to three injected planets, against the two ways of writing the same rounds without it.

For --n-lc light curves (2 048 and 16 384 by default):
  call      the whole find_transit_candidates call from Python (after a warm-up call);
  kernels   device time by kernel family from torch.profiler in a run of its own: K3 (the BLS search kernels), K14
            (bls_best / transit_count / transit_compact), K10 (bls_stats) and K6 (nanmedian_std), with K14 against its
            HBM byte model (bytes every K14 kernel must move, over its time);
  batch_api the same rounds with today's batch calls: to_periodogram("bls") + get_transit_mask_batch + slicing;
  loop      the single-curve loop (to_periodogram, get_transit_mask, slicing) on --loop-lc light curves, extrapolated
            to the batch by cadence count.
Prints one JSON line per measurement; card name, power limit and max SM clock from the same run come first.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_bls_ragged import card  # noqa: E402

N_CAND = 3


def make_lcs(B, seed=1005):
    """bench.py's config-5 times (TESS 2-min sector, 2 000 - 20 000 kept cadences) with 0 - 3 box transits each."""
    import bench
    import lightkurve_b200 as lk
    times, _, _ = bench.make_c5_workload(seed, B=B, F=8)
    lcs = []
    for b, t in enumerate(times):
        r = np.random.default_rng([seed, 78, b])
        sig = 10 ** r.uniform(np.log10(2e-4), -3)
        y = 1 + sig * r.standard_normal(len(t))
        for k in range(b % 4):
            per, dur, dep = r.uniform(1, 8) * 1.6 ** k, r.uniform(0.05, 0.3), 10 ** r.uniform(np.log10(5e-4), -2)
            y[np.abs((t - t[0] - r.uniform(0, per) + 0.5 * per) % per - 0.5 * per) < 0.5 * dur] -= dep
        lcs.append(lk.LightCurve(time=t, flux=y, flux_err=np.full(len(t), sig)))
    return lk.LightCurveCollection(lcs)


def family(name):
    n = name.lower()
    if "bls_best" in n or "transit_count" in n or "transit_compact" in n:
        return "K14"
    if "bls_stats" in n:
        return "K10"
    if "nanmedian_std" in n:
        return "K6"
    if "bls" in n:
        return "K3"
    return "other"


def k14_bytes(res_rounds):
    """Bytes K14 must move per call: the best kernel reads power (8 B per (light curve, period) pair) and gathers a few
    values; the compaction reads t, y, dy, the index and the in-transit flag of every cadence (8 + 8 + 8 + 4 + 1 B)
    twice (extremes, then the scatter) and writes t, y, dy, w, the index (36 B) and a time step (8 B) per survivor."""
    total = 0
    for pairs, n_in, n_out in res_rounds:
        total += 8 * pairs + 2 * 29 * n_in + 44 * n_out
    return total


def leg(coll, loop_lc, out_dir):
    import torch
    from lightkurve_b200 import engine
    from lightkurve_b200.periodogram import BoxLeastSquaresPeriodogram as BLS
    B = len(coll)
    n_cad = np.array([len(lc) for lc in coll])
    coll.find_transit_candidates(n_candidates=N_CAND)                  # warm-up (workspace growth)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = coll.find_transit_candidates(n_candidates=N_CAND)
    torch.cuda.synchronize()
    call_s = time.perf_counter() - t0
    # kernel time by family (a run of its own)
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        coll.find_transit_candidates(n_candidates=N_CAND)
        torch.cuda.synchronize()
    fam = {}
    for ev in prof.key_averages():
        dt = getattr(ev, "device_time_total", None)
        if dt is None:
            dt = getattr(ev, "cuda_time_total", 0)
        if dt and ev.key and not ev.key.startswith("Memcpy") and not ev.key.startswith("Memset"):
            fam[family(ev.key)] = fam.get(family(ev.key), 0.0) + dt / 1e3
    # the K14 byte model: periods per round from the grids, survivors per round from masked_in
    m = res["masked_in"]
    rounds = []
    from tools.bench_bls_ragged import default_grid
    for r in range(N_CAND):
        n_in = sum(int(np.sum((x == -1) | (x >= r))) for x in m)
        n_out = sum(int(np.sum((x == -1) | (x > r))) for x in m)
        pairs = sum(len(default_grid(np.asarray(lc.time.value)[(x == -1) | (x >= r)])) for lc, x in
                    zip(list(coll)[:64], m[:64])) * B / 64.0
        rounds.append((pairs, n_in, n_out))
    kb = k14_bytes(rounds)
    # the same rounds with the batch API of today
    t0 = time.perf_counter()
    cur = coll
    for r in range(N_CAND):
        pgs = cur.to_periodogram("bls")
        masks = BLS.get_transit_mask_batch(pgs, [pg.period_at_max_power for pg in pgs],
                                           [pg.duration_at_max_power for pg in pgs],
                                           [pg.transit_time_at_max_power for pg in pgs])
        cur = type(coll)([lc[~mk] for lc, mk in zip(cur, masks)])
    torch.cuda.synchronize()
    batch_api_s = time.perf_counter() - t0
    same_batch_api = all(np.array_equal(np.asarray(a.time.value), np.asarray(lc.remove_nans().time.value)[x == -1])
                         for a, lc, x in zip(cur, coll, m))
    # the single-curve loop on a subset
    n = min(loop_lc, B)
    t0 = time.perf_counter()
    for lc in list(coll)[:n]:
        lc = lc.remove_nans()
        for r in range(N_CAND):
            pg = lc.to_periodogram("bls")
            lc = lc[~pg.get_transit_mask(period=pg.period_at_max_power, duration=pg.duration_at_max_power,
                                         transit_time=pg.transit_time_at_max_power)]
    loop_s = time.perf_counter() - t0
    k14_ms = fam.get("K14", float("nan"))
    return {"workload": "find_transit_candidates: %d config-5 light curves (%d-%d cadences), 0-3 injected planets, "
                        "n_candidates=%d, default keywords" % (B, n_cad.min(), n_cad.max(), N_CAND),
            "call_s": call_s,
            "kernel_ms_by_family": fam,
            "k14": {"ms": k14_ms, "model_bytes": kb, "achieved_GBps": kb / (k14_ms * 1e-3) / 1e9,
                    "share_of_3.35TBps": kb / (k14_ms * 1e-3) / 3.35e12},
            "batch_api_s": batch_api_s, "batch_api_equals_call": bool(same_batch_api),
            "loop": {"measured_lc": n, "measured_s": loop_s,
                     "extrapolated_s": loop_s * n_cad.sum() / n_cad[:n].sum(),
                     "note": "extrapolated from %d light curves by cadence count" % n}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-lc", type=int, nargs="+", default=[2048, 16384])
    ap.add_argument("--loop-lc", type=int, default=64)
    ap.add_argument("--out", default=None, help="directory for the JSON lines (also printed)")
    a = ap.parse_args()
    from lightkurve_b200 import engine
    engine.init(0)
    lines = [card()]
    print(json.dumps(lines[0]), flush=True)
    for B in a.n_lc:
        lines.append(leg(make_lcs(B), a.loop_lc, a.out))
        print(json.dumps(lines[-1]), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_find_transits.jsonl"), "w") as f:
            for x in lines:
                f.write(json.dumps(x) + "\n")


if __name__ == "__main__":
    main()
