"""BLS vetting (K10): BoxLeastSquaresPeriodogram.compute_stats_batch / get_transit_mask_batch against the
per-periodogram loop, on bench.py's config-5 collection (tools/bench_bls_ragged.make_c5_bls).

Each light curve gets a candidate near its injected transit (an arbitrary one where there is none).  For each batch
size: the K10 kernel time from the library's CUDA events beside its byte model (t, y and dy read twice: 48 bytes per
cadence, plus 1 byte of mask with get_transit_mask_batch) and the HBM bound at 3.35 TB/s; the whole compute_stats_batch
and get_transit_mask_batch calls from Python; and the loops [pg.compute_stats(...)] / [pg.get_transit_mask(...)], timed
on --loop-lc periodograms and extrapolated by cadence count.  Prints one JSON line per measurement; card name, power
limit and max SM clock from the same run come first.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

HBM_BPS = 3.35e12            # H100 SXM data sheet


def workload(B, seed=1005):
    from bench_bls_ragged import make_c5_bls
    from _bls_stats_cases import make_pg
    times, fluxes, errs = make_c5_bls(seed=seed, B=B)
    rng = np.random.default_rng([seed, 5])
    pgs, cand = [], []
    for b, (t, y, e) in enumerate(zip(times, fluxes, errs)):
        r = np.random.default_rng([seed, 77, b])             # make_c5_bls's own draws: its injected transit
        r.uniform(np.log10(2e-4), -3)
        if b % 4 != 3:
            per, dur = r.uniform(1, 8), r.uniform(0.05, 0.3)
            tt = t[0] + 0.7
        else:
            per, dur, tt = rng.uniform(1, 8), rng.uniform(0.05, 0.3), t[0] + rng.uniform(0, 5)
        pgs.append(make_pg(t, y, e, per, dur, tt))
        cand.append((per, dur, tt))
    return pgs, [np.array(c) for c in zip(*cand)]


def leg(engine, B, loop_lc, reps):
    from lightkurve_b200.periodogram import BoxLeastSquaresPeriodogram as BLS
    pgs, (per, dur, tt) = workload(B)
    n_cad = float(sum(len(pg.time) for pg in pgs))
    BLS.compute_stats_batch(pgs, per, dur, tt)                 # warm-up (workspace growth)
    BLS.get_transit_mask_batch(pgs, per, dur, tt)
    out = {"workload": "c5 BLS vetting: %d light curves, %.0f cadences" % (B, n_cad)}
    for name, fn, bytes_per in (("compute_stats_batch", BLS.compute_stats_batch, 48.0),
                                ("get_transit_mask_batch", BLS.get_transit_mask_batch, 49.0)):
        engine.profile_enable(True)
        t0 = time.perf_counter()
        for _ in range(reps):
            res = fn(pgs, per, dur, tt)
        wall = (time.perf_counter() - t0) / reps
        kms = float(np.sum(engine.profile_read())) / reps
        engine.profile_enable(False)
        model = bytes_per * n_cad
        out[name] = {"call_s": wall, "kernel_ms": kms, "byte_model_GB": model / 1e9,
                     "achieved_GBps": model / (kms * 1e-3) / 1e9, "hbm_bound_ms": model / HBM_BPS * 1e3,
                     "share_of_hbm_bound": (model / HBM_BPS) / (kms * 1e-3)}
    n = min(loop_lc, B)
    loop_cad = float(sum(len(pg.time) for pg in pgs[:n]))
    for name, meth in (("compute_stats", "compute_stats"), ("get_transit_mask", "get_transit_mask")):
        t0 = time.perf_counter()
        loop = [getattr(pg, meth)(per[b], dur[b], tt[b]) for b, pg in enumerate(pgs[:n])]
        s = time.perf_counter() - t0
        out[name + "_loop"] = {"measured_lc": n, "measured_s": s, "extrapolated_s": s * n_cad / loop_cad,
                               "note": "extrapolated from %d periodograms by cadence count" % n}
    out["compute_stats_speedup"] = out["compute_stats_loop"]["extrapolated_s"] / out["compute_stats_batch"]["call_s"]
    out["get_transit_mask_speedup"] = (out["get_transit_mask_loop"]["extrapolated_s"]
                                       / out["get_transit_mask_batch"]["call_s"])
    same = all(np.array_equal(a, b) for a, b in zip(res[:n], loop))
    out["loop_masks_equal_batched"] = bool(same)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-lc", default="16384,2048", help="comma list of batch sizes")
    ap.add_argument("--loop-lc", type=int, default=300)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    from bench_bls_ragged import card
    from lightkurve_b200 import engine
    engine.init(0)
    print(json.dumps(card()), flush=True)
    for B in (int(x) for x in args.n_lc.split(",")):
        print(json.dumps(leg(engine, B, args.loop_lc, args.reps)), flush=True)


if __name__ == "__main__":
    main()
