"""Fold and bin (K13): LightCurveCollection.fold / bin against the per-light-curve loop, on bench.py's config-5
collection (tools/bench_bls_ragged.make_c5_bls).

For each batch size and each of three workloads - fold(2.3 d), fold(2.3 d) then bin(time_bin_size=0.02) of the phase,
and bin(time_bin_size=10 min) in time - it reports:
  - the K13 kernel time from the library's CUDA events (one event per lkb_fold / lkb_bin launch);
  - the whole collection call from Python (packing, transfers, kernels and result objects);
  - the loop [lc.fold(...) / lc.bin(...) for lc in coll], timed on --loop-lc light curves and extrapolated by their
    number;
  - the largest difference of the binned flux from the loop's on the timed light curves, relative to the flux.
Prints one JSON line per measurement; card name, power limit and max SM clock from the same run come first.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

PERIOD = 2.3
FOLD_BIN = 0.02
TIME_BIN = 10.0 / 1440.0


def _max_rel_diff(batch, loop):
    d = 0.0
    for a, b in zip(batch, loop):
        x, y = np.asarray(a.flux.value), np.asarray(b.flux.value)
        m = ~np.isnan(y)
        if m.any():
            d = max(d, float(np.max(np.abs(x[m] - y[m]) / np.abs(y[m]))))
    return d


def leg(engine, B, loop_lc, reps):
    import lightkurve_b200 as lk
    from bench_bls_ragged import make_c5_bls
    times, fluxes, errs = make_c5_bls(B=B)
    coll = lk.LightCurveCollection([lk.LightCurve(time=t, flux=f, flux_err=e) for t, f, e in zip(times, fluxes, errs)])
    n_cad = float(sum(len(t) for t in times))
    out = {"workload": "c5 fold/bin: %d light curves, %.0f cadences" % (B, n_cad)}
    sample = lk.LightCurveCollection(coll[:min(loop_lc, B)])
    legs = (("fold", lambda c: c.fold(period=PERIOD)),
            ("fold_bin_0.02", lambda c: c.fold(period=PERIOD).bin(time_bin_size=FOLD_BIN)),
            ("bin_10min", lambda c: c.bin(time_bin_size=TIME_BIN)))
    for name, fn in legs:
        fn(coll)                                                  # warm-up (workspace growth)
        engine.profile_enable(True)
        t0 = time.perf_counter()
        for _ in range(reps):
            res = fn(coll)
        wall = (time.perf_counter() - t0) / reps
        ev = engine.profile_read().reshape(reps, -1)
        engine.profile_enable(False)
        t0 = time.perf_counter()
        if name == "fold":
            loop = [lc.fold(period=PERIOD) for lc in sample]
        elif name == "fold_bin_0.02":
            loop = [lc.fold(period=PERIOD).bin(time_bin_size=FOLD_BIN) for lc in sample]
        else:
            loop = [lc.bin(time_bin_size=TIME_BIN) for lc in sample]
        s = time.perf_counter() - t0
        n = len(sample)
        out[name] = {"k13_kernel_ms": float(np.mean(ev.sum(axis=1))),
                     "k13_kernel_ms_each": [float(x) for x in np.mean(ev, axis=0)],
                     "call_s": wall,
                     "loop": {"measured_lc": n, "measured_s": s, "extrapolated_s": s * B / n,
                              "note": "extrapolated from %d light curves by their number" % n},
                     "speedup": s * B / n / wall,
                     "bins": int(sum(len(x) for x in res)),
                     "max_rel_flux_diff_to_loop": _max_rel_diff(res[:n], loop)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-lc", default="2048,16384", help="comma list of batch sizes")
    ap.add_argument("--loop-lc", type=int, default=32)
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
