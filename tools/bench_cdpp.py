"""CDPP and outlier removal (K4 + K11 + K12): LightCurveCollection.estimate_cdpp / remove_outliers against the
per-light-curve loop, on bench.py's config-5 collection (tools/bench_bls_ragged.make_c5_bls).

For each batch size:
  - the K11+K12 kernel time of estimate_cdpp from the library's CUDA events (the second event of an lkb_cdpp call; the
    first is K4), beside its byte model and the HBM bound at 3.35 TB/s.  Byte model: the flattened flux read once
    (8 bytes per cadence) and the [B, D] result; every light curve of config 5 fits in shared memory, so the clip rounds
    and the finish re-read it there;
  - the whole lkb_cdpp device time (K4 + K11 + K12 events);
  - the estimate_cdpp collection call from Python;
  - the loop [lc.estimate_cdpp() for lc in coll], timed on --loop-lc light curves and extrapolated by cadence count;
  - the same pair for remove_outliers (the K11 event: the flux read once, the mask written, 9 bytes per cadence).
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

HBM_BPS = 3.35e12            # H100 SXM data sheet


def leg(engine, B, loop_lc, reps):
    import lightkurve_b200 as lk
    from bench_bls_ragged import make_c5_bls
    times, fluxes, errs = make_c5_bls(B=B)
    coll = lk.LightCurveCollection([lk.LightCurve(time=t, flux=f, flux_err=e) for t, f, e in zip(times, fluxes, errs)])
    n_cad = float(sum(len(t) for t in times))
    out = {"workload": "c5 CDPP: %d light curves, %.0f cadences" % (B, n_cad)}
    coll.estimate_cdpp()                                          # warm-up (workspace growth)
    coll.remove_outliers()
    for name, fn, bytes_per, k_event in (("estimate_cdpp", lambda: coll.estimate_cdpp(), 8.0, 1),
                                         ("remove_outliers", lambda: coll.remove_outliers(), 9.0, 0)):
        engine.profile_enable(True)
        t0 = time.perf_counter()
        for _ in range(reps):
            res = fn()
        wall = (time.perf_counter() - t0) / reps
        ev = engine.profile_read().reshape(reps, -1)
        engine.profile_enable(False)
        kms = float(np.mean(ev[:, k_event]))
        model = bytes_per * n_cad
        out[name] = {"call_s": wall, "k11_k12_ms" if k_event else "k11_ms": kms, "byte_model_GB": model / 1e9,
                     "achieved_GBps": model / (kms * 1e-3) / 1e9, "hbm_bound_ms": model / HBM_BPS * 1e3,
                     "share_of_hbm_bound": (model / HBM_BPS) / (kms * 1e-3)}
        if k_event:
            out[name]["lkb_cdpp_device_ms"] = float(np.mean(ev.sum(axis=1)))
            out[name]["k4_ms"] = float(np.mean(ev[:, 0]))
            batch = res.value
    n = min(loop_lc, B)
    loop_cad = float(sum(len(t) for t in times[:n]))
    for name, meth in (("estimate_cdpp", "estimate_cdpp"), ("remove_outliers", "remove_outliers")):
        t0 = time.perf_counter()
        loop = [getattr(lc, meth)() for lc in coll[:n]]
        s = time.perf_counter() - t0
        out[name + "_loop"] = {"measured_lc": n, "measured_s": s, "extrapolated_s": s * n_cad / loop_cad,
                               "note": "extrapolated from %d light curves by cadence count" % n}
        out[name + "_speedup"] = out[name + "_loop"]["extrapolated_s"] / out[name]["call_s"]
        if meth == "estimate_cdpp":
            ref = np.array([q.value for q in loop])
            out["cdpp_max_rel_diff_to_loop"] = float(np.max(np.abs(batch[:n] / ref - 1)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-lc", default="2048,16384", help="comma list of batch sizes")
    ap.add_argument("--loop-lc", type=int, default=200)
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
