"""Box Least Squares over light curves with their own period grids: one batched call against the per-light-curve loop.

Workloads:
  c5     bench.py's config-5 times (make_c5_workload, seed 1005: TESS 2-min sector, 2 000-20 000 kept cadences,
         +-20 s jitter) with a box transit injected, finite flux_err, lightkurve's default durations and default
         per-light-curve period grids (BoxLeastSquaresPeriodogram._prepare).  --n-lc light curves (16 384 and 2 048).
  c3     bench.py's BLS workload (config 3: 256 light curves x 50 000 shared periods) through lkb_bls_power and
         through lkb_bls_power_ex with the shared grid given as 256 identical CSR rows (the cost of the descriptor path).

For each: kernel time from the library's CUDA events (the search kernels), (light curve, period) pairs/s, kernel
launches, and for c5 the whole LightCurveCollection.to_periodogram("bls") call from Python.  The per-light-curve loop
(LightCurve.to_periodogram("bls") for each light curve) is timed on --loop-lc light curves and extrapolated to the batch.
Prints one JSON line per measurement; card name, power limit and max SM clock from the same run come first.
--lib PATH times another build of liblkb200.so (for comparing builds; the c3 leg through lkb_bls_power only).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

DURATIONS = [0.05, 0.10, 0.15, 0.20, 0.25, 0.33]          # lightkurve's default BLS durations


def make_c5_bls(seed=1005, B=16384):
    """(times, fluxes, flux_errs) of bench.py's config-5 light curves with a box transit in 3 of 4."""
    import bench
    times, _, _ = bench.make_c5_workload(seed, B=B, F=8)
    fluxes, errs = [], []
    for b, t in enumerate(times):
        r = np.random.default_rng([seed, 77, b])
        sig = 10 ** r.uniform(np.log10(2e-4), -3)
        y = 1 + sig * r.standard_normal(len(t))
        if b % 4 != 3:
            per, dur, dep = r.uniform(1, 8), r.uniform(0.05, 0.3), 10 ** r.uniform(np.log10(5e-4), -2)
            y[np.abs((t - t[0] - 0.7 + 0.5 * per) % per - 0.5 * per) < 0.5 * dur] -= dep
        fluxes.append(y)
        errs.append(np.full(len(t), sig))
    return times, fluxes, errs


def default_grid(t, durations=DURATIONS, frequency_factor=10):
    """lightkurve's default BLS period grid of one light curve (BoxLeastSquaresPeriodogram._prepare)."""
    from lightkurve_b200.periodogram import BoxLeastSquaresPeriodogram as BLS
    dt = np.median(np.diff(t))
    pmin = np.max([dt * 4, np.max(durations) + dt])
    pmax = (np.max(t) - np.min(t)) / 3.0
    return BLS.autoperiod(t, durations, minimum_period=pmin, maximum_period=pmax, frequency_factor=frequency_factor)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, pl, clk = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception as e:                                            # pragma: no cover
        return {"gpu": "unknown (%r)" % (e,)}


def timed(engine, fn, reps):
    """(mean kernel ms from the library's events, launches per call, wall s per call, last result)"""
    fn()                                                              # warm-up (workspace growth)
    engine.profile_enable(True)
    l0 = engine.launch_count()
    t0 = time.perf_counter()
    for _ in range(reps):
        res = fn()
    wall = (time.perf_counter() - t0) / reps
    launches = (engine.launch_count() - l0) / reps
    kms = engine.profile_read()
    engine.profile_enable(False)
    return float(np.sum(kms)) / reps, launches, wall, res


def leg_c5(engine, B, loop_lc, reps):
    import lightkurve_b200 as lk
    times, fluxes, errs = make_c5_bls(B=B)
    grids = [default_grid(t) for t in times]
    pairs = float(sum(len(g) for g in grids))
    k_ms, launches, wall, _ = timed(engine, lambda: engine.bls_power(times, fluxes, errs, grids, DURATIONS), reps)
    lcs = [lk.LightCurve(time=t, flux=f, flux_err=e) for t, f, e in zip(times, fluxes, errs)]
    coll = lk.LightCurveCollection(lcs)
    coll.to_periodogram("bls")
    t0 = time.perf_counter()
    pgs = coll.to_periodogram("bls")
    coll_s = time.perf_counter() - t0
    n = min(loop_lc, B)
    lcs[0].to_periodogram("bls")
    engine.profile_enable(True)
    l0 = engine.launch_count()
    t0 = time.perf_counter()
    loop = [lc.to_periodogram("bls") for lc in lcs[:n]]
    loop_s = time.perf_counter() - t0
    loop_launches = engine.launch_count() - l0
    loop_kms = float(np.sum(engine.profile_read()))
    engine.profile_enable(False)
    same = all(np.array_equal(a.power.value, b.power.value) for a, b in zip(pgs[:n], loop))
    loop_pairs = float(sum(len(g) for g in grids[:n]))
    return {"workload": "c5 BLS: %d light curves, default lightkurve grids (%d-%d periods), %d durations"
                        % (B, min(len(g) for g in grids), max(len(g) for g in grids), len(DURATIONS)),
            "pairs": pairs,
            "batched": {"kernel_ms": k_ms, "pairs_per_s": pairs / (k_ms * 1e-3), "launches": launches,
                        "engine_call_s": wall, "collection_call_s": coll_s},
            "loop": {"measured_lc": n, "measured_s": loop_s, "measured_kernel_ms": loop_kms,
                     "measured_launches": loop_launches,
                     "extrapolated_s": loop_s * pairs / loop_pairs, "extrapolated_kernel_ms": loop_kms * pairs / loop_pairs,
                     "note": "extrapolated from %d light curves by (light curve, period) pairs" % n},
            "loop_equals_batched_bitwise": bool(same)}


def leg_c3(engine, reps):
    import bench
    from lightkurve_b200 import _lib as L
    B, N, P = 256, 20000, 50000
    t, fluxes, errs, period, duration = bench.make_bls_workload(1003, B, N, P)
    times = [t] * B
    pairs = float(B) * P
    out = {"workload": "c3 BLS: %d light curves x %d cadences x %d shared periods x %d durations" % (B, N, P, len(duration))}
    k_ms, launches, wall, shared = timed(engine, lambda: engine.bls_power(times, fluxes, errs, period, duration), reps)
    out["shared_entry"] = {"kernel_ms": k_ms, "pairs_per_s": pairs / (k_ms * 1e-3), "launches": launches, "call_s": wall}
    if "lkb_bls_power_ex" in L.SIGNATURES:
        k_ms, launches, wall, csr = timed(engine, lambda: engine.bls_power(times, fluxes, errs, [period] * B, duration),
                                          reps)
        out["csr_entry"] = {"kernel_ms": k_ms, "pairs_per_s": pairs / (k_ms * 1e-3), "launches": launches,
                            "call_s": wall}
        out["csr_equals_shared_bitwise"] = bool(all(np.array_equal(np.stack(csr[k]), shared[k]) for k in shared
                                                    if k != "period"))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--legs", default="c5,c3")
    ap.add_argument("--n-lc", default="16384,2048", help="comma list of c5 batch sizes")
    ap.add_argument("--loop-lc", type=int, default=300)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--lib", default=None, help="path of another liblkb200.so build to time")
    args = ap.parse_args()
    from lightkurve_b200 import _lib as L
    if args.lib:
        L.LIB_PATH = args.lib
        try:
            L.load()
        except AttributeError:                                        # a build without lkb_bls_power_ex
            L.SIGNATURES.pop("lkb_bls_power_ex")
            L.load()
    from lightkurve_b200 import engine
    engine.init(0)
    print(json.dumps(dict(card(), lib=L.LIB_PATH)), flush=True)
    for leg in args.legs.split(","):
        if leg == "c3":
            print(json.dumps(leg_c3(engine, args.reps)), flush=True)
        elif leg == "c5":
            for B in (int(x) for x in args.n_lc.split(",")):
                print(json.dumps(leg_c5(engine, B, args.loop_lc, args.reps)), flush=True)


if __name__ == "__main__":
    main()
