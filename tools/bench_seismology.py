"""Seismology spectra of a red-giant catalogue: LightCurveCollection.to_seismology (one GPU call) against the
single-curve loop Seismology.from_lightcurve, timed on a few stars and extrapolated.  Workload: Kepler-long-cadence-
like light curves (29.4 min cadence, ~4 years with a 10-day gap every quarter), normalization="psd", the grid to the
283 uHz Nyquist frequency.  Prints one JSON line; with --profile also the kernel split from torch.profiler.  The card
name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def catalogue(B, years, seed=0):
    import lightkurve_b200 as lk
    dt = 1765.5 / 86400.0
    N = int(years * 365.25 / dt)
    t = np.arange(N) * dt
    keep = np.ones(N, bool)
    q = int(93.0 / dt)
    for s in range(q, N, q):
        keep[s:s + int(10.0 / dt)] = False
    rng = np.random.default_rng(seed)
    tk = t[keep]
    base = np.sin(2 * np.pi * 1e-6 * 86400 * tk[None, :] * np.array([[100.0], [150.0]]))
    out = []
    for b in range(B):
        y = 1 + 3e-5 * base[b % 2] + 2e-5 * rng.normal(size=len(tk))
        out.append(lk.LightCurve(time=tk, flux=y, flux_err=np.full(len(tk), 2e-5)))
    return out


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                        "--format=csv,noheader"], text=True).strip()
    except Exception as e:                             # noqa: BLE001
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stars", type=int, default=2048)
    ap.add_argument("--years", type=float, default=4.0)
    ap.add_argument("--loop-stars", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    import torch
    import lightkurve_b200 as lk
    from lightkurve_b200 import engine
    from lightkurve_b200.seismology import Seismology
    engine.init(0)
    lcs = catalogue(a.stars, a.years)
    coll = lk.LightCurveCollection(lcs)
    np.random.seed(0)
    lk.LightCurveCollection(lcs[:8]).to_seismology(normalization="psd")        # warm-up of every kernel
    Seismology.from_lightcurve(lcs[0], normalization="psd")
    times = []
    for _ in range(a.repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        seis = coll.to_seismology(normalization="psd")
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    t0 = time.perf_counter()
    for lc in lcs[:a.loop_stars]:
        Seismology.from_lightcurve(lc, normalization="psd")
    loop = (time.perf_counter() - t0) / a.loop_stars * a.stars
    res = dict(workload="to_seismology", stars=a.stars, cadences=len(lcs[0]),
               bins=len(seis[0].periodogram.frequency), collection_s=min(times), collection_all_s=times,
               loop_extrapolated_s=loop, loop_stars_timed=a.loop_stars, speedup=loop / min(times), card=card())
    if a.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            coll.to_seismology(normalization="psd")
            torch.cuda.synchronize()
        split = {}
        for ev in prof.key_averages():
            if ev.device_type.name == "CUDA" or getattr(ev, "self_device_time_total", 0):
                split[ev.key] = getattr(ev, "self_device_time_total", 0.0) / 1e3
        res["kernel_ms"] = dict(sorted(split.items(), key=lambda kv: -kv[1])[:12])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
