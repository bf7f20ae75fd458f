"""K7 windowed autocorrelation (seismology ACF2D): CUDA-event time of lkb_acf_windows with device-resident inputs on
red-giant catalogs of Kepler 4-year long-cadence SNR spectra (grid up to 283.2 uHz: 35 749 bins at oversample 1,
178 749 at oversample 5), the host wall time of the whole batched estimators, and the host estimators on a few stars
extrapolated to the batch.  The fp64 FMA count is sum over windows of n(n+1)/2 (the valid index pairs); the ceiling
is SM count x max SM clock x 64 fp64 FMA/clk/SM.  Prints the card, its power limit and max SM clock, one JSON line
per workload and a markdown table; --out FILE also writes the rows as a JSON list.

    python tools/bench_acf.py [--out results/bench_acf.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NYQ = 283.2                                   # uHz, Kepler long cadence
F_OS1 = 35749
# (name, stars, oversample, estimator, host stars timed)
WORKLOADS = [
    ("numax os1", 2048, 1, "numax", 2),
    ("numax os5", 128, 5, "numax", 1),
    ("deltanu os1", 2048, 1, "deltanu", 4),
    ("deltanu os5", 512, 5, "deltanu", 2),
]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        plimit, clk = [s.strip() for s in q.split(",")]
    except (OSError, subprocess.SubprocessError, ValueError):
        plimit, clk = "unknown", "unknown"
    return name, plimit, clk


def catalog(B, oversample, seed=2024):
    """B seeded red-giant SNR spectra: four mode templates (numax 45/80/130/200 uHz) times per-star chi^2 noise."""
    from lightkurve_b200 import units as u
    from lightkurve_b200.periodogram import SNRPeriodogram
    F = F_OS1 * oversample
    fs = NYQ / F
    f = fs * (1 + np.arange(F))
    rng = np.random.default_rng(seed)
    templates = []
    for numax in (45.0, 80.0, 130.0, 200.0):
        dnu, sig = 0.294 * numax ** 0.772, 0.66 * numax ** 0.88 / 2.355
        comb = np.zeros(F)
        for eps, h in ((0.0, 1.0), (0.5, 1.2), (-0.12, 0.6)):
            for m in numax + dnu * (np.arange(-8, 9) + eps):
                comb += h / (1 + ((f - m) / 0.08) ** 2)
        templates.append(1 + 30.0 * np.exp(-0.5 * ((f - numax) / sig) ** 2) * comb)
    fq = u.Quantity(f, u.microhertz)
    return [SNRPeriodogram(fq, u.Quantity(templates[b % 4] * rng.exponential(size=F), None)) for b in range(B)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--min-window", type=float, default=1.0, help="seconds of timed kernel work per measurement")
    args = ap.parse_args()
    import torch
    from lightkurve_b200 import _lib as L, engine
    from lightkurve_b200 import seismology as S
    engine.init(0)
    lib = L.load()
    name, plimit, clk = card()
    sms = engine.sm_count()
    try:
        peak = sms * float(clk.split()[0]) * 1e6 * 64
    except ValueError:
        peak = float("nan")
    print("card: %s, power limit: %s, max SM clock: %s, %d SMs, fp64 FMA ceiling %.2f TFMA/s"
          % (name, plimit, clk, sms, peak / 1e12), flush=True)
    rows = []
    dev = torch.device("cuda", 0)
    for wname, B, os_, est, nhost in WORKLOADS:
        pgs = catalog(B, os_)
        if est == "numax":
            setups = [S._numax_setup(pg, None, None, None) for pg in pgs]
            starts = [s["starts"] for s in setups]
            lens = [s["nlags"] for s in setups]
        else:
            setups = [S._deltanu_setup(pg, 150.0) for pg in pgs]
            starts = [np.array([s["start"]]) for s in setups]
            lens = [s["length"] for s in setups]
        x = np.concatenate([s["power"] for s in setups])
        xoff = np.zeros(B + 1, np.int64)
        np.cumsum([len(s["power"]) for s in setups], out=xoff[1:])
        woff = np.zeros(B + 1, np.int64)
        np.cumsum([len(s) for s in starts], out=woff[1:])
        ws = np.ascontiguousarray(np.concatenate(starts), dtype=np.int64)
        wl = np.ascontiguousarray(lens, dtype=np.int64)
        W = int(woff[-1])
        fmas = float(sum(len(s) * n * (n + 1) / 2 for s, n in zip(starts, lens)))
        x_d = torch.from_numpy(x).to(dev)
        m_d = torch.empty(W, dtype=torch.float64, device=dev)

        def call():
            L.check(lib.lkb_acf_windows(L.ptr(x_d), L.ptr(xoff), B, L.ptr(woff), L.ptr(ws), L.ptr(wl), L.ptr(m_d),
                                        None, L.MEM_DEVICE, torch.cuda.current_stream().cuda_stream))
        call()                                               # warm-up (module load, workspace growth)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        torch.cuda.synchronize()
        one = e0.elapsed_time(e1) / 1e3
        steps = max(2, int(np.ceil(args.min_window / max(one, 1e-6))))
        e0.record()
        for _ in range(steps):
            call()
        e1.record()
        torch.cuda.synchronize()
        kern = e0.elapsed_time(e1) / 1e3 / steps
        del x_d, m_d
        torch.cuda.empty_cache()
        # the whole batched estimator from the host (validation, staging, kernels, smoothing / peak search)
        t0 = time.perf_counter()
        if est == "numax":
            S.estimate_numax_acf2d_batch(pgs)
        else:
            S.estimate_deltanu_acf2d_batch(pgs, [150.0] * B)
        wall = time.perf_counter() - t0
        # the host estimator on a few stars, extrapolated to the batch
        t0 = time.perf_counter()
        for pg in pgs[:nhost]:
            S.estimate_numax_acf2d(pg) if est == "numax" else S.estimate_deltanu_acf2d(pg, 150.0)
        host_star = (time.perf_counter() - t0) / nhost
        res = {"workload": wname, "B": B, "F": int(xoff[1]), "windows": W, "lags": int(lens[0]), "fp64_fma": fmas,
               "kernel_s": kern, "steps": steps, "gfma_s": fmas / kern / 1e9, "share_of_fp64_fma_ceiling": fmas / kern / peak,
               "batch_call_wall_s": wall, "host_s_per_star": host_star, "host_stars_timed": nhost,
               "host_extrapolated_s": host_star * B, "card": name, "power_limit": plimit, "max_sm_clock": clk}
        rows.append(res)
        print(json.dumps(res), flush=True)
        del pgs, setups, x
    print("\n| workload | stars x bins | windows x lags | fp64 FMA | lkb_acf_windows (events) | GFMA/s | of ceiling "
          "| batched estimator (host wall) | host estimator (extrapolated) |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %s | %d x %d | %d x %d | %.3g | %.1f ms | %.0f | %.0f %% | %.2f s | %.0f s (%.3f s/star x %d) |"
              % (r["workload"], r["B"], r["F"], r["windows"], r["lags"], r["fp64_fma"], 1e3 * r["kernel_s"], r["gfma_s"],
                 100 * r["share_of_fp64_fma_ceiling"], r["batch_call_wall_s"], r["host_extrapolated_s"],
                 r["host_s_per_star"], r["B"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
