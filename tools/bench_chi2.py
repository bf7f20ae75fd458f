"""Multi-term Lomb-Scargle (nterms 1..4): CUDA-event time of lkb_ls_power_chi2_ex with device-resident inputs, direct
sums against the NUFFT path, on ragged batches from the config-5 generator (bench.make_c5_workload) - one GPU's share of
config 5 and smaller batches down to config 1 (1 light curve x 1000 cadences x 2497 bins) - plus the worst parity
excess of the NUFFT rows against the direct ones.  Prints the card and its power limit, then one JSON line per
(workload, nterms); --out FILE also writes them as a JSON list.  The crossover sets `auto`'s threshold (ls.cu:
LS_CHI2_NUFFT_MIN_WORK).

    python tools/bench_chi2.py [--out results/bench_chi2.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (name, light curves, cadences per light curve (None: the config-5 generator's own), bins)
WORKLOADS = [
    ("c5-share", 2048, None, 20000),
    ("c5-256", 256, None, 20000),
    ("32x4000x10000", 32, 4000, 10000),
    ("4x4000x5000", 4, 4000, 5000),
    ("1x4000x5000", 1, 4000, 5000),
    ("c1", 1, 1000, 2497),
]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def workload(B, n, F):
    if n is None:
        from bench import make_c5_workload
        return make_c5_workload(1005, B=B, F=F)
    # fixed length: n random times over the config-5 span, the same grid rule (up to 50 / d, f0 = df)
    rng = np.random.default_rng(n)
    times = [np.sort(1325 + rng.uniform(0, 27.8, n)) for _ in range(B)]
    fluxes = [(1 + 1e-3 * np.sin(2 * np.pi * rng.uniform(0.05, 20) * t) + 1e-3 * rng.standard_normal(n)).astype(np.float32)
              for t in times]
    return times, fluxes, np.linspace(50.0 / F, 50.0, F)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--min-window", type=float, default=1.0, help="seconds of timed work per measurement")
    args = ap.parse_args()
    import torch
    from lightkurve_b200 import _lib as L, engine
    engine.init(0)
    lib = L.load()
    name, plimit = card()
    print("card: %s, power limit: %s" % (name, plimit), flush=True)
    algos = {"direct": L.LS_ALGO_SIMT, "nufft": L.LS_ALGO_NUFFT}
    rows = []
    for wname, B, n, F in WORKLOADS:
        times, fluxes, freq = workload(B, n, F)
        offsets = np.zeros(B + 1, np.int64)
        np.cumsum([len(t) for t in times], out=offsets[1:])
        dev = torch.device("cuda", 0)
        t_cat = torch.from_numpy(np.concatenate(times)).to(dev)
        y_cat = torch.from_numpy(np.concatenate(fluxes).astype(np.float32)).to(dev)
        f_d = torch.from_numpy(np.ascontiguousarray(freq, np.float64)).to(dev)
        work = float(offsets[-1]) * F
        for nterms in (1, 2, 3, 4):
            res = {"workload": wname, "B": B, "sum_N": int(offsets[-1]), "F": F, "sumN_x_F": work, "nterms": nterms,
                   "card": name, "power_limit": plimit}
            outs = {}
            for a, code in algos.items():
                out = torch.empty((B, F), dtype=torch.float32, device=dev)

                def call():
                    L.check(lib.lkb_ls_power_chi2_ex(L.ptr(t_cat), L.ptr(y_cat), L.DTYPE_F32, L.ptr(offsets), B, L.ptr(f_d),
                                                     None, F, nterms, L.LS_NORM_AMPLITUDE, None, L.ptr(out), None,
                                                     L.MEM_DEVICE, torch.cuda.current_stream().cuda_stream, code))
                call()                                           # warm-up (module load, workspace growth)
                torch.cuda.synchronize()
                res["ran_" + a] = engine.ls_last_algo()
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
                res["ms_" + a] = e0.elapsed_time(e1) / steps
                res["steps_" + a] = steps
                outs[a] = out.cpu().numpy().astype(np.float64)
            d, nf = outs["direct"], outs["nufft"]
            ex = np.abs(nf - d) / (1e-5 * d.max(axis=1, keepdims=True) + 1e-4 * d)
            ex = ex[np.isfinite(ex)]
            res["worst_excess_vs_direct"] = float(ex.max()) if ex.size else float("nan")
            res["speedup"] = res["ms_direct"] / res["ms_nufft"]
            rows.append(res)
            print(json.dumps(res), flush=True)
        del t_cat, y_cat, f_d
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
