"""K8 elastic net (CBVCorrector.correct_elasticnet): CUDA-event times of lkb_elasticnet with device-resident inputs at
the config-4 shape (4096 light curves x 65 000 cadences, K = 17 correlated CBVs, e-/s flux), split into the Gram pass
(rg_rows excluded), the coordinate descent and the model, for the default penalties and for alpha=1, l1_ratio=0.9.

The Gram pass's useful fp64 FMAs are B N (K+1)(K+2)/2 (upper triangle of [X | y]^T [X | y]); its compulsory bytes are
the flux (B N 8), the design matrix (N K 8) and the row list + weights rg_rows writes and the Gram kernel reads back
(B N 12, twice).  Ceilings: SM count x max SM clock x 128 fp64 tensor-core FMA/clk/SM, and 3.35 TB/s of HBM3.  The host
reference (scikit-learn's ElasticNet, or oracle/enet.py without it) is timed on a few light curves and extrapolated.
Prints the card, its power limit and max SM clock, one JSON line per workload and a markdown table.

    python tools/bench_enet.py [--out results/bench_enet.json]
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

B, N, K = 4096, 65000, 17
HBM_BYTES_S = 3.35e12
WORKLOADS = [("defaults", dict(alpha=1e-20, l1_ratio=0.01)), ("alpha=1 l1_ratio=0.9", dict(alpha=1.0, l1_ratio=0.9))]


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


def fixture(seed=4):
    rng = np.random.default_rng(seed)
    V = np.cumsum(rng.normal(size=(N, K - 1)), axis=0) / np.sqrt(N)
    X = np.hstack([V, np.ones((N, 1))])
    W = rng.normal(size=(B, K - 1)) * np.geomspace(1, 1e-2, K - 1)
    Y = 1e4 * (1 + 0.01 * (W @ V.T)) + 3.0 * rng.normal(size=(B, N))
    return X, Y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-lcs", type=int, default=3)
    args = ap.parse_args()
    import torch
    from lightkurve_b200 import _lib as L, engine
    engine.init(0)
    lib = L.load()
    name, plimit, clk = card()
    sms = engine.sm_count()
    try:
        peak = sms * float(clk.split()[0]) * 1e6 * 128
    except ValueError:
        peak = float("nan")
    print("card: %s, power limit: %s, max SM clock: %s, %d SMs, fp64 tensor-core ceiling %.2f TFMA/s"
          % (name, plimit, clk, sms, peak / 1e12), flush=True)
    X, Y = fixture()
    dev = torch.device("cuda", 0)
    X_d, Y_d = torch.from_numpy(X).to(dev), torch.from_numpy(Y).to(dev)
    c_d = torch.empty((B, K), dtype=torch.float64, device=dev)
    m_d = torch.empty((B, N), dtype=torch.float64, device=dev)
    it_d = torch.empty(B, dtype=torch.int32, device=dev)
    g_d = torch.empty(B, dtype=torch.float64, device=dev)
    cv_d = torch.empty(B, dtype=torch.uint8, device=dev)
    fmas = float(B) * N * (K + 1) * (K + 2) / 2
    gram_bytes = 8.0 * B * N + 8.0 * N * K + 2 * 12.0 * B * N
    try:
        from sklearn.linear_model import ElasticNet
        host_name = "scikit-learn ElasticNet"
    except ImportError:
        ElasticNet = None
        host_name = "oracle/enet.py"
    rows = []
    for wname, kw in WORKLOADS:
        def call():
            L.check(lib.lkb_elasticnet(L.ptr(X_d), 0, L.ptr(Y_d), None, B, N, K, kw["alpha"], kw["l1_ratio"], 1000,
                                       1e-4, 0, L.ptr(c_d), L.ptr(m_d), L.ptr(it_d), L.ptr(g_d), L.ptr(cv_d),
                                       L.MEM_DEVICE, torch.cuda.current_stream().cuda_stream))
        call()                                               # warm-up (module load, workspace growth)
        torch.cuda.synchronize()
        parts = []
        for _ in range(args.reps):
            engine.profile_enable(True)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            torch.cuda.synchronize()
            ms = engine.profile_read(8)
            engine.profile_enable(False)
            parts.append([e0.elapsed_time(e1)] + list(ms[:3]))
        tot, gram, cd, model = np.median(np.asarray(parts), axis=0) / 1e3
        n_iter = it_d.cpu().numpy()
        conv = cv_d.cpu().numpy()
        t0 = time.perf_counter()
        for b in range(args.host_lcs):
            if ElasticNet is not None:
                ElasticNet(fit_intercept=False, **kw).fit(X, Y[b])
            else:
                from oracle import enet as oen
                oen.enet_fit(X, Y[b], **kw)
        host_lc = (time.perf_counter() - t0) / args.host_lcs
        res = {"workload": wname, "B": B, "N": N, "K": K, **kw, "call_s": tot, "gram_s": gram, "cd_s": cd,
               "model_s": model, "gram_fp64_fma": fmas, "gram_share_of_fp64_tc_ceiling": fmas / gram / peak,
               "gram_bytes": gram_bytes, "gram_share_of_hbm": gram_bytes / gram / HBM_BYTES_S,
               "sweeps_mean": float(n_iter.mean()), "sweeps_max": int(n_iter.max()),
               "converged": int(conv.sum()), "host": host_name, "host_s_per_lc": host_lc,
               "host_extrapolated_s": host_lc * B, "card": name, "power_limit": plimit, "max_sm_clock": clk}
        rows.append(res)
        print(json.dumps(res), flush=True)
    print("\n| workload | call (events) | Gram | of fp64 TC / HBM | CD | model | sweeps mean / max | host (extrapolated) |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %s | %.1f ms | %.1f ms | %.0f %% / %.0f %% | %.1f ms | %.1f ms | %.1f / %d | %.0f s (%.3f s/LC, %s) |"
              % (r["workload"], 1e3 * r["call_s"], 1e3 * r["gram_s"], 100 * r["gram_share_of_fp64_tc_ceiling"],
                 100 * r["gram_share_of_hbm"], 1e3 * r["cd_s"], 1e3 * r["model_s"], r["sweeps_mean"], r["sweeps_max"],
                 r["host_extrapolated_s"], r["host_s_per_lc"], r["host"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
