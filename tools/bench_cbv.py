"""CBVCorrector.correct_batch with both goodness metrics (the reference's default correct()) on TESS-like targets:
rounds, the time of each engine call family (CUDA events around each call: device work plus the call's own small
copies; the final scores' periodograms are host-mode calls and include their staging), the under-fitting kernel
against its byte model, the whole call, and a per-corrector loop of the same code (a sample timed, extrapolated).

    python tools/bench_cbv.py --targets 1024 --cadences 18000 --loop-sample 4
"""
import argparse
import json
import os
import sys
import time
from collections import defaultdict

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--targets", type=int, default=1024)
    ap.add_argument("--cadences", type=int, default=18000)
    ap.add_argument("--loop-sample", type=int, default=4)
    ap.add_argument("--max-iter", type=int, default=100)
    args = ap.parse_args()
    import subprocess
    from lightkurve_b200 import engine
    from lightkurve_b200.correctors import CBVCorrector
    from oracle.cbv import tess_like_batch
    engine.init(0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    lcs, cbvs, _ = tess_like_batch(n=args.targets, N=args.cadences)
    import torch
    spent = defaultdict(float)
    calls = defaultdict(int)
    k9_bytes = [0.0]
    for name in ("regress", "ls_power_ragged", "ls_power_ragged_device", "underfit_metric", "overfit_terms",
                 "ls_power_shared"):
        fn = getattr(engine, name)

        def timed(*a, _fn=fn, _name=name, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = _fn(*a, **k)
            e1.record()
            e1.synchronize()
            spent[_name] += e0.elapsed_time(e1) / 1e3
            calls[_name] += 1
            if _name == "underfit_metric":        # byte model: neighbour rows, the target (once) and the bit rows
                G = a[0].shape[1]
                M = np.diff(np.asarray(a[2]))
                k9_bytes[0] += float(np.sum(8.0 * M * G + 8.0 * G + (M + 1) * G / 8.0))
            return r
        setattr(engine, name, timed)
    kw = dict(cbv_type=["SingleScale"], cbv_indices=[np.arange(1, 9)], max_iter=args.max_iter)
    np.random.seed(0)
    cs = [CBVCorrector(lc, cbvs=[cbvs]) for lc in lcs]
    t0 = time.perf_counter()
    CBVCorrector.correct_batch(cs, **kw)
    total = time.perf_counter() - t0
    rounds = max(len(c.optimization_trace) for c in cs)
    batch = dict(spent), dict(calls)
    k9b = k9_bytes[0]
    spent.clear()
    calls.clear()
    t0 = time.perf_counter()
    for lc in lcs[:args.loop_sample]:
        c = CBVCorrector(lc, cbvs=[cbvs])
        CBVCorrector.correct_batch([c], neighbors=lcs, **kw)
    loop = (time.perf_counter() - t0) / args.loop_sample * args.targets
    k9 = batch[0].get("underfit_metric", 0.0)
    print(json.dumps(dict(card=card, targets=args.targets, cadences=args.cadences, rounds=rounds,
                          batch_seconds=total, device_seconds_by_call=batch[0], calls=batch[1],
                          underfit_bytes_model=k9b, underfit_seconds=k9,
                          underfit_share_of_3350GBs=(k9b / 3.35e12) / k9 if k9 else None,
                          loop_seconds_extrapolated=loop, loop_sample=args.loop_sample)))


if __name__ == "__main__":
    main()
