"""Per-kernel time of one device-resident Lomb-Scargle step (bench.py's configuration 2 by default).

    python tools/ls_step_anatomy.py --out DIR [--workload c2] [--steps 5] [--label NAME]

Runs the step `--warmup` times, then `--steps` times under torch.profiler with CUDA activities, and sums the device
time of every kernel by name.  Kernels are grouped into what they do to the flux (prep / spread / low rows /
escalation / transforms / other), and the card name and power limit are read in the same run.  Every kernel's launch
shape (grid, block, dynamic + static shared memory, registers per thread; from the profiler's trace, one entry per
distinct shape) is recorded beside its time, so that a kernel sized for more work than it has shows as such.  Writes
DIR/anatomy_<label>.json and prints a table; the JSON holds milliseconds per step.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# kernel-name substrings -> group (first match wins)
GROUPS = [
    ("escalation", ("nufft2_flag", "_list_kernel", "lowacc", "lowexact")),
    ("cols", ("nufft2_cols",)),
    ("rows", ("nufft2_rows",)),
    ("prep", ("ls_prep_shared", "nufft2_stats", "nufft2_centre")),
    ("spread", ("nufft2_spread",)),
    ("low_rows", ("nufft2_lowrows", "nufft2_lowfinish")),
]


def group_of(name):
    for g, keys in GROUPS:
        if any(k in name for k in keys):
            return g
    return "other"


def launch_shapes(prof):
    """kernel name -> distinct launch shapes, read from the profiler's Chrome trace (written to a temporary file)"""
    shapes = defaultdict(list)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f).get("traceEvents", [])
    for ev in events:
        if ev.get("cat") != "kernel":
            continue
        a = ev.get("args", {})
        shape = "grid %s block %s smem %s regs %s" % (
            "x".join(str(v) for v in a.get("grid", [])), "x".join(str(v) for v in a.get("block", [])),
            a.get("shared memory", "?"), a.get("registers per thread", "?"))
        if shape not in shapes[ev["name"]]:
            shapes[ev["name"]].append(shape)
    return shapes


def card_info(torch):
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except Exception as e:                       # the numbers stay valid; the record says why the field is missing
        info["power_limit_and_max_sm_clock"] = "unavailable: %r" % (e,)
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--workload", default="c2")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1002)
    ap.add_argument("--label", default="run")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from lightkurve_b200 import engine

    assert torch.cuda.is_available(), "ls_step_anatomy.py needs a CUDA device"
    engine.init(0)
    dev = torch.device("cuda", 0)
    w = bench.WORKLOADS[args.workload]
    t, Y, freq = bench.make_workload(args.workload, args.seed)
    d_t, d_f, d_Y = (torch.tensor(a, device=dev) for a in (t, freq, Y))
    d_P = torch.empty((w["B"], w["F"]), dtype=torch.float32, device=dev)

    def step():
        engine.ls_power_shared(d_t, d_Y, d_f, "amplitude", out=d_P)

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()

    per_kernel = defaultdict(lambda: [0.0, 0])
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA or ev.name.startswith("Memcpy") or ev.name.startswith("Memset"):
            continue
        k = per_kernel[ev.name]
        k[0] += ev.device_time / 1000.0           # us -> ms
        k[1] += 1
    shapes = launch_shapes(prof)
    kernels = {name: {"ms_per_step": v[0] / args.steps, "launches_per_step": v[1] / args.steps,
                      "launch_shapes": shapes.get(name, [])}
               for name, v in sorted(per_kernel.items(), key=lambda kv: -kv[1][0])}
    groups = defaultdict(float)
    for name, v in kernels.items():
        groups[group_of(name)] += v["ms_per_step"]
    replaced = sum(groups[g] for g in ("prep", "spread", "low_rows", "escalation"))
    rec = {"label": args.label, "workload": args.workload, "steps": args.steps, "family": engine.ls_last_algo(),
           "escalated_per_step": engine.ls_last_escalated(), "card": card_info(torch),
           "kernel_ms_per_step": sum(groups.values()), "groups_ms_per_step": dict(groups),
           "prep_spread_lowrows_escalation_ms": replaced, "kernels": kernels}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "anatomy_%s.json" % args.label), "w") as f:
        json.dump(rec, f, indent=1)
    print("%s  %s  %s" % (args.label, rec["card"]["name"], rec["card"]["power_limit_and_max_sm_clock"]))
    for name, v in kernels.items():
        print("  %8.4f ms  x%-5g %-10s %s" % (v["ms_per_step"], v["launches_per_step"], group_of(name), name[:110]))
        for shape in v["launch_shapes"]:
            print("  %31s %s" % ("", shape))
    for g, v in sorted(groups.items(), key=lambda kv: -kv[1]):
        print("  group %-10s %8.4f ms" % (g, v))
    print("  kernels total %.4f ms; prep + spread + low rows + escalation %.4f ms" % (rec["kernel_ms_per_step"], replaced))


if __name__ == "__main__":
    main()
