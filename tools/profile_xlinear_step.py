"""Where one resident eurlex-4k step goes, kernel by kernel (diagnostic; needs a GPU).

Loads bench.py's eurlex-4k workload (same model and query seeds, built in a temporary directory), uploads the query batch
once and runs K resident steps (pb200_xlinear_resident_predict, the step bench.py times) under torch.profiler with CUDA
activities, in a run of its own.  Prints every kernel's name, launches per step and mean duration, the summed busy time per
step and the summed gaps between consecutive kernels of a step on the engine stream.  The card's name, power limit and SM
clock are read in the same call (nvidia-smi).

    python tools/profile_xlinear_step.py [--steps K] [--mode M] [--json OUT]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], stdout=subprocess.PIPE, text=True)
    return dict(zip(q.split(","), [s.strip() for s in r.stdout.strip().split(",")])) if r.returncode == 0 else {}


def short(name):
    name = name.replace("void ", "").replace("pb200::(anonymous namespace)::", "")
    return name.split("(")[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--mode", type=int, default=1, help="kernel mode (pb200_xlinear_set_lookup), 1 = default")
    ap.add_argument("--json", default=None, help="also write the numbers to this file")
    args = ap.parse_args()

    import numpy as np
    import torch
    from ctypes import byref
    from torch.profiler import ProfilerActivity, profile

    from pecos_b200 import core, synth
    from pecos_b200.core import ScipyCsrF32
    from pecos_b200.xlinear import XLinearModel

    cfg = dict(synth.WORKLOADS["eurlex-4k"])
    lib = core.get_clib()
    lib.require_gpu()
    lib.set_device(0)
    torch.cuda.init()
    with tempfile.TemporaryDirectory() as tmp:
        folder, _, _ = synth.build_workload("eurlex-4k", os.path.join(tmp, "eurlex-4k"), scale_queries=8)
        X = synth.make_queries(cfg["query_seed"], cfg["Q"], cfg["D"], cfg["nnz_per_row"], None)  # bench.py's batch
        m = XLinearModel.load(folder, is_predict_only=True)
    c = lib.clib_float32
    h = m.model.model_chain
    c.pb200_xlinear_set_lookup(h, args.mode)
    cx = ScipyCsrF32.init_from(X)
    c.pb200_xlinear_resident_upload_csr(h, byref(cx))
    beam, topk = cfg["beam_size"], cfg["only_topk"]
    for _ in range(args.warmup):
        c.pb200_xlinear_resident_predict(h, beam, None, topk, 0)
    c.pb200_xlinear_reset_profile(h)
    step_ms = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step_ms.append(c.pb200_xlinear_resident_predict(h, beam, None, topk, 0))  # ends in an event synchronise
            time.sleep(0.002)  # a clear gap between steps in the trace
    launches = int(c.pb200_xlinear_launches(h)) / args.steps
    kern = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.time_range.elapsed_us() >= 0:
            kern.append((e.time_range.start, e.time_range.end, short(e.name)))
    kern.sort()
    # steps: split where the stream sat idle for more than 1 ms (the host sleeps 2 ms between steps)
    steps, cur = [], []
    for k in kern:
        if cur and k[0] - cur[-1][1] > 1000:
            steps.append(cur)
            cur = []
        cur.append(k)
    if cur:
        steps.append(cur)
    per = defaultdict(list)
    for s in steps:
        for k in s:
            per[k[2]].append(k[1] - k[0])
    n = max(len(steps), 1)
    rows = sorted(((name, len(v) / n, float(np.mean(v))) for name, v in per.items()), key=lambda r: -r[1] * r[2])
    busy = [sum(k[1] - k[0] for k in s) for s in steps]
    span = [s[-1][1] - s[0][0] for s in steps]
    gaps = [sp - b for sp, b in zip(span, busy)]  # kernels of a step run back to back on one stream
    out = {"card": card(), "mode": args.mode, "steps": args.steps, "steps_in_trace": len(steps),
           "step_ms_events": float(np.median(step_ms)), "launches_per_step": launches,
           "busy_us_per_step": float(np.median(busy)), "span_us_per_step": float(np.median(span)),
           "gaps_us_per_step": float(np.median(gaps)),
           "kernels": [{"name": r[0], "per_step": r[1], "mean_us": r[2], "us_per_step": r[1] * r[2]} for r in rows]}
    print("card: %s" % out["card"])
    print("kernel mode %d: %d steps, step %.3f ms (events, median), %.1f launches per step" % (
        args.mode, len(steps), out["step_ms_events"], launches))
    print("  %-70s %8s %10s %12s" % ("kernel", "per step", "mean us", "us per step"))
    for r in out["kernels"]:
        print("  %-70s %8.2f %10.2f %12.2f" % (r["name"][:70], r["per_step"], r["mean_us"], r["us_per_step"]))
    print("per step (median): kernels busy %.1f us, first start to last end %.1f us, gaps between kernels %.1f us" % (
        out["busy_us_per_step"], out["span_us_per_step"], out["gaps_us_per_step"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
