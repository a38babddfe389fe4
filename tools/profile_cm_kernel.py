"""Where the time of the chunk-major score kernel goes on the eurlex-4k leaf (diagnostic; needs a GPU).

Builds a side copy of the library with -DPB200_CM_TRACE into a temporary directory (pecos_b200/lib is not touched), runs
the eurlex-4k workload of bench.py (same model and query seeds) through it, and prints, for the last launch of
xl_cm_scores_kernel (the leaf layer):
  * per-CTA elapsed time from %globaltimer (max / mean / min over the CTAs, and max / mean);
  * per-warp clock64 cycles by phase: chunk switch (barrier + choice of the next chunk), bulk-copy wait, query staging
    wait, lookup + compaction, accumulate, slice set-up + output (mean over the warps, and the share of each phase);
  * accumulate trips per warp and lane efficiency: entries added / (trips x 32 lanes x 4 slots);
  * per CTA: slices claimed, images staged (chunk switches + 1) and pairs scored (mean / min / max).
It fails if the pairs scored, summed over the CTAs, differ from the pairs bucketed for the launch: every pair must be
claimed exactly once.  The product build never defines PB200_CM_TRACE.

    python tools/profile_cm_kernel.py [--queries N] [--json OUT]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ["switch_choice", "copy_wait", "staging_wait", "lookup_compact", "accumulate", "slice_setup_output"]
MAX_WARPS = 16  # kCmMaxWarps
TRACE_CTAS = 1024  # kCmTraceCtas
WARP_FIELDS = len(PHASES) + 4  # kCmTraceWarp: phase cycles, trips, useful slots, slices, pairs
HEAD, CTA_HEAD = 3, 3  # g_cm_trace: grid, warps, pairs of the launch; per CTA: start ns, end ns, images staged
SLOTS = 4  # kCmSlots


def build_traced(out_dir):
    from pecos_b200 import build as b

    lib = os.path.join(out_dir, "libpecos_b200_float32_cmtrace.so")
    cmd = [os.environ.get("NVCC", "nvcc")] + b.NVCC_FLAGS + ["-DPB200_CM_TRACE"] + b.sources() + ["-o", lib]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stdout.write(r.stdout)
        raise RuntimeError("nvcc failed building the traced library")
    return lib


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=None, help="default: the workload's batch (15,449 queries)")
    ap.add_argument("--repeats", type=int, default=3, help="predict calls; the trace is the last one's")
    ap.add_argument("--json", default=None, help="also write the numbers to this file")
    args = ap.parse_args()

    from pecos_b200 import core, synth
    from pecos_b200.xlinear import XLinearModel

    with tempfile.TemporaryDirectory() as tmp:
        core._clib = core.B200CoreLib(build_traced(tmp))
        c = core._clib.clib_float32
        c.pb200_cm_trace_fetch.restype = ctypes.c_int
        c.pb200_cm_trace_fetch.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_ulonglong]
        core._clib.require_gpu()
        core._clib.set_device(0)
        folder, X, cfg = synth.build_workload("eurlex-4k", os.path.join(tmp, "eurlex-4k"))
        if args.queries:
            X = X[: args.queries]
        m = XLinearModel.load(folder, is_predict_only=True)
        depth = len(cfg["layer_sizes"])
        for _ in range(args.repeats):
            m.predict(X, beam_size=cfg["beam_size"], only_topk=cfg["only_topk"])
        kid = (ctypes.c_int * (2 * depth))()
        c.pb200_xlinear_get_kernel_ids(m.model.model_chain, kid)
        if kid[2 * (depth - 1)] != 4:
            raise RuntimeError(f"the leaf layer did not run the chunk-major kernel (score kernel id {kid[2 * (depth - 1)]})")
        per_cta = CTA_HEAD + MAX_WARPS * WARP_FIELDS
        buf = (ctypes.c_ulonglong * (HEAD + TRACE_CTAS * per_cta))()
        if c.pb200_cm_trace_fetch(buf, len(buf)) != 0:
            raise RuntimeError("pb200_cm_trace_fetch failed")
    raw = np.frombuffer(buf, dtype=np.uint64)
    grid, warps, launch_pairs = int(raw[0]), int(raw[1]), int(raw[2])
    rec = raw[HEAD: HEAD + grid * per_cta].reshape(grid, per_cta)
    cta_us = (rec[:, 1].astype(np.float64) - rec[:, 0].astype(np.float64)) / 1e3
    images = rec[:, 2].astype(np.int64)
    per_warp = rec[:, CTA_HEAD:].reshape(grid, MAX_WARPS, WARP_FIELDS)[:, :warps, :].astype(np.float64)
    cyc = per_warp[:, :, : len(PHASES)]
    trips, slots = per_warp[:, :, len(PHASES)], per_warp[:, :, len(PHASES) + 1]
    slices = per_warp[:, :, len(PHASES) + 2].sum(axis=1).astype(np.int64)
    pairs = per_warp[:, :, len(PHASES) + 3].sum(axis=1).astype(np.int64)
    phase_mean = cyc.mean(axis=(0, 1))
    warp_total = cyc.sum(axis=2)
    out = {
        "queries": int(X.shape[0]), "grid": grid, "warps_per_cta": warps,
        "cta_us": {"max": float(cta_us.max()), "mean": float(cta_us.mean()), "min": float(cta_us.min()),
                   "max_over_mean": float(cta_us.max() / cta_us.mean())},
        "warp_cycles": {"mean_total": float(warp_total.mean()), "max_total": float(warp_total.max()),
                        "phases_mean": {p: float(v) for p, v in zip(PHASES, phase_mean)},
                        "phases_share": {p: float(v / phase_mean.sum()) for p, v in zip(PHASES, phase_mean)}},
        "accumulate": {"trips_per_warp": float(trips.mean()), "entries_per_warp": float(slots.mean()),
                       "lane_efficiency": float(slots.sum() / max(trips.sum() * 32 * SLOTS, 1.0))},
        "per_cta": {name: {"mean": float(v.mean()), "min": int(v.min()), "max": int(v.max())}
                    for name, v in (("slices", slices), ("images_staged", images), ("pairs", pairs))},
        "pairs": {"launch": launch_pairs, "scored": int(pairs.sum())},
    }
    print(f"leaf: {out['queries']} queries, {grid} CTAs x {warps} warps")
    print("CTA elapsed (us): max %.1f  mean %.1f  min %.1f  max/mean %.3f" % (
        out["cta_us"]["max"], out["cta_us"]["mean"], out["cta_us"]["min"], out["cta_us"]["max_over_mean"]))
    print("warp cycles: mean total %.0f, max total %.0f" % (out["warp_cycles"]["mean_total"], out["warp_cycles"]["max_total"]))
    for p in PHASES:
        print("  %-20s %12.0f  %5.1f %%" % (p, out["warp_cycles"]["phases_mean"][p], 100 * out["warp_cycles"]["phases_share"][p]))
    acc = out["accumulate"]
    print("accumulate: %.0f trips and %.0f entries per warp, lane efficiency %.3f" % (
        acc["trips_per_warp"], acc["entries_per_warp"], acc["lane_efficiency"]))
    for name, v in out["per_cta"].items():
        print("per CTA %-14s mean %8.1f  min %6d  max %6d" % (name, v["mean"], v["min"], v["max"]))
    print("pairs: %d bucketed, %d scored" % (launch_pairs, out["pairs"]["scored"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    if out["pairs"]["scored"] != launch_pairs:
        raise SystemExit(f"the CTAs scored {out['pairs']['scored']} pairs, the launch has {launch_pairs}")


if __name__ == "__main__":
    main()
