#!/usr/bin/env python3
"""Per-kernel device time of the headline step (bench.py `value`), pose by pose.

Builds the same 1M x 1M GICP pair as bench.py, walks its Gauss-Newton pose schedule with linearize_device (the identity pose
unseeded, later poses seeded by their predecessor, the L2 flushed before every step) and records every kernel with torch.profiler
(CUDA activities).  The kernels of each step are those between two flushes; they are grouped into the grid probe, the packet /
pending search, the factor kernel and everything else, and reported per pose as the median over the repetitions with the
min / max beside it.

  python scripts/profile_kernels.py [--points N] [--reps R] [--out DIR]

Writes DIR/profile_kernels.json (and the raw trace, DIR/trace.pt.trace.json) and prints one JSON line.  Needs a GPU.
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GROUPS = (("probe", "grid_probe"), ("packet", "packet_search"), ("factor", "factor_reduce"))


def group_of(name):
    for g, key in GROUPS:
        if key in name:
            return g
    return "other"


def is_flush(name):
    return "at::native" in name  # the flush buffer's zero_() is the only torch kernel inside a step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=20, help="passes over the pose schedule inside the profiled window")
    ap.add_argument("--out", default=None, help="output directory (default: a temporary directory)")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    import small_gicp_b200 as sg

    if not torch.cuda.is_available():
        raise SystemExit("profile_kernels.py: no CUDA device")
    out_dir = args.out or tempfile.mkdtemp(prefix="sgb_profile_")
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    out = torch.zeros(64, dtype=torch.float64, device=dev)
    GICP = dict(factor=sg.FACTOR_GICP, rejector=sg.REJECT_DISTANCE, max_dist_sq=1.0)

    ctx = sg.Context(0)
    ctx.set_stream(stream.cuda_stream)
    inp = bench.make_inputs(args.points, 0, "knn", lambda p4: ctx.estimate_features(p4, 20, normals=False)[1])
    ctx.set_target(inp["target"], None, inp["target_covs"])
    ctx.build_target_kdtree()
    ctx.set_source(inp["source"], inp["source_covs"])
    poses, _ = bench.gn_trajectory(lambda T: ctx.linearize(T, **GICP))
    P = len(poses)

    def step(k):
        flush.zero_()
        if k == 0:
            ctx.drop_seeds()
        ctx.linearize_device(poses[k], out.data_ptr(), **GICP)

    for _ in range(3):  # warm every pose
        for k in range(P):
            step(k)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            for k in range(P):
                step(k)
        torch.cuda.synchronize()
    trace = os.path.join(out_dir, "trace.pt.trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        ev = json.load(f)["traceEvents"]
    kern = sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    steps, cur = [], None
    for e in kern:
        if is_flush(e["name"]):
            cur = {}
            steps.append(cur)
            continue
        if cur is None:
            continue
        g = group_of(e["name"])
        cur[g] = cur.get(g, 0.0) + e["dur"] / 1e3  # ms
        cur.setdefault("_names", set()).add(e["name"].split("(")[0].split("<")[0])
    if len(steps) != args.reps * P:
        raise SystemExit(f"profile_kernels.py: found {len(steps)} steps in the trace, expected {args.reps * P}")
    names = sorted(set().union(*(s.pop("_names", set()) for s in steps)))
    per_pose = []
    for k in range(P):
        rows = steps[k::P]
        entry = {"pose": k}
        for g in [g for g, _ in GROUPS] + ["other", "total"]:
            v = np.array([sum(x for kk, x in r.items()) if g == "total" else r.get(g, 0.0) for r in rows])
            entry[g] = {"median_ms": float(np.median(v)), "min_ms": float(v.min()), "max_ms": float(v.max())}
        tot = entry["total"]["median_ms"]
        entry["share"] = {g: entry[g]["median_ms"] / tot if tot > 0 else 0.0 for g, _ in GROUPS}
        per_pose.append(entry)
    props = torch.cuda.get_device_properties(0)
    res = {
        "device": props.name,
        "points": args.points,
        "poses": P,
        "reps": args.reps,
        "kernels": names,
        "per_pose": per_pose,
        "what": "kernel time per step from torch.profiler (CUDA activities), L2 flushed before each step; median (min, max) over reps",
    }
    with open(os.path.join(out_dir, "profile_kernels.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
