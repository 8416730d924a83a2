"""What the per-point rows of a batched linearize cost: sgb_linearize_batch against sgb_linearize_batch_points, on one GPU.

Workloads, each at B in {1, 64, 512} (--sizes), GICP, max_dist_sq 1:
  pairs-kdtree: the LiDAR frame pairs of bench_align_async.py (frame i a kd-tree map, frame i + 1 the source), at the perturbed initial
      relative poses;
  room: members of 20k points against the 1M-point synthetic room of bench_align_batch.py (one device kd-tree), at perturbed poses.
Everything is built and resident, and one linearize has seeded the searches, before anything is timed.  The per-point calls are first
checked to return member sums bit-identical to the plain call.  Then, alternately, median of --reps, call to return (each call returns
with its results):
  plain_ms        Context.linearize_batch;
  e_host_ms       linearize_batch_points(hessians=False) into numpy (host) rows;
  e_dev_ms        the same into a CUDA tensor, written by the factor kernel;
  eHb_host_ms     linearize_batch_points with H | b rows, into numpy;
  eHb_dev_ms      the same into CUDA tensors.
row_bytes is what the rows hold (8 B of e + 336 B of H | b per point).  The card's name, power limit and maximum SM clock are read with
nvidia-smi (read-only) and written next to the numbers.

    python scripts/bench_batch_points.py [--sizes 1,64,512] [--reps 20] [--workloads pairs-kdtree,room] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_align_async import lidar_pairs  # noqa: E402
from bench_align_batch import gpu_info, se3_exp  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,64,512")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--workloads", default="pairs-kdtree,room")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sizes = [int(x) for x in args.sizes.split(",")]
    workloads = args.workloads.split(",")

    import torch

    import small_gicp_b200 as sg
    from small_gicp_b200.synthetic import make_pair

    info = gpu_info()
    print(json.dumps(info), flush=True)
    dev = torch.device("cuda:0")
    results = []

    def measure(name, B, ctx, inits):
        kw = dict(factor=sg.FACTOR_GICP, max_dist_sq=1.0)
        n = int(ctx._batch_offsets[-1])
        de = torch.empty(n, dtype=torch.float64, device=dev)
        dhb = torch.empty((n, 42), dtype=torch.float64, device=dev)
        he, hhb = np.empty(n), np.empty((n, 42))
        calls = {
            "plain": lambda: ctx.linearize_batch(inits, **kw),
            "e_host": lambda: ctx.linearize_batch_points(inits, hessians=False, out_e=he, **kw),
            "e_dev": lambda: ctx.linearize_batch_points(inits, hessians=False, out_e=de, **kw),
            "eHb_host": lambda: ctx.linearize_batch_points(inits, out_e=he, out_Hb42=hhb, **kw),
            "eHb_dev": lambda: ctx.linearize_batch_points(inits, out_e=de, out_Hb42=dhb, **kw),
        }
        H, b, e, _ = calls["plain"]()  # seeds the searches, as every later call is seeded
        for k in ("e_host", "eHb_host", "eHb_dev"):
            r = calls[k]()
            if not (np.array_equal(H, r.H) and np.array_equal(b, r.b) and np.array_equal(e, r.e)):
                raise SystemExit(f"{name} B = {B}: {k} sums differ from linearize_batch")
        if not (np.array_equal(de.cpu().numpy(), he) and np.array_equal(dhb.cpu().numpy(), hhb)):
            raise SystemExit(f"{name} B = {B}: device rows differ from host rows")
        times = {k: [] for k in calls}
        for _ in range(args.reps + 2):  # the first two of each are warm-up
            for k, f in calls.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                f()
                times[k].append(time.perf_counter() - t0)
        launches = {}
        for k, f in calls.items():
            k0 = ctx.kernel_launches
            f()
            launches[k] = ctx.kernel_launches - k0
        med = lambda x: 1e3 * float(np.median(x[2:]))
        rec = {"workload": name, "B": B, "points": n, "row_bytes": 344 * n, "launches": launches,
               **{f"{k}_ms": med(v) for k, v in times.items()},
               **{f"{k}_range_ms": [1e3 * min(v[2:]), 1e3 * max(v[2:])] for k, v in times.items()}, **info}
        print(json.dumps(rec), flush=True)
        results.append(rec)

    if "pairs-kdtree" in workloads:
        P, Cv, starts, inits = lidar_pairs(sg, torch, max(sizes), dev)
        ctx = sg.Context(0)
        for B in sizes:
            ctx.build_target_kdtrees((P[: starts[B]], starts[: B + 1]), None, Cv[: starts[B]])
            ctx.set_source_batch((P[starts[1] : starts[B + 1]], starts[1 : B + 2] - starts[1]), Cv[starts[1] : starts[B + 1]])
            measure("pairs-kdtree", B, ctx, np.ascontiguousarray(inits[:B]))
        ctx.close()
    if "room" in workloads:
        pool, n = 8, 20_000
        tgt, src, Tgt = make_pair(1_000_000, n_source=pool * n)
        ctx = sg.Context(0)
        ctx.set_target(tgt)
        ctx.build_target_kdtree()
        ctx.estimate_target_features(20)
        slices = [src[j * n : (j + 1) * n] for j in range(pool)]
        pts = [torch.from_numpy(np.c_[s, np.ones(len(s))]).to(dev) for s in slices]
        covs = [ctx.estimate_features(p, 20, normals=False)[1] for p in pts]
        ctx.set_source_batch((torch.cat(pts), np.arange(pool + 1, dtype=np.uint64) * n), torch.cat(covs))
        for B in sizes:
            rng = np.random.default_rng(B)
            inits = np.empty((B, 4, 4))
            for m in range(B):
                d = np.r_[rng.normal(size=3) * np.deg2rad(1.5), rng.uniform(-1, 1, 3) * 0.15]
                inits[m] = se3_exp(d[None])[0] @ Tgt
            ctx.set_source_pairs([m % pool for m in range(B)])
            measure("room", B, ctx, inits)
        ctx.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"setup": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
