"""What the device-driven GNC loop (sgb_align_batch_gnc_async) saves against the host-driven one (sgb_align_batch_gnc), on one GPU.

Workloads: those of bench_align_gnc.py -- the LiDAR frame pairs (frame i a kd-tree map, frame i + 1 the source, 0.25 m voxel grid, GICP,
max_dist_sq 1, LM with 20 iterations, initial poses ground truth times 0.5 degree of yaw and 0.1 m), each source frame corrupted by a
moved rigid object (moved15 / moved30) or uniform clutter (clutter30 / clutter50 / clutter70), at B in {64, 512}, GNC-GM and GNC-TLS
with stage_iterations 3 and max_stages 64, c^2 the 90th percentile of r^2 of the clean pairs at the ground truth.
Per workload and GNC kind, on one context with its stream set to a torch stream: first every async output (T, info, H | b, stages and
mu, each point's g) is checked bit-identical to the synchronous call's; then sync and async calls alternate, --reps of each after one
warm-up, and the medians are reported in ms per call:
  sync      align_batch_gnc (it synchronises);
  async     align_batch_gnc_async to the end of the context's synchronize();
  return    align_batch_gnc_async to its return (the binding's pose transposition included);
  first     the first async call of the kind, to the end of synchronize(): it captures and instantiates the graph.
The card's name, power limit and maximum SM clock are read with nvidia-smi (read-only) in the same run and written next to the numbers.

    python scripts/bench_align_gnc_async.py [--sizes 64,512] [--reps 7] [--corruptions moved30,clutter50] [--out FILE]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_align_batch import gpu_info, se3_exp  # noqa: E402
from bench_align_gnc import corrupt  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="64,512")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--corruptions", default="moved30,clutter50")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sizes = [int(x) for x in args.sizes.split(",")]

    import torch

    import small_gicp_b200 as sg
    from small_gicp_b200 import synthetic as syn

    info = gpu_info()
    print(json.dumps(info), flush=True)
    dev = torch.device("cuda:0")
    K = max(sizes)
    world = syn.make_world(16_000_000, 42)
    side = syn.world_side(16_000_000)
    poses = [syn.lidar_pose(f, side) for f in range(K + 1)]
    prep = sg.Context(0)
    frames = [prep.voxelgrid_sampling(syn.lidar_frame_torch(world, poses[f], 45 + f, dev).cpu().numpy(), 0.25) for f in range(K + 1)]
    cov = lambda p: prep.estimate_features(p, 20, normals=False)[1]
    covs = [cov(p) for p in frames]
    noise = se3_exp(np.array([[0.0, 0.0, np.deg2rad(0.5), 0.1, 0.0, 0.0]]))[0]
    gt = np.array([np.linalg.inv(poses[i]) @ poses[i + 1] for i in range(K)])
    inits = np.array([g @ noise for g in gt])
    kw = dict(factor=sg.FACTOR_GICP, max_dist_sq=1.0, max_iterations=20, stage_iterations=3, max_stages=64)
    stream = torch.cuda.Stream()
    results = []

    def batch(ctx, B, src, scov):
        off = np.zeros(B + 1, dtype=np.int64)
        off[1:] = np.cumsum([len(p) for p in src[:B]])
        ctx.set_source_batch((np.concatenate(src[:B]), off), np.concatenate(scov[:B]))

    def same(a, b):
        a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
        return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))

    for B in sizes:
        ctx = sg.Context(0)
        ctx.set_stream(stream.cuda_stream)
        off = np.zeros(B + 1, dtype=np.int64)
        off[1:] = np.cumsum([len(p) for p in frames[:B]])
        ctx.build_target_kdtrees((np.concatenate(frames[:B]), off), None, np.concatenate(covs[:B]))
        batch(ctx, B, frames[1:], covs[1:])
        t = ctx.linearize_batch_points(gt[:B], factor=sg.FACTOR_GICP, max_dist_sq=1.0, hessians=False)
        matched = np.concatenate(ctx.correspondences_batch()) != sg.NO_CORRESPONDENCE
        c2 = float(np.quantile(2.0 * t.point_e[matched], 0.9))
        Td = torch.from_numpy(np.ascontiguousarray(inits[:B])).to(dev)
        for corr in args.corruptions.split(","):
            rng = np.random.default_rng(B)
            src = [corrupt(p, corr, rng) for p in frames[1 : B + 1]]
            scov = [cov(p) for p in src]
            batch(ctx, B, src, scov)
            for name, kind in (("gm", sg.GNC_GEMAN_MCCLURE), ("tls", sg.GNC_TLS)):

                def sync():
                    return ctx.align_batch_gnc(inits[:B], c2, gnc=kind, **kw)

                def enqueue(point_weights=False, out=None):
                    with torch.cuda.stream(stream):
                        return ctx.align_batch_gnc_async(Td, c2, gnc=kind, point_weights=point_weights, out=out, **kw)

                # the first async call of the kind builds its graph; its result is the one checked against the synchronous call
                ctx.synchronize()
                t0 = time.perf_counter()
                a = enqueue(point_weights=True)
                ctx.synchronize()
                first = time.perf_counter() - t0
                r = ctx.align_batch_gnc(inits[:B], c2, gnc=kind, point_weights=True, **kw)
                ok = all(same(getattr(r, f), getattr(a, f).cpu().numpy()) for f in ("T_target_source", "H", "b", "error", "mu", "point_w"))
                ok = ok and all(same(np.asarray(getattr(r, f), dtype=np.float64), getattr(a, f).cpu().numpy())
                                for f in ("converged", "iterations", "num_inliers", "stages"))
                if not ok:
                    raise SystemExit(f"{corr} B={B} {name}: the async result differs from align_batch_gnc")
                out = enqueue()
                times = {"sync": [], "async": [], "return": []}
                for rep in range(args.reps + 1):  # the first is the warm-up
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    sync()
                    ts = time.perf_counter() - t0
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    enqueue(out=out)
                    tr = time.perf_counter() - t0
                    ctx.synchronize()
                    ta = time.perf_counter() - t0
                    if rep:
                        times["sync"].append(ts)
                        times["async"].append(ta)
                        times["return"].append(tr)
                rec = {"workload": corr, "B": B, "gnc": name, "points": int(ctx._batch_offsets[-1]), "c2": c2, "bit_identical": ok,
                       "stages_median": float(np.median(r.stages)), "stages_max": int(r.stages.max()), "first_ms": 1e3 * first, **info}
                for k, v in times.items():
                    rec[k + "_ms"] = 1e3 * float(np.median(v))
                    rec[k + "_ms_range"] = [1e3 * float(np.min(v)), 1e3 * float(np.max(v))]
                rec["sync_over_async"] = rec["sync_ms"] / rec["async_ms"]
                print(json.dumps(rec), flush=True)
                results.append(rec)
        ctx.set_stream(None)
        ctx.close()
    prep.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"setup": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
