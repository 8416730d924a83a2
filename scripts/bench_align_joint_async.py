"""Per-call latency of the stream-ordered joint window align (sgb_align_joint_async) against sgb_align_joint, on one GPU.

Workloads: the rows of DESIGN §11 "Joint windows" -- K consecutive frames of the synthetic LiDAR stream of bench_align_joint.py (16M-point
world, voxel-grid sampled at 0.25 m, k = 20 covariances, all outside the timed window), windows of W frames with c edges back, the first
frame of every window fixed at ground truth and the others perturbed by ~2 deg / 0.3 m; GICP, Levenberg-Marquardt, max_dist_sq 4, on many
kd-trees or many voxel maps (leaf 1.0).  Both calls run on one context, alternated, median of --reps after 2 warm-ups:
  sync_ms          Context.align_joint, call to return (it ends in a host synchronisation);
  async_ms         Context.align_joint_async, call to the end of ctx.synchronize();
  async_return_ms  call to return of align_joint_async (the host is free from then on);
  first_async_ms   the first async call of the workload, to the end of synchronize(): table upload, capture and instantiation of the loop.
Before timing, every async result (X and info) is checked bit-identical to align_joint's.  The card's name, power limit and maximum SM clock
(nvidia-smi, read-only) go with every row.

    python scripts/bench_align_joint_async.py [--rows K:W:c:kind,...] [--reps 7] [--out FILE]
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

from bench_align_batch import gpu_info, se3_exp  # noqa: E402

ROWS = "64:8:2:kdtree,64:8:4:kdtree,64:16:2:kdtree,64:16:4:kdtree,64:8:2:voxelmap,64:16:4:voxelmap,512:8:2:kdtree,512:16:4:kdtree,512:16:4:voxelmap"
LEAF, OFFSETS = 1.0, 1
LM = 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default=ROWS)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    rows = [(int(K), int(W), int(c), kind) for K, W, c, kind in (r.split(":") for r in args.rows.split(","))]

    import torch

    import small_gicp_b200 as sg
    from small_gicp_b200 import synthetic as syn

    info = gpu_info()
    print(json.dumps(info), flush=True)
    dev = torch.device("cuda:0")
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    K_max = max(r[0] for r in rows)
    world = syn.make_world(16_000_000, 42)
    side = syn.world_side(16_000_000)
    G = [syn.lidar_pose(f, side) for f in range(K_max)]
    prep = sg.Context(0)
    frames, covs = [], []
    for f in range(K_max):
        p = prep.voxelgrid_sampling(syn.lidar_frame_torch(world, G[f], 45 + f, dev).cpu().numpy(), 0.25)
        frames.append(torch.from_numpy(p).to(dev))
        covs.append(torch.from_numpy(prep.estimate_features(p, 20, normals=False)[1]).to(dev))
    prep.close()
    del world
    rng = np.random.default_rng(2026)
    noise = [se3_exp(np.r_[rng.normal(size=3) * np.deg2rad(2.0) / np.sqrt(3), rng.normal(size=3) * 0.3 / np.sqrt(3)][None])[0] for _ in range(K_max)]
    kw = dict(factor=sg.FACTOR_GICP, optimizer=LM, max_dist_sq=4.0)
    results = []
    for K, W, c, kind in rows:
        offs = np.zeros(K + 1, dtype=np.int64)
        offs[1:] = np.cumsum([len(frames[i]) for i in range(K)])
        pts, cv = (torch.cat(frames[:K]), offs), torch.cat(covs[:K])
        woff = list(range(0, K, W)) + [K]
        first = {k: woff[k // W] for k in range(K)}
        X0 = np.array([G[k] if k == first[k] else G[k] @ noise[k] for k in range(K)])
        edges = [(i, i - d) for i in range(K) for d in range(1, c + 1) if i - d >= first[i]]
        ctx = sg.Context(0)
        ctx.set_stream(stream.cuda_stream)
        if kind == "kdtree":
            ctx.build_target_kdtrees(pts, None, cv)
        else:
            ctx.build_target_voxelmaps(pts, cv, LEAF, OFFSETS)
        ctx.set_source_batch(pts, cv)
        ctx.set_source_pairs(np.array([e[0] for e in edges], dtype=np.uint32), np.array([e[1] for e in edges], dtype=np.uint32))
        Xd = torch.from_numpy(X0).to(dev)
        r = ctx.align_joint(X0, windows=woff, **kw)  # (also builds the pairing's view of the target)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = ctx.align_joint_async(Xd, windows=woff, **kw)
        ctx.synchronize()
        first_ms = 1e3 * (time.perf_counter() - t0)
        same = bool(np.array_equal(r.X.view(np.uint64), out.X.cpu().numpy().view(np.uint64)) and
                    np.array_equal(np.c_[r.converged, r.iterations, r.num_inliers, r.error], out.info4.cpu().numpy()))
        if not same:
            raise SystemExit(f"K={K} W={W} c={c} {kind}: the asynchronous joint align differs from align_joint")
        ts, ta, tr = [], [], []
        for _ in range(args.reps + 2):  # the first two of each are warm-up
            t0 = time.perf_counter()
            ctx.align_joint(X0, windows=woff, **kw)
            ts.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            ctx.align_joint_async(Xd, windows=woff, out=out, **kw)
            t1 = time.perf_counter()
            ctx.synchronize()
            t2 = time.perf_counter()
            tr.append(t1 - t0)
            ta.append(t2 - t0)
        med = lambda x: 1e3 * float(np.median(x[2:]))
        k0 = ctx.kernel_launches
        ctx.align_joint(X0, windows=woff, **kw)
        k1 = ctx.kernel_launches
        ctx.align_joint_async(Xd, windows=woff, out=out, **kw)
        k2 = ctx.kernel_launches
        ctx.synchronize()
        rec = {"workload": f"K={K} W={W} c={c} {kind}", "windows": len(woff) - 1, "edges": len(edges), "bit_identical": same,
               "iterations_max": int(r.iterations.max()), "launches_sync": k1 - k0, "launches_async": k2 - k1,
               "sync_ms": med(ts), "async_ms": med(ta), "async_return_ms": med(tr), "first_async_ms": first_ms,
               "sync_range_ms": [1e3 * min(ts[2:]), 1e3 * max(ts[2:])], "async_range_ms": [1e3 * min(ta[2:]), 1e3 * max(ta[2:])],
               "speedup": float(np.median(ts[2:]) / np.median(ta[2:])), **info}
        print(json.dumps(rec), flush=True)
        results.append(rec)
        ctx.close()
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"setup": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
