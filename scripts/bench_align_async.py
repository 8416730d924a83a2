"""Per-align latency of the stream-ordered batched align (sgb_align_batch_async) against sgb_align_batch, on one GPU.

Workloads, each at B in {1, 8, 64, 512} (--sizes), GICP:
  pairs-voxelmap / pairs-kdtree: the LiDAR frame pairs of bench_align_pairs.py (frame i the map, frame i + 1 the source, leaf 1.0 voxel
      maps or kd-trees of the frames, Levenberg-Marquardt);
  room: members of 20k points against the 1M-point synthetic room of bench_align_batch.py (one device kd-tree), Levenberg-Marquardt.
Everything is built and resident before anything is timed; poses are on the device for the asynchronous call, on the host for the
synchronous one (its interface).  The two are checked to reach bit-identical poses first, then timed alternately, median of --reps:
  sync_ms        Context.align_batch, call to return (it returns with the results);
  async_ms       Context.align_batch_async, call to the end of ctx.synchronize();
  async_return_ms  call to return of align_batch_async (the host is free from then on);
  first_async_ms   the first asynchronous call of a workload and size (the loop graph is captured and instantiated), call to synchronize.
The card's name, power limit and maximum SM clock are read with nvidia-smi (read-only) and written next to the numbers.

    python scripts/bench_align_async.py [--sizes 1,8,64,512] [--reps 10] [--workloads pairs-voxelmap,pairs-kdtree,room] [--out FILE]
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


def lidar_pairs(sg, torch, n_pairs, dev):
    """(points, covs) of n_pairs + 1 consecutive sampled LiDAR frames on the device, and the perturbed initial relative poses"""
    from small_gicp_b200 import synthetic as syn

    world = syn.make_world(16_000_000, 42)
    side = syn.world_side(16_000_000)
    poses = [syn.lidar_pose(f, side) for f in range(n_pairs + 1)]
    prep = sg.Context(0)
    frames, covs = [], []
    for f in range(n_pairs + 1):
        p = prep.voxelgrid_sampling(syn.lidar_frame_torch(world, poses[f], 45 + f, dev).cpu().numpy(), 0.25)
        frames.append(p)
        covs.append(prep.estimate_features(p, 20, normals=False)[1])
    noise = se3_exp(np.array([[0.0, 0.0, np.deg2rad(0.5), 0.1, 0.0, 0.0]]))[0]
    inits = np.array([np.linalg.inv(poses[i]) @ poses[i + 1] @ noise for i in range(n_pairs)])
    starts = np.zeros(n_pairs + 2, dtype=np.int64)
    starts[1:] = np.cumsum([len(p) for p in frames])
    return torch.from_numpy(np.concatenate(frames)).to(dev), torch.from_numpy(np.concatenate(covs)).to(dev), starts, inits


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,64,512")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--workloads", default="pairs-voxelmap,pairs-kdtree,room")
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
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    results = []

    def measure(name, B, ctx, inits, kw):
        ctx.set_stream(stream.cuda_stream)
        Td = torch.from_numpy(inits).to(dev)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = ctx.align_batch_async(Td, **kw)
        ctx.synchronize()
        first = time.perf_counter() - t0
        r = ctx.align_batch(inits, **kw)
        same = bool(np.array_equal(r.T_target_source, out.T_target_source.cpu().numpy()))
        if not same:
            raise SystemExit(f"{name} B = {B}: the asynchronous align differs from align_batch")
        ts, ta, tr = [], [], []
        for _ in range(args.reps + 2):  # the first two of each are warm-up
            t0 = time.perf_counter()
            ctx.align_batch(inits, **kw)
            ts.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            ctx.align_batch_async(Td, out=out, **kw)
            t1 = time.perf_counter()
            ctx.synchronize()
            t2 = time.perf_counter()
            tr.append(t1 - t0)
            ta.append(t2 - t0)
        med = lambda x: 1e3 * float(np.median(x[2:]))
        k0 = ctx.kernel_launches
        ctx.align_batch(inits, **kw)
        k1 = ctx.kernel_launches
        ctx.align_batch_async(Td, out=out, **kw)
        k2 = ctx.kernel_launches
        ctx.synchronize()
        rec = {"workload": name, "B": B, "bit_identical": same, "iterations_max": int(r.iterations.max()), "launches_sync": k1 - k0, "launches_async": k2 - k1,
               "sync_ms": med(ts), "async_ms": med(ta), "async_return_ms": med(tr), "first_async_ms": 1e3 * first,
               "sync_range_ms": [1e3 * min(ts[2:]), 1e3 * max(ts[2:])], "async_range_ms": [1e3 * min(ta[2:]), 1e3 * max(ta[2:])],
               "speedup": float(np.median(ts[2:]) / np.median(ta[2:])), **info}
        print(json.dumps(rec), flush=True)
        results.append(rec)

    if any(w.startswith("pairs") for w in workloads):
        P, Cv, starts, inits = lidar_pairs(sg, torch, max(sizes), dev)
        for w in [w for w in workloads if w.startswith("pairs")]:
            ctx = sg.Context(0)
            for B in sizes:
                tgt = ((P[: starts[B]], starts[: B + 1]), Cv[: starts[B]])
                if w == "pairs-kdtree":
                    ctx.build_target_kdtrees(tgt[0], None, tgt[1])
                else:
                    ctx.build_target_voxelmaps(*tgt, 1.0, 1)
                ctx.set_source_batch((P[starts[1] : starts[B + 1]], starts[1 : B + 2] - starts[1]), Cv[starts[1] : starts[B + 1]])
                measure(w, B, ctx, np.ascontiguousarray(inits[:B]), dict(factor=sg.FACTOR_GICP, optimizer=1))
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
            measure("room", B, ctx, inits, dict(factor=sg.FACTOR_GICP, optimizer=1))
        ctx.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"setup": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
