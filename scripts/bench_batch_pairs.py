"""Batched registration over (cloud, map) pairs (sgb_source_set_pairs) against repeating the clouds and maps, on one GPU.

Workloads:
  window       K in {64, 512} consecutive frames of the synthetic LiDAR stream (synthetic.lidar_frame_torch in the 16M-point world, 1 m
               forward + 1 deg yaw per frame), each voxel-grid sampled at 0.25 m with k = 20 covariances estimated on the device, all
               outside the timed window and kept on the device.  Frame i is aligned against each of its c in {4, 8} predecessors
               (pose-graph / sliding-window edges), from the ground-truth relative pose perturbed by 0.5 deg / 0.1 m.  GICP on kd-trees
               and VGICP on voxel maps (leaf 1.0), Levenberg-Marquardt.
  multi-start  64 clouds of 20k points of the 1M-point synthetic room (synthetic.make_pair) x 16 initial poses each (<= 0.5 m, <= 5 deg
               about the cloud's centre) against the room on a device kd-tree with device-estimated covariances, Gauss-Newton.

Compared in one process, repetitions alternated, median of --reps:
  (a) pairs: every map built once, every cloud stored once (set_source_batch), set_source_pairs, align_batch;
  (b) repeat: one map per edge (the frame repeated), one cloud per edge (the frame repeated), align_batch.
(a) and (b) are checked to reach bit-identical poses and iterations before anything is timed.  Reported: build, store, pairing and align
times (per edge), kernel launches per call, the device memory the set-up takes (torch.cuda.mem_get_info around it), and the card's name,
power limit and maximum SM clock (nvidia-smi, read-only).

    python scripts/bench_batch_pairs.py [--reps 5] [--out FILE]
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

LEAF, OFFSETS = 1.0, 1
GN, LM = 0, 1  # sgb_optimizer_kind


def timed(ctx, fn):
    ctx.synchronize()
    t0 = time.perf_counter()
    out = fn()
    ctx.synchronize()
    return time.perf_counter() - t0, out


def compare(sg, torch, name, run_a, run_b, n_edges, reps, info):
    """run_a / run_b (ctx) -> (dict of phase -> seconds, result); both on fresh contexts first (memory, launches, identity), then alternated"""
    free0 = torch.cuda.mem_get_info()[0]
    ctx_a = sg.Context(0)
    k0 = ctx_a.kernel_launches
    pa, ra = run_a(ctx_a)
    ka = ctx_a.kernel_launches - k0
    mem_a = free0 - torch.cuda.mem_get_info()[0]
    free1 = torch.cuda.mem_get_info()[0]
    ctx_b = sg.Context(0)
    k0 = ctx_b.kernel_launches
    pb, rb = run_b(ctx_b)
    kb = ctx_b.kernel_launches - k0
    mem_b = free1 - torch.cuda.mem_get_info()[0]
    same = bool(np.array_equal(ra.T_target_source, rb.T_target_source) and np.array_equal(ra.iterations, rb.iterations))
    print(json.dumps({"workload": name, "bit_identical": same}), flush=True)
    if not same:
        raise SystemExit(f"(a) and (b) differ: {name}")
    ta, tb = {k: [] for k in pa}, {k: [] for k in pb}
    for _ in range(reps):
        for t, run, ctx in ((ta, run_a, ctx_a), (tb, run_b, ctx_b)):
            ph, _ = run(ctx)
            for k, v in ph.items():
                t[k].append(v)
    med = lambda x: 1e3 * float(np.median(x))
    rec = {"workload": name, "edges": n_edges, "iterations_max": int(ra.iterations.max()), "converged": int(ra.converged.sum()),
           "launches_a": ka, "launches_b": kb, "device_mib_a": mem_a / 2**20, "device_mib_b": mem_b / 2**20}
    for tag, t in (("a", ta), ("b", tb)):
        total = np.sum([t[k] for k in t], axis=0)
        rec[f"{tag}_total_ms"] = med(total)
        rec[f"{tag}_per_edge_ms"] = med(total) / n_edges
        for k in t:
            rec[f"{tag}_{k}_per_edge_ms"] = med(t[k]) / n_edges
    rec["speedup_a_over_b"] = rec["b_total_ms"] / rec["a_total_ms"]
    rec.update(info)
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", default="64,512")
    ap.add_argument("--window", default="4,8")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    frames_list = [int(x) for x in args.frames.split(",")]
    windows = [int(x) for x in args.window.split(",")]

    import torch

    import small_gicp_b200 as sg
    from small_gicp_b200 import synthetic as syn

    info = gpu_info()
    print(json.dumps(info), flush=True)
    dev = torch.device("cuda:0")
    results = []

    # ---- window ----
    K_max = max(frames_list)
    world = syn.make_world(16_000_000, 42)
    side = syn.world_side(16_000_000)
    poses = [syn.lidar_pose(f, side) for f in range(K_max)]
    prep = sg.Context(0)
    frames, covs = [], []
    for f in range(K_max):
        p = prep.voxelgrid_sampling(syn.lidar_frame_torch(world, poses[f], 45 + f, dev).cpu().numpy(), 0.25)
        frames.append(torch.from_numpy(p).to(dev))
        covs.append(torch.from_numpy(prep.estimate_features(p, 20, normals=False)[1]).to(dev))
    del world
    noise = se3_exp(np.array([[0.0, 0.0, np.deg2rad(0.5), 0.1, 0.0, 0.0]]))[0]
    print(json.dumps({"frames": K_max, "points_per_frame_mean": float(np.mean([len(p) for p in frames]))}), flush=True)

    def concat(idx):
        offs = np.zeros(len(idx) + 1, dtype=np.int64)
        offs[1:] = np.cumsum([len(frames[i]) for i in idx])
        return (torch.cat([frames[i] for i in idx]), offs), torch.cat([covs[i] for i in idx])

    for K in frames_list:
        for c in windows:
            edges = [(i, i - j) for i in range(1, K) for j in range(1, c + 1) if i - j >= 0]  # (source frame, target frame)
            cl = np.array([e[0] for e in edges], dtype=np.uint32)
            mp = np.array([e[1] for e in edges], dtype=np.uint32)
            inits = np.array([np.linalg.inv(poses[t]) @ poses[s] @ noise for s, t in edges])
            all_pts, all_covs = concat(range(K))
            rep_tgt_pts, rep_tgt_covs = concat(mp)
            rep_src_pts, rep_src_covs = concat(cl)
            for kind in ("kdtree", "voxelmap"):
                kw = dict(factor=sg.FACTOR_GICP, optimizer=LM)

                def build(ctx, pts, cv):
                    if kind == "kdtree":
                        ctx.build_target_kdtrees(pts, None, cv)
                    else:
                        ctx.build_target_voxelmaps(pts, cv, LEAF, OFFSETS)

                def run_a(ctx):
                    tb, _ = timed(ctx, lambda: build(ctx, all_pts, all_covs))
                    ts, _ = timed(ctx, lambda: ctx.set_source_batch(all_pts, all_covs))
                    tp, _ = timed(ctx, lambda: ctx.set_source_pairs(cl, mp))
                    ta, r = timed(ctx, lambda: ctx.align_batch(inits, **kw))
                    return {"build": tb, "store": ts, "pairing": tp, "align": ta}, r

                def run_b(ctx):
                    tb, _ = timed(ctx, lambda: build(ctx, rep_tgt_pts, rep_tgt_covs))
                    ts, _ = timed(ctx, lambda: ctx.set_source_batch(rep_src_pts, rep_src_covs))
                    ta, r = timed(ctx, lambda: ctx.align_batch(inits, **kw))
                    return {"build": tb, "store": ts, "align": ta}, r

                results.append(compare(sg, torch, f"window K={K} c={c} {kind}", run_a, run_b, len(edges), args.reps, info))
                torch.cuda.empty_cache()
            del all_pts, all_covs, rep_tgt_pts, rep_tgt_covs, rep_src_pts, rep_src_covs
    del frames, covs
    torch.cuda.empty_cache()

    # ---- multi-start ----
    n_clouds, starts, n_pts = 64, 16, 20_000
    tgt, src, Tgt = syn.make_pair(1_000_000, n_source=n_clouds * n_pts)
    room = sg.Context(0)
    room.set_target(tgt)
    room.build_target_kdtree()
    room.estimate_target_features(20)
    clouds = [torch.from_numpy(np.c_[s, np.ones(len(s))]).to(dev) for s in np.split(src, n_clouds)]
    ccovs = [room.estimate_features(p, 20, normals=False)[1] for p in clouds]
    rng = np.random.default_rng(64)
    cl = np.repeat(np.arange(n_clouds, dtype=np.uint32), starts)
    inits = np.empty((len(cl), 4, 4))
    for m, c in enumerate(cl):
        ax = rng.normal(size=3)
        ax /= np.linalg.norm(ax)
        P = se3_exp(np.r_[ax * rng.uniform(0, np.deg2rad(5.0)), np.zeros(3)][None])[0]
        C = np.eye(4)
        s = src[c * n_pts : (c + 1) * n_pts]
        C[:3, 3] = Tgt[:3, :3] @ (0.5 * (s.min(0) + s.max(0))) + Tgt[:3, 3]
        P[:3, 3] = rng.uniform(-1, 1, 3) * (0.5 / np.sqrt(3))
        inits[m] = C @ P @ np.linalg.inv(C) @ Tgt
    off = np.arange(n_clouds + 1, dtype=np.int64) * n_pts
    once = ((torch.cat(clouds), off), torch.cat(ccovs))
    roff = np.arange(len(cl) + 1, dtype=np.int64) * n_pts
    rep = ((torch.cat([clouds[c] for c in cl]), roff), torch.cat([ccovs[c] for c in cl]))
    target_ctx = {}

    def with_target(ctx):
        if id(ctx) not in target_ctx:  # the target is built once per context, outside the timed parts of both paths
            ctx.set_target(tgt)
            ctx.build_target_kdtree()
            ctx.estimate_target_features(20)
            target_ctx[id(ctx)] = True

    def ms_a(ctx):
        with_target(ctx)
        ts, _ = timed(ctx, lambda: ctx.set_source_batch(*once))
        tp, _ = timed(ctx, lambda: ctx.set_source_pairs(cl, None))
        ta, r = timed(ctx, lambda: ctx.align_batch(inits, factor=sg.FACTOR_GICP, optimizer=GN))
        return {"store": ts, "pairing": tp, "align": ta}, r

    def ms_b(ctx):
        with_target(ctx)
        ts, _ = timed(ctx, lambda: ctx.set_source_batch(*rep))
        ta, r = timed(ctx, lambda: ctx.align_batch(inits, factor=sg.FACTOR_GICP, optimizer=GN))
        return {"store": ts, "align": ta}, r

    results.append(compare(sg, torch, f"multi-start {n_clouds} clouds x {starts} starts, 1M-point room, kd-tree, GN", ms_a, ms_b, len(cl), args.reps, info))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"setup": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
