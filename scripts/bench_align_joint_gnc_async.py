"""What the device-driven joint-window GNC loop (sgb_align_joint_gnc_async) saves against the host-driven one (sgb_align_joint_gnc), on one GPU.

Workloads: those of bench_align_joint_gnc.py -- K consecutive frames of the synthetic LiDAR stream (16M-point world, 0.25 m voxel grid,
k = 20 covariances), windows of W frames, each frame with c edges back inside its window, the first frame of every window fixed at ground
truth and the others perturbed by ~2 deg / 0.3 m, GICP, Levenberg-Marquardt, max_dist_sq 4, 20 iterations, on many kd-trees and on many
voxel maps (leaf 1.0), every frame corrupted (clutter50: half of it replaced by uniform clutter; moved30: 30 % of it moved as one rigid
object), covariances re-estimated after the corruption; c^2 the 90th percentile of r^2 of the clean edges at ground truth.  K = 64 with
W in {8, 16} and c in {2, 4}, and K = 512 with W = 16, c = 4; GNC-GM and GNC-TLS with stage_iterations 3 and max_stages 64.
Per workload and GNC kind, on one context with its stream set to a torch stream: first every async output (X, info, stages and mu, each
point's g) is checked bit-identical to the synchronous call's, both calls made from the same seed state (none); then sync and async calls alternate, --reps of each after one warm-up, and
the medians are reported in ms per call:
  sync      align_joint_gnc (it synchronises at every stage and joint round);
  async     align_joint_gnc_async to the end of the context's synchronize();
  return    align_joint_gnc_async to its return (the binding's pose transposition included);
  first     the first async call of the kind, to the end of synchronize(): it captures and instantiates the graph.
With them the stages (median and maximum over the windows) and the joint rounds of the call (joint step launches of one synchronous call,
counted with torch.profiler).  The card's name, power limit and maximum SM clock are read with nvidia-smi (read-only) in the same run and
written next to the numbers.

    python scripts/bench_align_joint_gnc_async.py [--frames 64,512] [--reps 7] [--kinds kdtree,voxelmap] [--corruptions clutter50,moved30]
                                                  [--out FILE]
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

LEAF, OFFSETS = 1.0, 1
LM = 1
WORKLOADS = [(64, 8, 2), (64, 8, 4), (64, 16, 2), (64, 16, 4), (512, 16, 4)]  # K, W, c


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--kinds", default="kdtree,voxelmap")
    ap.add_argument("--corruptions", default="clutter50,moved30")
    ap.add_argument("--frames", default="64,512", help="the workloads of these K")
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import small_gicp_b200 as sg
    from small_gicp_b200 import synthetic as syn

    info = gpu_info()
    print(json.dumps(info), flush=True)
    dev = torch.device("cuda:0")
    workloads = [w for w in WORKLOADS if str(w[0]) in args.frames.split(",")]
    K_max = max(w[0] for w in workloads)
    world = syn.make_world(16_000_000, 42)
    side = syn.world_side(16_000_000)
    Gt = [syn.lidar_pose(f, side) for f in range(K_max)]
    prep = sg.Context(0)
    frames = [prep.voxelgrid_sampling(syn.lidar_frame_torch(world, Gt[f], 45 + f, dev).cpu().numpy(), 0.25) for f in range(K_max)]
    del world
    cov = lambda p: prep.estimate_features(p, 20, normals=False)[1]
    covs = [cov(p) for p in frames]
    rng = np.random.default_rng(2026)
    noise = [se3_exp(np.r_[rng.normal(size=3) * np.deg2rad(2.0) / np.sqrt(3), rng.normal(size=3) * 0.3 / np.sqrt(3)][None])[0] for _ in range(K_max)]
    kw = dict(factor=sg.FACTOR_GICP, optimizer=LM, max_dist_sq=4.0, max_iterations=20, stage_iterations=3, max_stages=64)
    stream = torch.cuda.Stream()
    results = []

    def context(kind, pts, cv, edges):
        ctx = sg.Context(0)
        off = np.zeros(len(pts) + 1, dtype=np.int64)
        off[1:] = np.cumsum([len(p) for p in pts])
        P, C = (np.concatenate(pts), off), np.concatenate(cv)
        if kind == "kdtree":
            ctx.build_target_kdtrees(P, None, C)
        else:
            ctx.build_target_voxelmaps(P, C, LEAF, OFFSETS)
        ctx.set_source_batch(P, C)
        ctx.set_source_pairs(np.array([e[0] for e in edges], dtype=np.uint32), np.array([e[1] for e in edges], dtype=np.uint32))
        return ctx

    def window_edges(K, W, c):
        first = {k: (k // W) * W for k in range(K)}
        return first, [(i, i - d) for i in range(K) for d in range(1, c + 1) if i - d >= first[i]]

    def same(a, b):
        a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
        return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))

    c2s = {}
    for K, W, c in workloads:
        for kind in args.kinds.split(","):
            if (K, kind) not in c2s:  # c^2 from the clean frames at ground truth, once per K and target kind
                _, e2 = window_edges(K, K, 2)
                clean = context(kind, frames[:K], covs[:K], e2)
                t = clean.linearize_batch_points(np.array([np.linalg.inv(Gt[j]) @ Gt[i] for i, j in e2]), factor=sg.FACTOR_GICP, max_dist_sq=4.0,
                                                 hessians=False)
                matched = np.concatenate(clean.correspondences_batch()) != sg.NO_CORRESPONDENCE
                c2s[(K, kind)] = float(np.quantile(2.0 * t.point_e[matched], 0.9))
                clean.close()
            c2 = c2s[(K, kind)]
            for corr in args.corruptions.split(","):
                crng = np.random.default_rng(K)
                pts = [corrupt(p, corr, crng) for p in frames[:K]]
                cv = [cov(p) for p in pts]
                woff = list(range(0, K, W)) + [K]
                first, edges = window_edges(K, W, c)
                X0 = np.array([Gt[k] if k == first[k] else Gt[k] @ noise[k] for k in range(K)])
                Xd = torch.from_numpy(np.ascontiguousarray(X0)).to(dev)
                ctx = context(kind, pts, cv, edges)
                ctx.set_stream(stream.cuda_stream)
                for name, gkind in (("gm", sg.GNC_GEMAN_MCCLURE), ("tls", sg.GNC_TLS)):

                    def sync(point_weights=False):
                        return ctx.align_joint_gnc(X0, c2, windows=woff, gnc=gkind, point_weights=point_weights, **kw)

                    def enqueue(point_weights=False, out=None):
                        with torch.cuda.stream(stream):
                            return ctx.align_joint_gnc_async(Xd, c2, windows=woff, gnc=gkind, point_weights=point_weights, out=out, **kw)

                    # The first async call of the kind builds its graph; its result is the one checked against the synchronous call.  Both
                    # start without seeds: a search seeded by an earlier call's correspondences may pick the other of two target points at
                    # an exact FP32 distance tie (the header's caveat), so the two calls are compared from the same seed state.
                    ctx.drop_seeds()
                    ctx.synchronize()
                    t0 = time.perf_counter()
                    a = enqueue(point_weights=True)
                    ctx.synchronize()
                    first_s = time.perf_counter() - t0
                    ctx.drop_seeds()
                    r = sync(point_weights=True)
                    differ = [f for f in ("X", "error", "mu", "point_w") if not same(getattr(r, f), getattr(a, f).cpu().numpy())]
                    differ += [f for f in ("converged", "iterations", "num_inliers", "stages")
                               if not same(np.asarray(getattr(r, f), dtype=np.float64), getattr(a, f).cpu().numpy())]
                    ok = not differ
                    if not ok:
                        print(f"K={K} W={W} c={c} {kind} {corr} {name}: the async result differs from align_joint_gnc in {differ}", flush=True)
                    # the joint rounds of one call: its joint step launches
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        sync()
                        torch.cuda.synchronize()
                    rounds = sum(1 for e in prof.events() if e.device_time > 0 and "joint_gnc_step_kernel" in e.name)
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
                    rec = {"workload": f"K={K} W={W} c={c} {kind} {corr}", "gnc": name, "windows": len(woff) - 1, "edges": len(edges),
                           "points": int(ctx._batch_offsets[-1]), "c2": c2, "bit_identical": ok, "differing": differ, "stages_median": float(np.median(r.stages)),
                           "stages_max": int(r.stages.max()), "joint_rounds": rounds, "first_ms": 1e3 * first_s, **info}
                    for k, v in times.items():
                        rec[k + "_ms"] = 1e3 * float(np.median(v))
                        rec[k + "_ms_range"] = [1e3 * float(np.min(v)), 1e3 * float(np.max(v))]
                    rec["sync_over_async"] = rec["sync_ms"] / rec["async_ms"]
                    print(json.dumps(rec), flush=True)
                    results.append(rec)
                ctx.set_stream(None)
                ctx.close()
                torch.cuda.empty_cache()
    prep.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"setup": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
