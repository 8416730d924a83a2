"""What graduated non-convexity for joint windows (sgb_align_joint_gnc) buys and costs on corrupted LiDAR windows, on one GPU.

Workloads: the "Joint windows" workloads of bench_align_joint.py -- K in {64, 512} consecutive frames of the synthetic LiDAR stream (16M-point
world, 0.25 m voxel grid, k = 20 covariances), windows of W in {8, 16} frames, each frame with c in {2, 4} edges back inside its window,
the first frame of every window fixed at ground truth and the others perturbed by ~2 deg / 0.3 m, GICP, Levenberg-Marquardt,
max_dist_sq 4, on many kd-trees and on many voxel maps (leaf 1.0) -- with every frame corrupted by one of bench_align_gnc.py's kinds
(moved15 / moved30: a rigid object of that share of the frame moved 0.8 m and 10 deg; clutter30 / 50 / 70: that share replaced by
uniform clutter), covariances re-estimated after the corruption.  A frame is both a cloud and a map, so its outliers enter every edge
it belongs to on either side.
Arms, alternated call by call, median of --reps timed calls after one warm-up, each ending in a device synchronise:
  plain      align_joint (20 iterations);
  cauchy     align_joint with the Cauchy kernel (robust_c 1);
  gnc_gm / gnc_tls   align_joint_gnc (stage_iterations 3, max_stages 64, the last stage 20 iterations);
  pairs_gnc  align_batch_gnc over the same edges from the same perturbed frames (TLS), chained i -> i-1 from each window's first frame;
  host_tls   the TLS loop of align_joint_gnc driven from Python with public calls (tests/np_joint_gnc.host_joint_gnc) on contexts holding
             one window, over the first --host-windows windows, its X checked bit-identical to gnc_tls's before it is timed.
c^2: the 90th percentile of r^2 = 2 e over the matched points of the uncorrupted edges (c = 2) at ground truth, once per K and target kind.
--fresh-key runs one other case instead, the worst for the call's cached graph of its device loop: windows of the first --window size,
the first --edges count, clutter30, and before every timed call a new batch whose first frame has lost a different number of points
(set_source_batch and set_source_pairs, untimed), so that every call builds and instantiates its graph; gnc_gm and gnc_tls alternated.
Reported per workload and arm: median and worst rotation [deg] and translation [m] error of the free frames against ground truth,
converged windows (edges for pairs_gnc), median and maximum stages (GNC), and ms per window; for gnc_tls also the share of its device
time spent in the joint step kernel and the joint rounds it ran (torch.profiler, one call of its own).  The card's name, power limit and
maximum SM clock are read with nvidia-smi (read-only) in the same run and written next to the numbers.

    python scripts/bench_align_joint_gnc.py [--frames 64,512] [--window 8,16] [--edges 2,4] [--kinds kdtree,voxelmap]
                                            [--corruptions moved15,...] [--reps 5] [--host-windows 2] [--fresh-key] [--out FILE]
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
from bench_align_gnc import CORRUPTIONS, corrupt  # noqa: E402
from bench_align_joint import pose_error  # noqa: E402

LEAF, OFFSETS = 1.0, 1
LM = 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", default="64,512")
    ap.add_argument("--window", default="8,16")
    ap.add_argument("--edges", default="2,4")
    ap.add_argument("--kinds", default="kdtree,voxelmap")
    ap.add_argument("--corruptions", default=",".join(CORRUPTIONS))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-windows", type=int, default=2)
    ap.add_argument("--fresh-key", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import np_gnc as G
    import small_gicp_b200 as sg
    from np_joint_gnc import host_joint_gnc
    from small_gicp_b200 import synthetic as syn

    info = gpu_info()
    print(json.dumps(info), flush=True)
    dev = torch.device("cuda:0")
    sizes = [int(x) for x in args.frames.split(",")]
    K_max = max(sizes)
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
    kw = dict(factor=sg.FACTOR_GICP, optimizer=LM, max_dist_sq=4.0, max_iterations=20)
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

    for K in sizes:
        for kind in args.kinds.split(","):
            # c^2 from the clean frames at ground truth
            _, e2 = window_edges(K, K, 2)
            clean = context(kind, frames[:K], covs[:K], e2)
            t = clean.linearize_batch_points(np.array([np.linalg.inv(Gt[j]) @ Gt[i] for i, j in e2]), factor=sg.FACTOR_GICP, max_dist_sq=4.0,
                                             hessians=False)
            matched = np.concatenate(clean.correspondences_batch()) != sg.NO_CORRESPONDENCE
            c2 = float(np.quantile(2.0 * t.point_e[matched], 0.9))
            clean.close()
            if args.fresh_key:
                pts = [corrupt(p, "clutter30", np.random.default_rng(K)) for p in frames[:K]]
                cv = [cov(p) for p in pts]
                W, c = int(args.window.split(",")[0]), int(args.edges.split(",")[0])
                woff = list(range(0, K, W)) + [K]
                first, edges = window_edges(K, W, c)
                X0 = np.array([Gt[k] if k == first[k] else Gt[k] @ noise[k] for k in range(K)])
                ctx = context(kind, pts, cv, edges)
                arms = {"gnc_gm": sg.GNC_GEMAN_MCCLURE, "gnc_tls": sg.GNC_TLS}
                times = {k: [] for k in arms}
                calls = 0
                for rep in range(args.reps + 1):  # the first is the warm-up
                    for k, gnc in arms.items():
                        calls += 1
                        p0 = [pts[0][:-calls]] + pts[1:]
                        off = np.zeros(K + 1, dtype=np.int64)
                        off[1:] = np.cumsum([len(p) for p in p0])
                        ctx.set_source_batch((np.concatenate(p0), off), np.concatenate([cv[0][:-calls]] + cv[1:]))
                        ctx.set_source_pairs(np.array([e[0] for e in edges], dtype=np.uint32), np.array([e[1] for e in edges], dtype=np.uint32))
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        ctx.align_joint_gnc(X0, c2, windows=woff, gnc=gnc, **kw)
                        torch.cuda.synchronize()
                        if rep:
                            times[k].append(time.perf_counter() - t0)
                rec = {"workload": f"fresh_key K={K} W={W} c={c} {kind} clutter30", "windows": len(woff) - 1, "edges": len(edges), "c2": c2, **info}
                rec.update({k: {"ms_per_call": 1e3 * float(np.median(t)), "ms_per_call_max": 1e3 * float(np.max(t))} for k, t in times.items()})
                print(json.dumps(rec), flush=True)
                results.append(rec)
                ctx.close()
                continue
            for corr in args.corruptions.split(","):
                crng = np.random.default_rng(K)
                pts = [corrupt(p, corr, crng) for p in frames[:K]]
                cv = [cov(p) for p in pts]
                for W in [int(x) for x in args.window.split(",")]:
                    woff = list(range(0, K, W)) + [K]
                    n_win = len(woff) - 1
                    for c in [int(x) for x in args.edges.split(",")]:
                        first, edges = window_edges(K, W, c)
                        X0 = np.array([Gt[k] if k == first[k] else Gt[k] @ noise[k] for k in range(K)])
                        T0 = np.array([np.linalg.inv(X0[j]) @ X0[i] for i, j in edges])
                        ctx = context(kind, pts, cv, edges)
                        arms = {
                            "plain": lambda: ctx.align_joint(X0, windows=woff, **kw),
                            "cauchy": lambda: ctx.align_joint(X0, windows=woff, robust=sg.ROBUST_CAUCHY, robust_c=1.0, **kw),
                            "gnc_gm": lambda: ctx.align_joint_gnc(X0, c2, windows=woff, gnc=sg.GNC_GEMAN_MCCLURE, **kw),
                            "gnc_tls": lambda: ctx.align_joint_gnc(X0, c2, windows=woff, gnc=sg.GNC_TLS, **kw),
                            "pairs_gnc": lambda: ctx.align_batch_gnc(T0, c2, gnc=sg.GNC_TLS, **kw),
                        }
                        times = {k: [] for k in arms}
                        out = {}
                        for rep in range(args.reps + 1):  # the first is the warm-up
                            for k, f in arms.items():
                                torch.cuda.synchronize()
                                t0 = time.perf_counter()
                                out[k] = f()
                                torch.cuda.synchronize()
                                if rep:
                                    times[k].append(time.perf_counter() - t0)
                        # gnc_tls's device time by kernel, in a profiled call of its own
                        with profile(activities=[ProfilerActivity.CUDA]) as prof:
                            arms["gnc_tls"]()
                            torch.cuda.synchronize()
                        kern = [e for e in prof.events() if e.device_time > 0]
                        step = [e.device_time for e in kern if "joint_gnc_step_kernel" in e.name]
                        total_us = sum(e.device_time for e in kern)
                        rec = {"workload": f"K={K} W={W} c={c} {kind} {corr}", "windows": n_win, "edges": len(edges),
                               "points": int(ctx._batch_offsets[-1]), "c2": c2, **info}
                        free = [k for k in range(K) if k != first[k]]
                        for name, r in out.items():
                            if name == "pairs_gnc":
                                chain = {}
                                for k in range(K):
                                    chain[k] = Gt[k] if k == first[k] else chain[k - 1] @ r.T_target_source[edges.index((k, k - 1))]
                                X = chain
                            else:
                                X = r.X
                            e = np.array([pose_error(Gt[k], X[k]) for k in free])
                            a = {"rot_deg_median": float(np.median(e[:, 0])), "rot_deg_max": float(e[:, 0].max()),
                                 "trans_m_median": float(np.median(e[:, 1])), "trans_m_max": float(e[:, 1].max()),
                                 "converged": int(np.sum(r.converged)), "ms_per_window": 1e3 * float(np.median(times[name])) / n_win}
                            if "gnc" in name:
                                a["stages_median"], a["stages_max"] = float(np.median(r.stages)), int(r.stages.max())
                            rec[name] = a
                        rec["gnc_tls"]["joint_step_share_of_device_time"] = float(sum(step) / total_us) if total_us else None
                        rec["gnc_tls"]["joint_rounds"] = len(step)
                        rec["gnc_tls"]["device_ms"] = total_us / 1e3
                        # the host-driven loop on contexts holding one window each, checked bit-identical, then timed
                        H = min(args.host_windows, n_win)
                        host_t, same = [], True
                        for w in range(H):
                            f0, f1 = woff[w], woff[w + 1]
                            we = [(i - f0, j - f0) for i, j in edges if f0 <= i < f1]
                            solo = context(kind, pts[f0:f1], cv[f0:f1], we)
                            solo.align_joint(X0[f0:f1], **kw)  # warm: the pairing's view of the target
                            torch.cuda.synchronize()
                            t0 = time.perf_counter()
                            m = host_joint_gnc(solo, X0[f0:f1], c2, kind=G.TLS, **kw)
                            torch.cuda.synchronize()
                            host_t.append(time.perf_counter() - t0)
                            same = same and np.array_equal(m.X.view(np.uint64), out["gnc_tls"].X[f0:f1].view(np.uint64))
                            solo.close()
                        rec["host_tls"] = {"windows": H, "ms_per_window": 1e3 * float(np.mean(host_t)), "bit_identical_to_gnc_tls": bool(same)}
                        print(json.dumps(rec), flush=True)
                        results.append(rec)
                        ctx.close()
                        torch.cuda.empty_cache()
    prep.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"setup": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
