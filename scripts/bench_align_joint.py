"""Joint window registration (sgb_align_joint) against the same edges aligned independently (set_source_pairs + align_batch), on one GPU.

Workload: K in {64, 512} consecutive frames of the synthetic LiDAR stream of bench_batch_pairs.py (synthetic.lidar_frame_torch in the
16M-point world, 1 m forward + 1 deg yaw per frame), each voxel-grid sampled at 0.25 m with k = 20 covariances, all outside the timed
window.  Windows of W in {8, 16} consecutive frames, each frame with c in {2, 4} edges back inside its window, the first frame of every
window fixed at ground truth and the others perturbed by ~2 deg / 0.3 m.  GICP, Levenberg-Marquardt, on many kd-trees and on many voxel
maps (leaf 1.0).

Arms, alternated, median of --reps after one warm-up each:
  (a) align_joint over all windows in one call;
  (b) the same edges as independent members (align_batch from the relative poses of the same perturbed frames): the cost floor of the
      same linearize work.
Reported per workload: ms per window of each arm, rounds (one joint_step_kernel launch each, counted in the profiled run), joint_step_kernel time per
round (torch.profiler, in a run of its own), device MiB of each arm's set-up, the pose error of each arm against ground truth ((b)
chained along i -> i-1), and the card's name, power limit and maximum SM clock (nvidia-smi, read-only).

    python scripts/bench_align_joint.py [--frames 64,512] [--window 8,16] [--edges 2,4] [--reps 5] [--out FILE]
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
LM = 1


def pose_error(G, X):
    dr = np.rad2deg(np.arccos(np.clip((np.trace(G[:3, :3].T @ X[:3, :3]) - 1) / 2, -1, 1)))
    return float(dr), float(np.linalg.norm(G[:3, 3] - X[:3, 3]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", default="64,512")
    ap.add_argument("--window", default="8,16")
    ap.add_argument("--edges", default="2,4")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    import torch

    import small_gicp_b200 as sg
    from small_gicp_b200 import synthetic as syn

    info = gpu_info()
    print(json.dumps(info), flush=True)
    dev = torch.device("cuda:0")
    K_max = max(int(x) for x in args.frames.split(","))
    world = syn.make_world(16_000_000, 42)
    side = syn.world_side(16_000_000)
    G = [syn.lidar_pose(f, side) for f in range(K_max)]
    prep = sg.Context(0)
    frames, covs = [], []
    for f in range(K_max):
        p = prep.voxelgrid_sampling(syn.lidar_frame_torch(world, G[f], 45 + f, dev).cpu().numpy(), 0.25)
        frames.append(torch.from_numpy(p).to(dev))
        covs.append(torch.from_numpy(prep.estimate_features(p, 20, normals=False)[1]).to(dev))
    del world
    rng = np.random.default_rng(2026)
    noise = [se3_exp(np.r_[rng.normal(size=3) * np.deg2rad(2.0) / np.sqrt(3), rng.normal(size=3) * 0.3 / np.sqrt(3)][None])[0] for _ in range(K_max)]
    results = []
    kw = dict(factor=sg.FACTOR_GICP, optimizer=LM, max_dist_sq=4.0)
    for K in [int(x) for x in args.frames.split(",")]:
        offs = np.zeros(K + 1, dtype=np.int64)
        offs[1:] = np.cumsum([len(frames[i]) for i in range(K)])
        pts, cv = (torch.cat(frames[:K]), offs), torch.cat(covs[:K])
        for W in [int(x) for x in args.window.split(",")]:
            woff = list(range(0, K, W)) + [K]
            first = {k: woff[k // W] for k in range(K)}
            X0 = np.array([G[k] if k == first[k] else G[k] @ noise[k] for k in range(K)])
            for c in [int(x) for x in args.edges.split(",")]:
                edges = [(i, i - d) for i in range(K) for d in range(1, c + 1) if i - d >= first[i]]
                cl = np.array([e[0] for e in edges], dtype=np.uint32)
                mp = np.array([e[1] for e in edges], dtype=np.uint32)
                T0 = np.array([np.linalg.inv(X0[j]) @ X0[i] for i, j in edges])
                for kind in ("kdtree", "voxelmap"):
                    ctxs, mib = [], []
                    for _ in range(2):
                        free0 = torch.cuda.mem_get_info()[0]
                        ctx = sg.Context(0)
                        if kind == "kdtree":
                            ctx.build_target_kdtrees(pts, None, cv)
                        else:
                            ctx.build_target_voxelmaps(pts, cv, LEAF, OFFSETS)
                        ctx.set_source_batch(pts, cv)
                        ctx.set_source_pairs(cl, mp)
                        ctxs.append(ctx)
                        mib.append(free0)
                    arm_a = lambda: ctxs[0].align_joint(X0, windows=woff, **kw)
                    arm_b = lambda: ctxs[1].align_batch(T0, **kw)
                    ra, rb = arm_a(), arm_b()  # warm-up; also sizes every buffer of both arms
                    mem_after = torch.cuda.mem_get_info()[0]
                    k0 = ctxs[0].kernel_launches
                    arm_a()
                    launches = ctxs[0].kernel_launches - k0
                    ta, tb = [], []
                    for _ in range(args.reps):
                        for t, run, ctx in ((ta, arm_a, ctxs[0]), (tb, arm_b, ctxs[1])):
                            ctx.synchronize()
                            t0 = time.perf_counter()
                            run()
                            ctx.synchronize()
                            t.append(time.perf_counter() - t0)
                    # joint_step_kernel alone, from a profiled run of arm (a)
                    from torch.profiler import ProfilerActivity, profile

                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        arm_a()
                        torch.cuda.synchronize()
                    step_us = [e.device_time for e in prof.events() if "joint_step_kernel" in e.name]
                    n_win = len(woff) - 1
                    ea = [pose_error(G[k], ra.X[k]) for k in range(K) if k != first[k]]
                    chain, eb = {}, []
                    for k in range(K):
                        if k == first[k]:
                            chain[k] = G[k]
                        else:
                            chain[k] = chain[k - 1] @ rb.T_target_source[edges.index((k, k - 1))]
                            eb.append(pose_error(G[k], chain[k]))
                    rec = {"workload": f"K={K} W={W} c={c} {kind}", "windows": n_win, "edges": len(edges), "rounds": len(step_us), "launches_a": launches,
                           "a_ms_per_window": 1e3 * float(np.median(ta)) / n_win, "b_ms_per_window": 1e3 * float(np.median(tb)) / n_win,
                           "a_total_ms": 1e3 * float(np.median(ta)), "b_total_ms": 1e3 * float(np.median(tb)),
                           "joint_step_us_per_round_median": float(np.median(step_us)) if step_us else None,
                           "device_mib_a_and_b": (mib[0] - mem_after) / 2**20,
                           "a_rot_err_deg_max": max(e[0] for e in ea), "a_trans_err_m_max": max(e[1] for e in ea),
                           "b_chained_rot_err_deg_max": max(e[0] for e in eb), "b_chained_trans_err_m_max": max(e[1] for e in eb),
                           "a_converged_windows": int(ra.converged.sum()), "b_converged_edges": int(rb.converged.sum())}
                    rec.update(info)
                    print(json.dumps(rec), flush=True)
                    results.append(rec)
                    for ctx in ctxs:
                        ctx.close()
                    torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
