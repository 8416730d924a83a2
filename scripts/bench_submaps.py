"""Submap members (sgb_source_set_submaps) against building a kd-tree of every placed union, on one GPU.

Workload: K in {64, 512} consecutive frames of the synthetic LiDAR stream of bench_batch_pairs.py (16M-point world, 1 m forward + 1 deg
yaw per frame, voxel-grid sampled at 0.25 m, k = 20 covariances estimated on the device, all outside the timed window and kept on the
device).  Frame i is aligned against the UNION of its c in {4, 8} predecessors, each placed by its ground-truth pose, from its own
ground-truth pose perturbed by 0.5 deg / 0.1 m.  GICP, Levenberg-Marquardt.

Compared in one process, repetitions alternated, median and min - max of --reps:
  (a) submaps: one kd-tree per frame (build_target_kdtrees), every frame stored once (set_source_batch), set_source_submaps, align_batch;
  (b) unions:  what a caller had to do before: per member the placed union assembled on the device (points P q, covariances R C R^T,
               with torch), build_target_kdtrees over the unions, set_source_batch, align_batch;
  (c) edges:   for context, the c pairwise edges of every frame through set_source_pairs (c independent alignments, not a joint one).
Reported per member: assemble (b only), build, store + pairing, align, total; device MiB the set-up takes, LM rounds (max iterations),
the pose difference between (a) and (b), and the card's name, power limit and maximum SM clock (nvidia-smi, read-only).

    python scripts/bench_submaps.py [--frames 64,512] [--window 4,8] [--reps 5] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_align_batch import gpu_info, se3_exp  # noqa: E402
from bench_batch_pairs import timed  # noqa: E402

LM = 1  # sgb_optimizer_kind


def stats(x):
    x = 1e3 * np.asarray(x)
    return {"median": float(np.median(x)), "min": float(x.min()), "max": float(x.max())}


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
    del world, prep
    noise = se3_exp(np.array([[0.0, 0.0, np.deg2rad(0.5), 0.1, 0.0, 0.0]]))[0]
    poses_dev = [torch.from_numpy(P).to(dev) for P in poses]
    print(json.dumps({"frames": K_max, "points_per_frame_mean": float(np.mean([len(p) for p in frames]))}), flush=True)

    def concat(idx):
        offs = np.zeros(len(idx) + 1, dtype=np.int64)
        offs[1:] = np.cumsum([len(frames[i]) for i in idx])
        return (torch.cat([frames[i] for i in idx]), offs), torch.cat([covs[i] for i in idx])

    kw = dict(factor=sg.FACTOR_GICP, optimizer=LM)
    results = []
    for K in frames_list:
        all_pts, all_covs = concat(range(K))
        src_pts, src_covs = concat(range(1, K))
        for c in windows:
            members = list(range(1, K))
            lists = [[i - j for j in range(1, c + 1) if i - j >= 0] for i in members]
            entry_poses = [[poses[k] for k in l] for l in lists]
            inits = np.array([poses[i] @ noise for i in members])
            edges = [(i, k) for i, l in zip(members, lists) for k in l]
            edge_inits = np.array([np.linalg.inv(poses[k]) @ poses[i] @ noise for i, k in edges])

            def run_a(ctx):
                tb, _ = timed(ctx, lambda: ctx.build_target_kdtrees(all_pts, None, all_covs))
                ts, _ = timed(ctx, lambda: (ctx.set_source_batch(all_pts, all_covs), ctx.set_source_submaps(lists, entry_poses, members)))
                ta, r = timed(ctx, lambda: ctx.align_batch(inits, **kw))
                return {"build": tb, "store": ts, "align": ta}, r

            def assemble():
                pts, cvs, offs = [], [], [0]
                for l in lists:
                    for k in l:
                        P = poses_dev[k]
                        pts.append(frames[k] @ P.T)
                        cvs.append(P @ covs[k] @ P.T)  # the fourth row and column of a covariance are zero, so the translation drops out
                    offs.append(offs[-1] + sum(len(frames[k]) for k in l))
                return (torch.cat(pts), np.array(offs, dtype=np.int64)), torch.cat(cvs)

            def run_b(ctx):
                tu, (u_pts, u_covs) = timed(ctx, lambda: (assemble(), torch.cuda.synchronize())[0])
                tb, _ = timed(ctx, lambda: ctx.build_target_kdtrees(u_pts, None, u_covs))
                ts, _ = timed(ctx, lambda: ctx.set_source_batch(src_pts, src_covs))
                ta, r = timed(ctx, lambda: ctx.align_batch(inits, **kw))
                return {"assemble": tu, "build": tb, "store": ts, "align": ta}, r

            def run_c(ctx):
                tb, _ = timed(ctx, lambda: ctx.build_target_kdtrees(all_pts, None, all_covs))
                ts, _ = timed(ctx, lambda: (ctx.set_source_batch(all_pts, all_covs), ctx.set_source_pairs([e[0] for e in edges], [e[1] for e in edges])))
                ta, r = timed(ctx, lambda: ctx.align_batch(edge_inits, **kw))
                return {"build": tb, "store": ts, "align": ta}, r

            rec = {"workload": f"window K={K} c={c}", "members": len(members), "entries": len(edges)}
            arms = {}
            for tag, run in (("a", run_a), ("b", run_b), ("c", run_c)):
                # an arm's memory: what its set-up and one align take while nothing else is released -- the earlier arms' contexts stay
                # alive and untouched, the earlier windows' were closed, and torch's cache was emptied just before
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
                free = torch.cuda.mem_get_info()[0]
                ctx = sg.Context(0)
                try:
                    _, r = run(ctx)  # warm-up: every buffer of the arm reaches its size
                except (sg.SgbError, torch.cuda.OutOfMemoryError) as ex:
                    rec[f"{tag}_not_run"] = str(ex)[:120]
                    continue
                torch.cuda.synchronize()
                rec[f"{tag}_device_mib"] = (free - torch.cuda.mem_get_info()[0]) / 2**20
                rec[f"{tag}_rounds"] = int(r.iterations.max())
                rec[f"{tag}_converged"] = int(r.converged.sum())
                arms[tag] = (ctx, run, r, {})
            for _ in range(args.reps):
                for tag, (ctx, run, _, t) in arms.items():
                    ph, _ = run(ctx)
                    for k, v in ph.items():
                        t.setdefault(k, []).append(v)
            for tag, (ctx, run, r, t) in arms.items():
                n = len(members)
                total = np.sum([t[k] for k in t], axis=0)
                rec[f"{tag}_total_per_member_ms"] = stats(total / n)
                for k in t:
                    rec[f"{tag}_{k}_per_member_ms"] = stats(np.asarray(t[k]) / n)
            if "a" in arms and "b" in arms:
                d = np.linalg.inv(arms["b"][2].T_target_source) @ arms["a"][2].T_target_source
                rec["a_vs_b_max_rotation_rad"] = float(np.arccos(np.clip((np.trace(d[:, :3, :3], axis1=1, axis2=2) - 1) / 2, -1, 1)).max())
                rec["a_vs_b_max_translation_m"] = float(np.linalg.norm(d[:, :3, 3], axis=1).max())
                rec["a_vs_b_equal_iterations"] = int((arms["a"][2].iterations == arms["b"][2].iterations).sum())
            rec.update(info)
            print(json.dumps(rec), flush=True)
            results.append(rec)
            for arm in arms.values():
                arm[0].close()  # its device memory is back before the next window's set-up is measured
            del arms, ctx, r
        del all_pts, all_covs, src_pts, src_covs
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"setup": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
