"""What graduated non-convexity (sgb_align_batch_gnc) buys and costs on corrupted LiDAR pairs, on one GPU.

Workloads: the LiDAR frame pairs of bench_align_async.lidar_pairs (frame i a kd-tree map, frame i + 1 the source, 0.25 m voxel grid,
covariances re-estimated after the corruption), GICP, max_dist_sq 1, at B in {64, 512} (--sizes), each source frame corrupted by
  moved15 / moved30: the moved-object recipe of bench_batch_weights.py --accuracy (the points nearest a random point in the horizontal
      plane, 15 % / 30 % of the frame, moved rigidly by 0.8 m and 10 degrees);
  clutter30 / clutter50 / clutter70: that share of the frame's points replaced by uniform clutter in the frame's box.
Initial poses: ground truth times 0.5 degree of yaw and 0.1 m.  Arms, alternated call by call in one run:
  plain      align_batch, Levenberg-Marquardt, 20 iterations;
  cauchy     the same with the Cauchy kernel (robust_c 1);
  two_pass   align, error_batch_points, weight 0 for rows above 10x the member's median positive row, align again (bench_batch_weights);
  gnc_gm / gnc_tls   align_batch_gnc (stage_iterations 3, max_stages 64, the last stage 20 iterations);
  host_tls   the same TLS loop driven from Python with public calls on a context holding one member (tests/np_gnc.host_gnc), timed on the
             first --host-members members only: what the host round trips cost per pair.
c^2: the 90th percentile of r^2 = 2 e over the matched points of the uncorrupted pairs at ground truth (one value per size).
--fresh-key runs one other case instead, the worst for the call's cached graph of its device loop: before every timed call a new batch
(clutter30) whose first source frame has lost a different number of points (set_source_batch, untimed), so that every call builds and
instantiates its graph, as in odometry, where every frame brings a new point count; gnc_gm and gnc_tls alternated, --sizes 1,8,64 say.
Reported per workload and arm: median and worst rotation [deg] and translation [m] error against ground truth, converged count, median
and maximum stages (GNC), and ms per pair (the median of --reps timed calls after one warm-up, each ending in a device synchronise).
The card's name, power limit and maximum SM clock are read with nvidia-smi (read-only) in the same run and written next to the numbers.

    python scripts/bench_align_gnc.py [--sizes 64,512] [--reps 3] [--host-members 8] [--fresh-key] [--out FILE]
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
from bench_batch_weights import pose_error  # noqa: E402

CORRUPTIONS = ["moved15", "moved30", "clutter30", "clutter50", "clutter70"]


def corrupt(p, kind, rng):
    p = p.copy()
    if kind.startswith("moved"):
        move = se3_exp(np.array([[0.0, 0.0, np.deg2rad(10.0), 0.8, 0.0, 0.0]]))[0]
        c = p[rng.integers(len(p)), :2]
        d = np.linalg.norm(p[:, :2] - c, axis=1)
        obj = d <= np.quantile(d, int(kind[5:]) / 100.0)
        ctr = p[obj, :3].mean(0)
        p[obj, :3] = (p[obj, :3] - ctr) @ move[:3, :3].T + move[:3, 3] + ctr
    elif kind.startswith("clutter"):
        k = rng.permutation(len(p))[: int(len(p) * int(kind[7:]) / 100.0)]
        p[k, :3] = rng.uniform(p[:, :3].min(0), p[:, :3].max(0), (len(k), 3))
    return p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="64,512")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-members", type=int, default=8)
    ap.add_argument("--corruptions", default=",".join(CORRUPTIONS))
    ap.add_argument("--fresh-key", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sizes = [int(x) for x in args.sizes.split(",")]

    import torch

    import np_gnc as G
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
    kw = dict(factor=sg.FACTOR_GICP, max_dist_sq=1.0, max_iterations=20)
    results = []

    def batch(ctx, B, src, scov):
        off = np.zeros(B + 1, dtype=np.int64)
        off[1:] = np.cumsum([len(p) for p in src[:B]])
        ctx.set_source_batch((np.concatenate(src[:B]), off), np.concatenate(scov[:B]))

    for B in sizes:
        ctx = sg.Context(0)
        off = np.zeros(B + 1, dtype=np.int64)
        off[1:] = np.cumsum([len(p) for p in frames[:B]])
        ctx.build_target_kdtrees((np.concatenate(frames[:B]), off), None, np.concatenate(covs[:B]))
        batch(ctx, B, frames[1:], covs[1:])
        t = ctx.linearize_batch_points(gt[:B], factor=sg.FACTOR_GICP, max_dist_sq=1.0, hessians=False)
        matched = np.concatenate(ctx.correspondences_batch()) != sg.NO_CORRESPONDENCE
        c2 = float(np.quantile(2.0 * t.point_e[matched], 0.9))
        if args.fresh_key:
            rng = np.random.default_rng(B)
            src = [corrupt(p, "clutter30", rng) for p in frames[1 : B + 1]]
            scov = [cov(p) for p in src]
            arms = {"gnc_gm": sg.GNC_GEMAN_MCCLURE, "gnc_tls": sg.GNC_TLS}
            times = {k: [] for k in arms}
            calls = 0
            for rep in range(args.reps + 1):  # the first is the warm-up
                for k, gnc in arms.items():
                    calls += 1
                    batch(ctx, B, [src[0][:-calls]] + src[1:], [scov[0][:-calls]] + scov[1:])
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    ctx.align_batch_gnc(inits[:B], c2, gnc=gnc, **kw)
                    torch.cuda.synchronize()
                    if rep:
                        times[k].append(time.perf_counter() - t0)
            rec = {"workload": "fresh_key clutter30", "B": B, "c2": c2, **info}
            rec.update({k: {"ms_per_call": 1e3 * float(np.median(t)), "ms_per_call_max": 1e3 * float(np.max(t))} for k, t in times.items()})
            print(json.dumps(rec), flush=True)
            results.append(rec)
            ctx.close()
            continue
        for corr in args.corruptions.split(","):
            rng = np.random.default_rng(B)
            src = [corrupt(p, corr, rng) for p in frames[1 : B + 1]]
            scov = [cov(p) for p in src]
            batch(ctx, B, src, scov)

            def two_pass():
                ctx.set_source_weights(None)
                first = ctx.align_batch(inits[:B], **kw)
                _, pe = ctx.error_batch_points(first.T_target_source)
                bo = ctx._batch_offsets
                w = np.ones(len(pe))
                for m in range(B):
                    rows = pe[bo[m] : bo[m + 1]]
                    pos = rows[rows > 0]
                    if len(pos):
                        w[bo[m] : bo[m + 1]] = np.where(rows > 10.0 * np.median(pos), 0.0, 1.0)
                ctx.set_source_weights(w)
                r = ctx.align_batch(first.T_target_source, **kw)
                ctx.set_source_weights(None)
                return r

            arms = {
                "plain": lambda: ctx.align_batch(inits[:B], **kw),
                "cauchy": lambda: ctx.align_batch(inits[:B], robust=sg.ROBUST_CAUCHY, robust_c=1.0, **kw),
                "two_pass": two_pass,
                "gnc_gm": lambda: ctx.align_batch_gnc(inits[:B], c2, gnc=sg.GNC_GEMAN_MCCLURE, **kw),
                "gnc_tls": lambda: ctx.align_batch_gnc(inits[:B], c2, gnc=sg.GNC_TLS, **kw),
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
            # the host-driven TLS loop on a one-member pairing, over the first members
            H = min(args.host_members, B)
            host_T, host_t = [], []
            for m in range(H):
                ctx.set_source_pairs([m], [m])
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                mm = G.host_gnc(ctx, inits[m], c2, kind=G.TLS, **kw)
                torch.cuda.synchronize()
                host_t.append(time.perf_counter() - t0)
                host_T.append(mm.T_target_source)
            batch(ctx, B, src, scov)
            rec = {"workload": corr, "B": B, "points": int(ctx._batch_offsets[-1]), "c2": c2, **info}
            for k, r in out.items():
                e = np.array([pose_error(gt[m], r.T_target_source[m]) for m in range(B)])
                rec[k] = {"rot_deg_median": float(np.median(e[:, 0])), "rot_deg_max": float(e[:, 0].max()), "trans_m_median": float(np.median(e[:, 1])),
                          "trans_m_max": float(e[:, 1].max()), "converged": int(np.sum(r.converged)), "ms_per_pair": 1e3 * float(np.median(times[k])) / B}
                if k.startswith("gnc"):
                    rec[k]["stages_median"], rec[k]["stages_max"] = float(np.median(r.stages)), int(r.stages.max())
            same = all(np.array_equal(host_T[m], out["gnc_tls"].T_target_source[m]) for m in range(H))
            rec["host_tls"] = {"members": H, "ms_per_pair": 1e3 * float(np.mean(host_t)), "bit_identical_to_gnc_tls": bool(same)}
            print(json.dumps(rec), flush=True)
            results.append(rec)
        ctx.close()
    prep.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"setup": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
