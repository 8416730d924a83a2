"""Batched VGICP over many target maps (sgb_target_build_voxelmaps), or batched GICP over many kd-trees (sgb_target_build_kdtrees,
--target kdtree), against one pair after another, on one GPU.

Workload: consecutive frames of the synthetic LiDAR stream (synthetic.lidar_frame_torch in the 16M-point world, 1 m forward + 1 deg
yaw per frame), each voxel-grid sampled at 0.25 m with k = 20 covariances estimated on the device, all outside the timed window, and kept
on the device (all frames concatenated in one tensor; both paths pass device pointers, so no host copy is timed).  Pair i:
frame i is the target map, frame i + 1 the source, from the ground-truth relative pose perturbed by 0.5 deg / 0.1 m.  VGICP at leaf 1.0,
search_offsets 1 (--target kdtree: GICP against a kd-tree of the target frame), Levenberg-Marquardt and Gauss-Newton, B in
{1, 8, 64, 512} pairs.

Compared in one process, repetitions alternated, median of --reps:
  (a) build_target_voxelmaps (kdtree: build_target_kdtrees) + set_source_batch + align_batch over all B pairs;
  (b) one pair after another on one context: build_target_voxelmap (kdtree: set_target + build_target_kdtree) + set_source_batch of
      one member + align_batch;
  (c) (a) and (b) with the map building left out of both: the maps of (a) are built once beforehand, those of (b) before each pair's
      timed part.
(a) and (b) are checked to reach bit-identical poses before anything is timed.  Also reported: rounds, kernel launches per call and the
build on its own.  The card's name, power limit and maximum SM clock are read with nvidia-smi (read-only) and written next to the numbers.

    python scripts/bench_align_pairs.py [--target voxelmap|kdtree] [--sizes 1,8,64,512] [--reps 10] [--out FILE]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--target", choices=("voxelmap", "kdtree"), default="voxelmap")
    ap.add_argument("--sizes", default="1,8,64,512")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sizes = [int(x) for x in args.sizes.split(",")]

    import torch

    import small_gicp_b200 as sg
    from small_gicp_b200 import synthetic as syn

    info = gpu_info()
    print(json.dumps(info), flush=True)
    dev = torch.device("cuda:0")
    n_frames = max(sizes) + 1
    world = syn.make_world(16_000_000, 42)
    side = syn.world_side(16_000_000)
    poses = [syn.lidar_pose(f, side) for f in range(n_frames)]
    prep = sg.Context(0)
    frames, covs = [], []
    for f in range(n_frames):
        p = prep.voxelgrid_sampling(syn.lidar_frame_torch(world, poses[f], 45 + f, dev).cpu().numpy(), 0.25)
        frames.append(p)
        covs.append(prep.estimate_features(p, 20, normals=False)[1])
    noise = se3_exp(np.array([[0.0, 0.0, np.deg2rad(0.5), 0.1, 0.0, 0.0]]))[0]
    inits = np.array([np.linalg.inv(poses[i]) @ poses[i + 1] @ noise for i in range(n_frames - 1)])
    print(json.dumps({"frames": n_frames, "points_per_frame_mean": float(np.mean([len(p) for p in frames]))}), flush=True)

    # on the device, concatenated: frame f = rows starts[f] .. starts[f + 1]
    starts = np.zeros(n_frames + 1, dtype=np.int64)
    starts[1:] = np.cumsum([len(p) for p in frames])
    P = torch.from_numpy(np.concatenate(frames)).to(dev)
    Cv = torch.from_numpy(np.concatenate(covs)).to(dev)
    one_p = [P[starts[f] : starts[f + 1]] for f in range(n_frames)]
    one_c = [Cv[starts[f] : starts[f + 1]] for f in range(n_frames)]

    ctx_a, ctx_b = sg.Context(0), sg.Context(0)
    results = []
    for B in sizes:
        T0 = inits[:B]
        tgt = ((P[: starts[B]], starts[: B + 1]), Cv[: starts[B]])  # frames 0 .. B - 1
        src = ((P[starts[1] : starts[B + 1]], starts[1 : B + 2] - starts[1]), Cv[starts[1] : starts[B + 1]])  # frames 1 .. B
        for lm in (1, 0):
            name = "LM" if lm else "GN"
            kw = dict(factor=sg.FACTOR_GICP, optimizer=lm)

            def build_a():
                t0 = time.perf_counter()
                if args.target == "kdtree":
                    ctx_a.build_target_kdtrees(tgt[0], None, tgt[1])
                else:
                    ctx_a.build_target_voxelmaps(*tgt, LEAF, OFFSETS)
                ctx_a.synchronize()
                return time.perf_counter() - t0

            def align_a():
                t0 = time.perf_counter()
                ctx_a.set_source_batch(*src)
                r = ctx_a.align_batch(T0, **kw)
                return time.perf_counter() - t0, r

            def run_b():
                """(total, build part, align part, poses, iterations)"""
                total = build = 0.0
                T, it = np.empty((B, 4, 4)), np.empty(B, np.int64)
                for i in range(B):
                    t0 = time.perf_counter()
                    if args.target == "kdtree":
                        ctx_b.set_target(one_p[i], None, one_c[i])
                        ctx_b.build_target_kdtree()
                    else:
                        ctx_b.build_target_voxelmap(one_p[i], one_c[i], LEAF, OFFSETS)
                    ctx_b.synchronize()
                    t1 = time.perf_counter()
                    ctx_b.set_source_batch((one_p[i + 1], [0, len(one_p[i + 1])]), one_c[i + 1])
                    r = ctx_b.align_batch(T0[i : i + 1], **kw)
                    t2 = time.perf_counter()
                    build += t1 - t0
                    total += t2 - t0
                    T[i], it[i] = r.T_target_source[0], r.iterations[0]
                return total, build, total - build, T, it

            # (a) and (b) must reach bit-identical poses before anything is timed
            k0 = ctx_a.kernel_launches
            build_a()
            k1 = ctx_a.kernel_launches
            _, ra = align_a()
            k2 = ctx_a.kernel_launches
            kb0 = ctx_b.kernel_launches
            _, _, _, Tb, ib = run_b()
            kb = (ctx_b.kernel_launches - kb0) / B
            same = bool(np.array_equal(ra.T_target_source, Tb) and np.array_equal(ra.iterations, ib))
            print(json.dumps({"B": B, "optimizer": name, "bit_identical": same}), flush=True)
            if not same:
                raise SystemExit(f"(a) and (b) differ at B = {B}, {name}")
            ta, ta_build, ta_align, tb, tb_build, tb_align = [], [], [], [], [], []
            for _ in range(args.reps):
                tbuild = build_a()
                talign, _ = align_a()
                ta.append(tbuild + talign)
                ta_build.append(tbuild)
                ta_align.append(talign)
                total, build, align, _, _ = run_b()
                tb.append(total)
                tb_build.append(build)
                tb_align.append(align)
            med = lambda x: 1e3 * float(np.median(x))
            rec = {
                "B": B,
                "target": args.target,
                "optimizer": name,
                "iterations_max": int(ra.iterations.max()),
                "converged": int(ra.converged.sum()),
                "launches_build_a": k1 - k0,
                "launches_align_a": k2 - k1,
                "launches_per_pair_b": kb,
                "a_ms": med(ta),
                "b_ms": med(tb),
                "a_per_pair_ms": med(ta) / B,
                "b_per_pair_ms": med(tb) / B,
                "c_a_align_only_ms": med(ta_align),
                "c_b_align_only_ms": med(tb_align),
                "c_a_per_pair_ms": med(ta_align) / B,
                "c_b_per_pair_ms": med(tb_align) / B,
                "build_a_ms": med(ta_build),
                "build_b_ms": med(tb_build),
                "a_range_ms": [1e3 * min(ta), 1e3 * max(ta)],
                "b_range_ms": [1e3 * min(tb), 1e3 * max(tb)],
                "speedup_a_over_b": float(np.median(tb) / np.median(ta)),
                "speedup_c": float(np.median(tb_align) / np.median(ta_align)),
                **info,
            }
            print(json.dumps(rec), flush=True)
            results.append(rec)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"setup": info, "target": args.target, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
