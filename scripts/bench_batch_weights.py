"""What per-point weights cost and what they buy: batched calls with and without sgb_source_set_weights, on one GPU.

Workloads, each at B in {1, 64, 512} (--sizes), GICP, max_dist_sq 1 (those of bench_batch_points.py):
  pairs-kdtree: the LiDAR frame pairs of bench_align_async.py (frame i a kd-tree map, frame i + 1 the source), at the perturbed initial
      relative poses;
  room: members of 20k points against the 1M-point synthetic room of bench_align_batch.py (one device kd-tree), at perturbed poses.
Per call, median of --reps after two warm-ups, the arms alternating call by call (each call returns with its results):
  lin_{plain,ones,random}_ms    Context.linearize_batch without weights, with all weights 1, with random weights in [0, 3];
  align_{plain,ones,random}_ms  Context.align_batch (Levenberg-Marquardt, 20 iterations) likewise;
  set_host_ms / set_dev_ms      Context.set_source_weights from a numpy array / from a CUDA tensor.
The all-ones arm is first checked to be bit-identical to the plain one.
Accuracy (--accuracy): --acc-pairs LiDAR pairs whose source frame has a rigid object of about 15 % of its points (the points nearest
a random point, in the horizontal plane) moved by 0.8 m and 10 degrees before the covariances are estimated.  Against the ground-truth
relative pose: the plain LM align, and a two-pass align -- align, error_batch_points at the result, weight 0 for every row above 10x
its member's median positive row, align again from the first result.
The card's name, power limit and maximum SM clock are read with nvidia-smi (read-only) and written next to the numbers.

    python scripts/bench_batch_weights.py [--sizes 1,64,512] [--reps 20] [--workloads pairs-kdtree,room] [--accuracy] [--out FILE]
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

from bench_align_async import lidar_pairs  # noqa: E402
from bench_align_batch import gpu_info, se3_exp  # noqa: E402


def pose_error(T1, T2):
    e = np.linalg.inv(T1) @ T2
    return float(np.degrees(np.arccos(np.clip((np.trace(e[:3, :3]) - 1.0) / 2.0, -1.0, 1.0)))), float(np.linalg.norm(e[:3, 3]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,64,512")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--workloads", default="pairs-kdtree,room")
    ap.add_argument("--accuracy", action="store_true")
    ap.add_argument("--acc-pairs", type=int, default=32)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sizes = [int(x) for x in args.sizes.split(",")] if args.sizes else []
    workloads = args.workloads.split(",") if args.workloads else []

    import torch

    import small_gicp_b200 as sg
    from small_gicp_b200.synthetic import make_pair

    info = gpu_info()
    print(json.dumps(info), flush=True)
    dev = torch.device("cuda:0")
    results = []
    med = lambda x: 1e3 * float(np.median(x[2:]))

    def measure(name, B, ctx, inits):
        kw = dict(factor=sg.FACTOR_GICP, max_dist_sq=1.0)
        n = int(ctx._batch_offsets[-1])
        ones = np.ones(n)
        rnd = np.random.default_rng(B).uniform(0.0, 3.0, n)
        rnd_dev = torch.from_numpy(rnd).to(dev)

        def arm(w, call):
            def f():
                ctx.set_source_weights(w)  # (outside the timed call)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                call()
                return time.perf_counter() - t0
            return f

        lin = lambda: ctx.linearize_batch(inits, **kw)
        aln = lambda: ctx.align_batch(inits, **kw)
        ctx.set_source_weights(None)
        plain = lin(), aln()
        ctx.set_source_weights(ones)
        if not all(np.array_equal(a, b) for a, b in zip(plain[0], lin())) or not np.array_equal(plain[1].T_target_source, aln().T_target_source):
            raise SystemExit(f"{name} B = {B}: all-ones weights changed the results")
        arms = {f"{c}_{w}": arm(wv, f) for c, f in (("lin", lin), ("align", aln)) for w, wv in (("plain", None), ("ones", ones), ("random", rnd))}
        times = {k: [] for k in arms}
        times["set_host"], times["set_dev"] = [], []
        for _ in range(args.reps + 2):  # the first two of each are warm-up
            for k, f in arms.items():
                times[k].append(f())
            for k, w in (("set_host", rnd), ("set_dev", rnd_dev)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ctx.set_source_weights(w)
                times[k].append(time.perf_counter() - t0)
        ctx.set_source_weights(None)
        rec = {"workload": name, "B": B, "points": n, **{f"{k}_ms": med(v) for k, v in times.items()}, **info}
        rec["lin_random_over_plain"] = rec["lin_random_ms"] / rec["lin_plain_ms"]
        rec["align_ones_over_plain"] = rec["align_ones_ms"] / rec["align_plain_ms"]
        print(json.dumps(rec), flush=True)
        results.append(rec)

    if "pairs-kdtree" in workloads and sizes:
        P, Cv, starts, inits = lidar_pairs(sg, torch, max(sizes), dev)
        ctx = sg.Context(0)
        for B in sizes:
            ctx.build_target_kdtrees((P[: starts[B]], starts[: B + 1]), None, Cv[: starts[B]])
            ctx.set_source_batch((P[starts[1] : starts[B + 1]], starts[1 : B + 2] - starts[1]), Cv[starts[1] : starts[B + 1]])
            measure("pairs-kdtree", B, ctx, np.ascontiguousarray(inits[:B]))
        ctx.close()
    if "room" in workloads and sizes:
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
            measure("room", B, ctx, inits)
        ctx.close()

    if args.accuracy:
        from small_gicp_b200 import synthetic as syn

        K = args.acc_pairs
        world = syn.make_world(16_000_000, 42)
        side = syn.world_side(16_000_000)
        poses = [syn.lidar_pose(f, side) for f in range(K + 1)]
        prep = sg.Context(0)
        rng = np.random.default_rng(7)
        move = se3_exp(np.array([[0.0, 0.0, np.deg2rad(10.0), 0.8, 0.0, 0.0]]))[0]
        frames, covs, moved = [], [], []
        for f in range(K + 1):
            p = prep.voxelgrid_sampling(syn.lidar_frame_torch(world, poses[f], 45 + f, dev).cpu().numpy(), 0.25)
            if f > 0:  # the source frames: a rigid object of ~15 % of the points moved
                c = p[rng.integers(len(p)), :2]
                d = np.linalg.norm(p[:, :2] - c, axis=1)
                obj = d <= np.quantile(d, 0.15)
                ctr = np.r_[p[obj, :3].mean(0), 1.0]
                q = p[obj, :3] - ctr[:3]
                p[obj, :3] = q @ move[:3, :3].T + move[:3, 3] + ctr[:3]
                moved.append(float(obj.mean()))
            frames.append(p)
            covs.append(prep.estimate_features(p, 20, normals=False)[1])
        prep.close()
        noise = se3_exp(np.array([[0.0, 0.0, np.deg2rad(0.5), 0.1, 0.0, 0.0]]))[0]
        gt = np.array([np.linalg.inv(poses[i]) @ poses[i + 1] for i in range(K)])
        inits = np.array([g @ noise for g in gt])
        off = np.zeros(K + 2, dtype=np.int64)
        off[1:] = np.cumsum([len(p) for p in frames])
        Pa, Ca = np.concatenate(frames), np.concatenate(covs)
        ctx = sg.Context(0)
        ctx.build_target_kdtrees((Pa[: off[K]], off[: K + 1]), None, Ca[: off[K]])
        ctx.set_source_batch((Pa[off[1] : off[K + 1]], off[1 : K + 2] - off[1]), Ca[off[1] : off[K + 1]])
        kw = dict(factor=sg.FACTOR_GICP, max_dist_sq=1.0)
        first = ctx.align_batch(inits, **kw)
        _, pe = ctx.error_batch_points(first.T_target_source)
        bo = ctx._batch_offsets
        w = np.ones(len(pe))
        for m in range(K):
            rows = pe[bo[m] : bo[m + 1]]
            pos = rows[rows > 0]
            if len(pos):
                w[bo[m] : bo[m + 1]] = np.where(rows > 10.0 * np.median(pos), 0.0, 1.0)
        ctx.set_source_weights(w)
        second = ctx.align_batch(first.T_target_source, **kw)
        ctx.set_source_weights(None)
        errs = {"plain": [pose_error(gt[m], first.T_target_source[m]) for m in range(K)],
                "two_pass": [pose_error(gt[m], second.T_target_source[m]) for m in range(K)]}
        rec = {"workload": "accuracy-moving-object", "pairs": K, "moved_fraction": float(np.mean(moved)), "zero_weight_fraction": float(1.0 - w.mean()),
               **info}
        for k, v in errs.items():
            v = np.array(v)
            rec[f"{k}_rot_deg_median"], rec[f"{k}_trans_m_median"] = float(np.median(v[:, 0])), float(np.median(v[:, 1]))
            rec[f"{k}_rot_deg_max"], rec[f"{k}_trans_m_max"] = float(v[:, 0].max()), float(v[:, 1].max())
        rec["two_pass_converged"] = int(second.converged.sum())
        print(json.dumps(rec), flush=True)
        results.append(rec)
        ctx.close()

    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"setup": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
