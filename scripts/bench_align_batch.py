"""Batched align() against what a caller has to write without it, on one GPU.

Workload: a 1M-point synthetic room (synthetic.make_pair) as the target, device kd-tree and device-estimated normals / covariances;
B in {1, 8, 64, 512, 4096} members of 20k source points each (8 distinct 20k samples of the room, cycled), every member from its own
initial pose: the ground truth perturbed by <= 0.5 m and <= 5 deg about the member's centre.  GICP, Gauss-Newton and Levenberg-Marquardt.

Compared in one process, repetitions alternated, median of --reps:
  (a) Context.align_batch: sgb_align_batch, the optimiser step on the device;
  (b) the lockstep loop in Python over linearize_batch / error_batch with the 6x6 solves and exponentials on the host (numpy, batched);
  (c) one member after another on a single-source context with the target resident: set_source, then the same loop with B = 1.
      (c) costs the same per member whatever B is, so it runs over the first --single-members members only; reported per member.
(a) and (b) are checked against each other before anything is timed.  Also reported: rounds, kernel launches per align, and the
sgb_source_set_batch upload, timed on its own.  The card's name, power limit and maximum SM clock are read with nvidia-smi (read-only)
and written next to the numbers.

    python scripts/bench_align_batch.py [--sizes 1,8,64,512,4096] [--reps 10] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    name, power, clock = [s.strip() for s in out.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def se3_exp(a):
    """(B, 6) twists -> (B, 4, 4), the reference's quaternion form (util/lie.hpp)"""
    w, v = a[:, :3], a[:, 3:]
    th2 = (w * w).sum(1)
    th = np.sqrt(th2)
    small = th2 < 1e-10
    ths = np.where(small, 1.0, th)
    im = np.where(small, 0.5 - th2 / 48.0 + th2 * th2 / 3840.0, np.sin(0.5 * ths) / ths)
    re = np.where(small, 1.0 - th2 / 8.0 + th2 * th2 / 384.0, np.cos(0.5 * ths))
    x, y, z = (im[:, None] * w).T
    R = np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * re), 2 * (x * z + y * re), 2 * (x * y + z * re), 1 - 2 * (x * x + z * z), 2 * (y * z - x * re),
                  2 * (x * z - y * re), 2 * (y * z + x * re), 1 - 2 * (x * x + y * y)], axis=1).reshape(-1, 3, 3)
    W = np.zeros((len(a), 3, 3))
    W[:, 0, 1], W[:, 0, 2], W[:, 1, 0], W[:, 1, 2], W[:, 2, 0], W[:, 2, 1] = -w[:, 2], w[:, 1], w[:, 2], -w[:, 0], -w[:, 1], w[:, 0]
    V = np.eye(3) + W * ((1 - np.cos(ths)) / np.where(small, 1.0, th2))[:, None, None] + (W @ W) * ((ths - np.sin(ths)) / np.where(small, 1.0, th2 * ths))[:, None, None]
    V[small] = R[small]
    T = np.tile(np.eye(4), (len(a), 1, 1))
    T[:, :3, :3] = R
    T[:, :3, 3] = (V @ v[:, :, None])[:, :, 0]
    return T


def lockstep(linearize, error, inits, lm, max_iterations=20, gn_lambda=1e-6, max_inner=10, init_lambda=1e-3, factor=10.0, reps=0.1 * np.pi / 180, teps=1e-3):
    """GaussNewtonOptimizer / LevenbergMarquardtOptimizer of every member in lockstep, the per-member solve and update on the host.
    linearize(T, active) -> (H, b, e, inliers); error(T, active) -> e.  Returns T, converged, iterations, error, rounds."""
    B = len(inits)
    T = inits.copy()
    conv = np.zeros(B, bool)
    alive = np.ones(B, bool)
    iters = np.zeros(B, np.int64)
    err = np.zeros(B)
    lam = np.full(B, init_lambda)
    rounds = 0
    I6 = np.eye(6)
    for it in range(max_iterations):
        act = alive & ~conv
        if not act.any():
            break
        H, b, e, _ = linearize(T, act)
        rounds += 1
        idx = np.nonzero(act)[0]
        iters[idx] = it
        err[idx] = e[idx]
        if not lm:
            d = np.linalg.solve(H[idx] + gn_lambda * I6, -b[idx][:, :, None])[:, :, 0]
            conv[idx] = (np.linalg.norm(d[:, :3], axis=1) <= reps) & (np.linalg.norm(d[:, 3:], axis=1) <= teps)
            T[idx] = T[idx] @ se3_exp(d)
            continue
        trial = act.copy()
        d = np.zeros((B, 6))
        cand = T.copy()
        for _ in range(max_inner):
            t = np.nonzero(trial)[0]
            if not len(t):
                break
            d[t] = np.linalg.solve(H[t] + lam[t, None, None] * I6, -b[t][:, :, None])[:, :, 0]
            cand[t] = T[t] @ se3_exp(d[t])
            ce = error(cand, trial)
            rounds += 1
            ok = trial & (ce <= err)
            k = np.nonzero(ok)[0]
            conv[k] = (np.linalg.norm(d[k, :3], axis=1) <= reps) & (np.linalg.norm(d[k, 3:], axis=1) <= teps)
            T[k] = cand[k]
            lam[k] /= factor
            err[k] = ce[k]
            rej = trial & ~ok
            lam[rej] *= factor
            trial = rej
        alive &= ~trial  # no trial accepted: the member stops (the reference's break)
    return T, conv, iters, err, rounds


def rot_trans(Ta, Tb):
    E = np.linalg.inv(Ta) @ Tb
    ang = np.arccos(np.clip((np.trace(E[:, :3, :3], axis1=1, axis2=2) - 1) / 2, -1, 1))
    return ang, np.linalg.norm(E[:, :3, 3], axis=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,64,512,4096")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--points", type=int, default=20000)
    ap.add_argument("--target", type=int, default=1_000_000)
    ap.add_argument("--single-members", type=int, default=64)
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    import torch

    import small_gicp_b200 as sg
    from small_gicp_b200.synthetic import make_pair

    info = gpu_info()
    print(json.dumps(info), flush=True)
    pool = 8
    tgt, src, Tgt = make_pair(args.target, n_source=pool * args.points)
    ctx = sg.Context(0)
    ctx.set_target(tgt)
    ctx.build_target_kdtree()
    ctx.estimate_target_features(20)
    ctx1 = sg.Context(0)  # (c): the same target, resident, one source at a time
    ctx1.set_target(tgt)
    ctx1.build_target_kdtree()
    ctx1.estimate_target_features(20)
    dev = torch.device("cuda:0")
    slices = [src[j * args.points : (j + 1) * args.points] for j in range(pool)]
    pts = [torch.from_numpy(np.c_[s, np.ones(len(s))]).to(dev) for s in slices]
    covs = [ctx.estimate_features(p, 20, normals=False)[1] for p in pts]
    centres = [0.5 * (s.min(0) + s.max(0)) for s in slices]

    results = []
    for B in [int(x) for x in args.sizes.split(",")]:
        rng = np.random.default_rng(B)
        inits = np.empty((B, 4, 4))
        for m in range(B):
            ax = rng.normal(size=3)
            ax /= np.linalg.norm(ax)
            P = se3_exp(np.r_[ax * rng.uniform(0, np.deg2rad(5.0)), np.zeros(3)][None])[0]
            C = np.eye(4)
            C[:3, 3] = Tgt[:3, :3] @ centres[m % pool] + Tgt[:3, 3]
            P[:3, 3] = rng.uniform(-1, 1, 3) * (0.5 / np.sqrt(3))  # |t| <= 0.5 m
            inits[m] = C @ P @ np.linalg.inv(C) @ Tgt  # rotated about the member's centre, then moved
        members = [m % pool for m in range(B)]
        offsets = np.arange(B + 1, dtype=np.uint64) * args.points
        P_all = torch.cat([pts[j] for j in members])
        C_all = torch.cat([covs[j] for j in members])
        up = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ctx.set_source_batch((P_all, offsets), C_all)
            ctx.synchronize()
            up.append(time.perf_counter() - t0)
        del P_all, C_all
        torch.cuda.empty_cache()
        n1 = min(B, args.single_members)
        pts1 = [pts[j].cpu().numpy() for j in range(pool)]
        covs1 = [covs[j].cpu().numpy() for j in range(pool)]

        for lm in (0, 1):
            name = "LM" if lm else "GN"

            def run_a():
                k0 = ctx.kernel_launches
                t0 = time.perf_counter()
                r = ctx.align_batch(inits, factor=2, optimizer=lm)
                return time.perf_counter() - t0, r, ctx.kernel_launches - k0

            def run_b():
                k0 = ctx.kernel_launches
                t0 = time.perf_counter()
                out = lockstep(lambda T, a: ctx.linearize_batch(T, active=a, factor=2), lambda T, a: ctx.error_batch(T, active=a), inits, lm)
                return time.perf_counter() - t0, out, ctx.kernel_launches - k0

            def run_c():
                t_run = 0.0
                for m in range(n1):
                    ctx1.set_source(pts1[members[m]], covs1[members[m]])
                    ctx1.synchronize()

                    def lin1(T, a):
                        H, b, e = ctx1.linearize(T[0], factor=2)
                        return H[None], b[None], np.array([e]), None

                    t0 = time.perf_counter()
                    lockstep(lin1, lambda T, a: np.array([ctx1.error(T[0])]), inits[m : m + 1], lm)
                    t_run += time.perf_counter() - t0
                return t_run

            # agreement of (a) and (b) before timing
            _, ra, launches_a = run_a()
            _, (Tb, cb, ib, eb, rounds), launches_b = run_b()
            rot, trans = rot_trans(ra.T_target_source, Tb)
            differ = int((ra.iterations != ib).sum() + (ra.converged != cb).sum())
            agree = {"worst_rot": float(rot.max()), "worst_trans": float(trans.max()), "members_differing_iterations_or_converged": differ}
            print(json.dumps({"B": B, "optimizer": name, "agreement": agree}), flush=True)
            if rot.max() > 1e-4 or trans.max() > 1e-3 or differ > max(1, B // 100):
                raise SystemExit(f"(a) and (b) disagree at B = {B}, {name}: {agree}")
            ta, tb, tc = [], [], []
            for _ in range(args.reps):
                ta.append(run_a()[0])
                tb.append(run_b()[0])
                tc.append(run_c())
            rec = {
                "B": B,
                "optimizer": name,
                "points_per_member": args.points,
                "rounds": rounds,
                "iterations_max": int(ra.iterations.max()),
                "converged": int(ra.converged.sum()),
                "launches_a": launches_a,
                "launches_b": launches_b,
                "a_align_batch_ms": 1e3 * float(np.median(ta)),
                "b_python_lockstep_ms": 1e3 * float(np.median(tb)),
                "c_single_per_member_ms": 1e3 * float(np.median(tc)) / n1,
                "a_per_member_ms": 1e3 * float(np.median(ta)) / B,
                "b_per_member_ms": 1e3 * float(np.median(tb)) / B,
                "a_range_ms": [1e3 * min(ta), 1e3 * max(ta)],
                "b_range_ms": [1e3 * min(tb), 1e3 * max(tb)],
                "c_members_timed": n1,
                "upload_set_source_batch_ms": 1e3 * float(np.median(up)),
                "agreement": agree,
                **info,
            }
            print(json.dumps(rec), flush=True)
            results.append(rec)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"setup": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
