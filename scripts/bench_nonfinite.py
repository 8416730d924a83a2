"""Cost of non-finite source rows (NaN, as organized LiDAR clouds mark missing returns) on one GPU.

A non-finite point is inert (include/sgicp_b200.h) and its query is never searched: the grid probe settles it without a correspondence,
the tree walks treat it as an idle lane, and the k-NN of feature estimation returns before walking.  This measures that such rows cost
nothing: one GICP linearize() (aligned pose: grid probe; misaligned pose: packet walk) and one estimate_features() of the source, with
0 rows, 1 row and 30 % of the rows replaced by NaN.  Synthetic pair of --points points each (make_pair); times are the median and
min - max of --reps calls after a warm-up, each ending in a device synchronisation (linearize returns H | b | e to the host).  One JSON
line, with the card's name, power limit and maximum SM clock (nvidia-smi, read-only).

    python scripts/bench_nonfinite.py [--points 200000] [--reps 30]
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


def _ms(fn, reps):
    fn()
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(1e3 * (time.perf_counter() - t0))
    return {"median_ms": float(np.median(t)), "min_ms": float(np.min(t)), "max_ms": float(np.max(t))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=200_000)
    ap.add_argument("--reps", type=int, default=30)
    a = ap.parse_args()
    import small_gicp_b200 as sg
    from small_gicp_b200.synthetic import make_pair

    tgt, src, T = make_pair(a.points)
    ctx = sg.Context(0)
    _, tcov = ctx.estimate_features(tgt, 20, normals=False)
    _, scov0 = ctx.estimate_features(src, 20, normals=False)
    ctx.set_target(tgt, None, tcov)
    ctx.build_target_kdtree()
    D = np.eye(4)
    D[:3, :3] = se3_exp(np.array([[0.01, -0.012, 0.008, 0.0, 0.0, 0.0]]))[0, :3, :3]
    D[:3, 3] = [0.25, -0.2, 0.15]
    rng = np.random.default_rng(0)
    out = {"points": a.points, "reps": a.reps, "gpu": gpu_info(), "cases": {}}
    for name, rows in (("none", []), ("one", [a.points // 2]), ("30pct", rng.choice(a.points, int(0.3 * a.points), replace=False))):
        s = np.array(src)
        s[np.asarray(rows, dtype=np.int64)] = np.nan
        ctx.set_source(s, scov0)
        res = {}
        for pose, Tp in (("aligned", T), ("misaligned", T @ D)):
            res[f"linearize_{pose}"] = _ms(lambda: ctx.linearize(Tp, factor=sg.FACTOR_GICP), a.reps)
            res[f"inliers_{pose}"] = ctx.num_inliers()
        res["estimate_features"] = _ms(lambda: ctx.estimate_features(s, 20, normals=False), max(3, a.reps // 5))
        out["cases"][name] = res
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
