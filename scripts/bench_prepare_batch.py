"""Batched preparation of many frames (sgb_voxelgrid_sampling_batch + sgb_estimate_features_batch) against preparing them one call at a
time, on one GPU, alone and as part of re-registering consecutive frame pairs.

Workload: raw frames of the synthetic LiDAR stream (synthetic.lidar_frame_torch in the 16M-point world, 64 x 1875 = 120k rays, 1 m
forward + 1 deg yaw per frame), kept on the device (all frames concatenated in one tensor; every path passes device pointers and gets
device outputs, so no host copy is timed).  B pairs use frames 0 .. B: voxel grid at 0.25 m, then k = 20 covariances.

Compared in one process, repetitions alternated, median of --reps:
  (a) prep: voxelgrid_sampling_batch + estimate_features_batch over the B + 1 frames;
  (b) prep: sgb_voxelgrid_sampling + sgb_estimate_features per frame;
  end-to-end per pair: the preparation, then build_target_kdtrees (frames 0 .. B - 1) + set_source_batch (frames 1 .. B) + GICP
  align_batch (Levenberg-Marquardt) from the ground-truth relative pose perturbed by 0.5 deg / 0.1 m, for (a) and for (b) (whose
  per-frame outputs are concatenated on the device first).
The end-to-end poses and iterations of (a) and (b) are compared bit for bit before anything is timed.  Also reported: kernel launches
and host synchronisations per call.  The card's name, power limit and maximum SM clock are read with nvidia-smi (read-only) and written
next to the numbers.

    python scripts/bench_prepare_batch.py [--sizes 1,8,64,512] [--reps 5] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_align_batch import gpu_info, se3_exp  # noqa: E402

LEAF, K = 0.25, 20
# host synchronisations per call, by construction (sgb_capi_preprocess.cu) with device-resident outputs
SYNCS_VOXELGRID_SINGLE, SYNCS_FEATURES_SINGLE, SYNCS_VOXELGRID_BATCH, SYNCS_FEATURES_BATCH = 2, 1, 1, 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,64,512")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    sizes = [int(x) for x in args.sizes.split(",")]

    import torch

    import small_gicp_b200 as sg
    from small_gicp_b200 import capi
    from small_gicp_b200 import synthetic as syn

    info = gpu_info()
    print(json.dumps(info), flush=True)
    dev = torch.device("cuda:0")
    n_frames = max(sizes) + 1
    world = syn.make_world(16_000_000, 42)
    side = syn.world_side(16_000_000)
    poses = [syn.lidar_pose(f, side) for f in range(n_frames)]
    raw = [syn.lidar_frame_torch(world, poses[f], 45 + f, dev) for f in range(n_frames)]
    starts = np.zeros(n_frames + 1, dtype=np.int64)
    starts[1:] = np.cumsum([len(r) for r in raw])
    R = torch.cat(raw).contiguous()
    del raw
    print(json.dumps({"frames": n_frames, "rays_per_frame_mean": float(np.mean(np.diff(starts)))}), flush=True)
    noise = se3_exp(np.array([[0.0, 0.0, np.deg2rad(0.5), 0.1, 0.0, 0.0]]))[0]
    inits = np.array([np.linalg.inv(poses[i]) @ poses[i + 1] @ noise for i in range(n_frames - 1)])

    ctx_a, ctx_b = sg.Context(0), sg.Context(0)
    reg_a, reg_b = sg.Context(0), sg.Context(0)
    vg_out = torch.empty((int(np.diff(starts).max()), 4), dtype=torch.float64, device=dev)

    def prep_a(B):
        pts, off = ctx_a.voxelgrid_sampling_batch((R[: starts[B + 1]], starts[: B + 2]), LEAF)
        _, covs = ctx_a.estimate_features_batch((pts, off), K, normals=False)
        return pts, off, covs

    def prep_b(B):
        """per frame: sgb_voxelgrid_sampling into a device buffer, then sgb_estimate_features of that cloud (device outputs)"""
        pts, covs = [], []
        m = C.c_size_t(0)
        for f in range(B + 1):
            p = R[starts[f] : starts[f + 1]]
            ctx_b._check(ctx_b._L.sgb_voxelgrid_sampling(ctx_b._h, p.shape[0], capi._d(p), LEAF, capi._d(vg_out), C.byref(m)))
            q = vg_out[: m.value].clone()
            _, c = ctx_b.estimate_features(q, K, normals=False)
            pts.append(q)
            covs.append(c)
        return pts, covs

    def register(ctx, pts, off, covs, B):
        ctx.build_target_kdtrees((pts[: off[B]], off[: B + 1]), None, covs[: off[B]])
        ctx.set_source_batch((pts[off[1] : off[B + 1]], off[1 : B + 2] - off[1]), covs[off[1] : off[B + 1]])
        return ctx.align_batch(inits[:B], factor=sg.FACTOR_GICP, optimizer=1)

    def end_to_end_a(B):
        t0 = time.perf_counter()
        pts, off, covs = prep_a(B)
        r = register(reg_a, pts, off, covs, B)
        return time.perf_counter() - t0, r

    def end_to_end_b(B):
        t0 = time.perf_counter()
        pts, covs = prep_b(B)
        off = np.r_[0, np.cumsum([len(p) for p in pts])]
        r = register(reg_b, torch.cat(pts), off, torch.cat(covs), B)
        return time.perf_counter() - t0, r

    def timed(fn, B):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn(B)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    results = []
    for B in sizes:
        # launches per call, and (a) against (b) end to end, bit for bit
        k0 = ctx_a.kernel_launches
        ctx_a.voxelgrid_sampling_batch((R[: starts[B + 1]], starts[: B + 2]), LEAF)
        k1 = ctx_a.kernel_launches
        prep_a(B)
        k2 = ctx_a.kernel_launches
        kb0 = ctx_b.kernel_launches
        prep_b(B)
        kb = ctx_b.kernel_launches - kb0
        _, ra = end_to_end_a(B)
        _, rb = end_to_end_b(B)
        same = bool(np.array_equal(ra.T_target_source, rb.T_target_source) and np.array_equal(ra.iterations, rb.iterations))
        print(json.dumps({"B": B, "bit_identical_end_to_end": same}), flush=True)
        pa, pb, ea, eb = [], [], [], []
        for _ in range(args.reps):
            pa.append(timed(prep_a, B))
            pb.append(timed(prep_b, B))
            ea.append(end_to_end_a(B)[0])
            eb.append(end_to_end_b(B)[0])
        med = lambda x: 1e3 * float(np.median(x))
        rec = {
            "B": B,
            "frames": B + 1,
            "launches_voxelgrid_batch": k1 - k0,
            "launches_features_batch": (k2 - k1) - (k1 - k0),
            "launches_per_frame_single": kb / (B + 1),
            "host_syncs_a": SYNCS_VOXELGRID_BATCH + SYNCS_FEATURES_BATCH,
            "host_syncs_b": (SYNCS_VOXELGRID_SINGLE + SYNCS_FEATURES_SINGLE) * (B + 1),
            "prep_a_ms": med(pa),
            "prep_b_ms": med(pb),
            "prep_a_per_frame_ms": med(pa) / (B + 1),
            "prep_b_per_frame_ms": med(pb) / (B + 1),
            "prep_speedup": float(np.median(pb) / np.median(pa)),
            "e2e_a_per_pair_ms": med(ea) / B,
            "e2e_b_per_pair_ms": med(eb) / B,
            "e2e_speedup": float(np.median(eb) / np.median(ea)),
            "prep_a_range_ms": [1e3 * min(pa), 1e3 * max(pa)],
            "prep_b_range_ms": [1e3 * min(pb), 1e3 * max(pb)],
            "iterations_max": int(ra.iterations.max()),
            "bit_identical_end_to_end": same,
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
