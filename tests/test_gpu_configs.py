"""The remaining BASELINE.json configurations as parity cases (sizes the oracle finishes in seconds):
  configs[2]  frame-to-frame GICP odometry stream (benchmark_odom.hpp:49-82 + odometry_benchmark_small_gicp_tbb.cpp:22-48):
              per frame 0.25 m voxel grid, k = 20 covariances, tree, LM GICP against the previous frame from identity
  configs[3]  VGICP (Gaussian voxel map target, leaf 1.0), LevenbergMarquardt
  configs[4]  size sweep: same sums at several sizes (here 20k / 60k; the 1M case lives in test_gpu_parity.py)"""
import numpy as np
import pytest

import oracle as O
from conftest import pose_error

pytestmark = pytest.mark.gpu


def lidar_like_frames(n_frames=4, n_points=60_000, seed=45):
    """A sensor moving 0.3 m + 0.5 deg yaw per frame through the synthetic room: every frame is an independent sample of the
    surfaces seen from the sensor pose, expressed in the sensor frame (stand-in for the KITTI stream, which is not available)."""
    from small_gicp_b200 import synthetic as syn

    world = syn.make_world(250_000, 42)
    frames, poses = [], []
    for f in range(n_frames):
        yaw = np.deg2rad(0.5 * f)
        T = np.eye(4)
        T[:3, :3] = [[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]]
        T[:3, 3] = [25.0 + 0.3 * f, 25.0, 1.5]
        pts = syn.sample_cloud(world, n_points, seed + f)
        Ti = np.linalg.inv(T)
        local = pts @ Ti[:3, :3].T + Ti[:3, 3]
        keep = np.linalg.norm(local, axis=1) < 20.0
        frames.append(local[keep].astype(np.float32).astype(np.float64))
        poses.append(T)
    return frames, poses


def test_odometry_stream_matches_oracle():
    import small_gicp_b200 as sg
    from small_gicp_b200 import host_api

    frames, poses = lidar_like_frames()
    ctx = sg.Context(0)
    prev = None
    T_gpu, T_cpu = np.eye(4), np.eye(4)
    for f, raw in enumerate(frames):
        # device pipeline
        pts = ctx.voxelgrid_sampling(raw, 0.25)
        _, covs = ctx.estimate_features(pts, 20, normals=False)
        # oracle pipeline
        oc = O.Cloud(raw).voxelgrid_sampling(0.25)
        ot = O.KdTree(oc)
        ot.estimate(20, O.FEAT_COV, max(1, O.max_threads()))
        np.testing.assert_allclose(pts, oc.points, atol=1e-9)
        if prev is not None:
            r = host_api.align(prev[0], pts, None, prev[1], covs, factor=sg.FACTOR_GICP, optimizer=host_api.OPT_LM, tree=host_api.TREE_DEVICE_KDTREE)
            ref = O.Registration(factor=O.FACTOR_GICP, num_threads=max(1, O.max_threads())).align(prev[2], prev[3], oc, np.eye(4))
            rot, trans = pose_error(ref.T_target_source, r.T_target_source)
            assert rot < 1e-4 and trans < 1e-3, (f, rot, trans)  # device covariances: same neighbour sets as the oracle's (exact re-rank)
            gt = np.linalg.inv(poses[f - 1]) @ poses[f]
            rot, trans = pose_error(gt, r.T_target_source)
            assert rot < 3e-3 and trans < 3e-2, (f, rot, trans)
            T_gpu, T_cpu = T_gpu @ r.T_target_source, T_cpu @ ref.T_target_source
        prev = (pts, covs, oc, ot)
    rot, trans = pose_error(T_cpu, T_gpu)
    assert rot < 1e-3 and trans < 1e-2
    ctx.close()


def test_vgicp_lm_synthetic():
    from small_gicp_b200 import host_api
    from small_gicp_b200.synthetic import make_pair

    tgt, src, Tgt = make_pair(100_000)
    nt = max(1, O.max_threads())
    tc, sc = O.Cloud(tgt), O.Cloud(src)
    tt, st = O.KdTree(tc), O.KdTree(sc)
    tt.estimate(20, O.FEAT_COV, nt)
    st.estimate(20, O.FEAT_COV, nt)
    vm = O.GaussianVoxelMap(tc, 1.0)
    ref = O.Registration(factor=O.FACTOR_GICP, num_threads=nt).align(vm, None, sc, np.eye(4))
    r = host_api.align(tc.points, sc.points, None, tc.covs, sc.covs, tree=host_api.TREE_VOXELMAP, voxel_resolution=1.0, optimizer=host_api.OPT_LM)
    rot, trans = pose_error(ref.T_target_source, r.T_target_source)
    assert rot < 1e-4 and trans < 1e-3, (rot, trans)
    assert r.iterations == ref.iterations and abs(r.num_inliers - ref.num_inliers) <= 3
    rot, trans = pose_error(Tgt, r.T_target_source)
    assert rot < 5e-3 and trans < 5e-2


@pytest.mark.parametrize("n", [20_000, 60_000])
@pytest.mark.parametrize("factor", [0, 2])
def test_size_sweep_first_and_converged_pose(n, factor):
    import np_factors as NF
    import small_gicp_b200 as sg
    from small_gicp_b200.synthetic import make_pair

    tgt, src, Tgt = make_pair(n)
    nt = max(1, O.max_threads())
    tc, sc = O.Cloud(tgt), O.Cloud(src)
    tt, st = O.KdTree(tc), O.KdTree(sc)
    tt.estimate(20, O.FEAT_NORMAL_COV, nt)
    st.estimate(20, O.FEAT_COV, nt)
    ctx = sg.Context(0)
    ctx.set_target(tc.points, tc.normals, tc.covs)
    ctx.build_target_kdtree()
    ctx.set_source(sc.points, sc.covs)
    reg = O.Registration(factor=factor, num_threads=0)
    model = NF.storage_model(sc.points, sc.covs, tc.points, tc.normals, tc.covs)
    for T in (np.eye(4), Tgt):  # iteration-0 pose and converged pose (traversal cost differs, sums must not)
        H0, b0, e0 = reg.linearize(tc, tt, sc, T)
        H, b, e = ctx.linearize(T, factor=factor)
        cg = ctx.correspondences()
        nm = NF.compare_correspondences(cg, reg.correspondences(len(sc)), tc.points, sc.points, T)
        # always: the GPU sums against numpy on the storage model over the GPU's own correspondences; when the sets agree also
        # against the oracle
        r = NF.tight_ratios((H, b, e), NF.linearize(T, cg, factor, 0, 1.0, *model))
        print(f"worst ratio to the storage model (n={n}, factor {factor}): {max(r):.2e}")
        assert max(r) <= NF.TIGHT, ("H, b, e:", r)
        if nm == 0:
            assert np.linalg.norm(H - H0) <= 2e-5 * np.linalg.norm(H0) and abs(e - e0) <= 2e-5 * e0
    ctx.close()
