"""Batched align() (sgb_align_batch, Context.align_batch, BatchRegistration / host_api.align_batch): every member of a multi-start batch
against the oracle's Registration<>::align and against the single-source align() of the host mirror from the same initial pose, a member's
results bit-identical whatever else is in the batch, the edge cases, and one step launch per round.

Each comparison prints the worst deviation it reached (run with -s to see it)."""
import numpy as np
import pytest

import np_factors as NF
import oracle as O
from conftest import noise_poses, pose_error
from test_gpu_storage_model import Data, about

pytestmark = pytest.mark.gpu


def _sg():
    import small_gicp_b200 as sg

    return sg


def _starts(n=16):
    """noise_poses() and more random poses <= 0.5 m / <= 10 deg (registration_test.cpp:60-71 analogue), n in all"""
    rng = np.random.default_rng(17)
    out = list(noise_poses())
    while len(out) < n:
        ax = rng.normal(size=3)
        ax /= np.linalg.norm(ax)
        out.append(about(np.zeros(3), np.r_[ax * rng.uniform(-1, 1) * np.deg2rad(10.0), rng.uniform(-1, 1, 3) * 0.5]))
    return np.array(out[:n])


def _golden_ctx(g, voxel=False):
    sg = _sg()
    tc, sc = g["target"], g["source"]
    ctx = sg.Context(0)
    if voxel:
        ctx.build_target_voxelmap(tc.points, tc.covs, 1.0, 1)
    else:
        ctx.set_target(tc.points, tc.normals, tc.covs)
        ctx.build_target_kdtree()
    return ctx


ORACLE_CASES = [  # name, factor, robust, optimizer, voxel map
    ("ICP_LM", 0, 0, 1, False),
    ("PLANE_ICP_LM", 1, 0, 1, False),
    ("GICP_LM", 2, 0, 1, False),
    ("GICP_GN", 2, 0, 0, False),
    ("VGICP_LM", 2, 0, 1, True),
]


@pytest.mark.parametrize("name,factor,robust,optimizer,voxel", ORACLE_CASES)
def test_multi_start_matches_oracle(golden_prepared, name, factor, robust, optimizer, voxel):
    g = golden_prepared
    tc, sc = g["target"], g["source"]
    starts = _starts()
    ctx = _golden_ctx(g, voxel)
    ctx.set_source_batch([sc.points] * len(starts), [sc.covs] * len(starts))
    r = ctx.align_batch(starts, factor=factor, robust=robust, optimizer=optimizer)
    reg = O.Registration(factor=factor, robust=robust, num_threads=0)
    reg.set_optimizer(type=optimizer)
    vm = O.GaussianVoxelMap(tc, 1.0, 1) if voxel else None
    worst = (0.0, 0.0)
    for m, T0 in enumerate(starts):
        ref = reg.align(vm, None, sc, T0) if voxel else reg.align(tc, g["target_tree"], sc, T0)
        rot, trans = pose_error(ref.T_target_source, r.T_target_source[m])
        worst = (max(worst[0], rot), max(worst[1], trans))
        assert rot < 1e-4 and trans < 1e-3, (name, m, rot, trans)
        assert r.iterations[m] == ref.iterations, (name, m, r.iterations[m], ref.iterations)
        assert abs(r.num_inliers[m] - ref.num_inliers) <= 2, (name, m, r.num_inliers[m], ref.num_inliers)
    print(f"{name}: worst vs oracle {worst[0]:.2e} rad / {worst[1]:.2e} m over {len(starts)} members, iterations {r.iterations.tolist()}")


SINGLE_CASES = [  # name, factor, robust, robust_c, optimizer, dof_mask
    ("GICP_LM", 2, 0, 1.0, 1, None),
    ("GICP_GN", 2, 0, 1.0, 0, None),
    ("HUBER_ICP_LM", 0, 1, 0.3, 1, None),
    ("CAUCHY_PLANE_ICP_GN", 1, 2, 0.5, 0, None),
    ("GICP_LM_DOF", 2, 0, 1.0, 1, [0, 0, 1, 1, 1, 0]),
    ("HUBER_GICP_GN_DOF", 2, 1, 0.5, 0, [1, 1, 0, 0, 0, 1]),
]


@pytest.mark.parametrize("name,factor,robust,c,optimizer,dof_mask", SINGLE_CASES)
def test_members_match_the_single_path(golden_prepared, name, factor, robust, c, optimizer, dof_mask):
    """every member against host_api.align (Registration<..., ParallelReductionCUDA, ...> on a device kd-tree) with the same options"""
    from small_gicp_b200 import host_api

    sg = _sg()
    g = golden_prepared
    tc, sc = g["target"], g["source"]
    starts = _starts()
    ctx = _golden_ctx(g)
    ctx.set_source_batch([sc.points] * len(starts), [sc.covs] * len(starts))
    kw = dict(factor=factor, robust=robust, robust_c=c, optimizer=optimizer, dof_mask=dof_mask)
    r = ctx.align_batch(starts, **kw)
    corrs = ctx.correspondences_batch()
    worst = (0.0, 0.0)
    for m, T0 in enumerate(starts):
        s = host_api.align(tc.points, sc.points, tc.normals, tc.covs, sc.covs, init_T=T0, tree=host_api.TREE_DEVICE_KDTREE, **kw)
        rot, trans = pose_error(s.T_target_source, r.T_target_source[m])
        worst = (max(worst[0], rot), max(worst[1], trans))
        assert rot < 1e-6 and trans < 1e-5, (name, m, rot, trans)
        assert bool(r.converged[m]) == s.converged and r.iterations[m] == s.iterations, (name, m, r.iterations[m], s.iterations)
        assert abs(r.num_inliers[m] - s.num_inliers) <= 2, (name, m)
        assert abs(r.error[m] - s.error) <= 1e-6 * s.error, (name, m, r.error[m], s.error)
        # the correspondences left behind are those of the member's last linearize
        assert int((corrs[m] != sg.NO_CORRESPONDENCE).sum()) == r.num_inliers[m]
    print(f"{name}: worst vs single path {worst[0]:.2e} rad / {worst[1]:.2e} m, iterations {r.iterations.tolist()}")


def test_host_mirror_equals_the_binding(golden_prepared):
    """host_api.align_batch (BatchRegistration through sgbh_align_batch) and Context.align_batch: bit for bit on the same inputs"""
    from small_gicp_b200 import host_api

    g = golden_prepared
    tc, sc = g["target"], g["source"]
    starts = _starts(6)
    sources = [sc.points[j::2] for j in range(3)] * 2
    covs = [sc.covs[j::2] for j in range(3)] * 2
    for kw in (dict(factor=2, optimizer=1), dict(factor=0, robust=1, robust_c=0.5, optimizer=0, dof_mask=[1, 1, 0, 1, 1, 1])):
        h = host_api.align_batch(tc.points, sources, tc.normals, tc.covs, covs, init_Ts=starts, tree=host_api.TREE_DEVICE_KDTREE, **kw)
        ctx = _golden_ctx(g)
        ctx.set_source_batch(sources, covs)
        r = ctx.align_batch(starts, **kw)
        for f in ("T_target_source", "converged", "iterations", "num_inliers", "error", "H", "b"):
            assert np.array_equal(getattr(h, f), getattr(r, f)), (kw, f)


# ---- independence, on the tie-free random-feature target of test_gpu_storage_model ----
@pytest.fixture(scope="module")
def data():
    return Data()


def _members(d):
    """name -> (points, covs, initial pose): two misaligned members of different sizes, one aligned, a far one, an empty one and one
    1 km away from the target (no inliers; these two stop at iteration 0)"""
    sl = lambda s, n: (d.sp[s : s + n], d.scv[s : s + n])
    out = {}
    for name, (s, n), T, delta in (("a", (0, 20000), d.misaligned, [0.002, -0.001, 0.0015, 0.03, 0.0, -0.02]), ("b", (20000, 5000), d.aligned, [0, 0, 0, 0, 0, 0]),
                                   ("far", (25000, 12000), d.misaligned, [0.02, -0.015, 0.01, 0.25, -0.2, 0.15])):
        p, cv = sl(s, n)
        out[name] = (p, cv, T @ about(NF.box_centre(p), delta))
    out["empty"] = (d.sp[:0], d.scv[:0], d.aligned)
    p, cv = sl(40000, 3000)
    out["none"] = (p + np.array([1000.0, 0, 0, 0]), cv, d.aligned)
    return out


def _run(ctx, M, names, **kw):
    ctx.set_source_batch([M[n][0] for n in names], [M[n][1] for n in names])
    r = ctx.align_batch(np.array([M[n][2] for n in names]), **kw)
    return {n: (r.T_target_source[j], r.converged[j], r.iterations[j], r.num_inliers[j], r.error[j], r.H[j], r.b[j]) for j, n in enumerate(names)}


@pytest.mark.parametrize("voxel,optimizer", [(False, 1), (False, 0), (True, 1)])
def test_members_are_independent_of_the_batch(data, voxel, optimizer):
    sg = _sg()
    ctx = sg.Context(0)
    if voxel:
        ctx.build_target_voxelmap(data.tp, data.tcv, 1.0, 7)
    else:
        ctx.set_target(data.tp, data.tn, data.tcv)
        ctx.build_target_kdtree()
    M = _members(data)
    kw = dict(factor=2, optimizer=optimizer)
    alone = {n: _run(ctx, M, [n], **kw)[n] for n in M}
    assert len({int(alone[n][2]) for n in M}) >= 2  # the batches mix members that stop early with members that run much longer
    for names in (["a", "empty", "none", "far"], ["far", "none", "b", "a"], ["empty", "a"], ["a", "b", "far", "none", "empty"], ["b", "a", "a"]):
        got = _run(ctx, M, names, **kw)
        for n in names:
            for k, (x, y) in enumerate(zip(got[n], alone[n])):
                assert np.array_equal(x, y), (names, n, k)
    print("iterations alone:", {n: int(alone[n][2]) for n in M})


def test_edge_members(data):
    sg = _sg()
    ctx = sg.Context(0)
    ctx.set_target(data.tp, data.tn, data.tcv)
    ctx.build_target_kdtree()
    M = _members(data)
    names = ["empty", "a", "none"]
    for optimizer in (0, 1):
        got = _run(ctx, M, names, factor=2, optimizer=optimizer)
        for n in ("empty", "none"):  # the reference's arithmetic: delta = 0 -> converged at iteration 0, pose unchanged, error 0
            T, conv, it, inl, e, H, b = got[n]
            assert np.array_equal(T, M[n][2]) and conv and it == 0 and inl == 0 and e == 0.0 and not H.any() and not b.any(), (n, optimizer)
        # max_iterations <= 0: the initial poses, not converged
        for mi in (0, -3):
            r = ctx.align_batch(np.array([M[n][2] for n in names]), factor=2, optimizer=optimizer, max_iterations=mi)
            assert np.array_equal(r.T_target_source, np.array([M[n][2] for n in names]))
            assert not r.converged.any() and not r.iterations.any() and not r.num_inliers.any() and not r.error.any()


def test_rejections(golden_prepared, data):
    sg = _sg()
    g = golden_prepared
    sc = g["source"]
    I = np.eye(4)[None]
    ctx = _golden_ctx(g)
    ctx.set_source(sc.points, sc.covs)
    ctx._batch_offsets = np.array([0, len(sc)])
    with pytest.raises(sg.SgbError, match="no batch"):
        ctx.align_batch(I)
    ctx.set_source_batch([sc.points], [sc.covs])
    for kw in (dict(factor=3), dict(robust=-1), dict(rejector=2), dict(optimizer=2)):
        with pytest.raises(sg.SgbError, match="invalid"):
            ctx.align_batch(I, **kw)
    peer = sg.Context(0)
    ctx.comm_connect_ptrs(0, 2, [ctx.comm_mailbox(), peer.comm_mailbox()])
    with pytest.raises(sg.SgbError, match="single-GPU"):
        ctx.align_batch(I)
    ctx.comm_disconnect()
    ctx.set_source_batch([sc.points])  # no covariances
    with pytest.raises(sg.SgbError, match="GICP needs"):
        ctx.align_batch(I, factor=2)
    vctx = _golden_ctx(g, voxel=True)
    vctx.set_source_batch([sc.points], [sc.covs])
    with pytest.raises(sg.SgbError, match="point-to-plane"):
        vctx.align_batch(I, factor=1)
    r = ctx.align_batch(I, factor=0)  # the context is still usable
    assert r.num_inliers[0] > 0


@pytest.mark.parametrize("voxel", [False, True])
def test_one_step_launch_per_round(golden_prepared, voxel):
    """Gauss-Newton: L = max(iterations) + 1 linearize rounds, each transform, probe, search, factor, segment, step (kd-tree) or factor,
    segment, step (voxel map), whatever the member count"""
    g = golden_prepared
    sc = g["source"]
    ctx = _golden_ctx(g, voxel)
    for B in (1, 16):
        starts = _starts(B)
        ctx.set_source_batch([sc.points] * B, [sc.covs] * B)
        k0 = ctx.kernel_launches
        r = ctx.align_batch(starts, factor=2, optimizer=0)
        L = int(r.iterations.max()) + 1
        assert ctx.kernel_launches - k0 == (3 if voxel else 6) * L, (B, ctx.kernel_launches - k0, L)
