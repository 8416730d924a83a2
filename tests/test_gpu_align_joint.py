"""Joint window registration (sgb_align_joint, Context.align_joint) on the GPU:
  1. a window of one free frame and one edge IS the pairwise align: bit-identical to align_batch of that pair member (T, converged,
     iterations, inliers, error, correspondences afterwards), on many kd-trees (ICP, point-to-plane, GICP) and many voxel maps (ICP,
     GICP), every robust kernel, GN and LM, a DoF mask, max_iterations 0 / 1 / 20;
  2. a star window (edges i -> 0, frame 0 fixed: H block diagonal) after one GN iteration is the pairwise align of every edge;
  3. round by round, GN and LM, every option and window shapes beyond these: tests/test_gpu_align_joint_replay.py;
  4. ground truth: 8 LiDAR frames perturbed by ~2 deg / 0.3 m come within 0.5 deg / 0.05 m (GICP on kd-trees and on voxel maps);
  5. a window's results do not depend on the other windows of the call; empty windows, edge-less frames, all-fixed windows;
  6. the launch count per round is the pairs round's plus one, for 1 and 1024 windows;
  7. misuse fails with its message and leaves the context usable."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GN, LM = 0, 1


def _sg():
    import small_gicp_b200 as sg

    return sg


def _exp(d):
    from test_np_joint import _exp as e

    return e(d)


def _p4(x):
    return np.c_[x, np.ones(len(x))]


class Frames:
    """K frames of one synthetic room: frame k's points in its own coordinates (ground-truth pose G[k], sensor -> world), with normals
    and covariances estimated on the device"""

    def __init__(self, K, n=2500, seed=7):
        from small_gicp_b200.synthetic import make_world, sample_cloud

        sg = _sg()
        world = make_world(300_000, seed)
        rng = np.random.default_rng(seed)
        self.G = [np.eye(4)]
        for _ in range(K - 1):
            self.G.append(self.G[-1] @ _exp(np.r_[rng.normal(size=3) * 0.01, 0.3 + rng.normal() * 0.05, rng.normal(size=2) * 0.05]))
        prep = sg.Context(0)
        self.pts, self.normals, self.covs = [], [], []
        for k in range(K):
            P = sample_cloud(world, n, 100 + k) + np.array([30.0, 30.0, 3.0])
            L = (np.linalg.inv(self.G[k]) @ _p4(P).T).T
            nr, cv = prep.estimate_features(L, 20)
            self.pts.append(L)
            self.normals.append(nr)
            self.covs.append(cv)
        prep.close()


@pytest.fixture(scope="module")
def frames():
    return Frames(40)


def _context(fr, idx, kind, clouds, maps):
    """frames idx of fr as the call's frames (cloud k and map k = frame idx[k]); the edges (clouds[p], maps[p])"""
    sg = _sg()
    ctx = sg.Context(0)
    pts = [fr.pts[i] for i in idx]
    if kind == "kdtree":
        ctx.build_target_kdtrees(pts, [fr.normals[i] for i in idx], [fr.covs[i] for i in idx])
    else:
        ctx.build_target_voxelmaps(pts, [fr.covs[i] for i in idx], 1.0, 1)
    ctx.set_source_batch(pts, [fr.covs[i] for i in idx])
    ctx.set_source_pairs(np.asarray(clouds, dtype=np.uint32), np.asarray(maps, dtype=np.uint32))
    return ctx


def _perturbed(fr, idx, seed, rot=0.01, trans=0.1):
    rng = np.random.default_rng(seed)
    G0 = np.linalg.inv(fr.G[idx[0]])
    return np.array([G0 @ fr.G[i] @ _exp(np.r_[rng.normal(size=3) * rot, rng.normal(size=3) * trans]) if k else np.eye(4) for k, i in enumerate(idx)])


def _bits(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.uint64), np.asarray(b, dtype=np.float64).view(np.uint64))


PAIR_CASES = [("kdtree", f) for f in (0, 1, 2)] + [("voxelmap", f) for f in (0, 2)]


@pytest.mark.parametrize("kind,factor", PAIR_CASES)
@pytest.mark.parametrize("robust,c", [(0, 1.0), (1, 0.5), (2, 0.5)], ids=["none", "huber", "cauchy"])
@pytest.mark.parametrize("opt", [GN, LM], ids=["gn", "lm"])
@pytest.mark.parametrize("max_it", [0, 1, 20])
def test_one_free_frame_is_the_pairwise_align(frames, kind, factor, robust, c, opt, max_it):
    idx = [3, 4]
    X = _perturbed(frames, idx, 1)
    kw = dict(factor=factor, robust=robust, robust_c=c, optimizer=opt, max_iterations=max_it, max_dist_sq=1.0)
    masks = [None, [1, 1, 0, 0, 0, 1]] if (robust == 0 and max_it == 20) else [None]
    for mask in masks:
        a = _context(frames, idx, kind, [1], [0])
        ra = a.align_joint(X, **kw, dof_mask=mask)
        b = _context(frames, idx, kind, [1], [0])
        rb = b.align_batch(X[1:2], **kw, dof_mask=mask)
        assert _bits(ra.X[0], X[0])
        assert _bits(ra.X[1], rb.T_target_source[0]), (ra.X[1], rb.T_target_source[0])
        assert ra.converged[0] == rb.converged[0] and ra.iterations[0] == rb.iterations[0]
        assert ra.num_inliers[0] == rb.num_inliers[0] and _bits(ra.error[0], rb.error[0])
        for x, y in zip(a.correspondences_batch(), b.correspondences_batch()):
            np.testing.assert_array_equal(x, y)
        a.close()
        b.close()


@pytest.mark.parametrize("kind", ["kdtree", "voxelmap"])
def test_star_window_one_gn_iteration_is_pairwise(frames, kind):
    idx = list(range(10, 16))
    X = _perturbed(frames, idx, 2)
    F = len(idx)
    clouds, maps = list(range(1, F)), [0] * (F - 1)
    kw = dict(factor=2, optimizer=GN, max_iterations=1)
    ra = _context(frames, idx, kind, clouds, maps).align_joint(X, **kw)
    rb = _context(frames, idx, kind, clouds, maps).align_batch(X[1:], **kw)
    for k in range(1, F):
        np.testing.assert_allclose(ra.X[k], rb.T_target_source[k - 1], rtol=1e-12, atol=1e-12 * np.abs(rb.T_target_source[k - 1]).max())


def _window_edges(F, loop=True):
    e = [(i, i - 1) for i in range(1, F)] + [(i, i - 2) for i in range(2, F)]
    if loop and F > 2:
        e.append((0, F - 1))
    return e


def _rot_deg(R):
    return np.rad2deg(np.arccos(np.clip((np.trace(R) - 1) / 2, -1, 1)))


@pytest.mark.parametrize("kind", ["kdtree", "voxelmap"])
def test_lidar_window_reaches_ground_truth(kind):
    import torch

    from small_gicp_b200 import synthetic as syn

    sg = _sg()
    dev = torch.device("cuda:0")
    world = syn.make_world(4_000_000, 42)
    side = syn.world_side(4_000_000)
    K = 8
    G = [syn.lidar_pose(f, side) for f in range(K)]
    prep = sg.Context(0)
    pts, covs = [], []
    for f in range(K):
        p = prep.voxelgrid_sampling(syn.lidar_frame_torch(world, G[f], 45 + f, dev).cpu().numpy(), 0.25)
        pts.append(p)
        covs.append(prep.estimate_features(p, 20, normals=False)[1])
    edges = [(i, i - d) for i in range(1, K) for d in (1, 2) if i - d >= 0]
    cl, mp = [e[0] for e in edges], [e[1] for e in edges]
    ctx = sg.Context(0)
    if kind == "kdtree":
        ctx.build_target_kdtrees(pts, None, covs)
    else:
        ctx.build_target_voxelmaps(pts, covs, 1.0, 1)
    ctx.set_source_batch(pts, covs)
    ctx.set_source_pairs(np.array(cl, dtype=np.uint32), np.array(mp, dtype=np.uint32))
    rng = np.random.default_rng(8)
    X0 = np.array([G[k] if k == 0 else G[k] @ _exp(np.r_[rng.normal(size=3) * np.deg2rad(2.0) / np.sqrt(3), rng.normal(size=3) * 0.3 / np.sqrt(3)])
                   for k in range(K)])
    r = ctx.align_joint(X0, factor=2, optimizer=LM, max_iterations=30, max_dist_sq=4.0)
    # the pairwise alternative: every edge alone, then i -> i-1 chained
    rp = ctx.align_batch(np.array([np.linalg.inv(X0[j]) @ X0[i] for i, j in edges]), factor=2, optimizer=LM, max_iterations=30, max_dist_sq=4.0)
    chain = [G[0]]
    for i in range(1, K):
        chain.append(chain[-1] @ rp.T_target_source[edges.index((i, i - 1))])
    for k in range(K):
        dr, dt = _rot_deg(G[k][:3, :3].T @ r.X[k][:3, :3]), np.linalg.norm(G[k][:3, 3] - r.X[k][:3, 3])
        cr, ct = _rot_deg(G[k][:3, :3].T @ chain[k][:3, :3]), np.linalg.norm(G[k][:3, 3] - chain[k][:3, 3])
        print(f"{kind} frame {k}: joint {dr:.4f} deg {dt:.4f} m   chained pairwise {cr:.4f} deg {ct:.4f} m")
        assert dr < 0.5 and dt < 0.05, (k, dr, dt)


def _windows_call(frames, wins, kind, **kw):
    """several windows (each a list of frame indices of `frames` and its local edges) in one call"""
    idx, cl, mp, off, X = [], [], [], [0], []
    for w, (fidx, edges, seed) in enumerate(wins):
        base = len(idx)
        idx += fidx
        cl += [base + i for i, _ in edges]
        mp += [base + j for _, j in edges]
        off.append(len(idx))
        X.append(_perturbed(frames, fidx, seed))
    ctx = _context(frames, idx, kind, cl, mp)
    r = ctx.align_joint(np.concatenate(X), windows=off, **kw)
    ctx.close()
    return r, off


@pytest.mark.parametrize("kind", ["kdtree", "voxelmap"])
def test_windows_are_independent(frames, kind):
    A = (list(range(0, 5)), _window_edges(5), 11)
    B = (list(range(20, 23)), [(1, 0), (2, 1)], 12)
    C = (list(range(30, 38)), _window_edges(8), 13)
    kw = dict(factor=2, optimizer=LM)
    alone = {n: _windows_call(frames, [w], kind, **kw)[0] for n, w in zip("ABC", (A, B, C))}
    for order in ("ABC", "CAB", "BCA"):
        r, off = _windows_call(frames, [dict(zip("ABC", (A, B, C)))[n] for n in order], kind, **kw)
        for w, n in enumerate(order):
            assert _bits(r.X[off[w] : off[w + 1]], alone[n].X)
            for f in ("converged", "iterations", "num_inliers", "error"):
                assert _bits(np.asarray(getattr(r, f)[w], dtype=np.float64), np.asarray(getattr(alone[n], f)[0], dtype=np.float64)), (order, n, f)
    small = ([1, 2], [(1, 0)], 14)
    one = _windows_call(frames, [small], kind, **kw)[0]
    for count in (17, 1024):
        r, off = _windows_call(frames, [small] * count, kind, **kw)
        assert _bits(r.X, np.concatenate([one.X] * count))
        assert np.all(r.iterations == one.iterations[0]) and _bits(r.error, np.full(count, one.error[0]))


def test_degenerate_windows(frames):
    sg = _sg()
    idx = [5, 6, 7, 8, 9, 10]
    # windows: [] (empty) | [0, 1, 2] with edge 1 -> 0 and edge-less frame 2 | [3, 4] all fixed with an edge | [5] alone
    ctx = _context(frames, idx, "kdtree", [1, 4], [0, 3])
    X = _perturbed(frames, idx, 4)
    r = ctx.align_joint(X, windows=[0, 0, 3, 5, 6], fixed=[1, 0, 0, 1, 1, 0], factor=2, optimizer=LM)
    assert r.X.shape == (6, 4, 4) and r.converged.shape == (4,)
    assert _bits(r.X[2], X[2]) and _bits(r.X[3:], X[3:])
    assert r.iterations[1] > 0 and not _bits(r.X[1], X[1])
    for w in (0, 2, 3):
        assert not r.converged[w] and r.iterations[w] == 0 and r.error[w] == 0 and r.num_inliers[w] == 0
    # the frame-2-less window gives the same as a window without that frame
    ctx2 = _context(frames, idx[:2], "kdtree", [1], [0])
    r2 = ctx2.align_joint(X[:2], factor=2, optimizer=LM)
    assert _bits(r.X[1], r2.X[1]) and r.iterations[1] == r2.iterations[0]
    del sg


@pytest.mark.parametrize("kind,per_round", [("kdtree", 3), ("voxelmap", 2)])
@pytest.mark.parametrize("count", [1, 1024])
def test_launches_per_round(frames, kind, per_round, count):
    """GN, identical windows: every round is a linearize of all edges; rounds = iterations + 1"""
    small = ([1, 2, 3], [(1, 0), (2, 1), (2, 0)], 15)
    idx, cl, mp, off = [], [], [], [0]
    for w in range(count):
        base = len(idx)
        idx += small[0]
        cl += [base + i for i, _ in small[1]]
        mp += [base + j for _, j in small[1]]
        off.append(len(idx))
    ctx = _context(frames, idx, kind, cl, mp)
    X = np.concatenate([_perturbed(frames, small[0], small[2])] * count)
    ctx.align_joint(X, windows=off, factor=2, optimizer=GN, max_iterations=1)  # the pairing's view of the target is built here
    for max_it in (3, 10):
        k0 = ctx.kernel_launches
        r = ctx.align_joint(X, windows=off, factor=2, optimizer=GN, max_iterations=max_it)
        rounds = int(r.iterations[0]) + 1
        assert np.all(r.iterations == r.iterations[0])
        assert ctx.kernel_launches - k0 == 1 + rounds * (per_round + 1), (kind, count, max_it, rounds)


def test_misuse_fails_and_leaves_the_context_usable(frames):
    sg = _sg()
    idx = [0, 1, 2, 3]
    X = _perturbed(frames, idx, 5)

    def ok(ctx, **kw):
        r = ctx.align_joint(X, factor=2, **kw)
        assert r.iterations[0] > 0

    def bad(ctx, msg, Xs=X, **kw):
        with pytest.raises(sg.SgbError, match=msg):
            ctx.align_joint(Xs, factor=2, **kw)

    ctx = sg.Context(0)
    with pytest.raises(sg.SgbError, match="no batch"):
        ctx.align_joint(np.zeros((0, 4, 4)))
    pts = [frames.pts[i] for i in idx]
    cv = [frames.covs[i] for i in idx]
    ctx.build_target_kdtrees(pts, None, cv)
    ctx.set_source_batch(pts, cv)
    bad(ctx, "pairing with a maps table")
    ctx.set_source_pairs(np.array([1, 2], dtype=np.uint32), None)
    bad(ctx, "pairing with a maps table")
    ctx.set_source_submaps([[0], [1]], clouds=np.array([1, 2], dtype=np.uint32))
    bad(ctx, "submap")
    ctx.set_source_pairs(np.array([1, 2, 3], dtype=np.uint32), np.array([0, 1, 2], dtype=np.uint32))
    ok(ctx)
    bad(ctx, "must run from 0", windows=[0, 3])
    bad(ctx, "ascending", windows=[0, 3, 2, 4])
    bad(ctx, "both frames of an edge", windows=[0, 2, 4])
    bad(ctx, "no fixed frame", fixed=[0, 0, 0, 0])
    ok(ctx)
    ctx.set_source_pairs(np.array([1, 2], dtype=np.uint32), np.array([0, 2], dtype=np.uint32))
    bad(ctx, "of its own frame")
    ctx.set_source_pairs(np.array([1, 2, 3], dtype=np.uint32), np.array([0, 1, 2], dtype=np.uint32))
    ok(ctx)
    # more than 32 frames in a window
    big = list(range(34))
    ctx34 = _context(frames, big, "kdtree", [1], [0])
    with pytest.raises(sg.SgbError, match="at most 32"):
        ctx34.align_joint(_perturbed(frames, big, 6))
    ctx34.align_joint(_perturbed(frames, big, 6), windows=[0, 2, 34])
    # cloud count != map count
    ctx.build_target_kdtrees(pts[:3], None, cv[:3])
    bad(ctx, "3 maps")
    ctx.build_target_kdtrees(pts, None, cv)
    ok(ctx)
    # a one-target context
    ctx.set_target(pts[0][:, :3], None, cv[0])
    ctx.build_target_kdtree()
    bad(ctx, "many-kd-trees or many-voxel-maps")
    ctx.build_target_kdtrees(pts, None, cv)
    ok(ctx)
    # what sgb_align_batch refuses: invalid kinds, missing normals
    with pytest.raises(sg.SgbError, match="invalid"):
        ctx.align_joint(X, factor=7)
    with pytest.raises(sg.SgbError):
        ctx.align_joint(X, factor=1)
    ok(ctx)
