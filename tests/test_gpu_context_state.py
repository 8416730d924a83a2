"""The context's target and source state across calls: whatever a context held before, installing a target or a source leaves it
exactly as a fresh context that installed only that (H|b|e, inliers, correspondences and error(), bitwise), and a kd-tree cannot be
put over a voxel-map target, whose voxels are not the points the tree would index."""
import itertools

import numpy as np
import pytest

import oracle as O

pytestmark = pytest.mark.gpu

LEAF = 0.5


def _sg():
    import small_gicp_b200 as sg

    return sg


class Data:
    def __init__(self):
        from small_gicp_b200.synthetic import make_pair

        self.tp, self.sp, Tgt = make_pair(20_000)
        tc, sc = O.Cloud(self.tp), O.Cloud(self.sp)
        self.tree = O.KdTree(tc)
        self.tree.estimate(20, O.FEAT_NORMAL_COV, 2)
        O.KdTree(sc).estimate(20, O.FEAT_COV, 2)
        self.tn, self.tcv, self.scv = tc.normals, tc.covs, sc.covs
        self.vox = O.GaussianVoxelMap(tc, LEAF, 7).export()[:3]
        d = np.eye(4)
        d[:3, 3] = [0.02, -0.01, 0.015]
        self.poses = (Tgt @ d, Tgt, Tgt @ np.linalg.inv(d))  # first and second linearize, error(): source onto target
        self.self_poses = (d, np.eye(4), np.linalg.inv(d))  # a cloud onto itself


@pytest.fixture(scope="module")
def data():
    return Data()


# every way of installing a target
TARGETS = {
    "reference_tree": lambda c, d: (c.set_target(d.tp, d.tn, d.tcv), c.set_target_kdtree(*d.tree.export())),
    "device_tree": lambda c, d: (c.set_target(d.tp, d.tn, d.tcv), c.build_target_kdtree()),
    "set_voxelmap": lambda c, d: c.set_target_voxelmap(LEAF, *d.vox, 7),
    "build_voxelmap": lambda c, d: c.build_target_voxelmap(d.tp, d.tcv, LEAF, 7),
    "adopted_source": lambda c, d: (c.set_source(d.tp, d.tcv), c.adopt_source_as_target()),
}


def _result(ctx, d, factor=2, poses=None):
    """two linearizes (the second seeded by the first), then error() at a third pose"""
    poses = d.poses if poses is None else poses
    out = {}
    for j, T in enumerate(poses[:2]):
        H, b, e = ctx.linearize(T, factor=factor)
        out.update({f"H{j}": H, f"b{j}": b, f"e{j}": e, f"inliers{j}": ctx.num_inliers(), f"corr{j}": ctx.correspondences()})
    out["error"] = ctx.error(poses[2])
    return out


def _batch_result(ctx, d):
    Ts = np.array(d.poses[:2])
    H, b, e, inl = ctx.linearize_batch(Ts, factor=2)
    return {"H": H, "b": b, "e": e, "inliers": inl, "corr": ctx.correspondences_batch(), "error": ctx.error_batch(np.array(d.poses[1:]))}


def _assert_same(got, want, what):
    assert got.keys() == want.keys()
    for k in want:
        if isinstance(want[k], list):
            assert len(got[k]) == len(want[k]) and all(np.array_equal(g, w) for g, w in zip(got[k], want[k])), (what, k)
        else:
            assert np.array_equal(got[k], want[k]), (what, k)


def _fresh(d, target):
    sg = _sg()
    ctx = sg.Context(0)
    TARGETS[target](ctx, d)
    ctx.set_source(d.sp, d.scv)
    r = _result(ctx, d)
    ctx.close()
    return r


def test_target_transitions(data):
    """A, linearize, B == B alone, for every ordered pair of target installs (A == B included)"""
    sg = _sg()
    fresh = {t: _fresh(data, t) for t in TARGETS}
    for t, r in fresh.items():
        assert r["inliers0"] > 100 and r["inliers1"] > 100, (t, r["inliers0"], r["inliers1"])
    for a, b in itertools.product(TARGETS, TARGETS):
        ctx = sg.Context(0)
        TARGETS[a](ctx, data)
        ctx.set_source(data.sp, data.scv)
        _result(ctx, data)
        TARGETS[b](ctx, data)
        ctx.set_source(data.sp, data.scv)
        _assert_same(_result(ctx, data), fresh[b], (a, b))
        ctx.close()


def test_source_transitions_single_batch_single(data):
    sg = _sg()
    halves = [data.sp[:7000], data.sp[7000:]]
    covs = [data.scv[:7000], data.scv[7000:]]
    fresh_batch = sg.Context(0)
    TARGETS["device_tree"](fresh_batch, data)
    fresh_batch.set_source_batch(halves, covs)
    want_batch = _batch_result(fresh_batch, data)
    fresh_batch.close()
    want_single = _fresh(data, "device_tree")

    ctx = sg.Context(0)
    TARGETS["device_tree"](ctx, data)
    ctx.set_source(data.sp, data.scv)
    _assert_same(_result(ctx, data), want_single, "single")
    ctx.set_source_batch(halves, covs)
    _assert_same(_batch_result(ctx, data), want_batch, "single -> batch")
    ctx.set_source(data.sp, data.scv)
    _assert_same(_result(ctx, data), want_single, "single -> batch -> single")
    ctx.close()


def test_source_transitions_estimate_then_adopt(data):
    """single -> estimate_source_features -> adopt, with linearizes in between, == the same installs on a fresh context"""
    sg = _sg()

    def run(ctx, linearize):
        TARGETS["device_tree"](ctx, data)
        ctx.set_source(data.sp)
        got = [_result(ctx, data, factor=0)] if linearize else []  # no covariances yet: ICP
        ctx.estimate_source_features(20)
        if linearize:
            got.append(_result(ctx, data))
        ctx.adopt_source_as_target()
        ctx.set_source(data.sp, data.scv)  # the adopted cloud onto itself
        return got + [_result(ctx, data, poses=data.self_poses)]

    ctx, fresh = sg.Context(0), sg.Context(0)
    got = run(ctx, True)
    _assert_same(got[-1], run(fresh, False)[-1], "adopted after estimate_source_features")
    for r in got:
        assert r["inliers1"] > 100
    ctx.close()
    fresh.close()


@pytest.mark.parametrize("target", ["set_voxelmap", "build_voxelmap"])
def test_kdtree_over_a_voxelmap_is_refused(data, target):
    sg = _sg()
    from small_gicp_b200.capi import SgbError

    ctx = sg.Context(0)
    TARGETS[target](ctx, data)
    ctx.set_source(data.sp, data.scv)
    before = _result(ctx, data)
    with pytest.raises(SgbError, match="sgb_target_set_points"):
        ctx.build_target_kdtree()
    with pytest.raises(SgbError, match="sgb_target_set_points"):
        ctx.set_target_kdtree(*data.tree.export())
    _assert_same(_result(ctx, data), before, "voxel map after the refusals")
    TARGETS["device_tree"](ctx, data)
    _assert_same(_result(ctx, data), _fresh(data, "device_tree"), "kd-tree target after the refusals")
    ctx.close()
