"""The two facts submap members (sgb_source_set_submaps) rest on, in FP64 and without a GPU:
  * ICP and GICP -- H, b, e of linearize() and error() with the precision matrix frozen at the linearisation pose -- evaluated at
    P_k^-1 T against the un-placed map k and summed over the entries equal the factor at T against the placed union; point-to-plane does
    not (the reference's residual n o r is not rotation invariant), which is why the library refuses it;
  * the union search model of np_submaps.check_union accepts the exhaustive nearest neighbour over the entries, the earlier entry at an
    exact tie, and nothing else."""
import numpy as np
import pytest

import np_factors as NF
import np_search as NS
import np_submaps as SM


def _pose(rng, rot=0.6, trans=5.0):
    w = rng.normal(size=3)
    w *= rot * rng.uniform(0.2, 1.0) / np.linalg.norm(w)
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    th = np.linalg.norm(w)
    T = np.eye(4)
    T[:3, :3] = np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th**2 * K @ K
    T[:3, 3] = rng.uniform(-trans, trans, 3)
    return T


def _covs(rng, n):
    A = rng.normal(size=(n, 3, 3)) * 0.1
    out = np.zeros((n, 4, 4))
    out[:, :3, :3] = A @ A.transpose(0, 2, 1) + 1e-3 * np.eye(3)
    return out


def _p4(x):
    return np.c_[x, np.ones(len(x))]


def _scene(seed, n_src=400, sizes=(300, 1, 500, 200)):
    rng = np.random.default_rng(seed)
    src = _p4(rng.uniform(-10, 10, (n_src, 3)))
    scov = _covs(rng, n_src)
    maps = []
    for n in sizes:
        nrm = rng.normal(size=(n, 3))
        maps.append((_p4(rng.uniform(-10, 10, (n, 3))), np.c_[nrm / np.linalg.norm(nrm, axis=1, keepdims=True), np.zeros(n)], _covs(rng, n)))
    poses = [_pose(rng) for _ in sizes]
    e = rng.integers(0, len(sizes), n_src)
    k = np.array([rng.integers(0, sizes[j]) for j in e])
    corr = (e.astype(np.uint64) << np.uint64(32)) | k.astype(np.uint64)
    corr[rng.random(n_src) < 0.1] = NF.NO
    return src, scov, maps, poses, corr, _pose(rng, 0.3, 2.0), _pose(rng, 0.3, 2.0)


def _rel(a, b):
    return np.linalg.norm(np.asarray(a) - np.asarray(b)) / np.linalg.norm(b)


@pytest.mark.parametrize("factor", [0, 2])
@pytest.mark.parametrize("robust,c", [(0, 1.0), (1, 0.5), (2, 0.5)])
def test_sum_over_entries_equals_the_placed_union(factor, robust, c):
    for seed in range(3):
        src, scov, maps, poses, corr, T, T2 = _scene(seed)
        upts, unrm, ucov, first = SM.placed_union(maps, poses)
        ucorr = SM.to_union(corr, first)
        H, b, e = SM.union_linearize(T, corr, factor, robust, c, src, scov, maps, poses)
        H0, b0, e0 = NF.linearize(T, ucorr, factor, robust, c, src, scov, upts, unrm, ucov)
        assert _rel(H, H0) <= 1e-12 and _rel(b, b0) <= 1e-12 and abs(e - e0) <= 1e-12 * e0, (seed, _rel(H, H0), _rel(b, b0))
        err = SM.union_error(T2, T, corr, factor, robust, c, src, scov, maps, poses)
        err0 = NF.error(T2, T, ucorr, factor, robust, c, src, scov, upts, unrm, ucov)
        assert abs(err - err0) <= 1e-12 * err0, seed


def test_point_to_plane_is_not_invariant():
    """n o r changes with the frame: the sum over the entries differs from the placed union by far more than rounding"""
    src, scov, maps, poses, corr, T, _ = _scene(7)
    upts, unrm, ucov, first = SM.placed_union(maps, poses)
    H, b, e = SM.union_linearize(T, corr, 1, 0, 1.0, src, scov, maps, poses)
    H0, b0, e0 = NF.linearize(T, SM.to_union(corr, first), 1, 0, 1.0, src, scov, upts, unrm, ucov)
    assert abs(e - e0) > 1e-2 * e0 and _rel(H, H0) > 1e-2
    # with identity placements there is nothing to be invariant under
    eye = [np.eye(4)] * len(maps)
    upts, unrm, ucov, first = SM.placed_union(maps, eye)
    H, b, e = SM.union_linearize(T, corr, 1, 0, 1.0, src, scov, maps, eye)
    H0, b0, e0 = NF.linearize(T, SM.to_union(corr, first), 1, 0, 1.0, src, scov, upts, unrm, ucov)
    assert abs(e - e0) <= 1e-12 * e0 and _rel(H, H0) <= 1e-12


def _exhaustive(T, src, targets, poses, max_d):
    """nearest over the entries by brute force on the model's own FP32 operands, the earlier entry at ties"""
    n = len(src)
    best_d, best = np.full(n, np.inf), np.full(n, NF.NO, dtype=np.uint64)
    for e, (t, P) in enumerate(zip(targets, poses)):
        if not t.n:
            continue
        q, q32, _, _ = NS.queries(SM.relative(P, T), src, t.centre)
        d = ((q32[:, None, :] - t.f[None]) ** 2).sum(-1)
        j = d.argmin(1)
        dj = d[np.arange(n), j]
        r2 = ((t.f[j] - q) ** 2).sum(-1)
        take = dj < best_d
        best_d = np.where(take, dj, best_d)
        best = np.where(take, np.where((max_d is None) | (r2 <= (max_d or 0)), (np.uint64(e) << np.uint64(32)) | j.astype(np.uint64), NF.NO), best)
    return best


@pytest.mark.parametrize("max_d", [1.0, 0.05, None])
def test_union_search_model(max_d):
    rng = np.random.default_rng(3)
    src = _p4(rng.uniform(-6, 6, (1500, 3)) + [100.0, -50.0, 10.0])
    clouds = [_p4(rng.uniform(-6, 6, (n, 3)) + [100.0, -50.0, 10.0]) for n in (900, 0, 33, 1200)]
    poses = [_pose(rng, 0.2, 1.0) for _ in clouds]
    # every map is stored in its own frame: what the caller hands over is P^-1 of the common-frame cloud
    maps = [_p4(c[:, :3] @ SM.inverse(P)[:3, :3].T + SM.inverse(P)[:3, 3]) for c, P in zip(clouds, poses)]
    targets = [NS.Target(m) for m in maps]
    T = _pose(rng, 0.01, 0.05)
    corr = _exhaustive(T, src, targets, poses, max_d)
    rep = NS.Report()
    assert SM.check_union(corr, T, src, targets, poses, max_d, report=rep) == len(src)
    assert rep.worst_band == 0.0
    # a neighbour that is not the nearest, a wrong entry, a missing match and an invented one are all refused
    hit = np.nonzero(corr != NF.NO)[0]
    for mutate in ("index", "entry", "drop", "invent"):
        bad = corr.copy()
        i = hit[5]
        if mutate == "index":
            bad[i] = (bad[i] & ~SM.LOW) | np.uint64((int(bad[i] & SM.LOW) + 1) % targets[int(bad[i] >> np.uint64(32))].n)
        elif mutate == "entry":
            bad[i] = (np.uint64(3 - int(bad[i] >> np.uint64(32))) << np.uint64(32)) | np.uint64(0)
        elif mutate == "drop":
            bad[i] = NF.NO
        else:
            miss = np.nonzero(corr == NF.NO)[0]
            if len(miss) == 0:
                continue
            bad[miss[0]] = np.uint64(0)
        with pytest.raises(AssertionError):
            SM.check_union(bad, T, src, targets, poses, max_d, report=NS.Report())


def test_union_search_model_empty_lists_and_ties():
    rng = np.random.default_rng(4)
    src = _p4(rng.uniform(-3, 3, (200, 3)))
    m = _p4(rng.uniform(-3, 3, (300, 3)))
    t = NS.Target(m)
    none = np.full(len(src), NF.NO, dtype=np.uint64)
    assert SM.check_union(none, np.eye(4), src, [], [], 1.0, report=NS.Report()) == len(src)
    assert SM.check_union(none, np.eye(4), src, [NS.Target(np.zeros((0, 4)))], [np.eye(4)], None, report=NS.Report()) == len(src)
    # the same map twice at the same pose: every distance ties exactly and the exhaustive model keeps entry 0
    corr = _exhaustive(np.eye(4), src, [t, t], [np.eye(4)] * 2, None)
    assert (corr >> np.uint64(32) == 0).all()
    SM.check_union(corr, np.eye(4), src, [t, t], [np.eye(4)] * 2, None, report=NS.Report())
