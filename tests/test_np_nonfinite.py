"""Non-finite input points (a NaN or +-Inf in x, y or z) without a GPU: what the reference does with them, and the models pinned to the
contract of include/sgicp_b200.h -- such a point is inert, and the results for the finite rows equal the results for the cloud with the
non-finite rows removed, indices mapped back.

What the reference does (recorded here; O.reference_lib() where it was built, the oracle's restatement otherwise):
  * voxelgrid_sampling drops every non-finite point: fast_floor gives INT_MIN, outside the 21-bit range.  The voxels equal the
    filtered cloud's to the last bits of their sums (its sort is not stable, so a voxel's points may be added in another order).
  * its kd-tree is NOT the filtered cloud's: built over a cloud with bad rows, it gives finite queries a point that is not their
    nearest finite point, and the features of finite points change (test_reference_kdtree_with_bad_target_rows); a NaN source row
    is matched, and linearize() then sums NaN (test_reference_nan_source_rows).  The reference is therefore not well-defined on such
    clouds, and the device's contract stands on its own: the filtered cloud's result."""
import numpy as np
import pytest

import np_factors as NF
import np_preprocess as PP
import np_search as NS
import oracle as O

NAN_NEG = np.frombuffer(np.uint64(0xFFF8000000000000).tobytes(), dtype=np.float64)[0]  # NaN with its sign bit set
BAD = (np.nan, np.inf, -np.inf, NAN_NEG)


def _libs():
    out = [("oracle", O.lib())]
    ref = O.reference_lib()
    if ref is not None:
        out.append(("reference", ref))
    return out


def _inject(pts, rows, values=BAD, axes=None):
    out = np.array(pts, dtype=np.float64)
    for j, r in enumerate(rows):
        out[r, (r if axes is None else axes[j]) % 3] = values[j % len(values)]
    return out


def _cloud(seed=0, n=2000, scale=3.0):
    return np.random.default_rng(seed).normal(size=(n, 3)) * scale


def test_nan_sign_bit():
    assert np.isnan(NAN_NEG) and np.signbit(NAN_NEG)


@pytest.mark.parametrize("lib", [n for n, _ in _libs()])
def test_reference_voxelgrid_drops_nonfinite(lib):
    L = dict(_libs())[lib]
    pb = _inject(_cloud(), [0, 7, 500, 1001, 1999])
    fin = NF.finite_rows(pb)
    v = O.Cloud(pb, _lib=L).voxelgrid_sampling(0.5).points
    vf = O.Cloud(pb[fin], _lib=L).voxelgrid_sampling(0.5).points
    assert np.isfinite(v).all() and v.shape == vf.shape
    a, b = v[np.lexsort(v.T[::-1])], vf[np.lexsort(vf.T[::-1])]
    assert np.abs(a - b).max() <= 1e-14 * np.abs(b).max()
    # the model drops them explicitly and equals the filtered cloud's model bit for bit; its voxels are the reference's
    m = PP.voxelgrid_model(pb, 0.5)
    assert np.array_equal(m, PP.voxelgrid_model(pb[fin], 0.5))
    mm = m[np.lexsort(m.T[::-1])]
    assert np.abs(mm - b).max() <= 1e-14 * np.abs(b).max()


@pytest.mark.parametrize("lib", [n for n, _ in _libs()])
def test_reference_nan_source_rows(lib):
    """recorded behaviour (module docstring): the reference's sums with a NaN source row are NaN, so no drop-in call can hold it to
    the filtered cloud; the filtered cloud itself is finite"""
    L = dict(_libs())[lib]
    rng = np.random.default_rng(1)
    tc = O.Cloud(_cloud(1), _lib=L)
    tt = O.KdTree(tc)
    pb = _inject(_cloud(2), [0, 7, 500, 1999])
    fin = NF.finite_rows(pb)
    sc, scf = O.Cloud(pb, _lib=L), O.Cloud(pb[fin], _lib=L)
    reg = O.Registration(factor=O.FACTOR_ICP, _lib=L)
    T = np.eye(4)
    T[:3, 3] = rng.normal(size=3) * 0.05
    H, _, e = reg.linearize(tc, tt, sc, T)
    corr = reg.correspondences(len(pb))
    Hf, _, ef = reg.linearize(tc, tt, scf, T)
    corr_f = reg.correspondences(int(fin.sum()))
    assert np.isfinite(Hf).all() and np.isfinite(ef)
    assert np.array_equal(corr[fin], corr_f)  # finite source rows: the same correspondences
    assert (corr[~fin] != O.NO_INDEX).any() and not np.isfinite(e)  # a NaN query is matched, and its NaN residual summed


@pytest.mark.parametrize("lib", [n for n, _ in _libs()])
def test_reference_kdtree_with_bad_target_rows(lib):
    """recorded behaviour (module docstring): over a cloud with bad rows the reference's kd-tree misses the nearest finite point of some
    finite queries, and the covariances of some finite points differ from the filtered cloud's; over the filtered cloud it is exact"""
    L = dict(_libs())[lib]
    pb = _inject(_cloud(1), [0, 7, 500, 1001, 1999])
    fin = NF.finite_rows(pb)
    q = _cloud(9, 500)
    best = ((q[:, None] - pb[fin][None]) ** 2).sum(-1).argmin(1)
    i_bad, _, _ = O.KdTree(O.Cloud(pb, _lib=L)).knn(q, 1)
    i_flt, _, _ = O.KdTree(O.Cloud(pb[fin], _lib=L)).knn(q, 1)
    assert np.array_equal(i_flt[:, 0].astype(np.int64), best)
    assert (i_bad[:, 0].astype(np.int64) != np.nonzero(fin)[0][best]).any()
    c, cf = O.Cloud(pb, _lib=L), O.Cloud(pb[fin], _lib=L)
    O.KdTree(c).estimate(10, O.FEAT_COV)
    O.KdTree(cf).estimate(10, O.FEAT_COV)
    assert not np.all(c.covs[fin] == cf.covs, axis=(1, 2)).all()


def test_box_centre_and_storage_skip_nonfinite():
    p = _cloud(3, 500)
    pb = _inject(p, [0, 1, 250, 499], (np.inf, -np.inf, np.nan, NAN_NEG))
    fin = NF.finite_rows(pb)
    assert fin.sum() == 496
    assert np.array_equal(NF.box_centre(pb), NF.box_centre(pb[fin]))
    s = NF.stored_points(pb)
    assert np.isnan(s[~fin, :3]).all()
    assert np.array_equal(s[fin], NF.stored_points(pb[fin]))
    assert np.array_equal(NF.box_centre(np.full((4, 3), np.inf)), np.zeros(3))  # nothing finite: the empty box's centre


def _nearest(tgt, src):
    d = ((src[:, None, :3] - tgt[None, :, :3]) ** 2).sum(-1)
    d = np.where(np.isnan(d), np.inf, d)
    return d.argmin(1)


def test_search_model_accepts_filtered_answer_and_refuses_a_bad_row():
    rng = np.random.default_rng(4)
    H = 1.0 / 64
    tgt = rng.integers(-256, 256, (400, 3)) * H
    src = rng.integers(-256, 256, (300, 3)) * H + rng.integers(-3, 4, (300, 3)) * H / 8
    tb = _inject(tgt, [0, 3, 200, 399])
    sb = _inject(src, [0, 150, 299, 42], axes=[1, 1, 1, 1])  # NaN / Inf in y only
    tfin, sfin = NF.finite_rows(tb), NF.finite_rows(sb)
    t = NS.Target(tb)
    assert t.n == 400 and t.n_finite == 396
    best = _nearest(tb[tfin], sb)
    corr = np.where(sfin, np.nonzero(tfin)[0][best], -1).astype(np.int64).astype(np.uint64)
    corr[~sfin] = NF.NO
    rep = NS.Report()
    assert NS.check_correspondences(corr, np.eye(4), sb, t, None, report=rep) == 300
    # a bad source row given a neighbour
    wrong = corr.copy()
    wrong[0] = 5
    with pytest.raises(AssertionError, match="non-finite queries"):
        NS.check_correspondences(wrong, np.eye(4), sb, t, None, report=rep)
    # a finite query given a non-finite target row
    wrong = corr.copy()
    wrong[1] = 3
    with pytest.raises(AssertionError, match="1 of"):
        NS.check_correspondences(wrong, np.eye(4), sb, t, None, report=rep)
    # a target of non-finite rows only: every query unmatched
    allbad = NS.Target(np.full((10, 3), np.nan))
    assert NS.check_correspondences(np.full(300, NF.NO), np.eye(4), sb, allbad, None, report=rep) == 300


def test_knn_model_nonfinite_rows():
    rng = np.random.default_rng(5)
    tgt = _inject(rng.normal(size=(300, 3)), [0, 100, 299])
    q = _inject(rng.normal(size=(50, 3)), [3, 40])
    t = NS.Target(tgt)
    k = 6
    tf = np.nonzero(NF.finite_rows(tgt))[0]
    idx = np.full((50, k), NF.NO)
    d2 = np.full((50, k), NS.DBL_MAX)
    qc = q - t.centre
    for i in np.nonzero(NF.finite_rows(q))[0]:
        dd = ((t.f[tf] - qc[i]) ** 2).sum(1)
        o = np.argsort(dd, kind="stable")[:k]
        idx[i], d2[i] = tf[o], dd[o]
    assert NS.check_knn(idx, d2, q, k, t, report=NS.Report()) == int(NF.finite_rows(q).sum())
    wrong = idx.copy()
    wrong[3, 0] = 7  # a non-finite query with a neighbour
    with pytest.raises(AssertionError, match="non-finite queries"):
        NS.check_knn(wrong, d2, q, k, t, report=NS.Report())
    wrong = idx.copy()
    wrong[0, 0] = 100  # a non-finite target row as a neighbour
    with pytest.raises(AssertionError):
        NS.check_knn(wrong, d2, q, k, t, report=NS.Report())


def test_factor_model_inert_rows():
    """the sums of a cloud with non-finite rows (no correspondence there) equal the filtered cloud's, and a bad row with a
    correspondence is refused"""
    rng = np.random.default_rng(6)
    tgt = rng.normal(size=(200, 3))
    src = tgt[:150] + rng.normal(size=(150, 3)) * 0.01
    sb = _inject(src, [0, 75, 149])
    tb = _inject(tgt, [10, 199])
    sfin, tfin = NF.finite_rows(sb), NF.finite_rows(tb)
    tmap = np.full(200, -1)
    tmap[tfin] = np.arange(int(tfin.sum()))
    corr = np.arange(150).astype(np.uint64)
    corr[~sfin] = NF.NO
    corr[np.isin(np.arange(150), [10])] = NF.NO  # the target row 10 is bad
    sp, _, tp, _, _ = NF.storage_model(sb, None, tb, None, None)
    spf, _, tpf, _, _ = NF.storage_model(sb[sfin], None, tb[tfin], None, None)
    cf = corr[sfin]
    cf = np.where(cf == NF.NO, NF.NO, tmap[np.minimum(cf, 199).astype(np.int64)].astype(np.uint64))
    T = np.eye(4)
    T[:3, 3] = [0.01, 0.0, -0.02]
    got = NF.linearize(T, corr, 0, 0, 1.0, sp, None, tp, None, None)
    want = NF.linearize(T, cf, 0, 0, 1.0, spf, None, tpf, None, None)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and got[2] == want[2]
    assert NF.error(T, T, corr, 0, 0, 1.0, sp, None, tp, None, None) == NF.error(T, T, cf, 0, 0, 1.0, spf, None, tpf, None, None)
    wrong = corr.copy()
    wrong[0] = 1
    with pytest.raises(AssertionError, match="non-finite source"):
        NF.linearize(T, wrong, 0, 0, 1.0, sp, None, tp, None, None)
    wrong = corr.copy()
    wrong[1] = 199
    with pytest.raises(AssertionError, match="non-finite target"):
        NF.error(T, T, wrong, 0, 0, 1.0, sp, None, tp, None, None)
