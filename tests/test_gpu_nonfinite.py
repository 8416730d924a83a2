"""Non-finite input points (NaN or +-Inf in x, y or z) are inert (include/sgicp_b200.h): every call on a cloud with such rows is checked
against the same call on the cloud with those rows removed, indices mapped back.

The storage-model checks cannot see a wrong box: a centre taken over an infinite coordinate changes the device and its model together.
Here the model is built from the FILTERED clouds, so the finite points must be stored exactly as they are without the bad rows (same
centre, same FP32 coordinates) for the sums to agree to NF.TIGHT.  Each scene injects bad rows at the first and last row, as a run of 33
(a whole 32-point leaf and a 32-query chunk), scattered over ~1 % of the rows, NaN in y only, +Inf, -Inf, both, positive NaN and NaN
with its sign bit set; a source member that is entirely non-finite is part of the batched checks.

Fixes and the tests that fail without them: one +Inf row (target or source) made the box centre infinite, so no point had a
correspondence (test_one_inf_row, and every +-Inf case); voxel-grid sampling and the voxel-map build put a NaN point into voxel 0
(test_voxel_paths); NaN target points all fell into grid cell 0, whose block then exceeded kGridMaxList and disabled the grid front end
(test_grid_front_end_kept).  Two changes alter no result and are not claimed by a failing test: the tree-box reductions of the kd
refinement skip NaN (those boxes only choose split axes), and NaN lanes leave leaf boxes empty (a NaN box would only be walked, never
answered from).  Non-finite queries now skip the search outright; that is a cost, not a result (measured in scripts/bench_nonfinite.py)."""
import numpy as np
import pytest

import np_factors as NF
import np_preprocess as PP
import np_search as NS
from conftest import pose_error
from test_gpu_align_batch import _starts
from test_gpu_preprocess_model import check_features
from test_gpu_storage_model import about

pytestmark = pytest.mark.gpu

N = 60_000
NAN_NEG = np.frombuffer(np.uint64(0xFFF8000000000000).tobytes(), dtype=np.float64)[0]
NO = NF.NO


def _sg():
    import small_gicp_b200 as sg

    return sg


def _rows(case, n, rng):
    """(rows, values, axes) of a case; axes None = every coordinate of the row"""
    if case == "first_last":
        return [0, n - 1], [np.nan, np.inf], None
    if case == "run33":
        return list(range(n // 2, n // 2 + 33)), [np.nan], None
    if case == "scattered":
        return sorted(rng.choice(n, n // 100, replace=False).tolist()), [np.nan, np.inf, -np.inf, NAN_NEG], None
    if case == "nan_y":
        return sorted(rng.choice(n, 50, replace=False).tolist()), [np.nan], [1]
    if case == "inf_pos":
        return [n // 3], [np.inf], [0]
    if case == "inf_neg":
        return [n // 3, 2 * n // 3], [-np.inf], [2]
    if case == "inf_both":
        return [5, n // 2, n - 7], [np.inf, -np.inf], [0, 1, 2]
    if case == "nan_pos":
        return sorted(rng.choice(n, 40, replace=False).tolist()), [np.nan], None
    if case == "nan_neg":
        return sorted(rng.choice(n, 40, replace=False).tolist()), [NAN_NEG], None
    raise ValueError(case)


CASES = ["first_last", "run33", "scattered", "nan_y", "inf_pos", "inf_neg", "inf_both", "nan_pos", "nan_neg"]


def inject(pts, case, seed):
    rng = np.random.default_rng(seed)
    out = np.array(pts, dtype=np.float64)
    rows, vals, axes = _rows(case, len(out), rng)
    for j, r in enumerate(rows):
        v = vals[j % len(vals)]
        if axes is None:
            out[r, :3] = v
        else:
            out[r, axes[j % len(axes)]] = v
    return out


@pytest.fixture(scope="module")
def scene():
    from small_gicp_b200.synthetic import make_pair

    tgt, src, T = make_pair(N, n_source=N // 2)
    return tgt, src, T


def _features(ctx, pts, k=10):
    """device features of a cloud with bad rows: those rows get the < 5 neighbours value, the finite rows are held to the FP64 model of
    the filtered cloud (check_features: the exact neighbour sets, unless the k-th and (k+1)-th are tied)"""
    fin = NF.finite_rows(pts)
    nrm, cov = ctx.estimate_features(pts, k)
    assert np.array_equal(nrm[~fin], np.zeros((int((~fin).sum()), 4)))
    assert np.array_equal(cov[~fin], np.broadcast_to(np.diag([1.0, 1.0, 1.0, 0.0]), (int((~fin).sum()), 4, 4)))
    check_features(pts[fin][:, :3], nrm[fin], cov[fin], k, "finite rows")
    return nrm, cov


def _ctx(tgt, tcov, src, scov, profiling=False):
    ctx = _sg().Context(0, profiling=profiling)
    ctx.set_target(tgt, None, tcov)
    ctx.build_target_kdtree()
    ctx.set_source(src, scov)
    return ctx


def _map(fin):
    """filtered index -> original row"""
    return np.nonzero(fin)[0]


def _check_call(ctx, T, tb, tcov, sb, scov, max_d=1.0):
    """one linearize / error on the bad clouds: every query against the exact search model, bad rows unmatched, the sums against the
    storage model of the FILTERED clouds to NF.TIGHT"""
    sg = _sg()
    H, b, e = ctx.linearize(T, factor=sg.FACTOR_GICP, max_dist_sq=max_d)
    corr = ctx.correspondences()
    sfin, tfin = NF.finite_rows(sb), NF.finite_rows(tb)
    assert (corr[~sfin] == NO).all()
    hit = corr != NO
    assert NF.finite_rows(tb[corr[hit].astype(np.int64)]).all()
    NS.check_correspondences(corr, T, sb, NS.Target(tb), max_d)
    inl = ctx.num_inliers()
    assert inl == int(hit.sum())
    # filtered model, the device's correspondences mapped to filtered target indices
    tmap = np.full(len(tb), -1, dtype=np.int64)
    tmap[tfin] = np.arange(int(tfin.sum()))
    cf = corr[sfin]
    cf = np.where(cf == NO, NO, tmap[np.where(cf == NO, 0, cf).astype(np.int64)].astype(np.uint64))
    sp, scv, tp, _, tcv = NF.storage_model(sb[sfin], scov[sfin], tb[tfin], None, tcov[tfin])
    if inl == 0:
        assert (H == 0).all() and (b == 0).all() and e == 0.0
        return corr, inl
    want = NF.linearize(T, cf, 2, 0, 1.0, sp, scv, tp, None, tcv)
    assert max(NF.tight_ratios((H, b, e), want)) <= NF.TIGHT
    T2 = T @ about(NF.box_centre(sb), [0.001, 0.0, -0.001, 0.01, 0.0, 0.005])
    e2 = ctx.error(T2)
    w2 = NF.error(T2, T, cf, 2, 0, 1.0, sp, scv, tp, None, tcv)
    assert abs(e2 - w2) <= NF.TIGHT * w2
    return corr, inl


@pytest.mark.parametrize("case", CASES)
def test_single_kdtree(scene, case):
    """bad rows in target and source: every finite query exact, bad rows unmatched, sums = the filtered clouds' model, inlier counts =
    the filtered context's, at identity, the converged pose and a misaligned pose"""
    tgt, src, Tgt = scene
    tb, sb = inject(tgt, case, 1), inject(src, case, 2)
    sfin, tfin = NF.finite_rows(sb), NF.finite_rows(tb)
    ctx = _sg().Context(0)
    _, tcov = _features(ctx, tb)
    _, scov = _features(ctx, sb)
    ctx.close()
    bad, flt = _ctx(tb, tcov, sb, scov), _ctx(tb[tfin], tcov[tfin], sb[sfin], scov[sfin])
    for T in (np.eye(4), Tgt, Tgt @ about(NF.box_centre(sb), [0.01, -0.012, 0.008, 0.25, -0.2, 0.15])):
        corr, inl = _check_call(bad, T, tb, tcov, sb, scov)
        flt.linearize(T, factor=_sg().FACTOR_GICP)
        assert inl == flt.num_inliers() and inl > 0
        cf = flt.correspondences()
        same = _map(tfin)[cf[cf != NO].astype(np.int64)]
        assert (corr[sfin][cf != NO] == same).mean() >= 0.999  # equal but for exact distance ties
    bad.close()
    flt.close()


@pytest.mark.parametrize("where", ["target", "source"])
def test_one_inf_row(scene, where):
    """one +Inf coordinate made the whole cloud's centre infinite: no correspondence anywhere, zero sums"""
    tgt, src, Tgt = scene
    tb, sb = np.array(tgt), np.array(src)
    (tb if where == "target" else sb)[17, 0] = np.inf
    sg = _sg()
    ctx = sg.Context(0)
    ctx.set_target(tb)
    ctx.build_target_kdtree()
    ctx.set_source(sb)
    H, b, e = ctx.linearize(Tgt, factor=sg.FACTOR_ICP)
    corr = ctx.correspondences()
    assert ctx.num_inliers() > 0.9 * NF.finite_rows(sb).sum()
    NS.check_correspondences(corr, Tgt, sb, NS.Target(tb), 1.0)
    sfin, tfin = NF.finite_rows(sb), NF.finite_rows(tb)
    tmap = np.full(len(tb), -1, dtype=np.int64)
    tmap[tfin] = np.arange(int(tfin.sum()))
    cf = corr[sfin]
    cf = np.where(cf == NO, NO, tmap[np.where(cf == NO, 0, cf).astype(np.int64)].astype(np.uint64))
    sp, _, tp, _, _ = NF.storage_model(sb[sfin], None, tb[tfin], None, None)
    assert max(NF.tight_ratios((H, b, e), NF.linearize(Tgt, cf, 0, 0, 1.0, sp, None, tp, None, None))) <= NF.TIGHT
    ctx.close()


REGIMES = [("SGB_PENDING_DIV", "1"), ("SGB_PENDING_DIV", "1000000"), ("SGB_GRID", "0")]


@pytest.mark.parametrize("var,value", REGIMES)
@pytest.mark.parametrize("case", ["run33", "scattered", "inf_both", "nan_neg"])
def test_search_regimes(scene, case, var, value, monkeypatch):
    """every finite query exact in the regimes test_gpu_search_exhaustive forces (grid probe + ring / packet walk, tree only)"""
    monkeypatch.setenv(var, value)
    tgt, src, Tgt = scene
    tb, sb = inject(tgt, case, 3), inject(src, case, 4)
    sg = _sg()
    ctx = sg.Context(0, profiling=True)
    ctx.set_target(tb)
    ctx.build_target_kdtree()
    ctx.set_source(sb)
    t = NS.Target(tb)
    for T in (np.eye(4), Tgt, Tgt @ about(NF.box_centre(sb), [0.0, 0.0, 0.0087, 0.2, 0.0, 0.0])):
        ctx.linearize(T, factor=sg.FACTOR_ICP)
        NS.check_correspondences(ctx.correspondences(), T, sb, t, 1.0)
    ctx.close()


def test_all_nonfinite_clouds(scene):
    """a target or a source of bad rows only: no correspondence, zero sums, no error"""
    tgt, src, Tgt = scene
    sg = _sg()
    ctx = sg.Context(0)
    allbad = np.full((5000, 3), np.nan)
    allbad[::2, 1] = np.inf
    ctx.set_target(allbad)
    ctx.build_target_kdtree()
    ctx.set_source(src)
    H, b, e = ctx.linearize(Tgt, factor=sg.FACTOR_ICP)
    assert (H == 0).all() and (b == 0).all() and e == 0.0 and (ctx.correspondences() == NO).all()
    ctx.set_target(tgt)
    ctx.build_target_kdtree()
    ctx.set_source(allbad)
    H, b, e = ctx.linearize(Tgt, factor=sg.FACTOR_ICP)
    assert (H == 0).all() and (b == 0).all() and e == 0.0 and (ctx.correspondences() == NO).all()
    ctx.close()


@pytest.mark.parametrize("case", ["scattered", "inf_both", "nan_y"])
def test_voxel_paths(scene, case):
    """voxelgrid_sampling(_batch) and the device-built voxel map(s): bit-identical to the filtered cloud's; VGICP sums equal"""
    tgt, src, Tgt = scene
    tb, sb = inject(tgt, case, 5), inject(src, case, 6)
    tfin, sfin = NF.finite_rows(tb), NF.finite_rows(sb)
    sg = _sg()
    ctx = sg.Context(0)
    v = ctx.voxelgrid_sampling(tb, 0.3)
    assert np.isfinite(v).all()
    assert np.array_equal(v, ctx.voxelgrid_sampling(tb[tfin], 0.3))
    assert np.array_equal(v, PP.voxelgrid_model(tb[tfin], 0.3))
    vb, off = ctx.voxelgrid_sampling_batch([tb, np.full((40, 3), np.nan), sb], 0.3)
    vf, offf = ctx.voxelgrid_sampling_batch([tb[tfin], np.zeros((0, 3)), sb[sfin]], 0.3)
    assert np.array_equal(off, offf) and np.array_equal(vb, vf)
    _, tcov = _features(ctx, tb)
    _, scov = _features(ctx, sb)
    out = []
    for t_, tc_, s_, sc_ in ((tb, tcov, sb, scov), (tb[tfin], tcov[tfin], sb[sfin], scov[sfin])):
        for offsets in (1, 7, 27):
            ctx.build_target_voxelmap(t_, tc_, 1.0, offsets)
            ctx.set_source(s_, sc_)
            H, b, e = ctx.linearize(Tgt, factor=sg.FACTOR_GICP)
            corr = ctx.correspondences()
            if s_ is sb:
                assert (corr[~sfin] == NO).all()
                corr = corr[sfin]
            out.append((H, b, e, ctx.num_inliers(), corr))
    for a, f in zip(out[:3], out[3:]):
        assert a[3] == f[3] > 0 and np.array_equal(a[4], f[4])
        assert max(NF.tight_ratios(a[:3], f[:3])) <= NF.TIGHT
    ctx.close()


def _batch_results(ctx, Ts, n_members):
    sg = _sg()
    H, b, e, inl = ctx.linearize_batch(Ts, factor=sg.FACTOR_GICP)
    eb = ctx.error_batch(Ts)
    pts = ctx.linearize_batch_points(Ts, factor=sg.FACTOR_GICP)
    return H, b, e, inl, eb, pts, ctx.correspondences_batch()


@pytest.mark.parametrize("target", ["kdtree", "kdtrees", "voxelmap", "voxelmaps"])
@pytest.mark.parametrize("weights", [False, True])
def test_batch_members(scene, target, weights):
    """batched calls over members with bad rows and a member that is entirely non-finite, against every target kind: member sums and
    inliers equal the filtered batch's (the all-bad member: an empty member), per-point rows of bad rows zero, finite rows equal"""
    tgt, src, Tgt = scene
    sg = _sg()
    n4 = len(src) // 4
    members = [inject(src[:n4], "scattered", 7), np.full((50, 3), np.nan), inject(src[n4 : 2 * n4], "run33", 8), inject(src[2 * n4 :], "inf_both", 9)]
    maps = [inject(tgt, "scattered", 10), inject(tgt, "first_last", 11), inject(tgt, "nan_y", 12), inject(tgt, "inf_both", 13)]
    ctx = sg.Context(0)
    covs = [_features(ctx, m)[1] if NF.finite_rows(m).any() else np.tile(np.diag([1.0, 1.0, 1.0, 0.0]), (len(m), 1, 1)) for m in members]
    mcovs = [_features(ctx, m)[1] for m in maps]
    ctx.close()
    fins = [NF.finite_rows(m) for m in members]
    mfins = [NF.finite_rows(m) for m in maps]
    rng = np.random.default_rng(14)
    Ts = np.array([Tgt @ about(NF.box_centre(m) if f.any() else np.zeros(3), rng.normal(0, [0.002] * 3 + [0.02] * 3)) for m, f in zip(members, fins)])
    w = [rng.uniform(0.2, 2.0, len(m)) for m in members]
    res = []
    for filt in (False, True):
        ms = [m[f] if filt else m for m, f in zip(members, fins)]
        cs = [c[f] if filt else c for c, f in zip(covs, fins)]
        ts = [m[f] if filt else m for m, f in zip(maps, mfins)]
        tcs = [c[f] if filt else c for c, f in zip(mcovs, mfins)]
        ctx = sg.Context(0)
        if target == "kdtree":
            ctx.set_target(ts[0], None, tcs[0])
            ctx.build_target_kdtree()
        elif target == "kdtrees":
            ctx.build_target_kdtrees(ts, None, tcs)
        elif target == "voxelmap":
            ctx.build_target_voxelmap(ts[0], tcs[0], 1.0, 7)
        else:
            ctx.build_target_voxelmaps(ts, tcs, 1.0, 7)
        ctx.set_source_batch(ms, cs)
        if weights:
            ctx.set_source_weights(np.concatenate([x[f] if filt else x for x, f in zip(w, fins)]))
        res.append(_batch_results(ctx, Ts, len(members)))
        ctx.close()
    (H, b, e, inl, eb, pts, corr), (Hf, bf, ef, inlf, ebf, ptsf, corrf) = res
    assert np.array_equal(inl, inlf) and inl[1] == 0 and (inl[[0, 2, 3]] > 0).all()
    assert (H[1] == 0).all() and (b[1] == 0).all() and e[1] == 0.0 and eb[1] == 0.0
    for m in (0, 2, 3):
        assert max(NF.tight_ratios((H[m], b[m], e[m]), (Hf[m], bf[m], ef[m]))) <= NF.TIGHT
        assert abs(eb[m] - ebf[m]) <= NF.TIGHT * ebf[m]
    fin_all = np.concatenate(fins)
    assert (pts.point_e[~fin_all] == 0).all() and (pts.point_Hb42[~fin_all] == 0).all()
    assert np.allclose(pts.point_e[fin_all], ptsf.point_e, rtol=1e-12, atol=0)
    for m in range(len(members)):
        assert (corr[m][~fins[m]] == NO).all()
        c, cf = corr[m][fins[m]], corrf[m]
        assert np.array_equal(c == NO, cf == NO)
        if not (cf != NO).any():
            continue
        if target in ("kdtree", "kdtrees"):
            mf = mfins[0] if target == "kdtree" else mfins[m]
            assert (c[cf != NO] == _map(mf)[cf[cf != NO].astype(np.int64)]).mean() >= 0.999
        else:
            assert np.array_equal(c, cf)


def test_knn_and_features_batch(scene):
    """target_batch_knn: NaN / Inf queries get empty rows, finite queries the filtered target's k-NN; estimate_features_batch: bad
    rows invalid, finite rows held to the filtered clouds' FP64 model"""
    tgt, src, Tgt = scene
    sg = _sg()
    tb = inject(tgt, "scattered", 15)
    q = inject(src[:5000] @ Tgt[:3, :3].T + Tgt[:3, 3], "inf_both", 16)
    q[100:133] = np.nan
    ctx = sg.Context(0)
    ctx.set_target(tb)
    ctx.build_target_kdtree()
    idx, d2 = ctx.target_batch_knn(q, 8)
    NS.check_knn(idx, d2, q, 8, NS.Target(tb))
    clouds = [tb, inject(src, "run33", 17), np.full((20, 3), np.inf)]
    n_b, c_b = ctx.estimate_features_batch(clouds, 10)
    ok = np.concatenate([NF.finite_rows(c) for c in clouds])
    assert (n_b[~ok] == 0).all() and np.array_equal(c_b[~ok], np.broadcast_to(np.diag([1.0, 1.0, 1.0, 0.0]), (int((~ok).sum()), 4, 4)))
    off = np.concatenate([[0], np.cumsum([len(c) for c in clouds])])
    for j, c in enumerate(clouds[:2]):
        f = NF.finite_rows(c)
        check_features(c[f][:, :3], n_b[off[j] : off[j + 1]][f], c_b[off[j] : off[j + 1]][f], 10, f"cloud {j}")
    ctx.close()


def _many_maps(scene):
    """two maps and three source clouds with bad rows (one entirely non-finite), the maps' and clouds' covariances"""
    tgt, src, Tgt = scene
    n3 = len(src) // 3
    maps = [inject(tgt, "scattered", 30), inject(tgt[::2], "inf_both", 31)]
    clouds = [inject(src[:n3], "run33", 32), np.full((40, 3), np.nan), inject(src[n3:], "nan_neg", 33)]
    return maps, clouds


def _remap_entries(c, lists_p, mfins):
    """(entry << 32 | index within the filtered map) -> the same with the index within the map as given"""
    out = np.full(len(c), NO)
    hit = c != NO
    ent = (c[hit] >> np.uint64(32)).astype(np.int64)
    loc = (c[hit] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    rows = np.array([_map(mfins[lists_p[e]])[j] for e, j in zip(ent, loc)], dtype=np.int64)
    out[hit] = (ent.astype(np.uint64) << np.uint64(32)) | rows.astype(np.uint64)
    return out


@pytest.mark.parametrize("kind", ["pairs", "submaps"])
def test_pairs_and_submaps(scene, kind):
    """(cloud, map) pairs and submap members over many kd-trees with bad rows on both sides: member sums, inliers and per-point rows
    (linearize_batch_points, error_batch_points) equal the filtered clouds' and maps'; bad rows unmatched"""
    tgt, src, Tgt = scene
    sg = _sg()
    maps, clouds = _many_maps(scene)
    mfins, cfins = [NF.finite_rows(m) for m in maps], [NF.finite_rows(c) for c in clouds]
    pcl, pmp = np.array([0, 1, 2, 2, 0]), np.array([0, 0, 1, 0, 1])
    lists = [[0, 1], [1], [1, 0], [0]]
    slc = np.array([0, 1, 2, 2])
    poses = [[np.eye(4), about(np.zeros(3), [0.0, 0.0, 1e-3, 0.01, 0.0, 0.0])], [np.eye(4)], [np.eye(4), np.eye(4)], [np.eye(4)]]
    members = pcl if kind == "pairs" else slc
    rng = np.random.default_rng(34)
    Ts = np.array([Tgt @ about(NF.box_centre(clouds[c]) if cfins[c].any() else np.zeros(3), rng.normal(0, [0.002] * 3 + [0.02] * 3)) for c in members])
    res = []
    for filt in (False, True):
        ctx = sg.Context(0)
        ctx.build_target_kdtrees([m[f] if filt else m for m, f in zip(maps, mfins)])
        ctx.set_source_batch([c[f] if filt else c for c, f in zip(clouds, cfins)])
        if kind == "pairs":
            ctx.set_source_pairs(pcl, pmp)
        else:
            ctx.set_source_submaps(lists, poses, slc)
        H, b, e, inl = ctx.linearize_batch(Ts, factor=sg.FACTOR_ICP)
        pts = ctx.linearize_batch_points(Ts, factor=sg.FACTOR_ICP)
        eb, pe = ctx.error_batch_points(Ts)
        res.append((H, b, e, inl, pts, eb, pe, ctx.correspondences_batch()))
        ctx.close()
    (H, b, e, inl, pts, eb, pe, corr), (Hf, bf, ef, inlf, ptsf, ebf, pef, corrf) = res
    assert np.array_equal(inl, inlf) and (inl[members == 1] == 0).all() and (inl[members != 1] > 0).all()
    for m in range(len(members)):
        fin = cfins[members[m]]
        assert (corr[m][~fin] == NO).all()
        if inl[m] == 0:
            assert (H[m] == 0).all() and e[m] == 0.0 and eb[m] == 0.0
            continue
        assert max(NF.tight_ratios((H[m], b[m], e[m]), (Hf[m], bf[m], ef[m]))) <= NF.TIGHT
        assert abs(eb[m] - ebf[m]) <= NF.TIGHT * ebf[m]
        c, cf = corr[m][fin], corrf[m]
        assert np.array_equal(c == NO, cf == NO)
        if kind == "pairs":
            want = np.where(cf == NO, NO, _map(mfins[pmp[m]])[np.where(cf == NO, 0, cf).astype(np.int64)].astype(np.uint64))
        else:
            want = _remap_entries(cf, lists[m], mfins)
        assert (c == want).mean() >= 0.999  # equal but for exact distance ties
    fin_all = np.concatenate([cfins[c] for c in members])
    for rows, rows_f in ((pts.point_e, ptsf.point_e), (pe, pef)):
        assert (rows[~fin_all] == 0).all()
        assert np.allclose(rows[fin_all], rows_f, rtol=1e-12, atol=0)
    assert (pts.point_Hb42[~fin_all] == 0).all()


def test_knn_maps_and_submaps(scene):
    """target_knn_maps / target_knn_submaps over many kd-trees with bad rows: bad queries get empty rows, finite queries the filtered
    maps' neighbours (indices mapped back, the same squared distances)"""
    tgt, src, Tgt = scene
    sg = _sg()
    maps, _ = _many_maps(scene)
    mfins = [NF.finite_rows(m) for m in maps]
    qs = [inject(src[:3000] @ Tgt[:3, :3].T + Tgt[:3, 3], "scattered", 35), inject(src[3000:5000] @ Tgt[:3, :3].T + Tgt[:3, 3], "inf_both", 36)]
    qfin = np.concatenate([NF.finite_rows(q) for q in qs])
    lists = [[0, 1], [1]]
    out = []
    for filt in (False, True):
        ctx = sg.Context(0)
        ctx.build_target_kdtrees([m[f] if filt else m for m, f in zip(maps, mfins)])
        out.append((ctx.target_knn_maps(qs, 6, maps=[1, 0]), ctx.target_knn_submaps(qs, lists, None, 6)))
        ctx.close()
    for which in (0, 1):
        (idx, d2), (idxf, d2f) = out[0][which], out[1][which]
        assert (idx[~qfin] == NO).all() and (d2[~qfin] == NS.DBL_MAX).all()
        assert np.array_equal(d2[qfin], d2f[qfin])
        n0 = len(qs[0])
        for s, (a, b_) in enumerate(((0, n0), (n0, n0 + len(qs[1])))):
            rows = np.arange(a, b_)[qfin[a:b_]]
            if which == 0:
                mf = mfins[[1, 0][s]]
                want = np.where(idxf[rows] == NO, NO, _map(mf)[np.where(idxf[rows] == NO, 0, idxf[rows]).astype(np.int64)].astype(np.uint64))
            else:
                want = _remap_entries(idxf[rows].ravel(), lists[s], mfins).reshape(idxf[rows].shape)
            assert (idx[rows] == want).mean() >= 0.999


def test_align_joint(scene):
    """a window of three frames whose clouds have bad rows (every frame also its own map): align_joint equals the filtered window's run"""
    tgt, src, Tgt = scene
    sg = _sg()
    frames = [inject(tgt, "scattered", 37), inject(src, "inf_both", 38), inject(tgt[1::2], "run33", 39)]
    fins = [NF.finite_rows(f) for f in frames]
    X0 = np.array([np.eye(4), Tgt @ about(NF.box_centre(src), [0.002, -0.001, 0.002, 0.03, -0.02, 0.01]), about(np.zeros(3), [0.0, 0.001, 0.0, 0.02, 0.0, 0.0])])
    out = []
    for filt in (False, True):
        fs = [f[m] if filt else f for f, m in zip(frames, fins)]
        ctx = sg.Context(0)
        ctx.build_target_kdtrees(fs)
        ctx.set_source_batch(fs)
        ctx.set_source_pairs([1, 2, 2, 1], [0, 0, 1, 2])
        out.append(ctx.align_joint(X0, factor=sg.FACTOR_ICP))
        ctx.close()
    a, f = out
    assert np.array_equal(a.iterations, f.iterations) and np.array_equal(a.num_inliers, f.num_inliers) and np.array_equal(a.converged, f.converged)
    assert a.num_inliers[0] > 0
    assert np.abs(a.X - f.X).max() <= 1e-6


def test_golden_pair(golden_prepared):
    """the golden pair with ~1 % NaN rows and one +Inf row on each side still meets test_gpu_align_batch's golden bars: every start
    within 1e-4 rad / 1e-3 m of the oracle's alignment of the filtered pair, the same iterations, inliers within 2"""
    import oracle as O

    sg = _sg()
    g = golden_prepared
    tc, sc = g["target"], g["source"]
    tp, sp = inject(tc.points, "scattered", 40), inject(sc.points, "scattered", 41)
    tp[len(tp) // 2, 0], sp[len(sp) // 3, 1] = np.inf, np.inf
    tf, sf = NF.finite_rows(tp), NF.finite_rows(sp)
    starts = _starts()
    ctx = sg.Context(0)
    ctx.set_target(tp, tc.normals, tc.covs)
    ctx.build_target_kdtree()
    ctx.set_source_batch([sp] * len(starts), [sc.covs] * len(starts))
    r = ctx.align_batch(starts, factor=sg.FACTOR_GICP)
    ctx.close()
    ot, os_ = O.Cloud(tc.points[tf]), O.Cloud(sc.points[sf])
    ot.set_features(tc.normals[tf], tc.covs[tf])
    os_.set_features(sc.normals[sf], sc.covs[sf])
    tree = O.KdTree(ot)
    reg = O.Registration(factor=O.FACTOR_GICP, num_threads=0)
    for m, T0 in enumerate(starts):
        ref = reg.align(ot, tree, os_, T0)
        rot, trans = pose_error(ref.T_target_source, r.T_target_source[m])
        assert rot < 1e-4 and trans < 1e-3, (m, rot, trans)
        assert r.iterations[m] == ref.iterations, (m, r.iterations[m], ref.iterations)
        assert abs(r.num_inliers[m] - ref.num_inliers) <= 2, (m, r.num_inliers[m], ref.num_inliers)


def test_grid_front_end_kept(scene, capfd, monkeypatch):
    """3000 NaN target rows: before they were kept out of the grid they all fell into cell 0, that block exceeded kGridMaxList and the
    front end was dropped for the whole target; now the grid is built and every query is still exact"""
    monkeypatch.setenv("SGB_DEBUG_PENDING", "1")
    tgt, src, Tgt = scene
    tb = np.array(tgt)
    tb[1000:4000] = np.nan
    sg = _sg()
    capfd.readouterr()
    ctx = sg.Context(0, profiling=True)
    ctx.set_target(tb)
    ctx.build_target_kdtree()
    ctx.set_source(src)
    ctx.linearize(Tgt, factor=sg.FACTOR_ICP)
    NS.check_correspondences(ctx.correspondences(), Tgt, src, NS.Target(tb), 1.0)
    ctx.close()
    err = capfd.readouterr().err
    assert "grid front end: cell" in err and "dropped" not in err, err[-2000:]


def test_align_batch_and_gnc(scene):
    """align_batch and align_batch_gnc on members with bad rows: the filtered batch's iterations and inliers, poses to 1e-6"""
    tgt, src, Tgt = scene
    sg = _sg()
    n3 = len(src) // 3
    members = [inject(src[:n3], "scattered", 18), inject(src[n3 : 2 * n3], "inf_both", 19), inject(src[2 * n3 :], "nan_neg", 20)]
    tb = inject(tgt, "scattered", 21)
    fins, tfin = [NF.finite_rows(m) for m in members], NF.finite_rows(tb)
    rng = np.random.default_rng(22)
    Ts = np.array([Tgt @ about(NF.box_centre(m), rng.normal(0, [0.01] * 3 + [0.1] * 3)) for m in members])
    out = []
    for filt in (False, True):
        ctx = sg.Context(0)
        ctx.set_target(tb[tfin] if filt else tb)
        ctx.build_target_kdtree()
        ctx.set_source_batch([m[f] if filt else m for m, f in zip(members, fins)])
        r = ctx.align_batch(Ts, factor=sg.FACTOR_ICP)
        g = ctx.align_batch_gnc(Ts, 0.25, factor=sg.FACTOR_ICP)
        out.append((r, g))
        ctx.close()
    (r, g), (rf, gf) = out
    for a, f in ((r, rf), (g, gf)):
        assert np.array_equal(a.iterations, f.iterations) and np.array_equal(a.num_inliers, f.num_inliers)
        assert np.array_equal(a.converged, f.converged)
        assert np.abs(a.T_target_source - f.T_target_source).max() <= 1e-6
