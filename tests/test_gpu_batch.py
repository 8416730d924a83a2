"""Batched registration (sgb_source_set_batch / sgb_{linearize,error,correspondences}_batch): every member of a batch against the
storage model of that member alone, against a single-source context given the same cloud and pose, and against itself in other
batches.

Members are disjoint slices of the 200k-target / 600k-source scene of test_gpu_storage_model (random features, 300 m from the
origin), with sizes on both sides of the 32-query chunk and the 128-point tile, an empty member and one above 65536 points.
Each test prints the worst ratio it reached (run with -s to see it)."""
import numpy as np
import pytest

import np_factors as NF
from test_gpu_storage_model import TRIALS, Data, about

pytestmark = pytest.mark.gpu

MEMBER_SIZES = [0, 1, 31, 32, 33, 127, 128, 129, 4095, 4096, 65537]
COMBOS = [(f, r) for f in (0, 1, 2) for r in (0, 1, 2)]


def _sg():
    import small_gicp_b200 as sg

    return sg


@pytest.fixture(scope="module")
def data():
    d = Data()
    starts = np.concatenate([[0], np.cumsum(MEMBER_SIZES)])
    d.members = [(int(starts[m]), int(MEMBER_SIZES[m])) for m in range(len(MEMBER_SIZES))]
    return d


def _ctx(d, voxel=False):
    sg = _sg()
    ctx = sg.Context(0)
    if voxel:
        ctx.build_target_voxelmap(d.tp, d.tcv, 1.0, 7)
    else:
        ctx.set_target(d.tp, d.tn, d.tcv)
        ctx.build_target_kdtree()
    return ctx


def _member(d, m):
    s, n = d.members[m]
    return d.sp[s : s + n], d.scv[s : s + n]


def _poses(d, members, shift=0):
    """aligned and misaligned poses alternating, each about the member's own centre"""
    out = []
    for j, m in enumerate(members):
        p, _ = _member(d, m)
        c = NF.box_centre(p)
        T = d.aligned if (j + shift) % 2 == 0 else d.misaligned
        out.append(T @ about(c, [0.002 * (m % 5), -0.001 * (m % 3), 0.0015, 0.01 * (m % 4), 0.0, -0.02]))
    return np.array(out)


def _single(ctx1, d, m, T, factor, robust, c, voxel=False):
    p, cv = _member(d, m)
    ctx1.set_source(p, cv)
    H, b, e = ctx1.linearize(T, factor=factor, robust=robust, robust_c=c)
    corr = ctx1.correspondences() if len(p) else np.zeros(0, dtype=np.uint64)
    return H, b, e, corr


def _model(d, m, tgt_model):
    p, cv = _member(d, m)
    tp, tn, tcv = tgt_model
    return NF.stored_points(p), NF.stored_covs(cv) if len(cv) else cv, tp, tn, tcv


def _check_batch(ctx, ctx1, d, members, factor, robust, c, voxel=False, tgt_model=None):
    """one linearize_batch + error_batch at two trial poses, every member against the single context and the storage model"""
    sg = _sg()
    Ts = _poses(d, members)
    H, b, e, inl = ctx.linearize_batch(Ts, factor=factor, robust=robust, robust_c=c)
    corrs = ctx.correspondences_batch()
    trials = [np.array([T @ about(NF.box_centre(_member(d, m)[0]), a) for T, m in zip(Ts, members)]) for a in TRIALS]
    errs = [ctx.error_batch(T2) for T2 in trials]
    worst = 0.0
    for j, m in enumerate(members):
        n = d.members[m][1]
        assert np.array_equal(H[j], H[j].T), (m, "H not bitwise symmetric")
        assert inl[j] == int((corrs[j] != sg.NO_CORRESPONDENCE).sum())
        Hs, bs, es, cs = _single(ctx1, d, m, Ts[j], factor, robust, c, voxel)
        assert np.array_equal(corrs[j], cs), (m, "correspondences differ from the single-source context")
        if n == 0 or inl[j] == 0:
            assert not H[j].any() and not b[j].any() and e[j] == 0.0
            continue
        if not voxel:
            p, _ = _member(d, m)
            check_correspondences_member(corrs[j], d, p, Ts[j])
        model = _model(d, m, tgt_model or d.tgt_model)
        ids = np.where(corrs[j] == NF.NO, NF.NO, corrs[j] >> np.uint64(32)) if voxel else corrs[j]  # voxel id << 32 (calc_index)
        ratios = NF.tight_ratios((H[j], b[j], e[j]), NF.linearize(Ts[j], ids, factor, robust, c, *model))
        assert max(ratios) <= NF.TIGHT, (m, factor, robust, "vs model", ratios)
        ratios_s = NF.tight_ratios((H[j], b[j], e[j]), (Hs, bs, es))
        assert max(ratios_s) <= NF.TIGHT, (m, factor, robust, "vs single context", ratios_s)
        worst = max(worst, *ratios, *ratios_s)
        for T2, eb in zip(trials, errs):
            e_model = NF.error(T2[j], Ts[j], ids, factor, robust, c, *model)
            r = abs(eb[j] - e_model) / e_model
            assert r <= NF.TIGHT, (m, "error_batch", eb[j], e_model, r)
            worst = max(worst, r)
    return worst


def check_correspondences_member(corr, d, p, T):
    """FP64 brute force on a sample (near ties and rejection-boundary cases allowed)"""
    sample = np.arange(len(p)) if len(p) <= 2000 else np.sort(d.rng.choice(len(p), 2000, replace=False))
    q = p[sample, :3] @ T[:3, :3].T + T[:3, 3]
    dist, k = d.tree.query(q, distance_upper_bound=1.0 + 1e-6)
    bf = np.where(np.isinf(dist), NF.NO, k.astype(np.uint64))
    bf[dist * dist > 1.0] = NF.NO
    NF.compare_correspondences(corr[sample], bf, d.tp, p[sample], T, 1.0)


@pytest.mark.parametrize("factor,robust", COMBOS)
def test_kdtree_batch_matches_model_and_single_context(data, factor, robust):
    ctx, ctx1 = _ctx(data), _ctx(data)
    members = list(range(len(MEMBER_SIZES)))
    ctx.set_source_batch([_member(data, m)[0] for m in members], [_member(data, m)[1] for m in members])
    c = 1.0 if robust == 0 else 0.3
    worst = 0.0
    for _ in range(2):  # the second call is seeded by the first
        worst = max(worst, _check_batch(ctx, ctx1, data, members, factor, robust, c))
    print(f"worst ratio (kd-tree, factor {factor}, robust {robust}): {worst:.2e}")


@pytest.mark.parametrize("factor,robust", [(0, 0), (2, 0), (2, 1), (2, 2)])
def test_voxelmap_batch_matches_model_and_single_context(data, factor, robust):
    from np_preprocess import voxelmap_model

    ctx, ctx1 = _ctx(data, voxel=True), _ctx(data, voxel=True)
    members = list(range(len(MEMBER_SIZES)))
    ctx.set_source_batch([_member(data, m)[0] for m in members], [_member(data, m)[1] for m in members])
    _, means, covs, _ = voxelmap_model(data.tp, data.tcv, 1.0)
    tgt_model = (NF.stored_points(means), None, NF.stored_covs(covs))
    c = 1.0 if robust == 0 else 0.3
    worst = _check_batch(ctx, ctx1, data, members, factor, robust, c, voxel=True, tgt_model=tgt_model)
    print(f"worst ratio (voxel map, factor {factor}, robust {robust}): {worst:.2e}")


def _run_batch(ctx, data, members, Ts, active=None, factor=2, robust=0):
    ctx.set_source_batch([_member(data, m)[0] for m in members], [_member(data, m)[1] for m in members])
    out = ctx.linearize_batch(Ts, active=active, factor=factor, robust=robust, robust_c=0.3)
    corr = ctx.correspondences_batch()
    e = ctx.error_batch(np.array([T @ about(NF.box_centre(_member(data, m)[0]), TRIALS[0]) for T, m in zip(Ts, members)]), active=active)
    return out, corr, e


@pytest.mark.parametrize("voxel,factor,robust", [(False, 2, 0), (False, 1, 1), (False, 0, 2), (True, 2, 2), (True, 0, 1)])
def test_members_are_independent_of_the_batch(data, voxel, factor, robust):
    """bit-identical H|b|e|inliers, correspondences and error() for a member wherever it sits, next to whatever, alone, duplicated,
    and with the others inactive"""
    ctx = _ctx(data, voxel)
    kw = dict(factor=factor, robust=robust)
    base = [10, 3, 8, 0, 5, 9]
    Tmap = {m: T for m, T in zip(base, _poses(data, base))}
    ref_out, ref_corr, ref_e = _run_batch(ctx, data, base, np.array([Tmap[m] for m in base]), **kw)

    def same(members, out, corr, e, active=None):
        for j, m in enumerate(members):
            if (active is not None and not active[j]) or m not in base:
                continue
            i = base.index(m)
            for a, r in zip(out, ref_out):
                assert np.array_equal(a[j], r[i]), (members, m)
            assert np.array_equal(corr[j], ref_corr[i]), (members, m)
            assert e[j] == ref_e[i], (members, m)

    for members in ([9, 5, 0, 8, 3, 10], [8, 8, 10, 8], [8], [3, 7, 2, 8, 10, 1, 6, 4, 9, 5, 0]):
        if any(m not in Tmap for m in members):
            Tmap.update({m: T for m, T in zip(members, _poses(data, members, shift=1)) if m not in Tmap})
        out, corr, e = _run_batch(ctx, data, members, np.array([Tmap[m] for m in members]), **kw)
        same(members, out, corr, e)
    active = np.array([1, 0, 1, 0, 0, 1], dtype=np.uint8)
    out, corr, e = _run_batch(ctx, data, base, np.array([Tmap[m] for m in base]), active=active, **kw)
    same(base, out, corr, e, active)
    for j in np.nonzero(active == 0)[0]:
        assert not out[0][j].any() and not out[1][j].any() and out[2][j] == 0 and out[3][j] == 0 and e[j] == 0


@pytest.mark.parametrize("B", [1, 2, 3, 17, 64])
@pytest.mark.parametrize("factor,robust", [(0, 0), (2, 1)])
def test_batch_sizes_match_model_and_single_context(data, B, factor, robust):
    """batches of B members drawn cyclically from the member sizes (duplicates included), every member against the storage model and a
    single-source context"""
    ctx, ctx1 = _ctx(data), _ctx(data)
    members = [(3 * j + B) % len(MEMBER_SIZES) for j in range(B)]
    ctx.set_source_batch([_member(data, m)[0] for m in members], [_member(data, m)[1] for m in members])
    worst = _check_batch(ctx, ctx1, data, members, factor, robust, 1.0 if robust == 0 else 0.3)
    print(f"worst ratio (B = {B}, factor {factor}, robust {robust}): {worst:.2e}")


def test_correspondences_forgotten_with_the_target(data):
    """a new target clears every member's cached correspondences; a member linearised against it gets its own again"""
    sg = _sg()
    ctx = _ctx(data)
    members = [8, 9]
    ctx.set_source_batch([_member(data, m)[0] for m in members], [_member(data, m)[1] for m in members])
    assert all((c == sg.NO_CORRESPONDENCE).all() for c in ctx.correspondences_batch())  # never linearised
    Ts = _poses(data, members)
    ctx.linearize_batch(Ts, factor=0)
    assert all((c != sg.NO_CORRESPONDENCE).any() for c in ctx.correspondences_batch())
    ctx.set_target(data.tp[::2], data.tn[::2], data.tcv[::2])
    ctx.build_target_kdtree()
    assert all((c == sg.NO_CORRESPONDENCE).all() for c in ctx.correspondences_batch())
    with pytest.raises(sg.SgbError, match="sgb_linearize_batch"):
        ctx.error_batch(Ts)
    ctx.linearize_batch(Ts, active=np.array([0, 1], dtype=np.uint8), factor=0)
    corr = ctx.correspondences_batch()
    assert (corr[0] == sg.NO_CORRESPONDENCE).all() and (corr[1] != sg.NO_CORRESPONDENCE).any()


def test_launches_and_inactive_members(data):
    sg = _sg()
    ctx, ctx1 = _ctx(data), _ctx(data)
    launches = set()
    for B in (1, 2, 3, 17, 64):
        members = [4 + (j % 7) for j in range(B)]
        ctx.set_source_batch([_member(data, m)[0] for m in members], [_member(data, m)[1] for m in members])
        Ts = _poses(data, members)
        ctx.linearize_batch(Ts, factor=2)
        k0 = ctx.kernel_launches
        ctx.linearize_batch(Ts, factor=2)
        launches.add(ctx.kernel_launches - k0)
    assert len(launches) == 1, launches
    # every member inactive: zeros
    H, b, e, inl = ctx.linearize_batch(Ts, active=np.zeros(64, dtype=np.uint8), factor=2)
    assert not H.any() and not b.any() and not e.any() and not inl.any()
    # an inactive member keeps its correspondences and linearisation pose: error_batch afterwards uses them
    members = [8, 10]
    ctx.set_source_batch([_member(data, m)[0] for m in members], [_member(data, m)[1] for m in members])
    T1 = _poses(data, members)
    ctx.linearize_batch(T1, factor=2)
    T2 = _poses(data, members, shift=1)
    ctx.linearize_batch(T2, active=np.array([0, 1], dtype=np.uint8), factor=2)
    T3 = np.array([T @ about(NF.box_centre(_member(data, m)[0]), TRIALS[1]) for T, m in zip(T1, members)])
    e = ctx.error_batch(T3)
    p, cv = _member(data, 8)
    ctx1.set_source(p, cv)
    ctx1.linearize(T1[0], factor=2)
    e_single = ctx1.error(T3[0])
    assert abs(e[0] - e_single) <= NF.TIGHT * e_single, (e[0], e_single)
    corr = ctx.correspondences_batch()
    assert np.array_equal(corr[0], ctx1.correspondences())
    assert not (corr[1] == sg.NO_CORRESPONDENCE).all()


def test_rejections_leave_the_context_usable(data):
    sg = _sg()
    ctx = _ctx(data)
    p, cv = _member(data, 8)
    I4 = np.eye(4)
    with pytest.raises(sg.SgbError, match="ascending"):
        ctx.set_source_batch((np.concatenate([p, p]), np.array([0, 10, 5, 2 * len(p)])), np.concatenate([cv, cv]))
    with pytest.raises(sg.SgbError, match="offsets"):
        ctx.set_source_batch((p, np.array([0, len(p) - 1])), cv)
    with pytest.raises(sg.SgbError, match="at most"):
        ctx.set_source_batch((p[:0], np.zeros(65538, dtype=np.uint64)))
    # batch calls without a batch, single calls with one
    ctx.set_source(p, cv)
    with pytest.raises(sg.SgbError, match="no batch"):
        ctx._batch_offsets = np.array([0, len(p)])
        ctx.linearize_batch(I4[None])
    ctx.linearize(data.aligned, factor=2)
    ctx.set_source_batch([p], [cv])
    for call in (lambda: ctx.linearize(data.aligned), lambda: ctx.error(data.aligned), ctx.correspondences, ctx.num_inliers):
        with pytest.raises(sg.SgbError, match="batch"):
            call()
    with pytest.raises(sg.SgbError, match="sgb_linearize_batch"):
        ctx.error_batch(data.aligned[None])
    # multi-GPU wiring refuses batches
    peer = sg.Context(0)
    ctx.comm_connect_ptrs(0, 2, [ctx.comm_mailbox(), peer.comm_mailbox()])
    with pytest.raises(sg.SgbError, match="single-GPU"):
        ctx.linearize_batch(data.aligned[None], factor=2)
    ctx.comm_disconnect()
    H, b, e, inl = ctx.linearize_batch(data.aligned[None], factor=2)
    ctx1 = _ctx(data)
    ctx1.set_source(p, cv)
    H1, b1, e1 = ctx1.linearize(data.aligned, factor=2)
    assert max(NF.tight_ratios((H[0], b[0], e[0]), (H1, b1, e1))) <= NF.TIGHT
