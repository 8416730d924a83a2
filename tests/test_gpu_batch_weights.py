"""Per-point weights of batched registration (sgb_source_set_weights, Context.set_source_weights): every batched call scales each source
point's terms by the caller's weight, on every target kind.

  1. all-ones weights change nothing: every batched call bit for bit, on every kind, factor and several align options;
  2. random weights in [0, 3] with exact zeros: every row is w times the unweighted row bit for bit (a numpy FP64 multiply), the
     correspondences and num_inliers are the unweighted call's, each member's rows add up to its sums, and the rows match the FP64
     storage model times w;
  3. weighted align_batch is the reference optimiser on the weighted H | b (the round-by-round replay of test_gpu_align_batch_replay),
     and zero weights on a subset align as the cloud without those points does;
  4. layout: permuted cloud and weights give permuted rows, a member is bit-identical at B = 1, 17 and 4096, and two members of one cloud
     carry weights of their own;
  5. lifetime: the source setters clear the weights, target rebuilds keep them, and weights set again between asynchronous aligns or
     graph replays are read there;
  6. CUDA and page-locked weights equal host weights bit for bit;
  7. launch counts;
  8. misuse fails with a message and leaves the weights in force."""
import numpy as np
import pytest

import np_factors as NF
from conftest import pose_error
from test_gpu_align_batch_replay import DEFAULTS, Stats, prefix_runs, replay
from test_gpu_batch_points import ROBUST, Scene, _factors, _kdtree, _p4, _same, kinds, model_member, row_ratios
from test_gpu_storage_model import OFFSET, _random_covs, about

pytestmark = pytest.mark.gpu

GN, LM = 0, 1
ALIGNS = [dict(optimizer=LM), dict(optimizer=GN, robust=1, robust_c=0.5), dict(optimizer=LM, robust=2, robust_c=0.5),
          dict(optimizer=LM, factor=0, dof_mask=[1, 1, 0, 1, 1, 1]), dict(optimizer=GN, max_iterations=1), dict(optimizer=LM, max_iterations=0)]
RESULT = ("T_target_source", "converged", "iterations", "num_inliers", "error", "H", "b")


def _sg():
    import small_gicp_b200 as sg

    return sg


def _torch():
    return pytest.importorskip("torch")


@pytest.fixture(scope="module")
def scene():
    return Scene()


@pytest.fixture(scope="module")
def all_kinds(scene):
    return kinds(scene)


@pytest.fixture(scope="module")
def stream():
    """one torch stream for the asynchronous calls of the module (the default stream is the null stream, which set_stream cannot name)"""
    torch = _torch()
    s = torch.cuda.Stream()
    yield s
    s.synchronize()


def _n(ctx):
    return int(ctx._batch_offsets[-1])


def random_weights(n, seed):
    """uniform in [0, 3], about 15 % exact zeros and a few -0.0"""
    rng = np.random.default_rng(seed)
    w = rng.uniform(0.0, 3.0, n)
    w[rng.random(n) < 0.15] = 0.0
    w[rng.random(n) < 0.02] = -0.0
    return w


def _lin(ctx, T, **kw):
    return ctx.linearize_batch(T, **kw)


def _align(r):
    return [np.asarray(getattr(r, f)) for f in RESULT]


def _async_host(a):
    return [a.T_target_source.cpu().numpy(), a.converged.cpu().numpy() != 0, a.iterations.cpu().numpy().astype(np.int64),
            a.num_inliers.cpu().numpy().astype(np.int64), a.error.cpu().numpy(), a.H.cpu().numpy(), a.b.cpu().numpy()]


def _joint_poses(K, k=0):
    return np.array([about(OFFSET, [0.002 * ((j + k) % 3), -0.001 * j, 0.001, 0.03 * ((j + k) % 2), -0.02, 0.01 * j]) for j in range(K)])


def battery(kind, s, stream):
    """every batched call on the kind's context: the plain calls, the _points calls, aligns, and their asynchronous and joint forms"""
    torch = _torch()
    ctx = kind.ctx
    T, T1, T2 = s.poses(kind.clouds), s.poses(kind.clouds, 1), s.poses(kind.clouds, 2)
    out = []
    for factor in _factors(kind):
        for robust, c in ROBUST:
            out += list(ctx.linearize_batch(T, factor=factor, robust=robust, robust_c=c))
            out += ctx.correspondences_batch()
            out += [ctx.error_batch(T1), ctx.error_batch(T2)]
        r = ctx.linearize_batch_points(T, factor=factor, robust=1, robust_c=0.05)
        out += [r.H, r.b, r.e, r.num_inliers, r.point_e, r.point_Hb42]
        out += list(ctx.error_batch_points(T1))
    Td = torch.from_numpy(np.ascontiguousarray(T)).cuda()
    ctx.set_stream(stream.cuda_stream)
    try:
        for kw in ALIGNS:
            out += _align(ctx.align_batch(T, **kw)) + ctx.correspondences_batch()
            with torch.cuda.stream(stream):
                a = ctx.align_batch_async(Td, **kw)
            ctx.synchronize()
            out += _async_host(a)
        if kind.name == "pairs_maps":  # frames = the 5 clouds with the 5 maps, edges = the pairs
            X = _joint_poses(5)
            Xd = torch.from_numpy(X).cuda()
            for kw in ALIGNS[:3]:
                j = ctx.align_joint(X, **kw)
                out += [j.X, j.converged, j.iterations, j.num_inliers, j.error]
                with torch.cuda.stream(stream):
                    ja = ctx.align_joint_async(Xd, **kw)
                ctx.synchronize()
                out += [ja.X.cpu().numpy(), ja.iterations.cpu().numpy(), ja.error.cpu().numpy()]
    finally:
        ctx.set_stream(None)
    return out


# ---- 1. all-ones weights ----
def test_all_ones_change_nothing(scene, all_kinds, stream):
    for kind in all_kinds:
        ctx = kind.ctx
        ctx.set_source_weights(None)
        plain = battery(kind, scene, stream)
        ctx.set_source_weights(np.ones(_n(ctx)))
        ones = battery(kind, scene, stream)
        ctx.set_source_weights(None)
        assert len(plain) == len(ones)
        for i, (a, b) in enumerate(zip(plain, ones)):
            assert np.array_equal(a, b), (kind.name, i)


# ---- 2. random weights: rows, sums, correspondences, model ----
def test_random_weights_scale_every_row(scene, all_kinds):
    s = scene
    worst = {}
    for kind in all_kinds:
        ctx = kind.ctx
        B = len(kind.clouds)
        T, T1 = s.poses(kind.clouds), s.poses(kind.clouds, 1)
        w = random_weights(_n(ctx), 17)
        for factor in _factors(kind):
            for robust, c in ROBUST:
                tag = (kind.name, factor, robust)
                args = dict(factor=factor, robust=robust, robust_c=c)
                ctx.set_source_weights(None)
                r0 = ctx.linearize_batch_points(T, **args)
                corr = ctx.correspondences_batch()
                _, pe0 = ctx.error_batch_points(T1)
                ctx.set_source_weights(w)
                r = ctx.linearize_batch_points(T, **args)
                assert _same(corr, ctx.correspondences_batch()) and np.array_equal(r.num_inliers, r0.num_inliers), tag
                e1, pe = ctx.error_batch_points(T1)
                assert np.array_equal(r.point_e, w * r0.point_e), tag
                assert np.array_equal(r.point_Hb42, w[:, None] * r0.point_Hb42), tag
                assert np.array_equal(pe, w * pe0), tag
                off = r.offsets
                for p in range(B):
                    rows = slice(off[p], off[p + 1])
                    e, H, b, wp = r.point_e[rows], r.point_H[rows], r.point_b[rows], w[rows]
                    if not e.any():
                        assert not r.H[p].any() and r.e[p] == 0 and e1[p] == 0, (tag, p)
                        continue
                    sums = NF.tight_ratios((H.sum(0), b.sum(0), e.sum()), (r.H[p], r.b[p], r.e[p]))
                    assert max(sums) <= NF.TIGHT and abs(pe[rows].sum() - e1[p]) <= NF.TIGHT * e1[p], (tag, p, sums)
                    if robust == 2:  # the model for Cauchy is checked unweighted by test_gpu_batch_points; one robust kernel suffices here
                        continue
                    em, Hm, bm, eem = model_member(kind, s, p, T[p], T1[p], corr[p], factor, robust, c)
                    rat = row_ratios(e, H, b, wp * em, wp[:, None, None] * Hm, wp[:, None] * bm)
                    ew = wp * eem
                    rerr = float((np.abs(pe[rows] - ew) / (ew + ew.mean())).max())
                    assert max(rat) <= NF.TIGHT and rerr <= NF.TIGHT, (tag, p, rat, rerr)
                    worst[kind.name] = max(worst.get(kind.name, 0.0), *rat, rerr, *sums)
        ctx.set_source_weights(None)
    print("worst (weighted rows vs model, rows summed vs member):", worst)


# ---- 3. weighted align_batch ----
@pytest.mark.parametrize("optimizer", [GN, LM])
def test_weighted_align_replays_the_reference_optimiser(scene, optimizer):
    s = scene
    ctx, rep = _kdtree(s), _kdtree(s)
    w = random_weights(_n(ctx), 23)
    ctx.set_source_weights(w)
    rep.set_source_weights(w)
    starts = s.poses(range(len(s.srcs)), 3)
    kw = {**DEFAULTS, "optimizer": optimizer, "robust": 1, "robust_c": 0.5}
    _, runs, _ = prefix_runs(ctx, starts, kw)
    stats = Stats()
    replay(runs, kw, rep, False, stats)
    print("worst step ratio (GN, LM):", stats.gn, stats.lm)
    ctx.set_source_weights(None)
    assert not all(np.array_equal(a, b) for a, b in zip(_align(runs[-1]), _align(ctx.align_batch(starts, **kw)))), "the weights had no effect"


def test_zero_weights_align_as_the_cloud_without_those_points(scene):
    s = scene
    rng = np.random.default_rng(29)
    keep = [rng.random(len(c)) >= 0.2 for c in s.srcs]
    ctx = _kdtree(s)
    ctx.set_source_weights(np.concatenate(keep).astype(np.float64))
    cut = _kdtree(s)
    cut.set_source_batch([c[k] for c, k in zip(s.srcs, keep)], [c[k] for c, k in zip(s.scovs, keep)])
    starts = s.poses(range(len(s.srcs)), 2)
    for kw in (dict(optimizer=LM), dict(optimizer=GN, robust=1, robust_c=0.5), dict(optimizer=LM, factor=0)):
        kw = dict(kw, rotation_eps=0.01 * np.pi / 180.0, translation_eps=1e-4)
        a, b = ctx.align_batch(starts, **kw), cut.align_batch(starts, **kw)
        assert np.array_equal(a.converged, b.converged), kw
        for m in range(len(s.srcs)):
            ang, tr = pose_error(a.T_target_source[m], b.T_target_source[m])
            assert ang <= 1e-4 and tr <= 1e-3, (kw, m, ang, tr)


# ---- 4. layout ----
def test_permuted_cloud_with_permuted_weights_gives_permuted_rows(scene):
    s = scene
    perm = np.random.default_rng(5).permutation(len(s.srcs[0]))
    ctx = _kdtree(s)
    w = random_weights(_n(ctx), 31)
    ctx.set_source_weights(w)
    one = _sg().Context(0)
    one.set_target(s.tp, s.tn, s.tcv)
    one.build_target_kdtree()
    one.set_source_batch([s.srcs[0][perm]], [s.scovs[0][perm]])
    n = len(perm)
    one.set_source_weights(w[:n][perm])
    T, T1 = s.poses([0]), s.poses([0], 1)
    for factor in (0, 1, 2):
        a = ctx.linearize_batch_points(np.repeat(T, len(s.srcs), 0), factor=factor, robust=1, robust_c=0.05)
        _, ae = ctx.error_batch_points(np.repeat(T1, len(s.srcs), 0))
        b = one.linearize_batch_points(T, factor=factor, robust=1, robust_c=0.05)
        _, be = one.error_batch_points(T1)
        assert np.array_equal(b.point_e, a.point_e[:n][perm]) and np.array_equal(b.point_Hb42, a.point_Hb42[:n][perm]), factor
        assert np.array_equal(be, ae[:n][perm]), factor


def test_member_independent_of_the_batch(scene):
    s = scene
    from small_gicp_b200.synthetic import make_world, sample_cloud

    filler = _p4(sample_cloud(make_world(50_000), 9000, 7) + OFFSET)
    fcov = _random_covs(np.random.default_rng(3), len(filler))
    X, Xc = s.srcs[0], s.scovs[0]
    wX = random_weights(len(X), 37)
    TX, TX1 = s.poses([0])[0], s.poses([0], 1)[0]
    ref = None
    for B, at in ((1, 0), (17, 9), (4096, 4000)):
        sizes = [(37 * j) % 200 + 1 for j in range(B)]
        starts = np.concatenate([[0], np.cumsum(sizes)]) % (len(filler) - 200)
        srcs = [filler[starts[j] : starts[j] + sizes[j]] for j in range(B)]
        covs = [fcov[starts[j] : starts[j] + sizes[j]] for j in range(B)]
        srcs[at], covs[at] = X, Xc
        ctx = _sg().Context(0)
        ctx.set_target(s.tp, s.tn, s.tcv)
        ctx.build_target_kdtree()
        ctx.set_source_batch(srcs, covs)
        w = random_weights(_n(ctx), B)
        w[ctx._batch_offsets[at] : ctx._batch_offsets[at + 1]] = wX
        ctx.set_source_weights(w)
        T = np.array([about(NF.box_centre(p), [0.001 * (j % 7), 0.0, -0.002, 0.03, -0.01 * (j % 3), 0.02]) for j, p in enumerate(srcs)])
        T1 = T.copy()
        T[at], T1[at] = TX, TX1
        got = []
        for factor in (0, 1, 2):
            r = ctx.linearize_batch_points(T, factor=factor, robust=2, robust_c=0.01)
            _, pe = ctx.error_batch_points(T1)
            rows = slice(r.offsets[at], r.offsets[at + 1])
            got += [r.H[at], r.b[at], r.e[at], r.point_e[rows].copy(), r.point_Hb42[rows].copy(), pe[rows].copy()]
        a = ctx.align_batch(T)
        got += [getattr(a, f)[at] for f in RESULT]
        if ref is None:
            ref = got
        assert _same(ref, got), B


def test_two_members_of_one_cloud_carry_their_own_weights(scene):
    s = scene
    n = len(s.srcs[0])
    wa, wb = random_weights(n, 41), random_weights(n, 43)
    ctx = _kdtree(s)
    ctx.set_source_pairs([0, 0])
    ctx.set_source_weights(np.concatenate([wa, wb]))
    T = np.concatenate([s.poses([0]), s.poses([0], 1)])
    r = ctx.linearize_batch_points(T, factor=2, robust=1, robust_c=0.05)
    al = ctx.align_batch(T)
    for p, wp in enumerate((wa, wb)):
        one = _kdtree(s)
        one.set_source_pairs([0])
        one.set_source_weights(wp)
        q = one.linearize_batch_points(T[p : p + 1], factor=2, robust=1, robust_c=0.05)
        rows = slice(p * n, (p + 1) * n)
        assert _same((q.H[0], q.b[0], q.e[0], q.num_inliers[0], q.point_e, q.point_Hb42),
                     (r.H[p], r.b[p], r.e[p], r.num_inliers[p], r.point_e[rows], r.point_Hb42[rows])), p
        b = one.align_batch(T[p : p + 1])
        assert all(np.array_equal(getattr(b, f)[0], getattr(al, f)[p]) for f in RESULT), p


# ---- 5. lifetime ----
def test_source_setters_clear_and_targets_keep_the_weights(scene):
    s = scene
    ctx = _sg().Context(0)
    ctx.build_target_kdtrees(s.maps, s.mnormals, s.mcovs)
    T = s.poses(range(len(s.srcs)))
    lists = [[0], [1], [2], [3], [4]]
    setters = {
        "batch": lambda: ctx.set_source_batch(s.srcs, s.scovs),
        "pairs": lambda: ctx.set_source_pairs(None, [0, 1, 2, 3, 4]),
        "submaps": lambda: ctx.set_source_submaps(lists),
        "points": lambda: (ctx.set_source(s.srcs[0], s.scovs[0]), ctx.set_source_batch(s.srcs, s.scovs)),
    }
    for name, setter in setters.items():
        ctx.set_source_batch(s.srcs, s.scovs)
        setter()
        ref = _lin(ctx, T)
        ctx.set_source_weights(random_weights(_n(ctx), 47))
        assert not _same(ref, _lin(ctx, T)), name
        setter()
        assert _same(ref, _lin(ctx, T)), name
    # after set_source the context holds no batch: the weights are gone with it
    ctx.set_source_batch(s.srcs, s.scovs)
    ctx.set_source_weights(np.ones(_n(ctx)))
    ctx.set_source(s.srcs[0], s.scovs[0])
    with pytest.raises(_sg().SgbError, match="holds no batch"):
        ctx.set_source_weights(np.ones(_n(ctx)))
    # a target rebuild and sgb_drop_seeds keep them
    for build in ("kdtree", "voxelmap"):
        k = _kdtree(s) if build == "kdtree" else _sg().Context(0)
        if build == "voxelmap":
            k.build_target_voxelmap(s.tp, s.tcv, 1.0, 7)
            k.set_source_batch(s.srcs, s.scovs)
        k.set_source_weights(random_weights(_n(k), 53))
        weighted = _lin(k, T)
        wal = _align(k.align_batch(T))
        if build == "kdtree":
            k.set_target(s.tp, s.tn, s.tcv)
            k.build_target_kdtree()
        else:
            k.build_target_voxelmap(s.tp, s.tcv, 1.0, 7)
        k.drop_seeds()
        assert _same(weighted, _lin(k, T)) and _same(wal, _align(k.align_batch(T))), build


def test_weights_set_again_between_async_calls_and_replays(scene, stream):
    torch = _torch()
    s = scene
    ctx = _kdtree(s)
    ctx.set_stream(stream.cuda_stream)
    T = s.poses(range(len(s.srcs)))
    Td = torch.from_numpy(np.ascontiguousarray(T)).cuda()
    ws = [random_weights(_n(ctx), 60 + k) for k in range(4)]

    def sync_ref(w):
        ctx.set_source_weights(w)
        return _align(ctx.align_batch(T))

    refs = [sync_ref(w) for w in ws]
    assert not _same(refs[0], refs[1])
    out = None
    for k in (0, 1, 0):
        ctx.set_source_weights(ws[k])
        with torch.cuda.stream(stream):
            out = ctx.align_batch_async(Td, out=out)
        ctx.synchronize()
        assert _same(refs[k], _async_host(out)), ("async", k)
    # torch.cuda.graph: captured once, the weights set again before each replay
    ctx.set_source_weights(ws[0])
    with torch.cuda.stream(stream):
        out = ctx.align_batch_async(Td, out=out)  # warm-up outside the capture
    stream.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        ctx.align_batch_async(Td, out=out)
    ctx.synchronize()
    for k in (2, 3, 2):
        ctx.set_source_weights(ws[k])
        with torch.cuda.stream(stream):
            g.replay()
        stream.synchronize()
        assert _same(refs[k], _async_host(out)), ("replay", k)
    ctx.set_stream(None)


def test_weights_set_again_between_joint_async_calls(all_kinds, stream):
    torch = _torch()
    kind = next(k for k in all_kinds if k.name == "pairs_maps")
    ctx = kind.ctx
    X = _joint_poses(5, 1)
    Xd = torch.from_numpy(X).cuda()
    ctx.set_stream(stream.cuda_stream)
    try:
        out = None
        for seed in (71, 72, 71):
            ctx.set_source_weights(random_weights(_n(ctx), seed))
            ref = ctx.align_joint(X)
            with torch.cuda.stream(stream):
                out = ctx.align_joint_async(Xd, out=out)
            ctx.synchronize()
            assert np.array_equal(ref.X, out.X.cpu().numpy()) and np.array_equal(ref.error, out.error.cpu().numpy()), seed
    finally:
        ctx.set_source_weights(None)
        ctx.set_stream(None)


# ---- 6. memory kinds ----
def test_device_and_page_locked_weights_equal_host_weights(scene, all_kinds):
    torch = _torch()
    s = scene
    for kind in all_kinds:
        ctx = kind.ctx
        T, T1 = s.poses(kind.clouds), s.poses(kind.clouds, 1)
        w = random_weights(_n(ctx), 83)
        ctx.set_source_weights(w)
        host = ctx.linearize_batch_points(T)
        _, host_pe = ctx.error_batch_points(T1)
        host_al = _align(ctx.align_batch(T))
        for wt in (torch.from_numpy(w).cuda(), torch.from_numpy(w).pin_memory()):
            ctx.set_source_weights(None)
            ctx.set_source_weights(wt)
            r = ctx.linearize_batch_points(T)
            _, pe = ctx.error_batch_points(T1)
            assert _same((host.H, host.b, host.e, host.point_e, host.point_Hb42, host_pe), (r.H, r.b, r.e, r.point_e, r.point_Hb42, pe)), kind.name
            assert _same(host_al, _align(ctx.align_batch(T))), kind.name
        ctx.set_source_weights(None)


# ---- 7. launch counts ----
def test_launch_counts(scene, all_kinds, stream):
    torch = _torch()
    s = scene
    for kind in all_kinds:
        ctx = kind.ctx
        T = s.poses(kind.clouds)
        Td = torch.from_numpy(np.ascontiguousarray(T)).cuda()
        active = np.arange(len(kind.clouds)) != 1
        ctx.set_stream(stream.cuda_stream)

        def async_align():
            with torch.cuda.stream(stream):
                ctx.align_batch_async(Td)
            ctx.synchronize()

        calls = (lambda: ctx.linearize_batch(T, active=active), lambda: ctx.linearize_batch_points(T, active=active),
                 lambda: ctx.error_batch(T, active=active), lambda: ctx.error_batch_points(T, active=active), lambda: ctx.align_batch(T), async_align)
        counts = []
        for weights in (None, np.ones(_n(ctx))):
            n0 = ctx.kernel_launches
            ctx.set_source_weights(weights)
            assert ctx.kernel_launches - n0 == (0 if weights is None else 1), kind.name
            for call in calls:
                call()  # once for any view rebuild or graph instantiation, then counted
                n0 = ctx.kernel_launches
                call()
                counts.append(ctx.kernel_launches - n0)
        assert counts[: len(calls)] == counts[len(calls) :], (kind.name, counts)
        ctx.set_source_weights(None)
        ctx.set_stream(None)


# ---- 8. misuse ----
def test_misuse_fails_with_a_message_and_keeps_the_weights(scene, stream):
    torch = _torch()
    sg = _sg()
    s = scene
    ctx = _kdtree(s)
    n = _n(ctx)
    T = s.poses(range(len(s.srcs)))
    w = random_weights(n, 89)
    ctx.set_source_weights(w)
    ref = _lin(ctx, T)

    def kept():
        assert _same(ref, _lin(ctx, T))

    with pytest.raises(sg.SgbError, match=r"need \(%d,\) weights" % n):
        ctx.set_source_weights(np.ones(n + 1))
    kept()
    for bad_row, bad in ((7, -1.0), (n - 1, np.nan), (0, np.inf), (1234, -np.inf), (5, -1e-300)):
        v = np.ones(n)
        v[bad_row] = bad
        v[bad_row + 1 :] = -2.0  # later rows fail too: the first one is named
        with pytest.raises(sg.SgbError, match=r"sgb_source_set_weights: the weight of row %d is " % bad_row):
            ctx.set_source_weights(v)
        kept()
        with pytest.raises(sg.SgbError, match=r"the weight of row %d is " % bad_row):
            ctx.set_source_weights(torch.from_numpy(v).cuda())
        kept()
    for wt in (torch.from_numpy(w).float().cuda(), torch.from_numpy(np.repeat(w, 2)).cuda()[::2]):
        with pytest.raises(sg.SgbError, match="contiguous float64"):
            ctx.set_source_weights(wt)
        kept()
    # inside a stream capture
    ctx.set_stream(stream.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with pytest.raises(sg.SgbError, match="being captured"):
        with torch.cuda.graph(g, stream=stream):
            ctx.set_source_weights(w[::-1].copy())
    torch.cuda.synchronize()
    ctx.set_stream(None)
    kept()
    # no batch: a fresh context, and one holding a single source
    fresh = sg.Context(0)
    with pytest.raises(sg.SgbError, match="holds no batch"):
        fresh.set_source_weights(np.ones(3))
    single = sg.Context(0)
    single.set_target(s.tp, s.tn, s.tcv)
    single.build_target_kdtree()
    single.set_source(s.srcs[0], s.scovs[0])
    with pytest.raises(sg.SgbError, match="holds no batch"):
        single.set_source_weights(None)
