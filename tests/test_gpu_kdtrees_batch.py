"""Batched registration over many kd-trees (sgb_target_build_kdtrees, Context.build_target_kdtrees, host_api.align_batch_pairs with
tree=TREE_DEVICE_KDTREE): member m against its own map m.  Every correspondence must pass the exhaustive exact search model of its own map
(np_search); every member's results must be bit-identical to a context that holds its map alone (sgb_target_set_points +
sgb_target_build_kdtree) and that member as a batch of one, and within TIGHT of the FP64 factor model; a member must not depend on the
rest of the batch, even at exact FP32 ties; the build's launch count must not depend on the map count; a round must take 3 / 2 launches;
and the misuses must fail with a message."""
import numpy as np
import pytest

import np_factors as NF
import np_search as NS
import oracle as O
from conftest import pose_error
from test_gpu_align_batch import _starts
from test_gpu_storage_model import OFFSET, _random_covs, _unit, about

pytestmark = pytest.mark.gpu

MAP_SIZES = [0, 1, 2, 31, 32, 33, 2048, 2049, 65537]
N_SRC = 3000
DUP = -1  # the map with duplicated points (exact FP32 distance ties) is the last one


def _sg():
    import small_gicp_b200 as sg

    return sg


def _p4(xyz):
    return np.c_[xyz, np.ones(len(xyz))]


def _n4(rng, n):
    return np.c_[_unit(rng, n), np.zeros(n)]


class Scene:
    """Maps drawn from regions of one synthetic world, shifted by OFFSET so that every map is centred far from the origin: the sizes of
    MAP_SIZES, two maps of one region sampled with two seeds (overlapping maps), and a map whose points each appear twice (exact ties).
    Random normals and covariances; one source per map, and a perturbed pose per member."""

    def __init__(self):
        from small_gicp_b200.synthetic import make_world, sample_cloud

        world = make_world(200_000)
        rng = np.random.default_rng(78)
        maps = [_p4(sample_cloud(world, n, 100 + j) + OFFSET) if n else np.zeros((0, 4)) for j, n in enumerate(MAP_SIZES)]
        for seed in (201, 202):
            p = sample_cloud(world, 60_000, seed)
            maps.append(_p4(p[(p[:, 0] < 20) & (p[:, 1] < 20)][:8000] + OFFSET))
        half = sample_cloud(world, 3000, 203) + OFFSET
        maps.append(_p4(np.r_[half, half[::-1]]))
        self.maps = maps
        self.normals = [_n4(rng, len(m)) for m in maps]
        self.covs = [_random_covs(rng, len(m)) for m in maps]
        self.srcs = [_p4(sample_cloud(world, N_SRC, 300 + j) + OFFSET) for j in range(len(maps))]
        self.scovs = [_random_covs(rng, N_SRC) for _ in maps]
        self.T = np.array([about(NF.box_centre(s), rng.uniform(-1, 1, 6) * [0.01, 0.01, 0.01, 0.1, 0.1, 0.1]) for s in self.srcs])
        self.trials = [np.array([T @ about(NF.box_centre(s), d) for T, s in zip(self.T, self.srcs)])
                       for d in ([0.002, -0.001, 0.003, 0.02, -0.01, 0.015], [-0.004, 0.002, 0.0, -0.03, 0.02, 0.0])]


@pytest.fixture(scope="module")
def scene():
    return Scene()


def _multi(s, pick=None, srcs=None, scovs=None):
    pick = list(range(len(s.maps))) if pick is None else pick
    ctx = _sg().Context(0)
    ctx.build_target_kdtrees([s.maps[k] for k in pick], [s.normals[k] for k in pick], [s.covs[k] for k in pick])
    ctx.set_source_batch(srcs if srcs is not None else [s.srcs[k] for k in pick], scovs if scovs is not None else [s.scovs[k] for k in pick])
    return ctx


def _single(s, m):
    ctx = _sg().Context(0)
    ctx.set_target(s.maps[m], s.normals[m], s.covs[m])
    ctx.build_target_kdtree()
    ctx.set_source_batch([s.srcs[m]], [s.scovs[m]])
    return ctx


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


# ---- 1. every correspondence against the exact search model of the member's own map ----
def test_every_query_against_its_own_map(scene):
    sg = _sg()
    s = scene
    ctx = _multi(s)
    assert ctx.target_size == sum(len(m) for m in s.maps)
    targets = [NS.Target(m) for m in s.maps]
    rep = NS.Report()
    # a perturbed pose and the converged one (from the batch's own align), unseeded and seeded, with and without a distance rejector
    conv = ctx.align_batch(s.T, factor=sg.FACTOR_GICP).T_target_source
    for T in (s.T, conv):
        for seeded in (False, True):
            for max_d in (1.0, None, 0.05):
                if not seeded:
                    ctx.drop_seeds()
                if max_d is None:
                    ctx.linearize_batch(T, factor=sg.FACTOR_ICP, rejector=sg.REJECT_NONE)
                else:
                    ctx.linearize_batch(T, factor=sg.FACTOR_ICP, rejector=sg.REJECT_DISTANCE, max_dist_sq=max_d)
                corr = ctx.correspondences_batch()
                for m, t in enumerate(targets):
                    c = corr[m]
                    assert ((c == NF.NO) | (c < max(t.n, 1))).all(), m  # never a point of another map
                    NS.check_correspondences(c, T[m], s.srcs[m], t, max_d, report=rep)
    print(f"many trees: {rep}")
    assert rep.worst_band <= 1.0


def test_overlapping_maps_stay_apart(scene):
    """two maps of one region: a member matches points of its own map only, even where the other map is nearer"""
    sg = _sg()
    s = scene
    a, b = len(s.maps) - 3, len(s.maps) - 2
    ctx = _multi(s, [a, b], srcs=[s.srcs[a], s.srcs[a]], scovs=[s.scovs[a], s.scovs[a]])
    ctx.linearize_batch(np.array([s.T[a], s.T[a]]), factor=sg.FACTOR_ICP, rejector=sg.REJECT_NONE)
    corr = ctx.correspondences_batch()
    for j, m in enumerate((a, b)):
        NS.check_correspondences(corr[j], s.T[a], s.srcs[a], NS.Target(s.maps[m]), None)
    assert not np.array_equal(corr[0], corr[1])


# ---- 2. every member bit-identical to its map alone, and the FP64 factor model ----
def test_members_equal_their_map_alone(scene):
    s = scene
    n = len(s.maps)
    ctx = _multi(s)
    refs = [_single(s, m) for m in range(n)]
    worst = 0.0
    for factor in (0, 1, 2):
        for robust, c in ((0, 1.0), (1, 0.3), (2, 0.5)):
            H, b, e, inl = ctx.linearize_batch(s.T, factor=factor, robust=robust, robust_c=c)
            corr = ctx.correspondences_batch()
            errs = [ctx.error_batch(T2) for T2 in s.trials]
            for m, r in enumerate(refs):
                if m == n + DUP:
                    continue  # exact ties: the single target's search may pick the other copy
                tag = (factor, robust, m)
                h1, b1, e1, i1 = r.linearize_batch(s.T[m : m + 1], factor=factor, robust=robust, robust_c=c)
                assert _same((H[m], b[m], e[m], inl[m]), (h1[0], b1[0], e1[0], i1[0])), tag
                assert np.array_equal(corr[m], r.correspondences_batch()[0]), tag
                for T2, eb in zip(s.trials, errs):
                    assert np.array_equal(eb[m], r.error_batch(T2[m : m + 1])[0]), tag
                if len(s.maps[m]) == 0:
                    assert (corr[m] == NF.NO).all() and not H[m].any() and e[m] == 0.0 and inl[m] == 0, tag
                    continue
                if (corr[m] == NF.NO).all():
                    assert not H[m].any(), tag
                    continue
                model = NF.storage_model(s.srcs[m], s.scovs[m], s.maps[m], s.normals[m], s.covs[m])
                rat = NF.tight_ratios((H[m], b[m], e[m]), NF.linearize(s.T[m], corr[m], factor, robust, c, *model))
                assert max(rat) <= NF.TIGHT, (tag, rat)
                worst = max(worst, max(rat))
                assert inl[m] == int((corr[m] != NF.NO).sum()), tag
    print(f"{n} maps, {ctx.target_size} points, worst TIGHT ratio {worst:.2e}")


# ---- 3. independence of the rest of the batch, exact ties included ----
def test_member_independent_of_the_batch(scene):
    s = scene
    n = len(s.maps)
    ctx = _multi(s)
    base = ctx.linearize_batch(s.T)
    base_corr = ctx.correspondences_batch()
    base_e = ctx.error_batch(s.trials[0])
    # permuted (maps with their members)
    perm = np.random.default_rng(5).permutation(n)
    pc = _multi(s, list(perm))
    got = pc.linearize_batch(s.T[perm])
    got_corr = pc.correspondences_batch()
    got_e = pc.error_batch(s.trials[0][perm])
    for j, k in enumerate(perm):
        assert _same([x[j] for x in got], [x[k] for x in base]), k
        assert np.array_equal(got_corr[j], base_corr[k]) and got_e[j] == base_e[k], k
    # other members inactive: the active ones unchanged, the inactive ones zero
    active = np.arange(n) % 2 == 0
    got = ctx.linearize_batch(s.T, active=active)
    for m in range(n):
        if active[m]:
            assert _same([x[m] for x in got], [x[m] for x in base]), m
        else:
            assert not got[0][m].any() and got[3][m] == 0, m
    # the duplicated-point map and the largest one in batches of 1, 3, 17 and 4096 pairs, at varying positions
    for m0 in (n + DUP, MAP_SIZES.index(65537)):
        ref = [x[m0] for x in base]
        for size in (1, 3, 17, 4096):
            pos = (size * 5) // 7
            pick = [(k * 7 + 3) % n for k in range(size)] if size < 4096 else [3] * size  # 4096: small fillers (map 3, 31 points)
            pick[pos] = m0
            srcs = [s.srcs[k] if k == m0 else s.srcs[k][:200] for k in pick]
            scovs = [s.scovs[k] if k == m0 else s.scovs[k][:200] for k in pick]
            c = _multi(s, pick, srcs, scovs)
            got = c.linearize_batch(s.T[pick])
            assert _same([x[pos] for x in got], ref), (m0, size)
            assert np.array_equal(c.correspondences_batch()[pos], base_corr[m0]), (m0, size)
            assert c.error_batch(s.trials[0][pick])[pos] == base_e[m0], (m0, size)


# ---- 4. batched align ----
ALIGN_CASES = [  # name, factor, robust, robust_c, optimizer, dof_mask
    ("GICP_GN", 2, 0, 1.0, 0, None),
    ("GICP_LM", 2, 0, 1.0, 1, None),
    ("GICP_LM_DOF", 2, 0, 1.0, 1, [1, 1, 0, 0, 1, 1]),
    ("HUBER_GICP_GN", 2, 1, 0.5, 0, None),
    ("HUBER_ICP_LM", 0, 1, 0.3, 1, None),
    ("CAUCHY_PLANE_ICP_GN", 1, 2, 0.5, 0, None),
]


@pytest.mark.parametrize("name,factor,robust,c,optimizer,dof_mask", ALIGN_CASES)
def test_align_members_equal_their_map_alone(scene, name, factor, robust, c, optimizer, dof_mask):
    s = scene
    kw = dict(factor=factor, robust=robust, robust_c=c, optimizer=optimizer, dof_mask=dof_mask)
    r = _multi(s).align_batch(s.T, **kw)
    for m in range(len(s.maps) + DUP):
        one = _single(s, m).align_batch(s.T[m : m + 1], **kw)
        for f in ("T_target_source", "converged", "iterations", "num_inliers", "error", "H", "b"):
            assert np.array_equal(getattr(r, f)[m], getattr(one, f)[0]), (name, m, f)
    print(f"{name}: iterations {r.iterations.tolist()}")


def test_golden_multi_start_against_the_oracle(golden_prepared):
    """GICP, 16 starts, each member holding its own copy of the golden target: the tolerances of test_gpu_align_batch"""
    g = golden_prepared
    tc, sc = g["target"], g["source"]
    starts = _starts()
    ctx = _sg().Context(0)
    ctx.build_target_kdtrees([tc.points] * len(starts), [tc.normals] * len(starts), [tc.covs] * len(starts))
    ctx.set_source_batch([sc.points] * len(starts), [sc.covs] * len(starts))
    for factor, optimizer in ((2, 1), (2, 0), (1, 1)):
        r = ctx.align_batch(starts, factor=factor, optimizer=optimizer)
        reg = O.Registration(factor=factor, num_threads=0)
        reg.set_optimizer(type=optimizer)
        worst = (0.0, 0.0)
        for m, T0 in enumerate(starts):
            ref = reg.align(tc, g["target_tree"], sc, T0)
            rot, trans = pose_error(ref.T_target_source, r.T_target_source[m])
            worst = (max(worst[0], rot), max(worst[1], trans))
            assert rot < 1e-4 and trans < 1e-3, (factor, optimizer, m, rot, trans)
            assert r.iterations[m] == ref.iterations, (factor, optimizer, m, r.iterations[m], ref.iterations)
            assert abs(r.num_inliers[m] - ref.num_inliers) <= 2, (factor, optimizer, m, r.num_inliers[m], ref.num_inliers)
        # the same as one tree and the members as a batch
        one = _sg().Context(0)
        one.set_target(tc.points, tc.normals, tc.covs)
        one.build_target_kdtree()
        one.set_source_batch([sc.points] * len(starts), [sc.covs] * len(starts))
        r1 = one.align_batch(starts, factor=factor, optimizer=optimizer)
        assert np.array_equal(r.T_target_source, r1.T_target_source) and np.array_equal(r.iterations, r1.iterations), (factor, optimizer)
        print(f"golden factor {factor} optimizer {optimizer} over 16 trees: worst vs oracle {worst[0]:.2e} rad / {worst[1]:.2e} m")


def test_host_mirror_equals_the_binding(scene):
    from small_gicp_b200 import host_api

    s = scene
    for kw in (dict(factor=2, optimizer=1), dict(factor=1, robust=2, robust_c=0.5, optimizer=0), dict(factor=0, robust=1, robust_c=0.5, optimizer=0,
                                                                                                     dof_mask=[1, 1, 0, 1, 1, 1])):
        h = host_api.align_batch_pairs(s.maps, s.srcs, s.covs, s.scovs, init_Ts=s.T, tree=host_api.TREE_DEVICE_KDTREE, target_normals=s.normals, **kw)
        r = _multi(s).align_batch(s.T, **kw)
        for f in ("T_target_source", "converged", "iterations", "num_inliers", "error", "H", "b"):
            assert np.array_equal(getattr(h, f), getattr(r, f)), (kw, f)


# ---- 5. launches ----
def test_build_launches_independent_of_map_count(scene):
    k = 3000  # points per map: above one shared-memory segment, so the build has a radix level
    pts, nrm, covs = scene.maps[8][:k], scene.normals[8][:k], scene.covs[8][:k]
    counts = {}
    for n_maps in (1, 64, 4096):
        ctx = _sg().Context(0)
        before = ctx.kernel_launches
        ctx.build_target_kdtrees([pts] * n_maps, [nrm] * n_maps, [covs] * n_maps)
        counts[n_maps] = ctx.kernel_launches - before
        assert ctx.target_size == k * n_maps
    assert len(set(counts.values())) == 1, counts
    print(f"build launches: {counts}")


def test_round_launches(scene):
    s = scene
    for pick in ([4, 5], list(range(len(s.maps)))):
        ctx = _multi(s, pick)
        T = s.T[pick]
        ctx.linearize_batch(T)
        before = ctx.kernel_launches
        ctx.linearize_batch(T)
        assert ctx.kernel_launches - before == 3, pick
        before = ctx.kernel_launches
        ctx.error_batch(T)
        assert ctx.kernel_launches - before == 2, pick


# ---- 6. errors and transitions ----
def test_errors_and_transitions(scene):
    sg = _sg()
    s = scene
    ctx = _multi(s, [4, 5, 6])
    ctx.linearize_batch(s.T[[4, 5, 6]])
    # member count != map count
    ctx.set_source_batch(s.srcs[:2], s.scovs[:2])
    for call in (lambda: ctx.linearize_batch(s.T[:2]), lambda: ctx.error_batch(s.T[:2]), lambda: ctx.align_batch(s.T[:2]),
                 lambda: ctx.correspondences_batch()):
        with pytest.raises(sg.SgbError, match="2 members but the target holds 3 kd-trees"):
            call()
    # the single-source calls and the single-tree calls on a forest, even of one map
    one = sg.Context(0)
    one.build_target_kdtrees(s.maps[6:7], s.normals[6:7], s.covs[6:7])
    one.set_source(s.srcs[6], s.scovs[6])
    buf = np.zeros(44)
    for call in (lambda: one.linearize(np.eye(4)), lambda: one.error(np.eye(4)), lambda: one.correspondences(), lambda: one.num_inliers(),
                 lambda: one.linearize_device(np.eye(4), buf.ctypes.data), lambda: one.error_device(np.eye(4), buf.ctypes.data)):
        with pytest.raises(sg.SgbError, match="kd-trees"):
            call()
    for call, msg in ((lambda: one.target_batch_knn(s.srcs[6][:10]), "kd-tree"), (lambda: one.estimate_target_features(), "kd-tree"),
                      (lambda: one.build_target_kdtree(), "many kd-trees"), (lambda: one.adopt_source_as_target(), "many kd-trees")):
        with pytest.raises(sg.SgbError, match=msg):
            call()
    # point-to-plane needs normals
    nn = sg.Context(0)
    nn.build_target_kdtrees(s.maps[6:7], None, s.covs[6:7])
    nn.set_source_batch(s.srcs[6:7], s.scovs[6:7])
    with pytest.raises(sg.SgbError, match="normals"):
        nn.linearize_batch(s.T[6:7], factor=sg.FACTOR_PLANE_ICP)
    # invalid builds
    c = sg.Context(0)
    with pytest.raises(sg.SgbError, match="offsets must be ascending"):
        c._check(c._L.sgb_target_build_kdtrees(c._h, 2, (sg.capi.C.c_size_t * 3)(0, 5, 3), s.maps[6].ctypes.data_as(sg.capi._dp), None, None))
    with pytest.raises(sg.SgbError, match="offsets\\[0\\] must be 0"):
        c._check(c._L.sgb_target_build_kdtrees(c._h, 1, (sg.capi.C.c_size_t * 2)(1, 5), s.maps[6].ctypes.data_as(sg.capi._dp), None, None))
    with pytest.raises(sg.SgbError, match="at most 65536"):
        c._check(c._L.sgb_target_build_kdtrees(c._h, 65537, (sg.capi.C.c_size_t * 65538)(), None, None, None))
    with pytest.raises(sg.SgbError, match="2\\^30"):
        c._check(c._L.sgb_target_build_kdtrees(c._h, 1, (sg.capi.C.c_size_t * 2)(0, 1 << 30), s.maps[6].ctypes.data_as(sg.capi._dp), None, None))
    # replacing the target in either direction drops the cached correspondences; a normal target works again
    ctx = _multi(s, [4, 5, 6])
    ctx.linearize_batch(s.T[[4, 5, 6]])
    ctx.error_batch(s.T[[4, 5, 6]])
    ctx.set_target(s.maps[6], s.normals[6], s.covs[6])
    ctx.build_target_kdtree()
    with pytest.raises(sg.SgbError, match="no preceding"):
        ctx.error_batch(s.T[[4, 5, 6]])
    ctx.linearize_batch(s.T[[4, 5, 6]])
    one.set_target(s.maps[6], s.normals[6], s.covs[6])
    one.build_target_kdtree()
    one.linearize(s.T[6])
    ctx.build_target_kdtrees([s.maps[k] for k in (4, 5, 6)], [s.normals[k] for k in (4, 5, 6)], [s.covs[k] for k in (4, 5, 6)])
    with pytest.raises(sg.SgbError, match="no preceding"):
        ctx.error_batch(s.T[[4, 5, 6]])
    assert all((c_ == sg.NO_CORRESPONDENCE).all() for c_ in ctx.correspondences_batch())
