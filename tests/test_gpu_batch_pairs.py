"""Batched registration over (cloud, map) pairs (sgb_source_set_pairs, Context.set_source_pairs) and the batched store of
sgb_source_set_batch.  The oracle is the repeat path: the same members built by uploading every member's cloud again
(set_source_batch([clouds[c_p] ...])) and, on a many-maps target, building every member's map again.  Every output -- linearize_batch,
error_batch, correspondences_batch, align_batch -- must be bit-identical to it, on every target kind; correspondences on many kd-trees
must pass the exact search model of the member's own map; the pairing must never go stale; the store must be bit-identical to
sgb_source_set_points of each cloud alone; the launch counts must not depend on the cloud or member count; misuse fails with a message."""
import numpy as np
import pytest

import np_factors as NF
import np_search as NS
from test_gpu_storage_model import OFFSET, _random_covs, _unit, about

pytestmark = pytest.mark.gpu

CLOUD_SIZES = [3000, 0, 1500, 2049, 700, 2500]
MAP_SIZES = [8000, 0, 5000, 3000, 6000]
ROBUST = [(0, 1.0), (1, 0.5), (2, 0.5)]  # none, Huber, Cauchy
GN, LM = 0, 1  # sgb_optimizer_kind


def _sg():
    import small_gicp_b200 as sg

    return sg


def _p4(xyz):
    return np.c_[xyz, np.ones(len(xyz))]


class Scene:
    def __init__(self):
        from small_gicp_b200.synthetic import make_world, sample_cloud

        world = make_world(200_000)
        rng = np.random.default_rng(91)
        self.maps = [_p4(sample_cloud(world, n, 10 + j) + OFFSET) if n else np.zeros((0, 4)) for j, n in enumerate(MAP_SIZES)]
        self.normals = [np.c_[_unit(rng, len(m)), np.zeros(len(m))] for m in self.maps]
        self.covs = [_random_covs(rng, len(m)) for m in self.maps]
        self.clouds = [_p4(sample_cloud(world, n, 50 + j) + OFFSET) if n else np.zeros((0, 4)) for j, n in enumerate(CLOUD_SIZES)]
        self.scovs = [_random_covs(rng, len(c)) for c in self.clouds]
        self.centres = [NF.box_centre(c) if len(c) else OFFSET for c in self.clouds]
        # one tie-free target of random points for the single kd-tree, and its voxel map
        self.single = _p4(rng.uniform(-30, 30, (200_000, 3)) + OFFSET)
        self.single_n = np.c_[_unit(rng, len(self.single)), np.zeros(len(self.single))]
        self.single_c = _random_covs(rng, len(self.single))

    def poses(self, cl, k=0):
        """a distinct perturbed pose per member (member p of cloud c), about the cloud's centre"""
        return np.array([about(self.centres[c], [0.003 * ((p + k) % 5) - 0.006, 0.002 * (p % 3), -0.002, 0.04 * ((p + k) % 4) - 0.06, 0.02, -0.03])
                         for p, c in enumerate(cl)])


@pytest.fixture(scope="module")
def scene():
    return Scene()


def _target(ctx, s, kind, maps=None):
    """the whole target (maps = None) or the repeat path's maps[t_p] ... (many maps only)"""
    pick = list(range(len(s.maps))) if maps is None else list(maps)
    if kind == "trees":
        ctx.build_target_kdtrees([s.maps[t] for t in pick], [s.normals[t] for t in pick], [s.covs[t] for t in pick])
    elif kind == "voxelmaps":
        ctx.build_target_voxelmaps([s.maps[t] for t in pick], [s.covs[t] for t in pick], leaf_size=0.5)
    elif kind == "tree":
        ctx.set_target(s.single, s.single_n, s.single_c)
        ctx.build_target_kdtree()
    else:
        ctx.build_target_voxelmap(s.single, s.single_c, 0.5)


def _paired(s, kind, cl, mp):
    ctx = _sg().Context(0)
    _target(ctx, s, kind)
    ctx.set_source_batch(s.clouds, s.scovs)
    ctx.set_source_pairs(cl, mp)
    return ctx


def _repeat(s, kind, cl, mp):
    ctx = _sg().Context(0)
    _target(ctx, s, kind, mp)
    ctx.set_source_batch([s.clouds[c] for c in cl], [s.scovs[c] for c in cl])
    return ctx


def _outputs(ctx, s, cl, factor, robust, c, align=True):
    """everything a batch computes, as a list of arrays"""
    sg = _sg()
    T = s.poses(cl)
    out = list(ctx.linearize_batch(T, factor=factor, robust=robust, robust_c=c))
    out += ctx.correspondences_batch()
    out += [ctx.error_batch(s.poses(cl, k)) for k in (1, 2)]
    if align:
        for opt in (GN, LM):
            dof = [1, 1, 0, 1, 1, 1] if opt == GN else None
            r = ctx.align_batch(T, factor=factor, robust=robust, robust_c=c, optimizer=opt, dof_mask=dof)
            out += [r.T_target_source, r.converged, r.iterations, r.num_inliers, r.error, r.H, r.b]
        out += ctx.correspondences_batch()
    return out


def _equal(a, b, tag):
    assert len(a) == len(b), tag
    for k, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape and np.array_equal(x, y), (tag, k)


# (cloud, map) pairings over 6 clouds (cloud 1 empty) and 5 maps (map 1 empty)
PAIRINGS = {
    "mixed_P_gt_N": [(0, 0), (0, 2), (2, 2), (3, 2), (5, 4), (1, 3), (0, 1)],  # cloud 0 thrice, 4 never; map 2 thrice
    "few_P_lt_N": [(3, 4), (2, 4), (4, 0), (0, 4)],  # maps 1, 2, 3 unused
    "reversed": [(k, 4 - k) for k in range(5)],
    "all_on_last": [(c, 4) for c in range(6)],
    "one_cloud_every_map": [(0, t) for t in range(5)],
}
TREE_CASES = [(f, r, c) for f in (0, 1, 2) for r, c in ROBUST]
VOXEL_CASES = [(f, r, c) for f in (0, 2) for r, c in ROBUST]


@pytest.mark.parametrize("factor,robust,c", TREE_CASES)
def test_many_trees_equal_the_repeat_path(scene, factor, robust, c):
    for name, pairs in PAIRINGS.items():
        cl, mp = [p[0] for p in pairs], [p[1] for p in pairs]
        _equal(_outputs(_paired(scene, "trees", cl, mp), scene, cl, factor, robust, c),
               _outputs(_repeat(scene, "trees", cl, mp), scene, cl, factor, robust, c), (name, factor, robust))


@pytest.mark.parametrize("factor,robust,c", VOXEL_CASES)
def test_many_voxelmaps_equal_the_repeat_path(scene, factor, robust, c):
    for name, pairs in PAIRINGS.items():
        cl, mp = [p[0] for p in pairs], [p[1] for p in pairs]
        _equal(_outputs(_paired(scene, "voxelmaps", cl, mp), scene, cl, factor, robust, c),
               _outputs(_repeat(scene, "voxelmaps", cl, mp), scene, cl, factor, robust, c), (name, factor, robust))


@pytest.mark.parametrize("kind", ["tree", "voxelmap"])
def test_multi_start_on_one_target_equals_the_repeat_path(scene, kind):
    """maps = None on one target: S copies of a cloud, each from its own start; the same member order gives the same virtual source"""
    for cl in ([0, 0, 0, 0, 2, 5, 5, 1, 3], [4], [3, 2, 0]):
        for factor in ((0, 2) if kind == "voxelmap" else (0, 1, 2)):
            _equal(_outputs(_paired(scene, kind, cl, None), scene, cl, factor, 1, 0.5),
                   _outputs(_repeat(scene, kind, cl, None), scene, cl, factor, 1, 0.5), (kind, cl, factor))


def test_own_map_search(scene):
    """on many kd-trees every correspondence of a pair member is an exact nearest neighbour in its own map"""
    sg = _sg()
    cl, mp = zip(*PAIRINGS["mixed_P_gt_N"])
    ctx = _paired(scene, "trees", list(cl), list(mp))
    T = scene.poses(cl)
    rep = NS.Report()
    for max_d in (1.0, None):
        if max_d is None:
            ctx.linearize_batch(T, factor=sg.FACTOR_ICP, rejector=sg.REJECT_NONE)
        else:
            ctx.linearize_batch(T, factor=sg.FACTOR_ICP, max_dist_sq=max_d)
        for p, corr in enumerate(ctx.correspondences_batch()):
            t = NS.Target(scene.maps[mp[p]])
            assert ((corr == NF.NO) | (corr < max(t.n, 1))).all(), p
            NS.check_correspondences(corr, T[p], scene.clouds[cl[p]], t, max_d, report=rep)
    assert rep.worst_band <= 1.0


def test_repairing_and_target_changes_never_go_stale(scene):
    sg = _sg()
    first, second = PAIRINGS["mixed_P_gt_N"], PAIRINGS["reversed"]
    cl2, mp2 = [p[0] for p in second], [p[1] for p in second]
    fresh = _outputs(_paired(scene, "trees", cl2, mp2), scene, cl2, 2, 0, 1.0)
    # pairing twice: the second pairing's results, as a fresh context gives them
    ctx = _paired(scene, "trees", [p[0] for p in first], [p[1] for p in first])
    _outputs(ctx, scene, [p[0] for p in first], 2, 0, 1.0, align=False)
    ctx.set_source_pairs(cl2, mp2)
    _equal(_outputs(ctx, scene, cl2, 2, 0, 1.0), fresh, "re-paired")
    # another target with other maps after the pairing (the view is rebuilt)
    other = [4, 3, 2, 0, 1]
    ctx.build_target_kdtrees([scene.maps[t] for t in other], [scene.normals[t] for t in other], [scene.covs[t] for t in other])
    ref = _sg().Context(0)
    ref.build_target_kdtrees([scene.maps[t] for t in other], [scene.normals[t] for t in other], [scene.covs[t] for t in other])
    ref.set_source_batch(scene.clouds, scene.scovs)
    ref.set_source_pairs(cl2, mp2)
    _equal(_outputs(ctx, scene, cl2, 2, 0, 1.0), _outputs(ref, scene, cl2, 2, 0, 1.0), "rebuilt target")
    # set_source_batch forgets the pairing: member m against map m again
    ctx.set_source_batch(scene.clouds[:5], scene.scovs[:5])
    ref2 = _sg().Context(0)
    ref2.build_target_kdtrees([scene.maps[t] for t in other], [scene.normals[t] for t in other], [scene.covs[t] for t in other])
    ref2.set_source_batch(scene.clouds[:5], scene.scovs[:5])
    _equal(_outputs(ctx, scene, range(5), 2, 0, 1.0), _outputs(ref2, scene, range(5), 2, 0, 1.0), "identity again")


def test_pair_order_and_inactive_members(scene):
    """permuting the pair list permutes every output bit for bit; inactive members change nothing for the others"""
    sg = _sg()
    pairs = PAIRINGS["mixed_P_gt_N"]
    perm = [3, 6, 0, 5, 1, 4, 2]
    cl, mp = [p[0] for p in pairs], [p[1] for p in pairs]
    a = _paired(scene, "voxelmaps", cl, mp)
    b = _paired(scene, "voxelmaps", [cl[k] for k in perm], [mp[k] for k in perm])
    T = scene.poses(cl)
    H, bb, e, inl = a.linearize_batch(T, factor=sg.FACTOR_GICP)
    H2, bb2, e2, inl2 = b.linearize_batch(T[perm], factor=sg.FACTOR_GICP)
    for x, y in ((H, H2), (bb, bb2), (e, e2), (inl, inl2)):
        assert np.array_equal(x[perm], y)
    ca, cb = a.correspondences_batch(), b.correspondences_batch()
    assert all(np.array_equal(ca[perm[k]], cb[k]) for k in range(len(perm)))
    ra = a.align_batch(T, factor=sg.FACTOR_GICP)
    rb = b.align_batch(T[perm], factor=sg.FACTOR_GICP)
    assert np.array_equal(ra.T_target_source[perm], rb.T_target_source) and np.array_equal(ra.iterations[perm], rb.iterations)
    active = np.array([1, 0, 1, 0, 1, 1, 0], dtype=bool)
    Hx, bx, ex, ix = a.linearize_batch(T, active=active, factor=sg.FACTOR_GICP)
    assert np.array_equal(Hx[active], H[active]) and np.array_equal(ex[active], e[active]) and not Hx[~active].any()


@pytest.mark.parametrize("n_clouds", [1, 3, 17, 4096])
def test_batched_store_equals_set_points(n_clouds):
    """each stored cloud is sgb_source_set_points of it alone: correspondences bit-identical to the single-source context; sums
    bit-identical to the same cloud stored with a batch of one; clouds of 0 - 65537 points, UTM-scale coordinates, duplicated points"""
    sg = _sg()
    rng = np.random.default_rng(n_clouds)
    utm = np.array([512_345.0, 5_412_678.0, 210.0])
    sizes_all = [0, 1, 2, 31, 128, 129, 2049, 65537]
    sizes = sizes_all if n_clouds == 17 else ([5] * n_clouds if n_clouds == 4096 else list(rng.choice(sizes_all, n_clouds)))
    if n_clouds == 17:
        sizes = (sizes * 3)[:17]
    tgt = _p4(rng.uniform(-20, 20, (100_000, 3)) + utm)
    tcv = _random_covs(rng, len(tgt))
    clouds, covs = [], []
    for k, n in enumerate(sizes):
        p = rng.uniform(-15, 15, (n, 3)) + utm
        if k % 3 == 2 and n > 1:
            p[n // 2:] = p[: n - n // 2]  # duplicated points
        clouds.append(_p4(p))
        covs.append(_random_covs(rng, n))
    T = np.array([about(NF.box_centre(c) if len(c) else utm, [0.002, -0.001, 0.001, 0.05, -0.02, 0.01]) for c in clouds])
    for with_covs in (True, False):
        factor = sg.FACTOR_GICP if with_covs else sg.FACTOR_ICP
        ctx = sg.Context(0)
        ctx.set_target(tgt, None, tcv)
        ctx.build_target_kdtree()
        ctx.set_source_batch(clouds, covs if with_covs else None)
        H, b, e, _ = ctx.linearize_batch(T, factor=factor)
        corr = ctx.correspondences_batch()
        one = sg.Context(0)
        one.set_target(tgt, None, tcv)
        one.build_target_kdtree()
        single = sg.Context(0)
        single.set_target(tgt, None, tcv)
        single.build_target_kdtree()
        check = range(len(clouds)) if n_clouds < 4096 else range(0, 4096, 511)
        for k in check:
            one.set_source_batch([clouds[k]], [covs[k]] if with_covs else None)
            H1, b1, e1, _ = one.linearize_batch(T[k:k + 1], factor=factor)
            assert np.array_equal(H1[0], H[k]) and np.array_equal(b1[0], b[k]) and e1[0] == e[k], (k, with_covs)
            if len(clouds[k]):
                single.set_source(clouds[k], covs[k] if with_covs else None)
                single.linearize(T[k], factor=factor)
                assert np.array_equal(single.correspondences(), corr[k]), (k, with_covs)


def test_launch_counts(scene):
    sg = _sg()
    rng = np.random.default_rng(5)
    counts = {}
    for n in (1, 64, 4096):
        ctx = sg.Context(0)
        clouds = [_p4(rng.uniform(-5, 5, (20, 3))) for _ in range(n)]
        before = ctx.kernel_launches
        ctx.set_source_batch(clouds, [_random_covs(rng, 20) for _ in range(n)])
        counts[n] = ctx.kernel_launches - before
    assert len(set(counts.values())) == 1, counts
    pair_counts = {}
    ctx = sg.Context(0)
    ctx.set_source_batch([_p4(rng.uniform(-5, 5, (4, 3))) for _ in range(3)])
    for P in (1, 64, 65536):
        before = ctx.kernel_launches
        ctx.set_source_pairs(np.arange(P) % 3, None)
        pair_counts[P] = ctx.kernel_launches - before
    assert len(set(pair_counts.values())) == 1, pair_counts
    # rounds: the same launches as without pairs, plus one view launch after a pairing or target change
    cl, mp = zip(*PAIRINGS["mixed_P_gt_N"])
    T = scene.poses(cl)
    for kind, lin, err in (("trees", 3, 2), ("voxelmaps", 2, 2)):
        ctx = _paired(scene, kind, list(cl), list(mp))
        before = ctx.kernel_launches
        ctx.linearize_batch(T, factor=sg.FACTOR_ICP)
        assert ctx.kernel_launches - before == lin + 1, kind
        for expect, call in ((lin, lambda: ctx.linearize_batch(T, factor=sg.FACTOR_ICP)), (err, lambda: ctx.error_batch(T))):
            before = ctx.kernel_launches
            call()
            assert ctx.kernel_launches - before == expect, kind
    for kind, lin, err in (("tree", 5, 2), ("voxelmap", 2, 2)):
        ctx = _paired(scene, kind, [0, 0, 3], None)
        T3 = scene.poses([0, 0, 3])
        ctx.linearize_batch(T3, factor=sg.FACTOR_ICP)
        before = ctx.kernel_launches
        ctx.linearize_batch(T3, factor=sg.FACTOR_ICP)
        assert ctx.kernel_launches - before == lin, kind
        before = ctx.kernel_launches
        ctx.error_batch(T3)
        assert ctx.kernel_launches - before == err, kind


def test_large_pairing_of_small_clouds():
    """P = 65536 members of small clouds, each against its own map: bit-identical to the repeat path"""
    sg = _sg()
    rng = np.random.default_rng(7)
    clouds = [_p4(rng.uniform(-3, 3, (int(n), 3)) + OFFSET) for n in rng.integers(0, 9, 300)]
    maps = [_p4(rng.uniform(-3, 3, (int(n), 3)) + OFFSET) for n in rng.integers(0, 40, 200)]
    P = 65536
    cl, mp = rng.integers(0, len(clouds), P), rng.integers(0, len(maps), P)
    T = np.array([about(OFFSET, [0.0, 0.0, 0.01 * (p % 7), 0.02 * (p % 5), 0.0, 0.01]) for p in range(P)])
    a = sg.Context(0)
    a.build_target_kdtrees(maps)
    a.set_source_batch(clouds)
    a.set_source_pairs(cl, mp)
    b = sg.Context(0)
    b.build_target_kdtrees([maps[t] for t in mp])
    b.set_source_batch([clouds[c] for c in cl])
    for ctx in (a, b):
        ctx.out = list(ctx.linearize_batch(T, factor=sg.FACTOR_ICP)) + [np.concatenate(ctx.correspondences_batch())]
        r = ctx.align_batch(T, factor=sg.FACTOR_ICP, optimizer=GN, max_iterations=5)
        ctx.out += [r.T_target_source, r.iterations]
    _equal(a.out, b.out, "65536 members")


def test_misuse_fails_with_a_message(scene):
    sg = _sg()
    ctx = sg.Context(0)
    with pytest.raises(sg.SgbError, match="no batch"):
        ctx._check(ctx._L.sgb_source_set_pairs(ctx._h, 0, None, None))
    _target(ctx, scene, "trees")
    ctx.set_source_batch(scene.clouds, scene.scovs)
    with pytest.raises(sg.SgbError, match="member 2 names cloud 6 but the batch holds 6 clouds"):
        ctx.set_source_pairs([0, 1, 6], [0, 0, 0])
    with pytest.raises(sg.SgbError, match="must equal the cloud count"):
        ctx.set_source_pairs(None, [0, 1, 2])
    with pytest.raises(sg.SgbError, match="at most 65536"):
        ctx.set_source_pairs(np.zeros(65537, dtype=np.uint32), None)
    with pytest.raises(sg.SgbError, match="too many member points"):
        big = sg.Context(0)
        big.set_source_batch([np.zeros((40_000, 4))])
        big.set_source_pairs(np.zeros(60_000, dtype=np.uint32), None)
    cl, mp = [0, 2, 3], [0, 4, 3]
    ctx.set_source_pairs(cl, mp)
    ctx.linearize_batch(scene.poses(cl), factor=sg.FACTOR_ICP)
    # a target with fewer maps after the pairing: caught at the call
    ctx.build_target_kdtrees(scene.maps[:4], scene.normals[:4], scene.covs[:4])
    with pytest.raises(sg.SgbError, match="member 1 is paired with map 4 but the target holds 4 maps"):
        ctx.linearize_batch(scene.poses(cl), factor=sg.FACTOR_ICP)
    with pytest.raises(sg.SgbError, match="member 1 is paired with map 4"):
        ctx.align_batch(scene.poses(cl), factor=sg.FACTOR_ICP)
    # a maps table on one target
    ctx.set_target(scene.single, scene.single_n, scene.single_c)
    ctx.build_target_kdtree()
    with pytest.raises(sg.SgbError, match="not a many-maps or many-kd-trees target"):
        ctx.linearize_batch(scene.poses(cl), factor=sg.FACTOR_ICP)
    # without a maps table: members == maps, as without pairs
    _target(ctx, scene, "voxelmaps")
    ctx.set_source_pairs([0, 0], None)
    with pytest.raises(sg.SgbError, match="2 members but the target holds 5 voxel maps"):
        ctx.linearize_batch(scene.poses([0, 0]), factor=sg.FACTOR_ICP)
    # an empty pairing is an empty batch
    ctx.set_source_pairs([], [])
    H, _, _, _ = ctx.linearize_batch(np.zeros((0, 4, 4)), factor=sg.FACTOR_ICP)
    assert H.shape == (0, 6, 6)


def test_host_mirror_matches_the_binding(scene):
    """BatchRegistration's pair-list and multi-start overloads (host_api) against Context.set_source_pairs + align_batch, bit for bit"""
    from small_gicp_b200 import host_api

    sg = _sg()
    cl, mp = [list(x) for x in zip(*PAIRINGS["mixed_P_gt_N"])]
    T = scene.poses(cl)
    kw = dict(factor=sg.FACTOR_GICP, optimizer=LM)
    for tree, kind, extra in ((host_api.TREE_DEVICE_KDTREE, "trees", {"target_normals": scene.normals}),
                              (host_api.TREE_VOXELMAP, "voxelmaps", {"voxel_resolution": 0.5})):
        h = host_api.align_batch_pairs(scene.maps, scene.clouds, scene.covs, scene.scovs, init_Ts=T, tree=tree, pairs=list(zip(cl, mp)), **extra, **kw)
        ctx = _paired(scene, kind, cl, mp)
        r = ctx.align_batch(T, **kw)
        assert np.array_equal(h.T_target_source, r.T_target_source) and np.array_equal(h.iterations, r.iterations), kind
        assert np.array_equal(h.H, r.H) and np.array_equal(h.error, r.error), kind
    starts = [0, 0, 3, 5, 5, 5]
    T = scene.poses(starts)
    h = host_api.align_batch(scene.single, scene.clouds, scene.single_n, scene.single_c, scene.scovs, init_Ts=T, tree=host_api.TREE_DEVICE_KDTREE,
                             cloud_of_member=starts, **kw)
    ctx = _paired(scene, "tree", starts, None)
    r = ctx.align_batch(T, **kw)
    assert np.array_equal(h.T_target_source, r.T_target_source) and np.array_equal(h.iterations, r.iterations)
