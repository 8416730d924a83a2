"""Submap members (sgb_source_set_submaps, Context.set_source_submaps): a stored cloud against the union of several maps of a
many-kd-trees target, each placed by its own rigid pose and none of them transformed.

  * a one-entry list at the identity is sgb_source_set_pairs with that map, bit for bit; at a pose P it is the pair member at P^-1 T;
  * every correspondence of every member passes the union search model (np_submaps.check_union): the nearest over the entries, each
    searched with its own FP32 query; an exact tie goes to the earlier entry;
  * H | b | e | inliers and error() match the FP64 storage model evaluated per entry at the relative pose, over the GPU's own
    correspondences, to np_factors.TIGHT;
  * the same member against ONE kd-tree built over the placed union (points and covariances carried into the common frame on the host)
    gives the same sums to the FP32 storage tolerance and the same converged poses and iteration counts;
  * a member's results do not depend on the other members, their order or their lists; re-pairing, pose changes and target rebuilds
    never leave anything stale; the launch counts equal the pairs path; misuse fails with a message and leaves the context usable;
  * the golden pair with its target cut into three posed maps agrees with the CPU oracle's GICP on the placed union; the C++ mirror's
    overload equals the binding."""
import numpy as np
import pytest

import np_factors as NF
import np_search as NS
import np_submaps as SM
from test_gpu_storage_model import OFFSET, _random_covs, about

pytestmark = pytest.mark.gpu

MAP_SIZES = [8000, 0, 5000, 3000, 6000, 1, 31, 32, 33, 2049, 65537]
CLOUD_SIZES = [3000, 0, 1500, 2049]
ROBUST = [(0, 1.0), (1, 0.5), (2, 0.5)]  # none, Huber, Cauchy
GN, LM = 0, 1
HIGH = np.uint64(32)


def _sg():
    import small_gicp_b200 as sg

    return sg


def _p4(xyz):
    return np.c_[xyz, np.ones(len(xyz))]


def _apply(T, p):
    return _p4(p[:, :3] @ T[:3, :3].T + T[:3, 3])


class Scene:
    """clouds and maps sampled from one world (so that they overlap in the common frame); map k is handed over in a frame of its own,
    P_k^-1 of its common-frame points, with a far-away frame for some"""

    def __init__(self):
        from small_gicp_b200.synthetic import make_world, sample_cloud

        world = make_world(200_000)
        rng = np.random.default_rng(17)
        self.P = [about(OFFSET, np.r_[rng.uniform(-0.4, 0.4, 3), rng.uniform(-3, 3, 3)]) for _ in MAP_SIZES]
        self.P[2] = self.P[2] @ about(np.zeros(3), [0, 0, 0.3, 5000.0, -3000.0, 100.0])  # map 2's own frame is far from the origin
        common = [_p4(sample_cloud(world, n, 10 + j) + OFFSET) if n else np.zeros((0, 4)) for j, n in enumerate(MAP_SIZES)]
        self.maps = [_apply(SM.inverse(P), c) for P, c in zip(self.P, common)]
        self.covs = [_random_covs(rng, len(m)) for m in self.maps]
        self.clouds = [_p4(sample_cloud(world, n, 50 + j) + OFFSET) if n else np.zeros((0, 4)) for j, n in enumerate(CLOUD_SIZES)]
        self.scovs = [_random_covs(rng, len(c)) for c in self.clouds]
        self.centres = [NF.box_centre(c) if len(c) else OFFSET for c in self.clouds]
        self.targets = [NS.Target(m) for m in self.maps]
        # a map far from everything: its tree is never entered past the root
        self.far = len(self.maps)
        self.maps.append(_p4(rng.uniform(-5, 5, (4000, 3)) + OFFSET + [900.0, 0.0, 0.0]))
        self.covs.append(_random_covs(rng, 4000))
        self.P.append(np.eye(4))
        self.targets.append(NS.Target(self.maps[-1]))

    def poses(self, cl, k=0):
        return np.array([about(self.centres[c], [0.003 * ((p + k) % 5) - 0.006, 0.002 * (p % 3), -0.002, 0.04 * ((p + k) % 4) - 0.06, 0.02, -0.03])
                         for p, c in enumerate(cl)])

    def context(self, maps=None):
        ctx = _sg().Context(0)
        pick = range(len(self.maps)) if maps is None else maps
        ctx.build_target_kdtrees([self.maps[t] for t in pick], None, [self.covs[t] for t in pick])
        ctx.set_source_batch(self.clouds, self.scovs)
        return ctx

    def submaps(self, ctx, cl, lists, poses=None):
        ctx.set_source_submaps(lists, [[self.P[k] for k in l] for l in lists] if poses is None else poses, cl)


@pytest.fixture(scope="module")
def scene():
    return Scene()


# members over 4 clouds (cloud 1 empty): lists of 1, 2, 5 and 33 entries, overlapping maps, map 0 twice (the second time misplaced),
# the empty map, an empty list, the far map, the one-point map
CL = [0, 2, 3, 0, 1, 2, 3]
LISTS = [[0], [2, 0], [4, 1, 0, 3, 2], [0, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11] * 3, [0, 2], [], [11, 5, 1]]


def _poses_of(s, lists):
    out = [[s.P[k] for k in l] for l in lists]
    out[3] = [P if j < 11 else P @ about(OFFSET, [0.0, 0.0, 0.002 * j, 0.05, 0.0, -0.01 * (j % 3)]) for j, P in enumerate(out[3])]
    return out


def _low(corr):
    return [np.where(c == NF.NO, c, c & SM.LOW) for c in corr]


def _outputs(ctx, T, T1, T2, factor, robust, c, low=False):
    out = list(ctx.linearize_batch(T, factor=factor, robust=robust, robust_c=c))
    corr = ctx.correspondences_batch()
    out += _low(corr) if low else corr
    out += [ctx.error_batch(T1), ctx.error_batch(T2)]
    for opt in (GN, LM):
        r = ctx.align_batch(T, factor=factor, robust=robust, robust_c=c, optimizer=opt)
        out += [r.T_target_source, r.converged, r.iterations, r.num_inliers, r.error, r.H, r.b]
    return out


@pytest.mark.parametrize("factor", [0, 2])
@pytest.mark.parametrize("robust,c", ROBUST)
def test_one_identity_entry_is_the_pair(scene, factor, robust, c):
    cl, mp = [0, 2, 3, 0, 1, 3], [0, 2, 4, 1, 3, 9]
    T, T1, T2 = scene.poses(cl), scene.poses(cl, 1), scene.poses(cl, 2)
    a = scene.context()
    a.set_source_submaps([[m] for m in mp], None, cl)
    b = scene.context()
    b.set_source_pairs(cl, mp)
    oa, ob = _outputs(a, T, T1, T2, factor, robust, c, low=True), _outputs(b, T, T1, T2, factor, robust, c)
    assert len(oa) == len(ob)
    for k, (x, y) in enumerate(zip(oa, ob)):
        assert x.shape == y.shape and np.array_equal(x, y), (factor, robust, k)


def test_one_posed_entry_is_the_pair_at_the_relative_pose(scene):
    sg = _sg()
    cl, mp = [0, 2, 3], [0, 2, 4]
    T = scene.poses(cl)
    a = scene.context()
    scene.submaps(a, cl, [[m] for m in mp])
    b = scene.context()
    b.set_source_pairs(cl, mp)
    Tb = np.array([SM.relative(scene.P[m], T[p]) for p, m in enumerate(mp)])
    for factor in (sg.FACTOR_ICP, sg.FACTOR_GICP):
        Ha, ba, ea, ia = a.linearize_batch(T, factor=factor)
        Hb, bb, eb, ib = b.linearize_batch(Tb, factor=factor)
        assert np.array_equal(ia, ib)
        for p in range(len(cl)):
            assert max(NF.tight_ratios((Ha[p], ba[p], ea[p]), (Hb[p], bb[p], eb[p]))) <= NF.TIGHT, (factor, p)
        assert all(np.array_equal(x, y) for x, y in zip(_low(a.correspondences_batch()), b.correspondences_batch()))
        ra, rb = a.error_batch(scene.poses(cl, 1)), b.error_batch(np.array([SM.relative(scene.P[m], t) for m, t in zip(mp, scene.poses(cl, 1))]))
        assert np.all(np.abs(ra - rb) <= NF.TIGHT * rb)


@pytest.mark.parametrize("max_d", [1.0, 0.05, None])
def test_every_correspondence_is_the_nearest_of_the_union(scene, max_d):
    sg = _sg()
    ctx = scene.context()
    poses = _poses_of(scene, LISTS)
    scene.submaps(ctx, CL, LISTS, poses)
    kw = dict(factor=sg.FACTOR_ICP, rejector=sg.REJECT_NONE) if max_d is None else dict(factor=sg.FACTOR_ICP, max_dist_sq=max_d)
    rep = NS.Report()
    # unseeded at a perturbed pose, seeded at another, seeded at the same (converged) pose again
    for T in (scene.poses(CL), scene.poses(CL, 1), scene.poses(CL, 1)):
        ctx.linearize_batch(T, **kw)
        for p, corr in enumerate(ctx.correspondences_batch()):
            SM.check_union(corr, T[p], scene.clouds[CL[p]], [scene.targets[k] for k in LISTS[p]], poses[p], max_d, report=rep)
    assert rep.worst_band <= 1.0
    corr = ctx.correspondences_batch()
    assert (corr[5] == NF.NO).all() and len(corr[4]) == 0
    used = np.unique(corr[3][corr[3] != NF.NO] >> HIGH)
    assert len(used) > 3, used  # the 33-entry member really draws on several maps
    print(rep)


@pytest.mark.parametrize("factor", [0, 2])
@pytest.mark.parametrize("robust,c", ROBUST)
def test_sums_match_the_storage_model(scene, factor, robust, c):
    ctx = scene.context()
    poses = _poses_of(scene, LISTS)
    scene.submaps(ctx, CL, LISTS, poses)
    T, T1 = scene.poses(CL), scene.poses(CL, 1)
    H, b, e, inl = ctx.linearize_batch(T, factor=factor, robust=robust, robust_c=c)
    corr = ctx.correspondences_batch()
    err = ctx.error_batch(T1)
    for p, cloud in enumerate(CL):
        if not (corr[p] != NF.NO).any():  # an empty list, an empty cloud, or (member 6) maps that nothing of the scan reaches
            assert p in (4, 5, 6)
            assert not H[p].any() and e[p] == 0 and inl[p] == 0 and err[p] == 0
            continue
        models = [NF.storage_model(scene.clouds[cloud], scene.scovs[cloud], scene.maps[k], None, scene.covs[k]) for k in LISTS[p]]
        sp, scv = models[0][0], models[0][1]
        maps = [(m[2], None, m[4]) for m in models]
        ref = SM.union_linearize(T[p], corr[p], factor, robust, c, sp, scv, maps, poses[p])
        assert inl[p] == (corr[p] != NF.NO).sum()
        assert max(NF.tight_ratios((H[p], b[p], e[p]), ref)) <= NF.TIGHT, (p, NF.tight_ratios((H[p], b[p], e[p]), ref))
        ref_e = SM.union_error(T1[p], T[p], corr[p], factor, robust, c, sp, scv, maps, poses[p])
        assert abs(err[p] - ref_e) <= NF.TIGHT * ref_e, p


def test_against_one_tree_over_the_placed_union(scene):
    """the caller's alternative: place every map on the host, build ONE kd-tree of the union per member, align against it"""
    sg = _sg()
    members = [0, 1, 2]
    lists, cl = [LISTS[p] for p in members], [CL[p] for p in members]
    poses = [[scene.P[k] for k in l] for l in lists]
    # (the fixtures' covariances carry junk below the diagonal, which the device never reads but R C R^T would mix in)
    sym = lambda c: np.triu(c) + np.triu(c, 1).transpose(0, 2, 1)
    unions = [SM.placed_union([(scene.maps[k], None, sym(scene.covs[k])) for k in l], P) for l, P in zip(lists, poses)]
    a = scene.context()
    scene.submaps(a, cl, lists, poses)
    b = sg.Context(0)
    b.build_target_kdtrees([u[0] for u in unions], None, [u[2] for u in unions])
    b.set_source_batch(scene.clouds, scene.scovs)
    b.set_source_pairs(cl, list(range(len(members))))
    T = scene.poses(cl)
    for factor in (sg.FACTOR_ICP, sg.FACTOR_GICP):
        Ha, ba, ea, ia = a.linearize_batch(T, factor=factor)
        Hb, bb, eb, ib = b.linearize_batch(T, factor=factor)
        ca, cb = a.correspondences_batch(), b.correspondences_batch()
        for p in range(len(members)):
            same = SM.to_union(ca[p], unions[p][3]) == cb[p]
            assert same.mean() > 0.995, (p, same.mean())  # the two store different FP32 roundings of the same points
            assert abs(int(ia[p]) - int(ib[p])) <= 0.005 * ib[p]
            # the union context's own sums, over its own correspondences (a few near-ties fall the other way)
            assert np.linalg.norm(Ha[p] - Hb[p]) <= 2e-3 * np.linalg.norm(Hb[p]) and abs(ea[p] - eb[p]) <= 2e-3 * eb[p]
            # the union as that context stores it (FP32 about the union's centre), evaluated over the submap member's correspondences:
            # what is left is the FP32 rounding of the same points about another centre
            c = cl[p]
            model = NF.storage_model(scene.clouds[c], scene.scovs[c], unions[p][0], None, unions[p][2])
            ref = NF.linearize(T[p], SM.to_union(ca[p], unions[p][3]), factor, 0, 1.0, *model)
            assert max(NF.tight_ratios((Ha[p], ba[p], ea[p]), ref)) <= 2e-5, (factor, p, NF.tight_ratios((Ha[p], ba[p], ea[p]), ref))
        for opt in (GN, LM):
            ra = a.align_batch(T, factor=factor, optimizer=opt)
            rb = b.align_batch(T, factor=factor, optimizer=opt)
            # (with the fixtures' random covariances Gauss-Newton GICP may run out of iterations: then on both paths alike)
            assert np.array_equal(ra.iterations, rb.iterations) and np.array_equal(ra.converged, rb.converged), (factor, opt, ra.iterations, rb.iterations)
            assert ra.converged.sum() >= 2
            for p in np.nonzero(ra.converged)[0]:
                d = np.linalg.inv(rb.T_target_source[p]) @ ra.T_target_source[p]
                rot = np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1))
                assert rot <= 1e-4 and np.linalg.norm(d[:3, 3]) <= 1e-3, (factor, opt, p, rot, d[:3, 3])


def test_independence_of_the_other_members(scene):
    sg = _sg()
    poses = _poses_of(scene, LISTS)
    a = scene.context()
    scene.submaps(a, CL, LISTS, poses)
    T = scene.poses(CL)
    H, b, e, inl = a.linearize_batch(T, factor=sg.FACTOR_GICP)
    corr = a.correspondences_batch()
    ra = a.align_batch(T, factor=sg.FACTOR_GICP)
    perm = [3, 6, 0, 5, 1, 4, 2]
    o = scene.context()
    scene.submaps(o, [CL[k] for k in perm], [LISTS[k] for k in perm], [poses[k] for k in perm])
    H2, b2, e2, inl2 = o.linearize_batch(T[perm], factor=sg.FACTOR_GICP)
    for x, y in ((H, H2), (b, b2), (e, e2), (inl, inl2)):
        assert np.array_equal(x[perm], y)
    c2 = o.correspondences_batch()
    assert all(np.array_equal(corr[perm[k]], c2[k]) for k in range(len(perm)))
    ro = o.align_batch(T[perm], factor=sg.FACTOR_GICP)
    assert np.array_equal(ra.T_target_source[perm], ro.T_target_source) and np.array_equal(ra.iterations[perm], ro.iterations)
    # each member alone, and with inactive neighbours
    for p in (2, 3):
        one = scene.context()
        scene.submaps(one, [CL[p]], [LISTS[p]], [poses[p]])
        H1, b1, e1, _ = one.linearize_batch(T[p:p + 1], factor=sg.FACTOR_GICP)
        assert np.array_equal(H1[0], H[p]) and np.array_equal(b1[0], b[p]) and e1[0] == e[p]
        assert np.array_equal(one.correspondences_batch()[0], corr[p])
    active = np.array([1, 0, 1, 0, 1, 1, 0], dtype=bool)
    a.drop_seeds()
    Hx, bx, ex, _ = a.linearize_batch(T, active=active, factor=sg.FACTOR_GICP)
    assert np.array_equal(Hx[active], H[active]) and np.array_equal(ex[active], e[active]) and not Hx[~active].any()
    # 4096 members of one small cloud, lists rotating over the maps: member p equals the same (cloud, list) in a batch of one
    big = scene.context()
    lists = [[(p + j) % 5 for j in range(1 + p % 3)] for p in range(4096)]
    scene.submaps(big, [2] * 4096, lists)
    Tb = np.repeat(scene.poses([2]), 4096, axis=0)
    Hb, _, eb, _ = big.linearize_batch(Tb, factor=sg.FACTOR_GICP)
    for p in (0, 1, 17, 4095):
        one = scene.context()
        scene.submaps(one, [2], [lists[p]])
        H1, _, e1, _ = one.linearize_batch(Tb[:1], factor=sg.FACTOR_GICP)
        assert np.array_equal(H1[0], Hb[p]) and e1[0] == eb[p], p


def test_an_exact_tie_goes_to_the_earlier_entry(scene):
    sg = _sg()
    ctx = scene.context()
    cl = [0, 2]
    scene.submaps(ctx, cl, [[0, 0], [2, 4, 2]])
    T = scene.poses(cl)
    for _ in range(2):  # unseeded, then seeded by its own result
        ctx.linearize_batch(T, factor=sg.FACTOR_ICP)
        c = ctx.correspondences_batch()
        assert ((c[0] == NF.NO) | (c[0] >> HIGH == 0)).all()
        assert ((c[1] == NF.NO) | (c[1] >> HIGH < 2)).all()
    single = scene.context()
    scene.submaps(single, cl, [[0], [2, 4]])
    single.linearize_batch(T, factor=sg.FACTOR_ICP)
    assert all(np.array_equal(x, y) for x, y in zip(c, single.correspondences_batch()))


def test_state_never_goes_stale(scene):
    sg = _sg()
    poses = _poses_of(scene, LISTS)
    T, T1, T2 = scene.poses(CL), scene.poses(CL, 1), scene.poses(CL, 2)

    def fresh(cl, lists, ps, maps=None):
        ctx = scene.context(maps)
        scene.submaps(ctx, cl, lists, ps)
        return _outputs(ctx, scene.poses(cl), scene.poses(cl, 1), scene.poses(cl, 2), 2, 0, 1.0)

    def equal(x, y, tag):
        assert len(x) == len(y) and all(np.array_equal(u, v) for u, v in zip(x, y)), tag

    want = fresh(CL, LISTS, poses)
    ctx = scene.context()
    # other lists first, then the lists; the poses alone changed; pairs in between; a batch in between
    scene.submaps(ctx, [0, 2], [[4, 3], [0]])
    ctx.linearize_batch(scene.poses([0, 2]), factor=sg.FACTOR_GICP)
    scene.submaps(ctx, CL, LISTS, poses)
    equal(_outputs(ctx, T, T1, T2, 2, 0, 1.0), want, "re-paired")
    moved = [[P @ about(OFFSET, [0, 0, 0.01, 0.1, 0, 0]) for P in ps] for ps in poses]
    scene.submaps(ctx, CL, LISTS, moved)
    equal(_outputs(ctx, T, T1, T2, 2, 0, 1.0), fresh(CL, LISTS, moved), "poses changed")
    ctx.set_source_pairs([0, 2], [0, 2])
    pairs = scene.context()
    pairs.set_source_pairs([0, 2], [0, 2])
    Tp = scene.poses([0, 2])
    equal(_outputs(ctx, Tp, Tp, Tp, 2, 0, 1.0), _outputs(pairs, Tp, Tp, Tp, 2, 0, 1.0), "pairs after submaps")
    scene.submaps(ctx, CL, LISTS, poses)
    equal(_outputs(ctx, T, T1, T2, 2, 0, 1.0), want, "submaps after pairs")
    ctx.set_source_batch(scene.clouds, scene.scovs)  # forgets the lists: member m against map m again, 4 members but 12 maps
    with pytest.raises(sg.SgbError, match="4 members but the target holds 12 kd-trees"):
        ctx.linearize_batch(scene.poses(range(4)), factor=sg.FACTOR_GICP)
    scene.submaps(ctx, CL, LISTS, poses)
    equal(_outputs(ctx, T, T1, T2, 2, 0, 1.0), want, "submaps after a batch")
    # the target rebuilt with the maps in another order: the same lists now name other maps
    order = [4, 3, 2, 0, 1, 5, 6, 7, 8, 9, 10, 11]
    ctx.build_target_kdtrees([scene.maps[t] for t in order], None, [scene.covs[t] for t in order])
    ref = scene.context(order)
    scene.submaps(ref, CL, LISTS, poses)
    equal(_outputs(ctx, T, T1, T2, 2, 0, 1.0), _outputs(ref, T, T1, T2, 2, 0, 1.0), "target rebuilt")


def test_launch_counts_equal_the_pairs_path(scene):
    sg = _sg()
    rng = np.random.default_rng(5)
    maps = [_p4(rng.uniform(-5, 5, (200, 3))) for _ in range(33)]
    clouds = [_p4(rng.uniform(-5, 5, (20, 3))) for _ in range(3)]
    counts = set()
    for P in (1, 64, 4096):
        for E in (1, 33):
            ctx = sg.Context(0)
            ctx.build_target_kdtrees(maps)
            ctx.set_source_batch(clouds)
            T = np.tile(np.eye(4), (P, 1, 1))
            rounds = []
            for pairing in (lambda: ctx.set_source_pairs(np.arange(P) % 3, np.arange(P) % 33),
                            lambda: ctx.set_source_submaps([[(p + j) % 33 for j in range(E)] for p in range(P)], None, np.arange(P) % 3)):
                k0 = ctx.kernel_launches
                pairing()
                k1 = ctx.kernel_launches
                ctx.linearize_batch(T, factor=sg.FACTOR_ICP)
                k2 = ctx.kernel_launches
                ctx.linearize_batch(T, factor=sg.FACTOR_ICP)
                k3 = ctx.kernel_launches
                ctx.error_batch(T)
                k4 = ctx.kernel_launches
                r = ctx.align_batch(T, factor=sg.FACTOR_ICP, optimizer=GN, max_iterations=3)
                k5 = ctx.kernel_launches
                rounds.append((k1 - k0, k2 - k1, k3 - k2, k4 - k3, (k5 - k4) / max(int(r.iterations.max()), 1)))
            assert rounds[0] == rounds[1], (P, E, rounds)
            counts.add(rounds[1][:4])
    assert counts == {(1, 4, 3, 2)}, counts


def test_misuse_fails_with_a_message(scene):
    sg = _sg()
    ctx = sg.Context(0)
    with pytest.raises(sg.SgbError, match="no batch"):
        ctx.set_source_submaps([[0]])
    ctx = scene.context()
    T = scene.poses([0, 2])
    with pytest.raises(sg.SgbError, match="not a rigid transformation"):
        ctx.set_source_submaps([[0], [2]], [[np.diag([1.0, 1.0, 1.001, 1.0])], [np.eye(4)]], [0, 2])
    with pytest.raises(sg.SgbError, match="not a rigid transformation"):
        ctx.set_source_submaps([[0], [2]], [[np.diag([1.0, 1.0, -1.0, 1.0])], [np.eye(4)]], [0, 2])
    with pytest.raises(sg.SgbError, match="member 1 names cloud 9 but the batch holds 4 clouds"):
        ctx.set_source_submaps([[0], [2]], None, [0, 9])
    ctx.set_source_submaps([[0], [2, 40]], None, [0, 2])
    with pytest.raises(sg.SgbError, match="entry 1 of member 1 names map 40 but the target holds 12 maps"):
        ctx.linearize_batch(T, factor=sg.FACTOR_ICP)
    ctx.set_source_submaps([[0], [2, 4]], None, [0, 2])
    for call in (lambda: ctx.linearize_batch(T, factor=sg.FACTOR_PLANE_ICP), lambda: ctx.align_batch(T, factor=sg.FACTOR_PLANE_ICP)):
        with pytest.raises(sg.SgbError, match="SGB_FACTOR_PLANE_ICP is not available against submaps"):
            call()
    with pytest.raises(sg.SgbError, match="no preceding sgb_linearize_batch"):
        ctx.error_batch(T)
    H, _, e, _ = ctx.linearize_batch(T, factor=sg.FACTOR_ICP)  # the context is still usable
    assert e[0] > 0 and e[1] > 0
    ctx.build_target_voxelmaps(scene.maps[:3], scene.covs[:3], leaf_size=0.5)
    with pytest.raises(sg.SgbError, match="submaps over voxel maps are not supported"):
        ctx.linearize_batch(T, factor=sg.FACTOR_ICP)
    ctx.set_target(scene.maps[0], None, scene.covs[0])
    ctx.build_target_kdtree()
    with pytest.raises(sg.SgbError, match="the current target is not one"):
        ctx.align_batch(T, factor=sg.FACTOR_ICP)
    ctx.build_target_kdtrees(scene.maps[:5], None, scene.covs[:5])
    H2, _, e2, _ = ctx.linearize_batch(T, factor=sg.FACTOR_ICP)
    assert np.array_equal(H, H2) and np.array_equal(e, e2)
    ctx.set_source_submaps([], None, [])
    assert ctx.linearize_batch(np.zeros((0, 4, 4)), factor=sg.FACTOR_ICP)[0].shape == (0, 6, 6)


def test_golden_pair_split_into_three_posed_maps_against_the_oracle(golden_prepared):
    """the golden target cut into three overlapping maps, each handed over in a frame of its own: the CPU oracle's GICP on the placed
    union (one cloud, one kd-tree) gives the same sums, to the oracle tolerance, and the same alignment"""
    import oracle as O

    sg = _sg()
    g = golden_prepared
    tp, tcv = g["target"].points, g["target"].covs
    sp, scv = g["source"].points, g["source"].covs
    x = tp[:, 0]
    q = np.quantile(x, [0.3, 0.4, 0.6, 0.7])
    masks = [x <= q[1], (x >= q[0]) & (x <= q[3]), x >= q[2]]
    mid = tp[:, :3].mean(0)
    P = [about(mid, [0.3, -0.2, 0.5, 4.0, -2.0, 1.0]), about(mid, [-0.1, 0.4, -0.7, -3.0, 5.0, 0.5]), about(mid, [0.0, 0.0, 1.2, 20.0, 10.0, -2.0])]
    maps, covs = [], []
    for m, Pk in zip(masks, P):
        R4 = np.eye(4)
        R4[:3, :3] = Pk[:3, :3].T
        maps.append(_apply(SM.inverse(Pk), tp[m]))
        covs.append(R4 @ tcv[m] @ R4.T)
    upts, _, ucov, _ = SM.placed_union([(m, None, c) for m, c in zip(maps, covs)], P)
    uc = O.Cloud(upts)
    uc.set_features(covs=ucov)
    ut = O.KdTree(uc)
    ctx = sg.Context(0)
    ctx.build_target_kdtrees(maps, None, covs)
    ctx.set_source_batch([sp], [scv])
    ctx.set_source_submaps([[0, 1, 2]], [P])
    reg = O.Registration(factor=O.FACTOR_GICP, num_threads=0)
    for T in (np.eye(4), NF.orthonormal(g["T"])):
        H, b, e, _ = ctx.linearize_batch(T[None], factor=sg.FACTOR_GICP)
        H0, b0, e0 = reg.linearize(uc, ut, g["source"], T)
        assert np.linalg.norm(H[0] - H0) <= 2e-5 * np.linalg.norm(H0) and abs(e[0] - e0) <= 2e-5 * e0
        assert np.all(np.abs(b[0] - b0) <= 2e-5 * np.sqrt(2.0 * e0 * np.diag(H0)))
    for opt, oopt in ((GN, O.OPT_GN), (LM, O.OPT_LM)):
        reg.set_optimizer(type=oopt)
        r0 = reg.align(uc, ut, g["source"], np.eye(4))
        r = ctx.align_batch(np.eye(4)[None], factor=sg.FACTOR_GICP, optimizer=opt)
        assert r.converged[0] and r0.converged and r.iterations[0] == r0.iterations, (opt, r.iterations, r0.iterations)
        d = np.linalg.inv(r0.T_target_source) @ r.T_target_source[0]
        rot = np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1))
        assert rot <= 1e-4 and np.linalg.norm(d[:3, 3]) <= 1e-3, (opt, rot, d[:3, 3])


def test_host_mirror_matches_the_binding(scene):
    """BatchRegistration's submap overload (host_api.align_batch_submaps) against Context.set_source_submaps + align_batch, bit for bit"""
    from small_gicp_b200 import host_api

    sg = _sg()
    poses = _poses_of(scene, LISTS)
    T = scene.poses(CL)
    ctx = scene.context()
    scene.submaps(ctx, CL, LISTS, poses)
    for kw in (dict(factor=sg.FACTOR_GICP, optimizer=LM), dict(factor=sg.FACTOR_ICP, optimizer=GN, robust=sg.ROBUST_HUBER, robust_c=0.5)):
        h = host_api.align_batch_submaps(scene.maps, scene.clouds, LISTS, poses, scene.covs, scene.scovs, init_Ts=T, cloud_of_member=CL, **kw)
        r = ctx.align_batch(T, **kw)
        assert np.array_equal(h.T_target_source, r.T_target_source) and np.array_equal(h.iterations, r.iterations)
        assert np.array_equal(h.H, r.H) and np.array_equal(h.error, r.error) and np.array_equal(h.converged, r.converged)
    with pytest.raises(sg.SgbError, match="point-to-plane is not available against submaps"):
        host_api.align_batch_submaps(scene.maps, scene.clouds, LISTS, poses, scene.covs, scene.scovs, init_Ts=T, cloud_of_member=CL, factor=sg.FACTOR_PLANE_ICP)
