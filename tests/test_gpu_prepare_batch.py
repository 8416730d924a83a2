"""Many clouds prepared at once: sgb_voxelgrid_sampling_batch / sgb_estimate_features_batch (Context.voxelgrid_sampling_batch /
estimate_features_batch) and the host mirror's preprocess_points_batch.

  1. every cloud's voxel grid bit-identical to sgb_voxelgrid_sampling of that cloud alone and to np_preprocess.voxelgrid_model, also
     across empty clouds, clouds of dropped points and the highest voxel of the 21-bit range between clouds that share voxels;
  2. every cloud's normals and covariances bit-identical to sgb_estimate_features of that cloud alone on tie-free clouds, and within
     check_features of np_preprocess.features_model on lines, planes, duplicated points and an integer grid;
  3. a cloud's results independent of the rest of the batch, exact ties included;
  4. neither call disturbs the context's target, source, batch or linearisation cache;
  5. launch counts independent of the cloud count;
  6. the whole pipeline (batched preparation -> forest -> batched GICP) equal to the per-frame one;
  7. the host mirror; 8. misuse."""
import numpy as np
import pytest

import np_preprocess as PP
from test_gpu_preprocess_model import FEAT_K, FEAT_N, OFFSET, _feat_cloud, _line, _plane, _vg_cloud, check_features
from test_gpu_storage_model import _random_covs, about

pytestmark = pytest.mark.gpu

VG_LEAVES = (0.1, 0.3, 2.0)
E20 = float(1 << 20)


def _sg():
    import small_gicp_b200 as sg

    return sg


@pytest.fixture(scope="module")
def ctx():
    c = _sg().Context(0)
    yield c
    c.close()


def _p4(xyz):
    return np.c_[xyz, np.ones(len(xyz))]


def _split(arr, offsets):
    return [arr[a:b] for a, b in zip(offsets[:-1], offsets[1:])]


def _vg_clouds():
    """the sizes of the single call's tests, one 2 m voxel of 300k points, a cloud outside the 21-bit range, clouds sharing voxels
    with empty clouds or a cloud of dropped points between them, and the highest voxel key followed by an empty cloud and dropped points"""
    rng = np.random.default_rng(5)
    far = np.full((50, 3), 4.0 * E20)  # voxel coordinates beyond 2^20 at every leaf below 4
    big = rng.uniform(0.05, 1.95, (300_000, 3)) + np.array([-310.0, -220.0, -46.0])
    a, b = _vg_cloud(3000, 21), _vg_cloud(3000, 22)  # one region: they share voxels
    empty = np.zeros((0, 3))
    clouds = [empty, _vg_cloud(1, 1), _vg_cloud(2, 2), _vg_cloud(255, 3), _vg_cloud(256, 4), _vg_cloud(257, 6), _vg_cloud(65537, 7), big, far]
    clouds += [a, empty, b, empty, empty, a, empty, empty, empty, b, far, a]
    # key 2^63 - 1 at leaf 2: voxel coordinate 2^20 - 1 on every axis; then an empty cloud, then dropped points and a point of that voxel
    top = np.full((4, 3), 2.0 * (E20 - 0.5)) + rng.uniform(-0.5, 0.5, (4, 3))
    clouds += [np.r_[a[:100], top], empty, np.r_[far[:5], top[:2], b[:100], far[5:9]]]
    return clouds


def test_voxelgrid_batch_equals_single_and_model(ctx):
    import torch

    clouds = _vg_clouds()
    for leaf in VG_LEAVES:
        got, off = ctx.voxelgrid_sampling_batch(clouds, leaf)
        assert off[0] == 0 and len(off) == len(clouds) + 1 and off[-1] == len(got)
        for c, (p, g) in enumerate(zip(clouds, _split(got, off))):
            one = ctx.voxelgrid_sampling(p, leaf)
            assert np.array_equal(g, one), (leaf, c, g.shape, one.shape)
            if len(p):
                assert np.array_equal(g, PP.voxelgrid_model(p, leaf)), (leaf, c)
            else:
                assert len(g) == 0
        if leaf == 2.0:
            assert len(_split(got, off)[-1]) >= 1 and int(PP.voxelmap_model(clouds[7], None, leaf)[3].max()) == 300_000
        # the (points, offsets) form, and CUDA tensors in -> a CUDA tensor out, the same bits
        cat = np.concatenate([_p4(p) for p in clouds])
        starts = np.r_[0, np.cumsum([len(p) for p in clouds])]
        g2, off2 = ctx.voxelgrid_sampling_batch((cat, starts), leaf)
        assert np.array_equal(g2, got) and np.array_equal(off2, off)
        g3, off3 = ctx.voxelgrid_sampling_batch((torch.from_numpy(cat).cuda(), starts), leaf)
        assert g3.is_cuda and np.array_equal(g3.cpu().numpy(), got) and np.array_equal(off3, off)
        print(f"voxel grid, leaf {leaf}: {len(clouds)} clouds, {len(got)} voxels, each bit-identical to its single call and the model")


def _grid(n_side):
    g = np.stack(np.meshgrid(*[np.arange(n_side, dtype=np.float64)] * 3, indexing="ij"), -1).reshape(-1, 3)
    return g + np.round(OFFSET)


def _tie_clouds():
    rng = np.random.default_rng(9)
    return [_line(rng, 4097), _plane(rng, 4097), np.repeat(_feat_cloud(2000, 51), 2, axis=0), _grid(13)]


FEAT_CLOUDS = [n for n in FEAT_N if n <= 65537]


def test_features_batch_equal_single_on_tie_free_clouds(ctx):
    clouds = [_feat_cloud(n, 100 + n % 997) for n in FEAT_CLOUDS]
    clouds = clouds + [np.zeros((0, 3))] + clouds[::-1]  # mixed sizes, an empty cloud between
    for k in FEAT_K:
        N, C = ctx.estimate_features_batch(clouds, k)
        off = np.r_[0, np.cumsum([len(p) for p in clouds])]
        for c, (p, n_, c_) in enumerate(zip(clouds, _split(N, off), _split(C, off))):
            if not len(p):
                continue
            n1, c1 = ctx.estimate_features(p, k)
            assert np.array_equal(n_, n1) and np.array_equal(c_, c1), (k, c, len(p))
        # one output only
        n_only, none = ctx.estimate_features_batch(clouds, k, covs=False)
        assert none is None and np.array_equal(n_only, N)
        none, c_only = ctx.estimate_features_batch(clouds, k, normals=False)
        assert none is None and np.array_equal(c_only, C)
    print(f"features: clouds of {FEAT_CLOUDS} points in one batch, bit-identical to their single calls for k in {FEAT_K}")


def test_features_batch_of_degenerate_clouds(ctx):
    clouds = _tie_clouds()
    off = np.r_[0, np.cumsum([len(p) for p in clouds])]
    worst = 0.0
    for k in (5, 10, 11, 20, 32):
        N, C = ctx.estimate_features_batch(clouds, k)
        for kind, p, n_, c_ in zip(("line", "plane", "duplicated", "grid"), clouds, _split(N, off), _split(C, off)):
            worst = max(worst, check_features(p, n_, c_, k, (kind, k)))
    print(f"features of degenerate clouds in one batch: worst gap-scaled error / bound {worst:.2e}")


def test_cuda_tensors_bitwise(ctx):
    import torch

    clouds = [_feat_cloud(n, 7 + n) for n in (65, 4097, 65537)]
    N, C = ctx.estimate_features_batch(clouds, 20)
    Nt, Ct = ctx.estimate_features_batch([torch.from_numpy(_p4(p)).cuda() for p in clouds], 20)
    assert Nt.is_cuda and Ct.is_cuda
    assert np.array_equal(Nt.cpu().numpy(), N) and np.array_equal(Ct.cpu().numpy(), C)


def test_independent_of_the_batch(ctx):
    """both calls under permutation and in batches of 1, 3, 17 and 4096 clouds, tie-heavy clouds included"""
    rng = np.random.default_rng(3)
    clouds = [_feat_cloud(n, 300 + n) for n in (33, 4097, 65537)] + _tie_clouds()
    base = ctx.estimate_features_batch(clouds, 20)
    off = np.r_[0, np.cumsum([len(p) for p in clouds])]
    ref = [(a, b) for a, b in zip(_split(base[0], off), _split(base[1], off))]
    vg_ref = [ctx.voxelgrid_sampling(p, 0.3) for p in clouds]
    perm = rng.permutation(len(clouds))
    pc = [clouds[j] for j in perm]
    N, C = ctx.estimate_features_batch(pc, 20)
    poff = np.r_[0, np.cumsum([len(p) for p in pc])]
    V, voff = ctx.voxelgrid_sampling_batch(pc, 0.3)
    for i, j in enumerate(perm):
        assert np.array_equal(N[poff[i] : poff[i + 1]], ref[j][0]) and np.array_equal(C[poff[i] : poff[i + 1]], ref[j][1]), j
        assert np.array_equal(V[voff[i] : voff[i + 1]], vg_ref[j]), j
    filler = [_feat_cloud(40, 900 + j) for j in range(8)]
    for j in range(len(clouds)):
        for size in (1, 3, 17, 4096):
            pos = (size * 5) // 7
            batch = [filler[(i * 3) % len(filler)] for i in range(size)]
            batch[pos] = clouds[j]
            boff = np.r_[0, np.cumsum([len(p) for p in batch])]
            N, C = ctx.estimate_features_batch(batch, 20)
            assert np.array_equal(N[boff[pos] : boff[pos + 1]], ref[j][0]) and np.array_equal(C[boff[pos] : boff[pos + 1]], ref[j][1]), (j, size)
            V, voff = ctx.voxelgrid_sampling_batch(batch, 0.3)
            assert np.array_equal(V[voff[pos] : voff[pos + 1]], vg_ref[j]), (j, size)


def test_context_state_untouched():
    """a point target with its grid, a forest target and a voxel-map target, each with a batch (and the point target with a single
    source): the registration results before and after both calls are bit-identical"""
    from small_gicp_b200.synthetic import make_world, sample_cloud

    sg = _sg()
    world = make_world(200_000)
    rng = np.random.default_rng(17)
    tgts = [_p4(sample_cloud(world, 20_000, 60 + j) + OFFSET) for j in range(3)]
    srcs = [_p4(sample_cloud(world, 3000, 70 + j) + OFFSET) for j in range(3)]
    tcov = [_random_covs(rng, len(t)) for t in tgts]
    scov = [_random_covs(rng, len(s)) for s in srcs]
    T = np.array([about(s[:, :3].mean(0), rng.uniform(-1, 1, 6) * [0.01, 0.01, 0.01, 0.1, 0.1, 0.1]) for s in srcs])
    others = [_feat_cloud(5000, 80), _vg_cloud(20_000, 81)]

    def disturb(c):
        c.voxelgrid_sampling_batch(others, 0.3)
        c.estimate_features_batch(others, 20)

    setups = {
        "points+grid": lambda c: (c.set_target(tgts[0], None, tcov[0]), c.build_target_kdtree()),
        "kdtrees": lambda c: c.build_target_kdtrees(tgts, None, tcov),
        "voxelmaps": lambda c: c.build_target_voxelmaps(tgts, tcov, 1.0, 1),
    }
    for name, setup in setups.items():
        c = sg.Context(0)
        setup(c)
        Ts = T
        c.set_source_batch(srcs, scov)
        lin0 = c.linearize_batch(Ts)
        e0 = c.error_batch(Ts)
        disturb(c)
        e1 = c.error_batch(Ts)  # the cached correspondences and linearisation poses survived
        lin1 = c.linearize_batch(Ts)
        assert np.array_equal(e0, e1), name
        assert all(np.array_equal(a, b) for a, b in zip(lin0, lin1)), name
        r0 = c.align_batch(Ts)
        disturb(c)
        r1 = c.align_batch(Ts)
        assert np.array_equal(r0.T_target_source, r1.T_target_source) and np.array_equal(r0.iterations, r1.iterations), name
        if name == "points+grid":
            c.set_source(srcs[0], scov[0])
            h0 = c.linearize(T[0])
            e0 = c.error(T[0] @ about(np.zeros(3), [0.001, 0, 0, 0.01, 0, 0]))
            disturb(c)
            assert c.error(T[0] @ about(np.zeros(3), [0.001, 0, 0, 0.01, 0, 0])) == e0
            assert all(np.array_equal(a, b) for a, b in zip(h0, c.linearize(T[0])))
        c.close()
    # adopting a source whose tree sgb_source_estimate_features built, after a batched call took the scratch tree buffers
    f0, f1 = _vg_cloud(30_000, 90), _vg_cloud(30_000, 91)
    res = []
    for batched in (False, True):
        c = sg.Context(0)
        c.set_source(f0)
        c.estimate_source_features(20)
        if batched:
            disturb(c)
        c.adopt_source_as_target()
        c.set_source(f1)
        c.estimate_source_features(20)
        res.append((c.linearize(np.eye(4)), c.correspondences()))
        c.close()
    assert all(np.array_equal(a, b) for a, b in zip(res[0][0], res[1][0])) and np.array_equal(res[0][1], res[1][1])


def test_launches_independent_of_the_cloud_count():
    p = _vg_cloud(3000, 31)  # above one shared-memory segment of the forest: the build has a radix level
    counts = {}
    for n in (1, 64, 4096):
        c = _sg().Context(0)
        k0 = c.kernel_launches
        c.voxelgrid_sampling_batch([p] * n, 0.3)
        k1 = c.kernel_launches
        c.estimate_features_batch([p] * n, 20)
        counts[n] = (k1 - k0, c.kernel_launches - k1)
        c.close()
    assert len(set(counts.values())) == 1, counts
    c = _sg().Context(0)
    k0 = c.kernel_launches
    c.voxelgrid_sampling(p, 0.3)
    k1 = c.kernel_launches
    c.estimate_features(p, 20)
    print(f"launches (voxel grid, features) per batched call: {counts}; single calls: ({k1 - k0}, {c.kernel_launches - k1})")
    c.close()


def _lidar_frames(n_frames):
    import torch

    from small_gicp_b200 import synthetic as syn

    world = syn.make_world(16_000_000, 42)
    side = syn.world_side(16_000_000)
    poses = [syn.lidar_pose(f, side) for f in range(n_frames)]
    raw = [syn.lidar_frame_torch(world, poses[f], 45 + f, torch.device("cuda:0")) for f in range(n_frames)]
    return poses, raw


def test_pipeline_equals_per_frame_preparation():
    """65 raw LiDAR frames: batched voxel grid -> batched covariances -> build_target_kdtrees + set_source_batch -> align_batch (GICP,
    LM and GN), against the same pipeline with the frames prepared one call at a time"""
    import oracle as O

    sg = _sg()
    poses, raw = _lidar_frames(65)
    c = sg.Context(0)
    # batched, on the device
    pts, off = c.voxelgrid_sampling_batch(raw, 0.25)
    _, covs = c.estimate_features_batch((pts, off), 20, normals=False)
    assert pts.is_cuda and covs.is_cuda
    # one frame at a time
    single = [c.voxelgrid_sampling(r.cpu().numpy(), 0.25) for r in raw]
    scovs = [c.estimate_features(p, 20, normals=False)[1] for p in single]
    c.close()
    P, Cv = pts.cpu().numpy(), covs.cpu().numpy()
    for f in range(65):
        assert np.array_equal(P[off[f] : off[f + 1]], single[f]), f
    diff = sum(int((Cv[off[f] : off[f + 1]] != scovs[f]).any(axis=(1, 2)).sum()) for f in range(65))
    noise = O.se3_exp(np.array([0.0, 0.0, np.deg2rad(0.5), 0.1, 0.0, 0.0]))
    inits = np.array([np.linalg.inv(poses[i]) @ poses[i + 1] @ noise for i in range(64)])
    results = {}
    for name, frames, fcovs in (("batched", _split(P, off), _split(Cv, off)), ("single", single, scovs)):
        r = sg.Context(0)
        r.build_target_kdtrees(frames[:64], None, fcovs[:64])
        r.set_source_batch(frames[1:], fcovs[1:])
        results[name] = [r.align_batch(inits, factor=sg.FACTOR_GICP, optimizer=opt) for opt in (1, 0)]
        r.close()
    for a, b in zip(results["batched"], results["single"]):
        assert np.array_equal(a.T_target_source, b.T_target_source) and np.array_equal(a.iterations, b.iterations)
    print(f"pipeline: 65 frames, {len(P)} voxels, {diff} covariances differ from the single calls (exact ties); "
          f"LM iterations {results['batched'][0].iterations.max()}, GN {results['batched'][1].iterations.max()}")


def test_host_mirror(golden):
    from small_gicp_b200 import host_api
    from small_gicp_b200.synthetic import make_world, sample_cloud

    tgt, src, _ = golden
    world = make_world(500_000)
    clouds = [tgt, src] + [sample_cloud(world, 40_000, 400 + j) for j in range(3)] + [np.zeros((0, 3))]
    one = host_api.preprocess_points(clouds, 0.25, 10, batch=False)
    many = host_api.preprocess_points(clouds, 0.25, 10, batch=True)
    for j, (a, b) in enumerate(zip(one, many)):
        assert all(np.array_equal(x, y) for x, y in zip(a, b)), j
    assert len(many[0][0]) > 0 and len(many[-1][0]) == 0


def test_misuse(ctx):
    sg = _sg()
    L, h = ctx._L, ctx._h
    p = _p4(_feat_cloud(100, 1))
    dp = p.ctypes.data_as(sg.capi._dp)
    out = np.empty_like(p)
    odp = out.ctypes.data_as(sg.capi._dp)
    szt = sg.capi.C.c_size_t
    oo = (szt * 65538)()

    def vg(n, offs, pts=dp, o=odp, oo_=oo, leaf=0.3):
        return ctx._check(L.sgb_voxelgrid_sampling_batch(h, n, (szt * len(offs))(*offs), pts, leaf, o, oo_))

    def ft(n, offs, k=10, pts=dp, on=odp, oc=None):
        return ctx._check(L.sgb_estimate_features_batch(h, n, (szt * len(offs))(*offs), pts, k, on, oc))

    for call in (vg, ft):
        with pytest.raises(sg.SgbError, match="offsets\\[0\\] must be 0"):
            call(1, [1, 100])
        with pytest.raises(sg.SgbError, match="offsets must be ascending \\(cloud 1\\)"):
            call(2, [0, 60, 50])
        with pytest.raises(sg.SgbError, match="65537 clouds, at most 65536"):
            call(65537, [0] * 65538)
        with pytest.raises(sg.SgbError, match="null points" if call is ft else "null buffer"):
            call(1, [0, 100], pts=None)
    with pytest.raises(sg.SgbError, match="null offsets"):
        ctx._check(L.sgb_voxelgrid_sampling_batch(h, 1, None, dp, 0.3, odp, oo))
    with pytest.raises(sg.SgbError, match="null out_offsets"):
        vg(1, [0, 100], oo_=None)
    with pytest.raises(sg.SgbError, match="null buffer"):
        vg(1, [0, 100], o=None)
    with pytest.raises(sg.SgbError, match="leaf_size must be positive"):
        vg(1, [0, 100], leaf=0.0)
    with pytest.raises(sg.SgbError, match="2\\^31"):
        vg(1, [0, 1 << 31])
    for k in (0, 33):
        with pytest.raises(sg.SgbError, match="num_neighbors must be in 1..32"):
            ft(1, [0, 100], k=k)
    with pytest.raises(sg.SgbError, match="2\\^30"):
        ft(2, [0, 1 << 29, 1 << 30])
    # nothing asked for, or nothing given: no work, no failure
    ft(1, [0, 100], on=None)
    ft(0, [0])
    vg(0, [0])
    with pytest.raises(sg.SgbError, match="offsets must have B \\+ 1 entries"):
        ctx.voxelgrid_sampling_batch((p, [0, 50]), 0.3)
    # the context still works
    got, off = ctx.voxelgrid_sampling_batch([p, p], 0.3)
    assert np.array_equal(got[off[1] : off[2]], ctx.voxelgrid_sampling(p, 0.3))
