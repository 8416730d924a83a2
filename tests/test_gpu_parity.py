"""GPU parity: the CUDA hot path (through the C-ABI) against the CPU oracle on identical inputs.

Each check is a triangle  oracle <-> numpy <-> GPU  (tests/np_factors.py):
  1. correspondences: GPU == oracle except FP32 near-ties (squared distances equal to 1e-5 rel + 1e-7) and points
     sitting on the rejection boundary (|d2 - max_dist_sq| < 1e-4);
  2. oracle sums == numpy sums over the ORACLE's correspondences to 1e-9 (pins the numpy leg to the oracle);
  3. GPU sums == numpy sums over the GPU's OWN correspondences, evaluated on the storage model of what the device holds
     (np_factors.storage_model: centred FP32 coordinates, FP32 normals and covariance entries) to np_factors.TIGHT = 1e-10;
     when (1) found no difference at all the GPU sums are also compared directly with the oracle's.

Tolerances against the oracle (FP32 coordinate/covariance storage, FP32 search, FP64 factor algebra and sums; DESIGN.md §5):
  H      : ||H_gpu - H_ref||_F <= 2e-5 ||H_ref||_F
  e      : |e_gpu - e_ref| <= 2e-5 e_ref
  b      : |b_gpu - b_ref|_k <= 2e-5 sqrt(2 e H_kk)           (Cauchy-Schwarz scale of b_k)
  step   : |H^-1 b|_gpu - |H^-1 b|_ref  <= 2e-6 (rad / m)
  pose   : converged SE(3) within 1e-4 rad / 1e-3 m of the oracle (BASELINE.json north_star)
The model leg needs exact rotations (the kernels work in the source frame, D = R^T M R): the 6-digit golden pose goes through
np_factors.orthonormal for the oracle and the GPU alike.
"""
import numpy as np
import pytest

import np_factors as NF
import oracle as O
from conftest import noise_poses, pose_error

pytestmark = pytest.mark.gpu

RTOL = 2e-5


def _sg():
    import small_gicp_b200 as sg

    return sg


def load_ctx(target, tree, source, own_tree=False, profiling=False):
    sg = _sg()
    ctx = sg.Context(0, profiling=profiling)
    ctx.set_target(target.points, target.normals, target.covs)
    if own_tree:
        ctx.build_target_kdtree(0)
    else:
        nodes, idx = tree.export()
        ctx.set_target_kdtree(nodes, idx)
    ctx.set_source(source.points, source.covs)
    return ctx


def check_linearized(got, ref, tag="", rtol=RTOL):
    (H, b, e), (H0, b0, e0) = got, ref
    assert np.linalg.norm(H - H0) <= rtol * np.linalg.norm(H0), (tag, np.linalg.norm(H - H0) / np.linalg.norm(H0))
    assert abs(e - e0) <= rtol * e0, (tag, e, e0)
    scale = np.sqrt(2.0 * e0 * np.diag(H0))
    assert np.all(np.abs(b - b0) <= rtol * scale), (tag, np.abs(b - b0) / scale)
    d, d0 = np.linalg.solve(H + 1e-6 * np.eye(6), -b), np.linalg.solve(H0 + 1e-6 * np.eye(6), -b0)
    assert np.abs(d - d0).max() <= max(2e-6, 100 * rtol * np.abs(d0).max() * 1e-2), (tag, np.abs(d - d0).max())


def check_tight(got, ref, tag=""):
    """GPU sums against numpy on the storage model (np_factors.TIGHT); returns the worst of the three ratios"""
    r = NF.tight_ratios(got, ref)
    assert max(r) <= NF.TIGHT, (tag, "H, b, e:", r)
    return max(r)


def check_tight_error(e_gpu, e_model, tag=""):
    r = abs(e_gpu - e_model) / e_model
    assert r <= NF.TIGHT, (tag, e_gpu, e_model, r)
    return r


class Arrays:
    """numpy views of an oracle (target, source) pair, and the storage model of the same pair uploaded whole"""

    def __init__(self, target, source):
        self.tp, self.tn, self.tc = target.points, target.normals, target.covs
        self.sp, self.sc = source.points, source.covs
        self.model = NF.storage_model(self.sp, self.sc, self.tp, self.tn, self.tc)


def triangle(ctx, reg, target, tree, source, arr, T, factor, robust, c, rejector=1, max_d=1.0, tag=""):
    sg = _sg()
    cpu = reg.linearize(target, tree, source, T)
    gpu = ctx.linearize(T, factor=factor, robust=robust, robust_c=c, rejector=rejector, max_dist_sq=max_d)
    np.testing.assert_array_equal(gpu[0], gpu[0].T)  # the kernel writes both triangles from one sum
    c_cpu = reg.correspondences(len(arr.sp))
    c_gpu = ctx.correspondences()
    nm = NF.compare_correspondences(c_gpu, c_cpu, arr.tp, arr.sp, T, max_d if rejector else None)
    assert ctx.num_inliers() == int((c_gpu != sg.NO_CORRESPONDENCE).sum())
    args = (factor, robust, c, arr.sp, arr.sc, arr.tp, arr.tn, arr.tc)
    check_linearized(cpu, NF.linearize(T, c_cpu, *args), (tag, "oracle-vs-numpy"), rtol=1e-9)
    worst = check_tight(gpu, NF.linearize(T, c_gpu, factor, robust, c, *arr.model), (tag, "gpu-vs-model"))
    if nm == 0:
        check_linearized(gpu, cpu, (tag, "gpu-vs-oracle"))
    return c_cpu, c_gpu, nm, worst


FACTORS = [
    ("ICP", 0, 0),
    ("PLANE_ICP", 1, 0),
    ("GICP", 2, 0),
    ("HUBER_GICP", 2, 1),
    ("CAUCHY_GICP", 2, 2),
    ("HUBER_ICP", 0, 1),
    ("CAUCHY_PLANE", 1, 2),
]


@pytest.fixture(scope="module")
def golden_ctx(golden_prepared):
    g = golden_prepared
    ctx = load_ctx(g["target"], g["target_tree"], g["source"])
    yield ctx
    ctx.close()


@pytest.mark.parametrize("name,factor,robust", FACTORS)
def test_linearize_and_error_golden(golden_prepared, golden_ctx, name, factor, robust):
    g = golden_prepared
    ctx = golden_ctx
    arr = Arrays(g["target"], g["source"])
    reg = O.Registration(factor=factor, robust=robust, robust_c=0.7, num_threads=0)
    worst = 0.0
    for j, T in enumerate([np.eye(4), NF.orthonormal(g["T"])] + noise_poses()[1:3]):
        c_cpu, c_gpu, nm, w = triangle(ctx, reg, g["target"], g["target_tree"], g["source"], arr, T, factor, robust, 0.7, tag=(name, j))
        worst = max(worst, w)
        # LM trial poses: cached correspondences, precision matrices frozen at the linearisation pose
        for a in ([0.01, -0.02, 0.005, 0.05, -0.03, 0.02], [0, 0, 0, 0, 0, 0]):
            T2 = T @ O.se3_exp(np.array(a, dtype=float))
            e_gpu = ctx.error(T2)
            e_np = NF.error(T2, T, c_gpu, factor, robust, 0.7, *arr.model)
            worst = max(worst, check_tight_error(e_gpu, e_np, (name, j)))
            e_cpu = reg.error(g["target"], g["source"], T2)
            assert abs(e_cpu - NF.error(T2, T, c_cpu, factor, robust, 0.7, arr.sp, arr.sc, arr.tp, arr.tn, arr.tc)) <= 1e-9 * e_cpu
            if nm == 0:
                assert abs(e_gpu - e_cpu) <= RTOL * e_cpu
    print(f"worst ratio to the storage model ({name}): {worst:.2e}")


def test_null_rejector_and_small_radius(golden_prepared, golden_ctx):
    g = golden_prepared
    arr = Arrays(g["target"], g["source"])
    for rej, md in ((O.REJECT_NONE, 1.0), (O.REJECT_DISTANCE, 0.05), (O.REJECT_DISTANCE, 25.0)):
        reg = O.Registration(factor=O.FACTOR_GICP, rejector=rej, max_dist_sq=md, num_threads=0)
        triangle(golden_ctx, reg, g["target"], g["target_tree"], g["source"], arr, np.eye(4), 2, 0, 1.0, rejector=rej, max_d=md, tag=("rejector", rej, md))
        if rej == O.REJECT_NONE:
            assert golden_ctx.num_inliers() == len(g["source"])


def test_seeded_search_is_exact(golden_prepared):
    """The second linearize on unchanged clouds seeds every search with the previous correspondence; the result must be
    the same exact nearest neighbours as an unseeded search (fresh context) at the new pose."""
    g = golden_prepared
    a = load_ctx(g["target"], g["target_tree"], g["source"])
    b = load_ctx(g["target"], g["target_tree"], g["source"])
    a.linearize(noise_poses()[1])  # seeds from a different pose
    Ha, ba, ea = a.linearize(g["T"])
    Hb, bb, eb = b.linearize(g["T"])
    assert np.array_equal(a.correspondences(), b.correspondences())
    assert np.array_equal(Ha, Hb) and np.array_equal(ba, bb) and ea == eb
    a.close()
    b.close()


def test_own_tree_gives_same_result(golden_prepared):
    """Exact NN does not depend on the tree's split choices (only exact ties do)."""
    g = golden_prepared
    a = load_ctx(g["target"], g["target_tree"], g["source"])
    b = load_ctx(g["target"], None, g["source"], own_tree=True)
    Ha, ba, ea = a.linearize(g["T"])
    Hb, bb, eb = b.linearize(g["T"])
    ca, cb = a.correspondences(), b.correspondences()
    assert (ca != cb).sum() <= 2
    assert np.linalg.norm(Ha - Hb) <= 1e-6 * np.linalg.norm(Ha) and abs(ea - eb) <= 1e-6 * ea
    a.close()
    b.close()


def _gn_align(ctx, sg, factor, robust, init_T, max_iter=20, lam=1e-6):
    """GaussNewtonOptimizer::optimize (registration/optimizer.hpp:24-63) on top of the C-ABI, host side in numpy."""
    T = init_T.copy()
    for i in range(max_iter):
        H, b, e = ctx.linearize(T, factor=factor, robust=robust)
        d = np.linalg.solve(H + lam * np.eye(6), -b)
        T = T @ O.se3_exp(d)
        if np.linalg.norm(d[:3]) <= 0.1 * np.pi / 180 and np.linalg.norm(d[3:]) <= 1e-3:
            break
    return T, i


@pytest.mark.parametrize("name,factor,robust", FACTORS[:5])
def test_converged_pose_matches_oracle(golden_prepared, golden_ctx, name, factor, robust):
    g = golden_prepared
    sg = _sg()
    reg = O.Registration(factor=factor, robust=robust, num_threads=0)
    reg.set_optimizer(type=O.OPT_GN)
    for Tn in noise_poses()[:2]:
        r = reg.align(g["target"], g["target_tree"], g["source"], Tn)
        T, it = _gn_align(golden_ctx, sg, factor, robust, Tn)
        rot, trans = pose_error(r.T_target_source, T)
        assert rot < 1e-4 and trans < 1e-3, (name, rot, trans)
        assert it == r.iterations
        rot, trans = pose_error(g["T"], T)
        assert rot < np.deg2rad(2.5) and trans < 0.2


def test_voxelmap_target(golden_prepared):
    g = golden_prepared
    sg = _sg()
    worst = 0.0
    for offsets in (1, 7, 27):
        vm = O.GaussianVoxelMap(g["target"], 1.0, offsets)
        coords, means, covs, _ = vm.export()
        ctx = sg.Context(0)
        ctx.set_target_voxelmap(1.0, coords, means, covs, offsets)
        ctx.set_source(g["source"].points, g["source"].covs)
        reg = O.Registration(factor=O.FACTOR_GICP, num_threads=0)
        # the voxel means are one upload of their own: centred on their box, stored like any target point
        model = NF.storage_model(g["source"].points, g["source"].covs, means, None, covs)
        for T in (np.eye(4), NF.orthonormal(g["T"])):
            cpu = reg.linearize(vm, None, g["source"], T)
            gpu = ctx.linearize(T, factor=sg.FACTOR_GICP)
            c = reg.correspondences(len(g["source"]))
            cg = ctx.correspondences()
            nm = int((cg != c).sum())
            assert nm <= 2
            # GPU sums against numpy on the storage model over the GPU's OWN correspondences (always), and against the oracle when they agree
            src = g["source"]
            vox_id = np.where(cg == sg.NO_CORRESPONDENCE, NF.NO, cg >> np.uint64(32))  # calc_index: voxel id << 32 (incremental_voxelmap.hpp:151)
            worst = max(worst, check_tight(gpu, NF.linearize(T, vox_id, 2, 0, 1.0, *model), ("vgicp-model", offsets)))
            T2 = T @ O.se3_exp(np.array([0.01, 0.0, -0.01, 0.02, 0.02, 0.0]))
            e_gpu = ctx.error(T2)
            e_npy = NF.error(T2, T, vox_id, 2, 0, 1.0, src.points, src.covs, means, None, covs)
            worst = max(worst, check_tight_error(e_gpu, NF.error(T2, T, vox_id, 2, 0, 1.0, *model), ("vgicp-model-error", offsets)))
            if nm == 0:
                check_linearized(gpu, cpu, ("vgicp", offsets))
                assert abs(e_gpu - reg.error(vm, g["source"], T2)) <= RTOL * e_npy
        ctx.close()
    print(f"worst ratio to the storage model (voxel map): {worst:.2e}")


def test_device_built_voxelmap_matches_oracle(golden_prepared):
    """sgb_target_build_voxelmap (voxel keys -> radix sort -> per-voxel mean / covariance -> hash table, all on the device)
    against the oracle's restatement of IncrementalVoxelMap<GaussianVoxel>::insert: same set of voxels, same means and
    covariances, and the same VGICP sums (voxel ids are numbered differently, so correspondences are compared by voxel)."""
    g = golden_prepared
    sg = _sg()
    tgt = g["target"]
    for leaf, offsets in ((1.0, 1), (0.5, 7), (2.0, 27)):
        vm = O.GaussianVoxelMap(tgt, leaf, offsets)
        coords, means, covs, _ = vm.export()
        adopted = sg.Context(0)
        adopted.set_target_voxelmap(leaf, coords, means, covs, offsets)
        built = sg.Context(0)
        built.build_target_voxelmap(tgt.points, tgt.covs, leaf, offsets)
        assert built.target_size == len(coords)
        for ctx in (adopted, built):
            ctx.set_source(g["source"].points, g["source"].covs)
        # the ids differ (ascending key order vs first-insertion order): map both to voxel coordinates
        order_ref = {tuple(int(v) for v in c): i for i, c in enumerate(coords)}
        keys_sorted = sorted(order_ref, key=lambda c: ((c[2] + (1 << 20)) << 42) | ((c[1] + (1 << 20)) << 21) | (c[0] + (1 << 20)))
        id_built_to_ref = np.array([order_ref[c] for c in keys_sorted], dtype=np.int64)
        for T in (np.eye(4), g["T"]):
            Ha, ba, ea = adopted.linearize(T, factor=sg.FACTOR_GICP)
            Hb, bb, eb = built.linearize(T, factor=sg.FACTOR_GICP)
            assert np.linalg.norm(Ha - Hb) <= 1e-9 * np.linalg.norm(Ha) and abs(ea - eb) <= 1e-9 * ea, (leaf, offsets)
            ca, cb = adopted.correspondences(), built.correspondences()
            none = ca == sg.NO_CORRESPONDENCE
            assert np.array_equal(none, cb == sg.NO_CORRESPONDENCE)
            ida = (ca[~none] >> np.uint64(32)).astype(np.int64)
            idb = (cb[~none] >> np.uint64(32)).astype(np.int64)
            assert np.array_equal(ida, id_built_to_ref[idb])
        adopted.close()
        built.close()
    # empty input and points outside the 21-bit voxel range
    ctx = sg.Context(0)
    ctx.build_target_voxelmap(np.zeros((0, 4)), None, 1.0)
    assert ctx.target_size == 0
    ctx.close()


def test_empty_and_tiny_inputs(golden_prepared):
    g = golden_prepared
    sg = _sg()
    ctx = sg.Context(0)
    # empty source / empty target: zeros, no crash (helper_test.cpp:53-59, kdtree_test.cpp:170-176)
    ctx.set_target(g["target"].points, g["target"].normals, g["target"].covs)
    ctx.build_target_kdtree()
    ctx.set_source(np.zeros((0, 4)), np.zeros((0, 4, 4)))
    H, b, e = ctx.linearize(np.eye(4))
    assert not H.any() and not b.any() and e == 0.0 and ctx.num_inliers() == 0
    assert ctx.error(np.eye(4)) == 0.0
    ctx.set_target(np.zeros((0, 4)), None, np.zeros((0, 4, 4)))
    ctx.build_target_kdtree()
    ctx.set_source(g["source"].points, g["source"].covs)
    H, b, e = ctx.linearize(np.eye(4))
    assert not H.any() and e == 0.0
    assert np.all(ctx.correspondences() == sg.NO_CORRESPONDENCE)
    # ragged sizes around the leaf size and the block size
    for n in (1, 5, 19, 20, 21, 127, 129, 1000):
        tc = O.Cloud(g["target"].points[:n])
        tt = O.KdTree(tc)
        tc.set_features(g["target"].normals[:n], g["target"].covs[:n])
        c2 = load_ctx(tc, tt, g["source"])
        reg = O.Registration(factor=O.FACTOR_GICP, rejector=O.REJECT_NONE, num_threads=0)
        triangle(c2, reg, tc, tt, g["source"], Arrays(tc, g["source"]), NF.orthonormal(g["T"]), 2, 0, 1.0, rejector=0, tag=("tiny", n))
        c2.close()
    # missing features are an error, not a silent fallback
    ctx.set_target(g["target"].points)
    ctx.build_target_kdtree()
    with pytest.raises(sg.SgbError):
        ctx.linearize(np.eye(4), factor=sg.FACTOR_GICP)
    with pytest.raises(sg.SgbError):
        ctx.linearize(np.eye(4), factor=sg.FACTOR_PLANE_ICP)
    ctx.linearize(np.eye(4), factor=sg.FACTOR_ICP)
    ctx.close()


@pytest.fixture(scope="module")
def synthetic_pair():
    from small_gicp_b200.synthetic import make_pair

    tgt, src, T = make_pair(200_000)
    nt = max(1, O.max_threads())
    tc, sc = O.Cloud(tgt), O.Cloud(src)
    tt, st = O.KdTree(tc), O.KdTree(sc)
    tt.estimate(20, O.FEAT_NORMAL_COV, nt)
    st.estimate(20, O.FEAT_COV, nt)
    return tc, tt, sc, T, nt


def test_synthetic_200k_gicp(synthetic_pair):
    """BASELINE config 2 shape (synthetic room pair, GICP, GN) at a size the oracle finishes in seconds."""
    tc, tt, sc, Tgt, nt = synthetic_pair
    sg = _sg()
    ctx = load_ctx(tc, tt, sc)
    reg = O.Registration(factor=O.FACTOR_GICP, num_threads=0)
    arr = Arrays(tc, sc)
    for T in (np.eye(4), Tgt):
        triangle(ctx, reg, tc, tt, sc, arr, T, 2, 0, 1.0, tag="synthetic")
    regp = O.Registration(factor=O.FACTOR_GICP, num_threads=nt)
    regp.set_optimizer(type=O.OPT_GN)
    r = regp.align(tc, tt, sc, np.eye(4))
    T, it = _gn_align(ctx, sg, sg.FACTOR_GICP, sg.ROBUST_NONE, np.eye(4))
    rot, trans = pose_error(r.T_target_source, T)
    assert rot < 1e-4 and trans < 1e-3, (rot, trans)
    rot, trans = pose_error(Tgt, T)
    assert rot < 2e-3 and trans < 2e-2, (rot, trans)
    # own tree: same sums
    ctx2 = load_ctx(tc, None, sc, own_tree=True)
    H1, b1, e1 = ctx.linearize(Tgt)
    H2, b2, e2 = ctx2.linearize(Tgt)
    assert np.linalg.norm(H1 - H2) <= 1e-6 * np.linalg.norm(H1) and abs(e1 - e2) <= 1e-6 * e1
    # determinism: bitwise identical on repeat
    H3, b3, e3 = ctx.linearize(Tgt)
    assert np.array_equal(H1, H3) and np.array_equal(b1, b3) and e1 == e3
    ctx.close()
    ctx2.close()


def test_search_structures_agree(synthetic_pair, monkeypatch):
    """Exact NN is independent of the search structure: device-built kd-tree (default), host-built median-split
    kd-tree, adopted reference kd-tree; grid front end with block lists / per-cell lists / off, ring search on / off,
    every pending query through the warp-per-query kernel or through the packet search, cells so small that most
    queries stay pending; packet, per-thread and fused kernels -- same correspondences, same sums."""
    tc, tt, sc, Tgt, nt = synthetic_pair
    sg = _sg()
    results = {}
    switches = ("SGB_TREE", "SGB_SEARCH", "SGB_GRID", "SGB_RING", "SGB_PENDING_DIV", "SGB_GRID_CELL", "SGB_PACKET_QUEUE", "SGB_TMA_LEAF",
                "SGB_CHUNK_CLASSES", "SGB_CLASS_FALLBACK_PCT", "SGB_KD_SMEM")
    for name, env, own in (
        ("device-kd/grid", {}, True),
        ("device-kd/no-grid", {"SGB_GRID": "0"}, True),
        ("device-kd/grid-no-ring", {"SGB_RING": "0"}, True),
        ("device-kd/grid-warp-per-pending", {"SGB_PENDING_DIV": "1"}, True),
        ("device-kd/grid-packet-pending", {"SGB_PENDING_DIV": "1000000"}, True),
        ("device-kd/grid-packet-pending-static-stride", {"SGB_PENDING_DIV": "1000000", "SGB_PACKET_QUEUE": "0"}, True),
        ("device-kd/no-grid-static-stride", {"SGB_GRID": "0", "SGB_PACKET_QUEUE": "0"}, True),
        ("device-kd/grid-small-cells", {"SGB_GRID_CELL": "0.7"}, True),
        ("device-kd/grid-small-cells-warp", {"SGB_GRID_CELL": "0.7", "SGB_PENDING_DIV": "1"}, True),
        ("device-kd/grid-large-cells", {"SGB_GRID_CELL": "6"}, True),
        ("device-kd/packet-tma-leaf", {"SGB_PENDING_DIV": "1000000", "SGB_TMA_LEAF": "1"}, True),
        ("device-kd/no-grid-tma-leaf", {"SGB_GRID": "0", "SGB_TMA_LEAF": "1"}, True),
        ("device-kd/packet-no-class-lists", {"SGB_PENDING_DIV": "1000000", "SGB_CHUNK_CLASSES": "0"}, True),
        ("device-kd/packet-class-lists-always", {"SGB_PENDING_DIV": "1000000", "SGB_CLASS_FALLBACK_PCT": "100"}, True),
        ("device-kd/packet-class-lists-never", {"SGB_PENDING_DIV": "1000000", "SGB_CLASS_FALLBACK_PCT": "0"}, True),
        ("device-lbvh/grid", {"SGB_TREE": "lbvh"}, True),
        ("device-kd-radix-levels/grid", {"SGB_KD_SMEM": "0"}, True),  # kd refinement with one radix sort per level all the way down
        ("device-kd-radix-levels/no-grid", {"SGB_KD_SMEM": "0", "SGB_GRID": "0"}, True),
        ("host-kd/packet", {"SGB_TREE": "host"}, True),
        ("reference-kd/packet", {}, False),
        ("reference-kd/per-thread", {"SGB_SEARCH": "1"}, False),
        ("host-kd/fused", {"SGB_SEARCH": "0"}, True),
    ):
        for k in switches:
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        ctx = load_ctx(tc, tt, sc, own_tree=own, profiling=True)  # the SGB_* switches only exist in libsgicp_b200_prof.so
        ctx.linearize(np.eye(4))  # also exercises the seeded second search
        H, b, e = ctx.linearize(Tgt)
        results[name] = (H, b, e, ctx.correspondences())
        ctx.close()
    for k in switches:
        monkeypatch.delenv(k, raising=False)
    for name, own in (("product/device-kd", True), ("product/reference-kd", False)):  # the shipped library (no switches) against all of them
        ctx = load_ctx(tc, tt, sc, own_tree=own)
        ctx.linearize(np.eye(4))
        H, b, e = ctx.linearize(Tgt)
        results[name] = (H, b, e, ctx.correspondences())
        ctx.close()
    H0, b0, e0, c0 = results["reference-kd/packet"]
    for name, (H, b, e, c) in results.items():
        assert (c != c0).sum() <= 3, name
        assert np.linalg.norm(H - H0) <= 1e-6 * np.linalg.norm(H0) and abs(e - e0) <= 1e-6 * e0, name


def test_grid_far_and_unbounded_queries(synthetic_pair, monkeypatch):
    """Queries the grid front end cannot settle: a source displaced by metres (nothing within the 2.5-cell ring), no
    rejector at all (unbounded search radius -> tree fallback), a tiny and a huge correspondence distance.  The grid
    path must return what the pure tree search returns."""
    tc, tt, sc, Tgt, nt = synthetic_pair
    sg = _sg()
    far = Tgt.copy()
    far[:3, 3] += np.array([2.5, -1.5, 0.7])
    cases = (
        (Tgt, sg.REJECT_NONE, 0.0),
        (far, sg.REJECT_NONE, 0.0),
        (far, sg.REJECT_DISTANCE, 1.0),
        (far, sg.REJECT_DISTANCE, 25.0),
        (Tgt, sg.REJECT_DISTANCE, 1e-3),
        (Tgt, sg.REJECT_DISTANCE, 400.0),
    )
    out = {}
    for name, env in (("grid", {}), ("tree", {"SGB_GRID": "0"}), ("grid-warp", {"SGB_PENDING_DIV": "1"}), ("grid-packet", {"SGB_PENDING_DIV": "1000000"})):
        for k in ("SGB_GRID", "SGB_PENDING_DIV"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        ctx = load_ctx(tc, tt, sc, own_tree=True, profiling=bool(env))  # "grid" = the product library, the variants need the switches
        res = []
        for T, rej, md in cases:
            H, b, e = ctx.linearize(T, factor=sg.FACTOR_GICP, rejector=rej, max_dist_sq=md)
            res.append((H, e, ctx.correspondences(), ctx.num_inliers()))
        out[name] = res
        ctx.close()
    for name in ("grid", "grid-warp", "grid-packet"):
        for k, ((H, e, c, ni), (H0, e0, c0, ni0)) in enumerate(zip(out[name], out["tree"])):
            assert (c != c0).sum() <= 3, (name, k, int((c != c0).sum()))
            assert abs(ni - ni0) <= 3, (name, k)
            assert np.linalg.norm(H - H0) <= 1e-6 * max(np.linalg.norm(H0), 1e-30) and abs(e - e0) <= 1e-6 * max(e0, 1e-30), (name, k)
    assert out["tree"][1][3] == len(sc)  # no rejector: every source point keeps a correspondence, however far


def test_degenerate_density_stays_exact_and_bounded():
    """Inputs the grid front end must not choke on (kdtree_synthetic_test.cpp:26-93 spirit: clusters, duplicates, huge range):
    half of the target in a 1 cm cluster (a block list of thousands of points: the front end is dropped, kGridMaxList), exact
    duplicates, and two outliers at +-1e5 m that stretch the box (the cell-count bound inflates the cell).  The search must stay
    exact -- brute force on a sample, ICP sums vs numpy -- and finish promptly."""
    import time

    from scipy.spatial import cKDTree

    import np_factors as NF

    sg = _sg()
    rng = np.random.default_rng(11)
    plane = np.c_[rng.uniform(-50, 50, (20_000, 2)), rng.normal(0, 0.01, 20_000)]
    cluster = np.array([3.0, -2.0, 0.5]) + rng.uniform(-0.005, 0.005, (20_000, 3))
    dup = np.repeat(plane[:500], 4, axis=0)
    for extra in (np.zeros((0, 3)), np.array([[1e5, 0.0, 0.0], [-1e5, 2e4, 0.0]])):
        tgt = np.concatenate([plane, cluster, dup, extra]).astype(np.float32).astype(np.float64)
        src = np.concatenate([plane[::2] + rng.normal(0, 0.02, (10_000, 3)), cluster[::4] + rng.normal(0, 0.002, (5_000, 3)), [[40.0, 40.0, 30.0]]])
        src = src.astype(np.float32).astype(np.float64)
        ctx = sg.Context(0)
        ctx.set_target(tgt)
        ctx.build_target_kdtree(0)
        ctx.set_source(src)
        t0 = time.perf_counter()
        T = np.eye(4)
        T[:3, 3] = [0.03, -0.02, 0.01]
        H, b, e = ctx.linearize(T, factor=sg.FACTOR_ICP, rejector=sg.REJECT_DISTANCE, max_dist_sq=1.0)
        dt = time.perf_counter() - t0
        assert dt < 2.0, dt  # a per-thread scan of a 20k-point list per query would take far longer
        corr = ctx.correspondences()
        q = src @ T[:3, :3].T + T[:3, 3]
        d, j = cKDTree(tgt).query(q)
        got = np.where(corr == NF.NO, np.inf, np.linalg.norm(tgt[np.minimum(corr, len(tgt) - 1).astype(np.int64)] - q, axis=1))
        want = np.where(d * d > 1.0, np.inf, d)
        clear = np.abs(d * d - 1.0) > 1e-4
        # same nearest DISTANCE (duplicates / near-ties may pick another index); FP32 search on coordinates centred on a box that the
        # outliers stretch to 2e5 m carries ~8 mm of rounding, on the un-stretched box ~4 um
        tol = 2e-2 if len(extra) else 1e-4
        fin = np.isfinite(want) & np.isfinite(got) & clear
        assert np.all(np.isfinite(want[clear]) == np.isfinite(got[clear]))
        assert np.all(np.abs(got[fin] - want[fin]) <= tol), float(np.abs(got[fin] - want[fin]).max())
        p4 = lambda a: np.c_[a, np.ones(len(a))]
        H2, b2, e2 = NF.linearize(T, corr, sg.FACTOR_ICP, 0, 1.0, p4(src), None, p4(tgt), None, None)
        assert np.linalg.norm(H - H2) <= (1e-3 if len(extra) else 2e-5) * np.linalg.norm(H2)
        assert abs(e - e2) <= (2e-2 if len(extra) else 2e-5) * e2
        assert corr[-1] == NF.NO  # 30 m above everything: rejected
        ctx.close()


def test_full_size_properties():
    """BASELINE config 2 full size (1M x 1M): size-independent properties instead of an oracle run.
      * own-tree NN == brute-force NN on a random sample of queries (exactness)
      * linearity: sums over two disjoint halves of the source add up to the sum over the whole
      * error(T_lin) == e of linearize; H symmetric positive definite
    """
    import torch

    from small_gicp_b200.synthetic import make_pair

    sg = _sg()
    n = 1_000_000
    tgt, src, Tgt = make_pair(n)
    ctx = sg.Context(0)
    ctx.set_target(tgt)
    ctx.build_target_kdtree()
    ctx.set_source(src)
    H, b, e = ctx.linearize(Tgt, factor=sg.FACTOR_ICP)
    corr = ctx.correspondences()
    assert abs(ctx.error(Tgt) - e) <= 1e-9 * e
    assert np.linalg.eigvalsh(H).min() > 0
    # exactness on a sample, brute force in torch on the GPU (float64)
    rng = np.random.default_rng(0)
    sample = rng.choice(n, 2000, replace=False)
    q = torch.tensor((src[sample] @ Tgt[:3, :3].T + Tgt[:3, 3]), device="cuda")
    P = torch.tensor(tgt, device="cuda")
    d2 = torch.cdist(q, P).min(dim=1)
    bf_idx = d2.indices.cpu().numpy()
    bf_d2 = (d2.values.cpu().numpy()) ** 2
    got = corr[sample]
    inl = bf_d2 <= 1.0
    flipped = (got != sg.NO_CORRESPONDENCE) != inl
    assert not flipped.any() or np.abs(bf_d2[flipped] - 1.0).max() < 1e-4
    both = inl & (got != sg.NO_CORRESPONDENCE)
    mism = both & (got != bf_idx.astype(np.uint64))
    if mism.any():
        qq = q.cpu().numpy()[mism]
        dg = ((tgt[got[mism].astype(np.int64)] - qq) ** 2).sum(1)
        assert np.all(np.abs(dg - bf_d2[mism]) <= 1e-5 * bf_d2[mism] + 1e-7)
    assert mism.sum() <= 5
    # linearity over a split of the source
    # (each call re-centres its source box, so FP32 roundings differ slightly between the split and the whole)
    half = n // 2
    ctx.set_source(src[:half])
    Ha, ba, ea = ctx.linearize(Tgt, factor=sg.FACTOR_ICP)
    ctx.set_source(src[half:])
    Hb, bb, eb = ctx.linearize(Tgt, factor=sg.FACTOR_ICP)
    assert np.linalg.norm(Ha + Hb - H) <= 1e-6 * np.linalg.norm(H)
    assert abs(ea + eb - e) <= 1e-6 * e
    ctx.close()
