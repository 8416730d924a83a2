"""The drop-in call by call on the GPU: the reference's Registration<> on ParallelReductionCUDA (include/small_gicp/registration/
reduction_cuda.hpp) logged by href_align_log, every linearize() / error() held to the FP64 models at np_factors.TIGHT by
tests/np_dropin.py, the same run on the reference's ParallelReductionOMP held to them at 1e-9, and the two logs held to each other.

The matrix covers every factor x robust kernel, GN and LM, NullRejector and DistanceRejector, every search structure the reference
offers (KdTree with max_leaf_size 1 / 20 / 33 / 64 / 300 / > n, UnsafeKdTree, a KdTreeBuilderOMP tree, GaussianVoxelMap with leaf 0.3 /
1.0, 1 / 7 / 27 offsets and LRU eviction), PointCloud and a cloud type reached only through traits, sync_every_linearize = false,
one reduction aligning against a kd-tree, a voxel map and the kd-tree again, and two Registrations sharing one context through
use_context(), on the golden pair, the golden pair at UTM-like coordinates, a scene in the negative octant, a target of duplicated
points (exact ties) and a 200k-point synthetic pair.  Each case prints its worst TIGHT ratio (run with -s)."""
import os
import time

import numpy as np
import pytest

import np_dropin as D
import np_factors as NF
from conftest import ROOT, noise_poses

pytestmark = pytest.mark.gpu

LIB = os.path.join(ROOT, "oracle", "_ref", "libsgb_host_ref.so")
OMP, CUDA = 0, 1
UTM = np.array([5e5, 5e6, 120.0])
# The FP64 model works in world coordinates: at |x| = 5e6 m its own residuals round by ~u |x| = 6e-10 m against residuals of a few
# cm, which puts its sums ~1e-8 off exact at worst; the device works relative to the clouds' centres.  Elsewhere: np_factors.TIGHT.
UTM_TOL = 1e-8
TOTALS = {"cases": 0, "calls": 0, "worst": 0.0, "seconds": 0.0}


@pytest.fixture(scope="module")
def lib():
    return D.load_harness(LIB)


def _moved(c, offset):
    p = np.array(c.points, dtype=np.float64)
    p[:, :3] += offset
    return p


@pytest.fixture(scope="module")
def scenes(golden_prepared):
    """scene name -> (target points, normals, covs, source points, covs)"""
    g = golden_prepared
    t, s = g["target"], g["source"]
    out = {"golden": (t.points, t.normals, t.covs, s.points, s.covs)}
    out["utm"] = (_moved(t, UTM), t.normals, t.covs, _moved(s, UTM), s.covs)
    neg = -np.maximum(t.points[:, :3].max(0), s.points[:, :3].max(0)) - 3.0  # every coordinate of both clouds below -3
    out["negative"] = (_moved(t, neg), t.normals, t.covs, _moved(s, neg), s.covs)
    out["duplicated"] = tuple(np.concatenate([a, a]) for a in (t.points, t.normals, t.covs)) + (s.points, s.covs)
    return out


@pytest.fixture(scope="module")
def big():
    import oracle as O
    from small_gicp_b200.synthetic import make_pair

    tgt, src, _ = make_pair(200_000)
    tc, sc = O.Cloud(tgt), O.Cloud(src)
    O.KdTree(tc).estimate(20, O.FEAT_NORMAL_COV, 4)
    O.KdTree(sc).estimate(20, O.FEAT_COV, 4)
    return (tc.points, tc.normals, tc.covs, sc.points, sc.covs)


LRU = dict(insert_poses=np.tile(np.eye(4), (4, 1, 1)), lru_horizon=1, lru_clear_cycle=2)
CASES = [
    ("golden", "gicp_lm_kd20", dict(init_T=noise_poses()[1])),
    ("golden", "icp_huber_gn_kd1", dict(factor=0, robust=1, robust_c=0.5, optimizer=0, max_leaf_size=1, init_T=noise_poses()[2])),
    ("golden", "icp_cauchy_lm_null_kdn", dict(factor=0, robust=2, robust_c=0.5, max_dist_sq=None, max_leaf_size=1 << 20, max_iterations=8)),
    ("golden", "plane_lm_unsafe64", dict(factor=1, structure=1, max_leaf_size=64, init_T=noise_poses()[3])),
    ("golden", "plane_cauchy_gn_null_kd300", dict(factor=1, robust=2, robust_c=0.5, optimizer=0, max_dist_sq=None, max_leaf_size=300, max_iterations=8)),
    ("golden", "gicp_cauchy_gn_omptree33_f32", dict(robust=2, robust_c=0.7, optimizer=0, structure=2, max_leaf_size=33, cloud_type=1)),
    ("golden", "gicp_huber_lm_unsafe1_f32", dict(robust=1, robust_c=0.7, structure=1, max_leaf_size=1, cloud_type=1, init_T=noise_poses()[1])),
    ("golden", "vgicp_lm_1.0_o1_f32", dict(structure=3, voxel_resolution=1.0, offsets=1, cloud_type=1)),
    ("golden", "vgicp_gn_0.3_o27_lru", dict(structure=3, voxel_resolution=0.3, offsets=27, optimizer=0, **LRU)),
    ("golden", "gicp_lm_nosync", dict(sync=False, init_T=noise_poses()[1])),
    ("utm", "gicp_lm_kd20", dict(init_T=noise_poses()[2])),
    ("utm", "vgicp_huber_gn_1.0_o27", dict(structure=3, voxel_resolution=1.0, offsets=27, robust=1, robust_c=0.7, optimizer=0)),
    ("negative", "plane_huber_gn_unsafe20", dict(factor=1, robust=1, robust_c=0.5, optimizer=0, structure=1)),
    ("negative", "vgicp_cauchy_lm_0.3_o7_lru", dict(structure=3, voxel_resolution=0.3, offsets=7, robust=2, robust_c=0.7, **LRU)),
    ("duplicated", "icp_lm_kd20", dict(factor=0)),
    ("duplicated", "plane_gn_kd33", dict(factor=1, optimizer=0, max_leaf_size=33)),
    ("golden", "kd_map_kd", dict(scenario=1, voxel_resolution=1.0, offsets=7)),
    ("golden", "kd_map_kd_gen7", dict(scenario=1, voxel_resolution=1.0, offsets=7, generation=7)),
    ("golden", "shared_ctx", dict(scenario=2, voxel_resolution=0.3, offsets=27, robust=1, robust_c=0.7)),
    ("golden", "shared_ctx_gen7", dict(scenario=2, voxel_resolution=0.3, offsets=27, robust=1, robust_c=0.7, generation=7)),
    ("big", "gicp_lm_kd20", dict(max_iterations=5, init_T=noise_poses()[1])),
    ("big", "vgicp_gn_1.0_o1", dict(structure=3, voxel_resolution=1.0, optimizer=0, max_iterations=5)),
]


def _scene(scenes, big, name):
    return big if name == "big" else scenes[name]


def run_case(lib, data, kw, tol):
    t0 = time.perf_counter()
    prob, log = D.run(lib, CUDA, *data, **kw)
    ck = D.check(prob, log, tol=tol)
    oprob, olog = D.run(lib, OMP, *data, **kw)
    D.check(oprob, olog, exact=True)
    agreed = D.compare_arms(prob, log, olog)
    return prob, log, ck, agreed, time.perf_counter() - t0


@pytest.mark.parametrize("scene,name,kw", CASES, ids=[f"{s}-{n}" for s, n, _ in CASES])
def test_every_call_against_the_models(lib, scenes, big, scene, name, kw):
    tol = UTM_TOL if scene == "utm" else NF.TIGHT
    if scene == "utm" and "init_T" in kw:  # the same initial error as at the origin: the noise pose taken about the moved scene
        shift = np.eye(4)
        shift[:3, 3] = UTM
        kw = dict(kw, init_T=shift @ kw["init_T"] @ np.linalg.inv(shift))
    prob, log, ck, agreed, secs = run_case(lib, _scene(scenes, big, scene), kw, tol)
    inliers = [int((c.corr != D.NO).sum()) for c in log.calls if c.kind == 0]
    assert min(inliers) > 0 and max(inliers) > len(prob.src_pts) // 10, (scene, name, inliers)  # sums worth checking in every call
    TOTALS["cases"] += 1
    TOTALS["calls"] += ck.checked
    TOTALS["worst"] = max(TOTALS["worst"], ck.worst / tol)
    TOTALS["seconds"] += secs
    print(f"{scene}/{name}: {ck.checked} calls, worst ratio {ck.worst / tol:.3g} of its limit {tol:.0e}, arms agree for {agreed} calls, {secs:.1f} s; "
          f"totals {TOTALS}")


def _logged(log):
    """every logged quantity of a run, for the non-vacuity comparisons"""
    parts = [np.r_[c.T.ravel(), c.H.ravel(), c.b, c.e] for c in log.calls]
    parts += [np.r_[c.source_index, c.target_index, c.corr].astype(np.float64) for c in log.calls if c.kind == 0]
    parts += [np.r_[a[0], a[1].ravel(), a[2:]] for a in log.aligns]
    return parts


def _differ(a, b):
    pa, pb = _logged(a), _logged(b)
    return len(pa) != len(pb) or any(x.shape != y.shape or not np.array_equal(x, y) for x, y in zip(pa, pb))


BASE = dict(init_T=noise_poses()[1], max_iterations=6)
FLIPS = {
    "factor": dict(factor=1), "robust": dict(robust=1, robust_c=0.5), "optimizer": dict(optimizer=0), "rejector": dict(max_dist_sq=None),
    "cloud type": dict(cloud_type=1), "sync": dict(sync=False), "voxel map": dict(structure=3), "scenario 1": dict(scenario=1),
    "scenario 2": dict(scenario=2),
}
MAP_FLIPS = {"leaf": dict(voxel_resolution=0.3), "offsets": dict(offsets=27), "eviction": LRU}


def test_every_option_changes_the_log(lib, scenes):
    """flipping one option at a time changes at least one logged quantity: none of them is ignored on the way to the device"""
    data = scenes["golden"]
    _, base = D.run(lib, CUDA, *data, **BASE)
    for what, kw in FLIPS.items():
        _, log = D.run(lib, CUDA, *data, **BASE, **kw)
        assert _differ(base, log), what
    vbase = dict(BASE, structure=3)
    _, vlog = D.run(lib, CUDA, *data, **vbase)
    for what, kw in MAP_FLIPS.items():
        _, log = D.run(lib, CUDA, *data, **vbase, **kw)
        assert _differ(vlog, log), what
