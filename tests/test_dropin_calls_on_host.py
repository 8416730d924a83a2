"""The call-by-call checker of the drop-in (tests/np_dropin.py) on the host: it accepts the logs of the reference's own
ParallelReductionOMP against the same FP64 models at 1e-9, and it rejects six planted faults, each with a message naming the call and
the quantity.  The CUDA arm's logs are checked in tests/test_gpu_dropin_calls.py."""
import copy
import os

import numpy as np
import pytest
from scipy.spatial import cKDTree

import np_dropin as D
import np_factors as NF
from conftest import ROOT, noise_poses

LIB = os.path.join(ROOT, "oracle", "_ref", "libsgb_host_ref.so")
OMP = 0


@pytest.fixture(scope="module")
def lib():
    return D.load_harness(LIB)


def omp_log(lib, g, **kw):
    t, s = g["target"], g["source"]
    return D.run(lib, OMP, t.points, t.normals, t.covs, s.points, s.covs, **kw)


CASES = {
    "gicp_lm_kdtree": dict(init_T=noise_poses()[1]),
    "icp_gn_unsafe_leaf1": dict(factor=0, optimizer=0, structure=1, max_leaf_size=1, init_T=noise_poses()[2]),
    "plane_huber_omp_tree": dict(factor=1, robust=1, robust_c=0.5, structure=2, max_leaf_size=33),
    "gicp_cauchy_null_f32": dict(robust=2, robust_c=0.5, max_dist_sq=None, cloud_type=1, max_iterations=6),
    "vgicp_27_lru": dict(structure=3, voxel_resolution=0.3, offsets=27, lru_horizon=1, lru_clear_cycle=2,
                         insert_poses=np.tile(np.eye(4), (4, 1, 1)), init_T=noise_poses()[1]),
    "kd_map_kd": dict(scenario=1, voxel_resolution=1.0, offsets=7, robust=1, robust_c=0.7, max_iterations=5),
}


@pytest.fixture(scope="module")
def logs(lib, golden_prepared):
    return {name: omp_log(lib, golden_prepared, **kw) for name, kw in CASES.items()}


@pytest.mark.parametrize("name", list(CASES))
def test_checker_accepts_the_omp_arm(logs, name):
    prob, log = logs[name]
    ck = D.check(prob, log, exact=True)
    lin = sum(c.kind == 0 for c in log.calls)
    assert lin >= 2 and ck.checked == len(log.calls), name
    assert ck.worst <= 1e-9
    if CASES[name].get("max_dist_sq", 1.0) is not None:
        assert any((c.corr == NF.NO).any() for c in log.calls if c.kind == 0) or name == "kd_map_kd"
    print(f"{name}: {ck.checked} calls, worst {ck.worst:.3g}")


def _copy(logs, name):
    """a planted fault goes into a copy: every test starts from the clean log"""
    prob, log = logs[name]
    return prob, copy.deepcopy(log)


def _first(log, kind, align=None):
    return next(j for j, c in enumerate(log.calls) if c.kind == kind and (align is None or c.align == align))


def _fails(prob, log, pattern):
    with pytest.raises(AssertionError, match=pattern):
        D.check(prob, log, exact=True)


def test_rejects_second_nearest_target_index(logs):
    prob, log = _copy(logs, "gicp_lm_kdtree")
    j = _first(log, 0)
    c = log.calls[j]
    q = prob.src_pts[:, :3] @ c.T[:3, :3].T + c.T[:3, 3]
    i = int(np.nonzero(c.corr != NF.NO)[0][5])
    _, k = cKDTree(prob.tgt_pts[:, :3]).query(q[i], k=2)
    c.corr[i] = c.target_index[i] = np.uint64(k[1])
    _fails(prob, log, rf"call {j} \(linearize\): correspondences")


def test_rejects_transposed_h_rt(logs):
    prob, log = _copy(logs, "gicp_lm_kdtree")
    j = _first(log, 0)
    H = log.calls[j].H
    H[0:3, 3:6], H[3:6, 0:3] = H[0:3, 3:6].T.copy(), H[3:6, 0:3].T.copy()
    _fails(prob, log, rf"call {j} \(linearize\): H off the model")


def test_rejects_a_dropped_point(logs):
    prob, log = _copy(logs, "icp_gn_unsafe_leaf1")
    ck = D.Checker(prob, log, exact=True)
    j = [k for k, c in enumerate(log.calls) if c.kind == 0][1]
    c = log.calls[j]
    ids = ck.ids(j).copy()
    ids[int(np.nonzero(ids != NF.NO)[0][-1])] = NF.NO
    c.H, c.b, c.e = NF.linearize(c.T, ids, prob.factor, prob.robust, prob.robust_c, *ck.inputs(False))
    _fails(prob, log, rf"call {j} \(linearize\): H off the model")


def test_rejects_error_at_the_linearisation_pose(logs):
    prob, log = _copy(logs, "gicp_lm_kdtree")
    ck = D.Checker(prob, log, exact=True)
    j = _first(log, 1)
    lin = max(k for k in range(j) if log.calls[k].kind == 0)
    L = log.calls[lin]
    log.calls[j].e = NF.error(L.T, L.T, ck.ids(lin), prob.factor, prob.robust, prob.robust_c, *ck.inputs(False))
    _fails(prob, log, rf"call {j} \(error\): e off the model")


def test_rejects_a_voxel_index_off_by_one(logs):
    prob, log = _copy(logs, "vgicp_27_lru")
    j = _first(log, 0)
    c = log.calls[j]
    i = int(np.nonzero(c.corr != NF.NO)[0][3])
    c.corr[i] = c.target_index[i] = c.corr[i] + np.uint64(1 << 32)
    _fails(prob, log, rf"call {j} \(linearize\): correspondences")


def test_rejects_a_lost_robust_weight(logs):
    prob, log = _copy(logs, "plane_huber_omp_tree")
    ck = D.Checker(prob, log, exact=True)
    j = [k for k, c in enumerate(log.calls) if c.kind == 0][-1]
    c = log.calls[j]
    c.H, c.b, c.e = NF.linearize(c.T, ck.ids(j), prob.factor, 0, prob.robust_c, *ck.inputs(False))
    _fails(prob, log, rf"call {j} \(linearize\): H off the model")


def test_voxel_map_was_evicted_and_reordered(logs):
    """the LRU case really evicts: a map of the whole cloud at once has voxels the evicted map lacks"""
    prob, log = _copy(logs, "vgicp_27_lru")
    from np_preprocess import voxelmap_model

    full = voxelmap_model(prob.tgt_pts, None, 0.3)[0]
    assert 0 < len(log.vox_coords) < len(full)
