import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


def pytest_sessionstart(session):
    """A fresh checkout has no built artefacts (they are git-ignored): build them once (nvcc cross-compiles without a GPU).  Only when
    something is MISSING -- libraries built elsewhere and copied in with the tree must not be rebuilt because of clock skew."""
    needed = [
        os.path.join(ROOT, "small_gicp_b200", "lib", "libsgicp_b200.so"),
        os.path.join(ROOT, "small_gicp_b200", "lib", "libsgicp_b200_prof.so"),
        os.path.join(ROOT, "small_gicp_b200", "lib", "libsgicp_b200_host.so"),
        os.path.join(ROOT, "oracle", "libsgicp_oracle.so"),
    ]
    if all(os.path.exists(p) for p in needed):
        return
    import __graft_entry__

    __graft_entry__.build()


def load_golden_xyz(name):
    return np.fromfile(os.path.join(GOLDEN, name + "_xyz.f32"), dtype="<f4").reshape(-1, 3).astype(np.float64)


def pose_error(T1, T2):
    """registration_test.cpp:139-151: angle of R1^T R2, norm of the translation of T1^-1 T2"""
    e = np.linalg.inv(T1) @ T2
    ang = np.arccos(np.clip((np.trace(e[:3, :3]) - 1.0) / 2.0, -1.0, 1.0))
    return float(ang), float(np.linalg.norm(e[:3, 3]))


@pytest.fixture(scope="session")
def golden():
    T = np.loadtxt(os.path.join(GOLDEN, "T_target_source.txt")).reshape(4, 4)
    return load_golden_xyz("target"), load_golden_xyz("source"), T


@pytest.fixture(scope="session")
def golden_prepared(golden):
    """registration_test.cpp:29-58 SetUp: 0.3 m voxelgrid, k=20 normals+covariances, trees, voxel maps."""
    import oracle as O

    tgt, src, T = golden
    tc = O.Cloud(tgt).voxelgrid_sampling(0.3)
    sc = O.Cloud(src).voxelgrid_sampling(0.3)
    tt, st = O.KdTree(tc), O.KdTree(sc)
    nt = max(1, min(4, O.max_threads()))
    tt.estimate(20, O.FEAT_NORMAL_COV, nt)
    st.estimate(20, O.FEAT_NORMAL_COV, nt)
    return {"target": tc, "source": sc, "target_tree": tt, "source_tree": st, "T": T}


def noise_poses():
    """registration_test.cpp:60-71 analogue: identity + 3 random poses <= 0.5 m / <= 10 deg (our own fixed seed)."""
    rng = np.random.default_rng(7)
    out = [np.eye(4)]
    for _ in range(3):
        T = np.eye(4)
        T[:3, 3] = rng.uniform(-1, 1, 3) * 0.5
        ang = rng.uniform(-1, 1) * np.deg2rad(10.0)
        ax = rng.uniform(-1, 1, 3)
        ax /= np.linalg.norm(ax)
        K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
        T[:3, :3] = np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * (K @ K)
        out.append(T)
    return out
