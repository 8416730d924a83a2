"""The per-point arithmetic the CUDA kernels inline (small_gicp_b200/csrc/sgb_math.cuh) compiled for the HOST from the same
source (tests/host_math) and held against the oracle and the numpy leg -- no GPU needed.

What this pins on a CPU-only machine: the source-frame factor algebra of factor_reduce_kernel (D = R^T M R), the target-frame
one of the fused / voxel kernels, the GICP precision matrix, the robust kernels, the rejector on the FP64 residual, the
error() semantics (precision frozen at the linearisation pose, gicp_factor.hpp:81-89), the layout of the 28 compact sums in
H | b | e, and the FP32 storage model (centred FP32 coordinates, 6 FP32 covariance entries).  What it cannot pin: the search,
the memory pipeline and the reductions -- those are the `-m gpu` tests."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import np_factors as NF
import oracle as O
from conftest import ROOT, noise_poses

HM_DIR = os.path.join(ROOT, "tests", "host_math")
c_dp = ctypes.POINTER(ctypes.c_double)


@pytest.fixture(scope="module")
def hm():
    subprocess.check_call(["make", "-s", "-C", HM_DIR])
    lib = ctypes.CDLL(os.path.join(HM_DIR, "libsgb_host_math.so"))
    lib.sgbm_linearize_pairs.restype = ctypes.c_int
    lib.sgbm_error_pairs.restype = ctypes.c_int
    return lib


def _p(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(c_dp)


def _colmajor(T):
    return np.ascontiguousarray(T.T, dtype=np.float64)


class Pairs:
    """matched pairs (source i <-> target corr[i]) of the golden clouds at pose T, in the reference's host layout"""

    def __init__(self, g, corr):
        tc, sc = g["target"], g["source"]
        self.idx = np.nonzero(corr != NF.NO)[0]
        k = corr[self.idx].astype(np.int64)
        self.sp = np.ascontiguousarray(sc.points[self.idx])
        self.sc = np.ascontiguousarray(sc.covs[self.idx])
        self.tp = np.ascontiguousarray(tc.points[k])
        self.tn = np.ascontiguousarray(tc.normals[k])
        self.tcv = np.ascontiguousarray(tc.covs[k])
        # the device centres every cloud on its bounding-box centre (FP64)
        self.cs = 0.5 * (sc.points[:, :3].min(0) + sc.points[:, :3].max(0))
        self.ct = 0.5 * (tc.points[:, :3].min(0) + tc.points[:, :3].max(0))
        self.n = len(self.idx)

    def linearize(self, lib, T, factor, robust, c, max_d2, frame, want_accepted=False):
        out = np.zeros(44)
        acc = np.zeros(self.n, dtype=np.uint8) if want_accepted else None
        # covariances travel as Matrix4d column-major; they are symmetric, so the row-major numpy block is the same bytes
        rc = lib.sgbm_linearize_pairs(
            factor, robust, ctypes.c_double(c), ctypes.c_double(max_d2), _p(_colmajor(T)), _p(self.cs), _p(self.ct), ctypes.c_size_t(self.n),
            _p(self.sp), _p(self.sc), _p(self.tp), _p(self.tn), _p(self.tcv), frame, _p(out), None if acc is None else acc.ctypes.data_as(ctypes.POINTER(ctypes.c_ubyte)))
        assert rc == 0
        return out[:36].reshape(6, 6), out[36:42], out[42], int(out[43]), acc

    def error(self, lib, T, Tlin, factor, robust, c):
        e = ctypes.c_double(0.0)
        rc = lib.sgbm_error_pairs(factor, robust, ctypes.c_double(c), _p(_colmajor(T)), _p(_colmajor(Tlin)), _p(self.cs), _p(self.ct), ctypes.c_size_t(self.n),
                                  _p(self.sp), _p(self.sc), _p(self.tp), _p(self.tn), _p(self.tcv), ctypes.byref(e))
        assert rc == 0
        return e.value


def storage_model(P):
    return NF.storage_model(P.sp, P.sc, P.tp, P.tn, P.tcv, P.cs, P.ct)


CASES = [(f, r) for f in (0, 1, 2) for r in (0, 1, 2)]


@pytest.mark.parametrize("factor,robust", CASES)
def test_kernel_arithmetic_matches_oracle_and_numpy(hm, golden_prepared, factor, robust):
    g = golden_prepared
    tc, sc = g["target"], g["source"]
    reg = O.Registration(factor=factor, robust=robust, robust_c=0.7, num_threads=0)
    for T in (np.eye(4), NF.orthonormal(g["T"]), noise_poses()[2]):
        H0, b0, e0 = reg.linearize(tc, g["target_tree"], sc, T)
        corr = reg.correspondences(len(sc))
        P = Pairs(g, corr)
        assert P.n > 1000
        for frame in (0, 1):
            H, b, e, n_in, _ = P.linearize(hm, T, factor, robust, 0.7, 1.0, frame)
            assert n_in == P.n
            assert np.array_equal(H, H.T)  # the expansion mirrors the upper triangle exactly (registration_test.cpp:220-224 asks for 1e-3)
            # 1. against the oracle on the FP64 inputs: the GPU parity tolerance (FP32 storage of coordinates / covariances)
            assert np.linalg.norm(H - H0) <= 2e-5 * np.linalg.norm(H0), (frame, np.linalg.norm(H - H0) / np.linalg.norm(H0))
            assert abs(e - e0) <= 2e-5 * e0
            assert np.abs(b - b0).max() <= 2e-5 * np.sqrt(2 * e0 * np.diag(H0)).max()
            # 2. against numpy on the SAME FP32-rounded inputs: pure algebra, FP64 rounding only
            sp, scv, tp, tn, tcv = storage_model(P)
            ident = np.arange(P.n).astype(np.uint64)
            H2, b2, e2 = NF.linearize(T, ident, factor, robust, 0.7, sp, scv, tp, tn, tcv)
            assert np.linalg.norm(H - H2) <= 1e-9 * np.linalg.norm(H2), (frame, np.linalg.norm(H - H2) / np.linalg.norm(H2))
            assert abs(e - e2) <= 1e-9 * e2
            assert np.abs(b - b2).max() <= 1e-9 * np.sqrt(2 * e2 * np.diag(H2)).max()
        # error(): trial pose, precision frozen at the linearisation pose; error(T_lin) == e of linearize
        T2 = T @ O.se3_exp(np.array([0.01, -0.02, 0.005, 0.05, -0.03, 0.02]))
        e_trial0 = reg.error(tc, sc, T2)
        e_trial = P.error(hm, T2, T, factor, robust, 0.7)
        assert abs(e_trial - e_trial0) <= 2e-5 * e_trial0
        sp, scv, tp, tn, tcv = storage_model(P)
        assert abs(e_trial - NF.error(T2, T, np.arange(P.n).astype(np.uint64), factor, robust, 0.7, sp, scv, tp, tn, tcv)) <= 1e-9 * e_trial
        e_same = P.error(hm, T, T, factor, robust, 0.7)
        H, b, e, _, _ = P.linearize(hm, T, factor, robust, 0.7, 1.0, 0)
        assert abs(e_same - e) <= 1e-12 * e


def test_rejector_is_strict_on_the_fp64_residual(hm, golden_prepared):
    """rejector.hpp:24: reject iff d2 > max_dist_sq.  Pairs are taken WITHOUT a rejector, then the arithmetic applies it."""
    g = golden_prepared
    tc, sc = g["target"], g["source"]
    T = noise_poses()[1]
    reg = O.Registration(factor=0, rejector=O.REJECT_NONE, num_threads=0)
    reg.linearize(tc, g["target_tree"], sc, T)
    P = Pairs(g, reg.correspondences(len(sc)))
    sp, _, tp, _, _ = storage_model(P)
    d2 = (((sp[:, :3] @ T[:3, :3].T + T[:3, 3]) - tp[:, :3]) ** 2).sum(1)
    for max_d2 in (0.05, 0.25, 1.0):
        _, _, _, n_in, acc = P.linearize(hm, T, 0, 0, 1.0, max_d2, 0, want_accepted=True)
        clear = np.abs(d2 - max_d2) > 1e-9  # pairs within rounding of the threshold may go either way
        assert np.array_equal(acc[clear].astype(bool), (d2 <= max_d2)[clear])
        assert n_in == int(acc.sum())
    # a pair exactly on the threshold is kept (strict >): one point at distance 1 along x, max_dist_sq = 1
    one = np.array([[0.0, 0.0, 0.0, 1.0]]), np.array([[1.0, 0.0, 0.0, 1.0]])
    out = np.zeros(44)
    z3, zc, zn = np.zeros(3), np.zeros((1, 4, 4)), np.zeros((1, 4))
    for max_d2, kept in ((1.0, 1), (np.nextafter(1.0, 0.0), 0)):
        assert hm.sgbm_linearize_pairs(0, 0, ctypes.c_double(1.0), ctypes.c_double(max_d2), _p(_colmajor(np.eye(4))), _p(z3), _p(z3), ctypes.c_size_t(1),
                                       _p(one[0]), _p(zc), _p(one[1]), _p(zn), _p(zc), 0, _p(out), None) == 0
        assert int(out[43]) == kept


def _random_rotation(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


@pytest.mark.parametrize("seed", range(6))
def test_kernel_arithmetic_on_random_inputs(hm, seed):
    """Beyond the golden clouds: arbitrary rotations (not just small ones), clouds hundreds of metres from the origin (the centring is what
    keeps FP32 storage accurate there), covariances with the reference's (1e-3, 1, 1) spectrum in random orientations, robust-kernel widths
    that put points on both sides of the Huber knee, and a rejector radius that cuts through the residual distribution."""
    rng = np.random.default_rng(100 + seed)
    n = 4000
    offset = rng.uniform(-400, 400, 3)
    tp = np.c_[rng.uniform(-30, 30, (n, 3)) + offset, np.ones(n)]
    T = np.eye(4)
    T[:3, :3] = _random_rotation(rng)
    T[:3, 3] = rng.uniform(-5, 5, 3)
    res = rng.normal(0, 0.3, (n, 3))  # residual target - T * source
    sp = np.c_[(tp[:, :3] - res - T[:3, 3]) @ T[:3, :3], np.ones(n)]  # R^T (q - t)

    def covs():
        out = np.zeros((n, 4, 4))
        for i in range(n):
            V = _random_rotation(rng)
            out[i, :3, :3] = V @ np.diag([1e-3, 1.0, 1.0]) @ V.T
        return out

    scv, tcv = covs(), covs()
    tn = np.c_[np.stack([_random_rotation(rng)[:, 0] for _ in range(n)]), np.zeros(n)]

    P = Pairs.__new__(Pairs)  # matched pairs given directly, not taken from the golden clouds
    P.sp, P.sc, P.tp, P.tn, P.tcv, P.n = sp, scv, tp, tn, tcv, n
    P.cs = 0.5 * (sp[:, :3].min(0) + sp[:, :3].max(0))
    P.ct = 0.5 * (tp[:, :3].min(0) + tp[:, :3].max(0))
    spm, scm, tpm, tnm, tcm = storage_model(P)
    d2 = (((spm[:, :3] @ T[:3, :3].T + T[:3, 3]) - tpm[:, :3]) ** 2).sum(1)
    max_d2 = float(np.quantile(d2, 0.8))
    keep = d2 <= max_d2
    clear = np.abs(d2 - max_d2) > 1e-9
    ident = np.arange(n).astype(np.uint64)
    corr = np.where(keep, ident, NF.NO)
    for factor in (0, 1, 2):
        for robust, c in ((0, 1.0), (1, 0.35), (2, 0.5)):
            for frame in (0, 1):
                H, b, e, n_in, acc = P.linearize(hm, T, factor, robust, c, max_d2, frame, want_accepted=(frame == 0))
                if frame == 0:
                    assert np.array_equal(acc[clear].astype(bool), keep[clear])
                assert abs(n_in - int(keep.sum())) <= int((~clear).sum())
                H2, b2, e2 = NF.linearize(T, corr, factor, robust, c, spm, scm, tpm, tnm, tcm)
                assert np.linalg.norm(H - H2) <= 1e-9 * np.linalg.norm(H2), (factor, robust, frame)
                assert abs(e - e2) <= 1e-9 * e2 and np.abs(b - b2).max() <= 1e-9 * np.sqrt(2 * e2 * np.diag(H2)).max()
            T2 = T @ O.se3_exp(rng.normal(0, 0.02, 6))
            e_t = P.error(hm, T2, T, factor, robust, c)
            assert abs(e_t - NF.error(T2, T, ident, factor, robust, c, spm, scm, tpm, tnm, tcm)) <= 1e-9 * e_t
