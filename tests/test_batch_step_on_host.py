"""The optimiser step of batched align() (sgb_math.cuh: solve_ldlt6, se3_exp6, pose_mul, align_init / align_after_linearize /
align_after_error, run by batch_step_kernel once per member and round) compiled for the HOST (tests/host_step) next to the C++ host
mirror's solve_ldlt / se3_exp (core.hpp) and GaussNewtonOptimizer / LevenbergMarquardtOptimizer (registration.hpp), both without FMA
contraction: every result must be bit-identical.  The optimisers are driven by one deterministic fake Reduction (H, b, e and error() as
functions of the pose), so the comparison covers the control flow -- lambda carried across outer iterations, `<=` acceptance, the break
when no trial is accepted, iterations = the last outer iteration -- not only the arithmetic.  No GPU needed."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

HS_DIR = os.path.join(ROOT, "tests", "host_step")
c_dp = ctypes.POINTER(ctypes.c_double)


@pytest.fixture(scope="module")
def hm():
    subprocess.check_call(["make", "-s", "-C", HS_DIR])
    return ctypes.CDLL(os.path.join(HS_DIR, "libsgb_host_step.so"))


def _p(a):
    return None if a is None else a.ctypes.data_as(c_dp)


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.uint64), np.asarray(b, dtype=np.float64).view(np.uint64))


def _spd(rng, n=6, cond=1e6):
    Q, _ = np.linalg.qr(rng.normal(size=(n, n)))
    A = Q @ np.diag(np.geomspace(1.0, 1.0 / cond, n) * rng.uniform(1, 1e4)) @ Q.T
    return 0.5 * (A + A.T)


def _solve(hm, H, b, lam, mask=None):
    x1, x2 = np.zeros(6), np.zeros(6)
    H = _f(H)  # symmetric: row- and column-major agree
    hm.sgbm_damped_step(_p(H), _p(_f(b)), ctypes.c_double(lam), _p(None if mask is None else _f(mask)), _p(x1), _p(x2))
    return x1, x2


def _systems():
    rng = np.random.default_rng(11)
    out = [("spd", _spd(rng), rng.normal(size=6) * 10 ** rng.uniform(-3, 3), lam) for lam in (0.0, 1e-6, 1e-3, 10.0) for _ in range(25)]
    for r in (0, 1, 3, 5):  # rank-deficient, all-zero at rank 0
        for lam in (0.0, 1e-6, 1e-3):
            V = rng.normal(size=(6, r))
            out.append((f"rank{r}", V @ V.T, rng.normal(size=6), lam))
    # an exactly singular diagonal (zero pivots) and a permuted-pivot order
    out.append(("zero_pivots", np.diag([0.0, 3.0, 0.0, 1.0, 0.0, 2.0]), np.ones(6), 0.0))
    out.append(("pivoting", np.diag([1e-3, 1e3, 1.0, 1e2, 1e-1, 1e4]) + 1e-4, rng.normal(size=6), 1e-6))
    return out


@pytest.mark.parametrize("mask", [None, [1, 1, 1, 1, 1, 1], [0, 0, 1, 1, 1, 0], [1, 1, 0, 0, 0, 1], [0.5, 1, 2, 1, 0, 1]])
def test_damped_solve_is_bit_identical_to_the_mirror(hm, mask):
    """(H + RestrictDoFFactor term + lambda I) x = -b: random SPD systems over 12 decades of scale, rank-deficient and all-zero H with
    and without damping, zero pivots, and DoF masks (all-ones = NullFactor adds exactly 0)"""
    for name, H, b, lam in _systems():
        x_step, x_mirror = _solve(hm, H, b, lam, mask)
        assert _bits_equal(x_step, x_mirror), (name, lam, mask, x_step, x_mirror)
    if mask is not None and all(m == 1 for m in mask):
        for name, H, b, lam in _systems():
            assert _bits_equal(_solve(hm, H, b, lam, mask)[0], _solve(hm, H, b, lam, None)[1]), name


def test_se3_exp_and_pose_update_are_bit_identical_to_the_mirror(hm):
    rng = np.random.default_rng(5)
    cases = [np.zeros(6), np.array([1e-12, 0, 0, 1, 2, 3]), np.array([1e-6, -2e-6, 3e-6, 0.1, 0, 0]), np.array([0, 0, np.pi, 0, 0, 0])]
    cases += [rng.normal(size=6) * s for s in (1e-5, 1e-3, 0.1, 1.0, 3.0) for _ in range(20)]
    for a in cases:
        T = np.eye(4)
        T[:3, :3] = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        T[:3, 3] = rng.normal(size=3) * 100
        Tc = _f(T.T)
        e1, e2, t1, t2 = np.zeros(16), np.zeros(16), np.zeros(16), np.zeros(16)
        hm.sgbm_pose_update(_p(Tc), _p(_f(a)), _p(e1), _p(e2), _p(t1), _p(t2))
        assert _bits_equal(e1, e2), a
        assert _bits_equal(t1, t2), a


DEFAULT = dict(lm=1, max_iterations=20, max_inner_iterations=10, gn_lambda=1e-6, init_lambda=1e-3, lambda_factor=10.0, rotation_eps=0.1 * np.pi / 180, translation_eps=1e-3)


def _align(hm, T0, target, gain=1.0, bump=0.0, reject_from=10**6, w=(3, 2, 1, 5, 4, 6), coupling=0.3, mask=None, **opt):
    o = dict(DEFAULT, **opt)
    opts = _f([o["lm"], o["max_iterations"], o["max_inner_iterations"], o["gn_lambda"], o["init_lambda"], o["lambda_factor"], o["rotation_eps"], o["translation_eps"],
               0 if mask is None else 1, 0, 0, 0])
    model = _f(list(target) + list(w) + [coupling, gain, bump, reject_from, 1000, 0, 0, 0])
    out1, out2, rounds = np.zeros(62), np.zeros(62), np.zeros(2)
    hm.sgbm_align_fake(_p(opts), _p(_f(np.ones(6) if mask is None else mask)), _p(model), _p(_f(T0.T)), _p(out1), _p(out2), _p(rounds))
    return out1, out2, rounds


def _pose(rng, rot=0.2, trans=1.0):
    T = np.eye(4)
    w = rng.normal(size=3) * rot
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    th = np.linalg.norm(w)
    T[:3, :3] = np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th**2 * K @ K
    T[:3, 3] = rng.normal(size=3) * trans
    return T


def _x(T):
    return np.array([0.5 * (T[2, 1] - T[1, 2]), 0.5 * (T[0, 2] - T[2, 0]), 0.5 * (T[1, 0] - T[0, 1]), *T[:3, 3]])


# name -> (fake model / options, what the script must exercise: converged, iterations, error rounds > 0 and rejections)
SCRIPTS = {
    "lm_plain": dict(gain=1.0),
    "lm_rejected_trials": dict(gain=2.6, bump=0.05),  # overshoot: trials rejected until lambda has grown, lambda carried on
    "lm_break_all_rejected": dict(gain=1.0, reject_from=3),  # from the 3rd linearize on every trial is rejected: the LM break
    "lm_converged_at_0": dict(gain=1.0, at_target=True),  # b = 0
    "lm_out_of_iterations": dict(gain=0.35, max_iterations=4),
    "lm_no_inner_iterations": dict(gain=1.0, max_inner_iterations=0),
    "lm_zero_iterations": dict(gain=1.0, max_iterations=0),
    "lm_dof_mask": dict(gain=1.0, mask=[0, 0, 1, 1, 1, 0]),
    "lm_dof_mask_rejected": dict(gain=2.6, bump=0.05, mask=[1, 1, 0, 0, 0, 1]),
    "gn_plain": dict(lm=0, gain=1.0),
    "gn_converged_at_0": dict(lm=0, gain=1.0, at_target=True),
    "gn_out_of_iterations": dict(lm=0, gain=0.35, max_iterations=5),
    "gn_dof_mask": dict(lm=0, gain=1.0, mask=[0, 0, 1, 1, 1, 0]),
    "gn_zero_iterations": dict(lm=0, gain=1.0, max_iterations=-1),
}


@pytest.mark.parametrize("script", sorted(SCRIPTS))
def test_state_machine_is_bit_identical_to_the_mirror_optimizers(hm, script):
    rng = np.random.default_rng(sum(map(ord, script)))
    kw = dict(SCRIPTS[script])
    at_target = kw.pop("at_target", False)
    lm = kw.get("lm", 1)
    for trial in range(8):
        T0 = _pose(rng)
        target = _x(T0) if at_target else _x(T0) + rng.normal(size=6) * np.array([0.05, 0.05, 0.05, 0.3, 0.3, 0.3])
        s, m, rounds = _align(hm, T0, target, **kw)
        names = ["T"] * 16 + ["converged", "iterations", "num_inliers", "error"] + ["H"] * 36 + ["b"] * 6
        bad = [names[i] for i in range(62) if not _bits_equal(s[i], m[i])]
        assert not bad, (script, trial, sorted(set(bad)), s[16:20], m[16:20])
        conv, it = bool(s[16]), int(s[17])
        if at_target:
            assert conv and it == 0 and _bits_equal(s[:16], _f(T0.T).ravel())
        if script.endswith("zero_iterations"):
            assert not conv and it == 0 and rounds.sum() == 0 and _bits_equal(s[:16], _f(T0.T).ravel()) and s[19] == 0
        if script.endswith("out_of_iterations"):
            assert not conv and it == kw["max_iterations"] - 1
        if script == "lm_rejected_trials":
            assert rounds[1] > rounds[0], rounds  # more trials than linearizes: some were rejected
        if script == "lm_break_all_rejected":
            assert not conv and it == 2 and rounds[0] == 3 and rounds[1] == 2 + DEFAULT["max_inner_iterations"], rounds
        if script == "lm_no_inner_iterations":
            assert not conv and it == 0 and rounds[1] == 0
        if not lm:
            assert rounds[1] == 0 and rounds[0] == (it + 1 if kw.get("max_iterations", 1) > 0 else 0)
