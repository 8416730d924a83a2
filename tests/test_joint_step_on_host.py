"""The joint window step of sgb_align_joint (sgb_math.cuh: solve_ldlt_n, edge_adjoint, joint_after_linearize / joint_after_error, run by
joint_step_kernel once per window and round) compiled for the HOST (tests/host_joint) with one thread standing for the CTA:
  * solve_ldlt_n at n = 6 is solve_ldlt6 bit for bit, and at n = 6F it matches an FP64 numpy solve to the backward-error bound of the
    replay tests;
  * the edge adjoint is np_joint's;
  * the window state machine, driven by a deterministic reduction (ICP terms of fixed correspondences), makes np_joint's decisions.
No GPU needed."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import np_joint as J
from conftest import ROOT
from np_align import Options
from test_np_joint import _exp

HJ_DIR = os.path.join(ROOT, "tests", "host_joint")
c_dp = ctypes.POINTER(ctypes.c_double)
c_ip = ctypes.POINTER(ctypes.c_int)


class WindowState(ctypes.Structure):
    _fields_ = [("e", ctypes.c_double), ("inliers", ctypes.c_double), ("lam", ctypes.c_double), ("phase", ctypes.c_int), ("it", ctypes.c_int),
                ("trial", ctypes.c_int), ("converged", ctypes.c_int), ("iterations", ctypes.c_int)]


@pytest.fixture(scope="module")
def hj():
    subprocess.check_call(["make", "-s", "-C", HJ_DIR])
    L = ctypes.CDLL(os.path.join(HJ_DIR, "libsgb_host_joint.so"))
    assert L.sgbj_state_size() == ctypes.sizeof(WindowState)
    return L


def _p(a):
    return a.ctypes.data_as(c_dp)


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.uint64), np.asarray(b, dtype=np.float64).view(np.uint64))


def _spd(rng, n, cond=1e6):
    Q, _ = np.linalg.qr(rng.normal(size=(n, n)))
    A = Q @ np.diag(np.geomspace(1.0, 1.0 / cond, n) * rng.uniform(1, 1e4)) @ Q.T
    return np.ascontiguousarray(0.5 * (A + A.T))


def _solve_n(hj, A, b):
    x = np.zeros(A.shape[0])
    hj.sgbj_solve_ldlt_n(A.shape[0], _p(np.ascontiguousarray(A)), _p(np.ascontiguousarray(b)), _p(x))
    return x


def test_solve_ldlt_n_at_6_is_solve_ldlt6_bit_for_bit(hj):
    rng = np.random.default_rng(1)
    systems = [(_spd(rng, 6, 10 ** rng.uniform(0, 8)), rng.normal(size=6) * 10 ** rng.uniform(-3, 3)) for _ in range(200)]
    for r in (0, 1, 3, 5):
        V = rng.normal(size=(6, r))
        systems.append((np.ascontiguousarray(V @ V.T), rng.normal(size=6)))
    systems.append((np.diag([0.0, 3.0, 0.0, 1.0, 0.0, 2.0]), np.ones(6)))
    systems.append((np.diag([1e-3, 1e3, 1.0, 1e2, 1e-1, 1e4]) + 1e-4, rng.normal(size=6)))
    for A, b in systems:
        x6 = np.zeros(6)
        hj.sgbj_solve_ldlt6(_p(np.ascontiguousarray(A)), _p(np.ascontiguousarray(b)), _p(x6))
        assert _bits_equal(_solve_n(hj, A, b), x6), (A, b)


@pytest.mark.parametrize("F", [1, 2, 5, 16, 32])
def test_solve_ldlt_n_matches_numpy(hj, F):
    """backward error |A x - b| <= 1e-10 |A| |x| (the bound of the replay tests' solves), on SPD systems and on a window-shaped system
    (block tridiagonal plus a loop block) of every size"""
    n = 6 * F
    rng = np.random.default_rng(F)
    for k in range(6):
        A = _spd(rng, n, 10 ** (2 + k))
        if k % 2:
            A = A * np.kron(np.eye(F) + np.eye(F, k=1) + np.eye(F, k=-1) + np.eye(F, k=F - 1) + np.eye(F, k=1 - F), np.ones((6, 6))) + n * np.eye(n)
        b = rng.normal(size=n)
        x = _solve_n(hj, A, b)
        ref = np.linalg.solve(A, b)
        assert np.linalg.norm(A @ x - b) <= 1e-10 * np.linalg.norm(A) * np.linalg.norm(x) + 1e-300
        np.testing.assert_allclose(x, ref, rtol=1e-6 * 10 ** (k / 2), atol=1e-8 * np.abs(ref).max())


def test_edge_adjoint_is_the_model(hj):
    rng = np.random.default_rng(2)
    for _ in range(50):
        T = _exp(rng.normal(size=6))
        A = np.zeros(36)
        hj.sgbj_edge_adjoint(_p(np.ascontiguousarray(T.T).reshape(-1)), _p(A))
        np.testing.assert_allclose(A.reshape(6, 6), J.adjoint(T), atol=1e-14)


def _opts(o):
    return np.array([1.0 if o.lm else 0.0, o.max_iterations, o.max_inner_iterations, o.gn_lambda, o.init_lambda, o.lambda_factor, o.rotation_eps,
                     o.translation_eps, *o.dof_mask], dtype=np.float64)


def _problem(seed, F, edges):
    rng = np.random.default_rng(seed)
    truth = [np.eye(4)] + [_exp(np.concatenate([rng.normal(size=3) * 0.2, rng.normal(size=3)])) for _ in range(F - 1)]
    data = []
    for i, j in edges:
        src = rng.normal(size=(15, 3)) * 3.0
        T = J.edge_pose(truth[i], truth[j])
        data.append((src, src @ T[:3, :3].T + T[:3, 3] + rng.normal(size=(15, 3)) * 0.02, None))
    X0 = [truth[0]] + [X @ _exp(rng.normal(size=6) * 0.08) for X in truth[1:]]
    return X0, data


def _host_run(hj, o, X0, fixed, edges, data):
    """the host loop of sgb_align_joint for one window, with the edge reductions computed in numpy at the poses the step writes"""
    F, E = len(X0), len(edges)
    fi, nf = J.free_index(fixed)
    free = np.array(fi, dtype=np.int32)
    ei = np.array([e[0] for e in edges], dtype=np.int32)
    ej = np.array([e[1] for e in edges], dtype=np.int32)
    X = np.ascontiguousarray(np.array([np.asarray(T).T.reshape(-1) for T in X0]))
    cand, delta, sums = X.copy(), np.zeros(6 * max(nf, 1)), np.zeros(44 * max(E, 1))
    s = WindowState()
    ov = _opts(o)
    hj.sgbj_init(_p(ov), nf, E, ctypes.byref(s))
    poses = np.array([J.edge_pose(X0[i], X0[j]).T.reshape(-1) for i, j in edges])
    trace = []
    while s.phase in (0, 1):
        Ts = [p.reshape(4, 4).T for p in poses]
        lin = s.phase == 0
        if lin:
            out = np.zeros((E, 44))
            for q, (T, d) in enumerate(zip(Ts, data)):
                H, b, e = J.edge_terms(T, *d)
                out[q, :36], out[q, 36:42], out[q, 42], out[q, 43] = H.reshape(-1), b, e, 15.0
            trace.append(("lin",))
        else:
            out = np.array([J.edge_error(T, *d) for T, d in zip(Ts, data)])
            lam = s.lam
        out = np.ascontiguousarray(out.reshape(-1))
        it_before = s.it
        hj.sgbj_step(_p(ov), F, free.ctypes.data_as(c_ip), E, ei.ctypes.data_as(c_ip), ej.ctypes.data_as(c_ip), _p(sums), _p(X), _p(cand), _p(delta),
                     ctypes.byref(s), int(lin), _p(out), _p(poses))
        if not lin:
            trace.append(("trial", lam, s.it != it_before))
    return [x.reshape(4, 4).T for x in X], s, trace


@pytest.mark.parametrize("lm", [False, True], ids=["gn", "lm"])
@pytest.mark.parametrize("shape", ["pair", "chain", "loop", "two_fixed"])
@pytest.mark.parametrize("max_iterations", [0, 1, 3, 20])
def test_window_state_machine_matches_the_model(hj, lm, shape, max_iterations):
    F, edges, fixed = {
        "pair": (2, [(1, 0)], [1, 0]),
        "chain": (5, [(1, 0), (2, 1), (3, 2), (4, 3), (2, 0)], [1, 0, 0, 0, 0]),
        "loop": (6, [(1, 0), (2, 1), (3, 2), (4, 3), (5, 4), (0, 5), (3, 1)], [1, 0, 0, 0, 0, 0]),
        "two_fixed": (4, [(0, 1), (2, 1), (3, 2)], [0, 1, 0, 1]),
    }[shape]
    X0, data = _problem(len(shape) * 7 + max_iterations, F, edges)
    o = Options(lm=lm, max_iterations=max_iterations, init_lambda=1e2 if lm else 1e-3)  # a large lambda: some trials are rejected
    lin = lambda Xs: [J.edge_terms(J.edge_pose(Xs[i], Xs[j]), *d) + (15.0,) for (i, j), d in zip(edges, data)]
    err = lambda Xs: [J.edge_error(J.edge_pose(Xs[i], Xs[j]), *d) for (i, j), d in zip(edges, data)]
    ref = J.optimize(lin, err, _exp, X0, fixed, edges, o)
    X, s, trace = _host_run(hj, o, X0, fixed, edges, data)
    ref_trace = [("lin",) if t[0] == "lin" else ("trial", t[1], t[2]) for t in ref.trace if t[0] != "gn"]
    assert len(trace) == len(ref_trace)
    for a, b in zip(trace, ref_trace):
        assert a[0] == b[0]
        if a[0] == "trial":
            assert a[2] == b[2]
            np.testing.assert_allclose(a[1], b[1], rtol=1e-12)
    assert s.phase == 2
    assert bool(s.converged) == ref.converged
    assert s.iterations == ref.iterations
    if max_iterations > 0:
        np.testing.assert_allclose(s.e, ref.error, rtol=1e-9)
        assert s.inliers == ref.inliers
    for k, (a, b) in enumerate(zip(X, ref.X)):
        if fixed[k]:
            assert _bits_equal(a, X0[k])
        np.testing.assert_allclose(a, b, atol=1e-9)


def test_edge_less_free_frame_stays_put(hj):
    """a free frame without an edge: its block is lambda I, its b 0, its step 0"""
    F, edges, fixed = 3, [(1, 0)], [1, 0, 0]
    X0, data = _problem(5, F, edges)
    X0.append(_exp(np.array([0.1, 0.2, 0.3, 1.0, 2.0, 3.0])))
    X, s, _ = _host_run(hj, Options(lm=False, max_iterations=5), X0[:2] + [X0[-1]], fixed, edges, data)
    np.testing.assert_array_equal(X[2], X0[-1])
    assert s.iterations >= 1
