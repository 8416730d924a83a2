"""The numpy model of joint window registration (np_joint) against finite differences: on small synthetic windows with fixed
correspondences, the assembled b is the gradient of E(X) = sum over edges of the factor error at X_j^-1 X_i with respect to every free
frame's right perturbation, and (ICP) the assembled H is J^T J of the finite-difference residual Jacobian.  This pins the sign and the
ordering conventions of A_e = -Ad(T_e^-1).  No GPU."""
import numpy as np
import pytest

import np_joint as J


def _exp(d):
    """SE(3) exp of [r; t] (the reference's se3_exp: the rotation's exponential and its left Jacobian)"""
    w, v = np.asarray(d[:3], dtype=np.float64), np.asarray(d[3:], dtype=np.float64)
    th = np.linalg.norm(w)
    K = J.skew(w)
    if th < 1e-12:
        R, V = np.eye(3) + K, np.eye(3) + 0.5 * K
    else:
        R = np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th**2 * K @ K
        V = np.eye(3) + (1 - np.cos(th)) / th**2 * K + (th - np.sin(th)) / th**3 * K @ K
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, V @ v
    return T


def _window(rng, F, edges, gicp):
    """frames at random poses, each edge with its own fixed correspondences (source in frame i, target in frame j) and weights"""
    Xs = [np.eye(4)] + [_exp(np.concatenate([rng.normal(size=3) * 0.3, rng.normal(size=3)])) for _ in range(F - 1)]
    data = []
    for i, j in edges:
        n = 12
        src = rng.normal(size=(n, 3)) * 2.0
        tgt = np.array([(J.edge_pose(Xs[i], Xs[j]) @ np.append(p, 1.0))[:3] for p in src]) + rng.normal(size=(n, 3)) * 0.05
        M = None
        if gicp:
            A = rng.normal(size=(n, 3, 3))
            M = np.einsum("nij,nkj->nik", A, A) + 0.1 * np.eye(3)
        data.append((src, tgt, M))
    # perturb the frames so that the gradient is not ~0
    Xs = [Xs[0]] + [X @ _exp(rng.normal(size=6) * 0.05) for X in Xs[1:]]
    return Xs, data


def _energy(Xs, edges, data):
    return sum(J.edge_error(J.edge_pose(Xs[i], Xs[j]), *d) for (i, j), d in zip(edges, data))


def _system(Xs, edges, fixed, data):
    terms = [J.edge_terms(J.edge_pose(Xs[i], Xs[j]), *d) for (i, j), d in zip(edges, data)]
    return J.assemble(Xs, edges, fixed, [t[0] for t in terms], [t[1] for t in terms])


WINDOWS = {
    "pair": (2, [(1, 0)], [1, 0]),
    "chain": (4, [(1, 0), (2, 1), (3, 2), (3, 1)], [1, 0, 0, 0]),
    "reversed_edges": (4, [(0, 1), (1, 2), (2, 3), (0, 3)], [1, 0, 0, 0]),
    "loop_two_fixed": (5, [(1, 0), (2, 1), (3, 2), (4, 3), (0, 4), (2, 4)], [1, 0, 1, 0, 0]),
}


@pytest.mark.parametrize("name", sorted(WINDOWS))
@pytest.mark.parametrize("gicp", [False, True], ids=["icp", "gicp"])
def test_assembled_b_is_the_gradient(name, gicp):
    F, edges, fixed = WINDOWS[name]
    rng = np.random.default_rng(len(name) + 10 * gicp)
    Xs, data = _window(rng, F, edges, gicp)
    _, b = _system(Xs, edges, fixed, data)
    fi, nf = J.free_index(fixed)
    h = 1e-6
    g = np.zeros(6 * nf)
    for k in range(F):
        if fi[k] < 0:
            continue
        for m in range(6):
            d = np.zeros(6)
            d[m] = h
            Xp, Xm = list(Xs), list(Xs)
            Xp[k], Xm[k] = Xs[k] @ _exp(d), Xs[k] @ _exp(-d)
            g[6 * fi[k] + m] = (_energy(Xp, edges, data) - _energy(Xm, edges, data)) / (2 * h)
    # E = sum 1/2 r^T M r and b = J^T M r with J = dr/d(delta): the gradient of E is b
    np.testing.assert_allclose(b, g, rtol=1e-6, atol=1e-6 * np.abs(g).max())


@pytest.mark.parametrize("name", sorted(WINDOWS))
def test_assembled_H_is_JtJ_of_the_residuals(name):
    F, edges, fixed = WINDOWS[name]
    rng = np.random.default_rng(100 + len(name))
    Xs, data = _window(rng, F, edges, False)
    H, _ = _system(Xs, edges, fixed, data)
    fi, nf = J.free_index(fixed)

    def residuals(Ys):
        out = []
        for (i, j), (src, tgt, _) in zip(edges, data):
            T = J.edge_pose(Ys[i], Ys[j])
            out.append((tgt - (src @ T[:3, :3].T + T[:3, 3])).reshape(-1))
        return np.concatenate(out)

    h = 1e-6
    Jac = np.zeros((residuals(Xs).size, 6 * nf))
    for k in range(F):
        if fi[k] < 0:
            continue
        for m in range(6):
            d = np.zeros(6)
            d[m] = h
            Xp, Xm = list(Xs), list(Xs)
            Xp[k], Xm[k] = Xs[k] @ _exp(d), Xs[k] @ _exp(-d)
            Jac[:, 6 * fi[k] + m] = (residuals(Xp) - residuals(Xm)) / (2 * h)
    JtJ = Jac.T @ Jac
    np.testing.assert_allclose(H, JtJ, rtol=1e-5, atol=1e-6 * np.abs(JtJ).max())


def test_gauss_newton_reaches_the_minimum_of_a_consistent_window():
    """noise-free correspondences: the joint GN converges to the frames that generated them"""
    from np_align import Options

    rng = np.random.default_rng(3)
    F, edges, fixed = 4, [(1, 0), (2, 1), (3, 2), (2, 0)], [1, 0, 0, 0]
    truth = [np.eye(4)] + [_exp(np.concatenate([rng.normal(size=3) * 0.2, rng.normal(size=3)])) for _ in range(F - 1)]
    data = []
    for i, j in edges:
        src = rng.normal(size=(20, 3)) * 3.0
        T = J.edge_pose(truth[i], truth[j])
        data.append((src, src @ T[:3, :3].T + T[:3, 3], None))
    X0 = [truth[0]] + [X @ _exp(rng.normal(size=6) * 0.05) for X in truth[1:]]
    lin = lambda Xs: [J.edge_terms(J.edge_pose(Xs[i], Xs[j]), *d) + (20.0,) for (i, j), d in zip(edges, data)]
    err = lambda Xs: [J.edge_error(J.edge_pose(Xs[i], Xs[j]), *d) for (i, j), d in zip(edges, data)]
    for lm in (False, True):
        r = J.optimize(lin, err, _exp, X0, fixed, edges, Options(lm=lm, max_iterations=30))
        assert r.converged
        for X, T in zip(r.X, truth):
            np.testing.assert_allclose(X, T, atol=1e-6)
