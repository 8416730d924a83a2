"""Joint window registration (sgb_align_joint) restated in numpy (FP64): the frames X_k of a window solved together against its edges (i, j),
edge e at T_e = X_j^-1 X_i, with the per-edge sums H_e | b_e | e_e of the pairs path as inputs.

  * adjoint: A_e = -Ad(T_e^-1), Ad(R, t) = [[R, 0], [[t]x R, R]], so that the right perturbations X <- X exp(delta) move the edge by
    delta_e = delta_i + A_e delta_j;
  * assemble: H_ii += H_e, H_ij += H_e A_e, H_ji += A_e^T H_e, H_jj += A_e^T H_e A_e, b_i += b_e, b_j += A_e^T b_e over the free frames, then
    the RestrictDoFFactor term on every free frame's diagonal block;
  * damped_solve: np_align.damped_solve at size n;
  * optimize: the GN / LM window state machine of joint_step_kernel, with the edge reductions passed in as callables, and a trace of its
    decisions.

No GPU: linearize(Xs) -> [(H_e, b_e, e_e, inliers_e)] per edge, error(Xs) -> [e_e] per edge, exp(delta) -> 4x4."""
from dataclasses import dataclass, field

import numpy as np

from np_align import criteria_converged, dof_term


def skew(v):
    return np.array([[0.0, -v[2], v[1]], [v[2], 0.0, -v[0]], [-v[1], v[0], 0.0]])


def inv_pose(T):
    R, t = T[:3, :3], T[:3, 3]
    out = np.eye(4)
    out[:3, :3] = R.T
    out[:3, 3] = -R.T @ t
    return out


def edge_pose(Xi, Xj):
    return inv_pose(Xj) @ Xi


def adjoint(T):
    """A_e = -Ad(T^-1) for twists [r; t]"""
    Ti = inv_pose(T)
    R, t = Ti[:3, :3], Ti[:3, 3]
    Ad = np.zeros((6, 6))
    Ad[:3, :3] = R
    Ad[3:, :3] = skew(t) @ R
    Ad[3:, 3:] = R
    return -Ad


def free_index(fixed):
    out, n = [], 0
    for f in fixed:
        out.append(-1 if f else n)
        n += 0 if f else 1
    return out, n


def assemble(Xs, edges, fixed, Hs, bs, mask=(1.0,) * 6):
    """the window's (H, b) over its free frames from each edge's H_e (6x6) and b_e (6), edges = [(i, j)] in member order"""
    fi, nf = free_index(fixed)
    n = 6 * nf
    H, b = np.zeros((n, n)), np.zeros(n)
    for (i, j), He, be in zip(edges, Hs, bs):
        A = adjoint(edge_pose(Xs[i], Xs[j]))
        a, c = fi[i], fi[j]
        if a >= 0:
            H[6 * a : 6 * a + 6, 6 * a : 6 * a + 6] += He
            b[6 * a : 6 * a + 6] += be
        if c >= 0:
            H[6 * c : 6 * c + 6, 6 * c : 6 * c + 6] += A.T @ He @ A
            b[6 * c : 6 * c + 6] += A.T @ be
        if a >= 0 and c >= 0:
            H[6 * a : 6 * a + 6, 6 * c : 6 * c + 6] += He @ A
            H[6 * c : 6 * c + 6, 6 * a : 6 * a + 6] += A.T @ He
    d = dof_term(mask)
    for k in range(nf):
        H[6 * k : 6 * k + 6, 6 * k : 6 * k + 6] += np.diag(d)
    return H, b


def damped_solve(H, b, lam):
    """np_align.damped_solve at size n"""
    n = H.shape[0]
    A = np.asarray(H, dtype=np.float64) + lam * np.eye(n)
    try:
        return np.linalg.solve(A, -np.asarray(b, dtype=np.float64))
    except np.linalg.LinAlgError:
        return np.linalg.pinv(A) @ -np.asarray(b, dtype=np.float64)


@dataclass
class WindowResult:
    X: list
    converged: bool = False
    iterations: int = 0
    error: float = 0.0
    inliers: float = 0.0
    trace: list = field(default_factory=list)  # per decision: ("lin", X) / ("gn", delta) / ("trial", lambda, accepted)


def _update(Xs, fixed, delta, exp):
    fi, _ = free_index(fixed)
    return [X.copy() if fi[k] < 0 else X @ exp(delta[6 * fi[k] : 6 * fi[k] + 6]) for k, X in enumerate(Xs)]


def _all_converged(delta, o):
    return all(criteria_converged(delta[6 * k : 6 * k + 6], o.rotation_eps, o.translation_eps) for k in range(delta.size // 6))


def optimize(linearize, error, exp, X0, fixed, edges, o):
    """the window's result from X0 (the edges' reductions given as callables of the frame poses)"""
    r = WindowResult(X=[np.array(X, dtype=np.float64) for X in X0])
    _, nf = free_index(fixed)
    if o.max_iterations <= 0 or nf == 0 or not edges:
        return r
    lam = o.init_lambda
    for it in range(o.max_iterations):
        if r.converged:
            break
        terms = linearize(r.X)
        H, b = assemble(r.X, edges, fixed, [t[0] for t in terms], [t[1] for t in terms], o.dof_mask)
        e = float(sum(t[2] for t in terms))
        r.inliers = float(sum(t[3] for t in terms))
        r.trace.append(("lin", [X.copy() for X in r.X]))
        if not o.lm:
            d = damped_solve(H, b, o.gn_lambda)
            r.trace.append(("gn", d))
            r.converged = _all_converged(d, o)
            r.X = _update(r.X, fixed, d, exp)
            r.iterations, r.error = it, e
            continue
        success = False
        for _ in range(o.max_inner_iterations):
            d = damped_solve(H, b, lam)
            Xn = _update(r.X, fixed, d, exp)
            en = float(sum(error(Xn)))
            accepted = en <= e
            r.trace.append(("trial", lam, accepted))
            if accepted:
                r.converged = _all_converged(d, o)
                r.X = Xn
                lam /= o.lambda_factor
                success = True
                e = en
                break
            lam *= o.lambda_factor
        r.iterations, r.error = it, e
        if not success:
            break
    return r


# ---- a small synthetic window with fixed correspondences: the per-edge terms exactly as the factor kernels form them ----


def edge_terms(T, src, tgt, M=None):
    """sum over the correspondences (src[n] in frame i, tgt[n] in frame j) of J^T M J | J^T M r | 1/2 r^T M r at T (r = tgt - T src,
    J = [R skew(p) | -R]); M: (n, 3, 3) weights in the target frame (None: identity, ICP)"""
    R, t = T[:3, :3], T[:3, 3]
    H, b, e = np.zeros((6, 6)), np.zeros(6), 0.0
    for n, (p, q) in enumerate(zip(src, tgt)):
        r = q - (R @ p + t)
        W = np.eye(3) if M is None else M[n]
        J = np.hstack([R @ skew(p), -R])
        H += J.T @ W @ J
        b += J.T @ W @ r
        e += 0.5 * r @ W @ r
    return H, b, e


def edge_error(T, src, tgt, M=None):
    return edge_terms(T, src, tgt, M)[2]
