"""The joint replay checker (np_joint_replay.replay_joint) on the host, no GPU:
  * it accepts the prefix runs of the host build of the joint step (tests/host_joint, one thread standing for the CTA) with numpy edge
    terms, GN and LM, on the pair, chain, loop and two-fixed windows together in one call, with and without a DoF mask;
  * it rejects the prefix runs of planted faults, each a mutated copy of np_joint.optimize below (the library is not touched), and names
    the window, the iteration and the quantity that disagreed.  A checker that passed these would pass a device with the same bug."""
import numpy as np
import pytest

import np_joint as J
import np_joint_replay as R
from np_align import Options
from test_joint_step_on_host import _host_run, _problem, hj  # noqa: F401  (hj: the host build's fixture)
from test_np_joint import _exp

SHAPES = {  # frames, edges (local), fixed
    "pair": (2, [(1, 0)], [1, 0]),
    "chain": (5, [(1, 0), (2, 1), (3, 2), (4, 3), (2, 0)], [1, 0, 0, 0, 0]),
    "loop": (6, [(1, 0), (2, 1), (3, 2), (4, 3), (5, 4), (0, 5), (3, 1)], [1, 0, 0, 0, 0, 0]),
    "two_fixed": (4, [(0, 1), (2, 1), (3, 2)], [0, 1, 0, 1]),
}


class Run:
    """what align_joint returns, for the windows of a call"""

    def __init__(self, X, converged, iterations, inliers, error):
        self.X = np.array(X)
        self.converged = np.array(converged, dtype=bool)
        self.iterations = np.array(iterations, dtype=np.int64)
        self.num_inliers = np.array(inliers, dtype=np.int64)
        self.error = np.array(error, dtype=np.float64)


class Call:
    """the windows of SHAPES side by side: global frames, edges, fixed flags, offsets, each edge's correspondences"""

    def __init__(self, names, seed, h_scale=1.0):
        self.h_scale = h_scale
        self.off, self.edges, self.fixed, self.X0, self.data, self.parts = [0], [], [], [], [], []
        for w, name in enumerate(names):
            F, le, lf = SHAPES[name]
            X0, data = _problem(seed + 7 * w, F, le)
            base = self.off[-1]
            self.parts.append((X0, lf, le, data))
            self.edges += [(base + i, base + j) for i, j in le]
            self.fixed += lf
            self.X0 += X0
            self.data += data
            self.off.append(base + F)
        self.X0 = np.array(self.X0)

    def terms(self, T, d):
        """np_joint.edge_terms, H scaled by h_scale: below 1 the model underestimates the curvature, so that small-lambda LM trials
        overshoot and are rejected"""
        H, b, e = J.edge_terms(T, *d)
        return self.h_scale * H, b, e

    def linearize(self, Xs, active):
        E = len(self.edges)
        H, b, e, n = np.zeros((E, 6, 6)), np.zeros((E, 6)), np.zeros(E), np.zeros(E)
        for q, ((i, j), d) in enumerate(zip(self.edges, self.data)):
            if active[q]:
                H[q], b[q], e[q] = self.terms(J.edge_pose(Xs[i], Xs[j]), d)
                n[q] = 15
        return H, b, e, n

    def error(self, Xs, active):
        return np.array([self.terms(J.edge_pose(Xs[i], Xs[j]), d)[2] if a else 0.0 for (i, j), d, a in zip(self.edges, self.data, active)])

    def runs(self, window_run, o, K):
        """prefix runs k = 0 .. K of window_run(o_k, X0, fixed, edges, data) -> (X list, converged, iterations, inliers, error)"""
        out = []
        for k in range(K + 1):
            ok = Options(**{**o.__dict__, "max_iterations": k})
            parts = [window_run(ok, *p) for p in self.parts]
            out.append(Run(np.concatenate([p[0] for p in parts]), *zip(*[p[1:] for p in parts])))
        return out


def _kw(o):
    return dict(optimizer=1 if o.lm else 0, max_iterations=o.max_iterations, gn_lambda=o.gn_lambda, max_inner_iterations=o.max_inner_iterations,
                init_lambda=o.init_lambda, lambda_factor=o.lambda_factor, rotation_eps=o.rotation_eps, translation_eps=o.translation_eps,
                dof_mask=list(o.dof_mask))


def _replay(call, runs, o):
    return R.replay_joint(runs, call.off, call.edges, call.fixed, _kw(o), call.linearize, call.error, exp=_exp)


PLANAR = (0.0, 0.0, 1.0, 1.0, 1.0, 0.0)


@pytest.mark.parametrize("lm", [False, True], ids=["gn", "lm"])
@pytest.mark.parametrize("mask", [None, PLANAR], ids=["nomask", "planar"])
def test_the_checker_accepts_the_host_step(hj, lm, mask):  # noqa: F811
    call = Call(list(SHAPES), 3)
    o = Options(lm=lm, max_iterations=12, dof_mask=mask or (1.0,) * 6)

    def host(ok, X0, lf, le, data):
        X, s, _ = _host_run(hj, ok, X0, lf, le, data)
        return X, bool(s.converged), s.iterations, s.inliers, s.e

    K = max(int(call.runs(host, o, 12)[-1].iterations.max()) + 1, 1)
    runs = call.runs(host, o, min(K, 12))
    st = _replay(call, runs, o)
    print(f"{'lm' if lm else 'gn'} {mask}: worst step ratio GN {st.gn:.2f} / LM {st.lm:.2f}, rejected {st.rejected}, rounds {len(st.rounds)}")
    assert st.linearizes.min() >= 1
    assert st.trials.sum() == (st.linearizes.sum() + st.rejected - st.all_rejected if lm else 0)


def test_round_sequence_puts_trials_first():
    """window 0: lin, err, err, lin; window 1: lin, lin: the second linearize of window 1 waits for window 0's trials"""
    assert R.round_sequence([["lin", "err", "err", "lin"], ["lin", "lin"]]) == ["lin", "err", "err", "lin"]
    assert R.round_sequence([["lin", "err"], ["lin", "lin", "lin"]]) == ["lin", "err", "lin", "lin"]
    assert R.round_sequence([[], []]) == []


# ---- planted faults: np_joint.optimize with one mistake each ----
FAULTS = {
    1: "the trial edge pose built from X_j instead of cand_j",
    2: "the DoF term added to the first free frame only",
    3: "lambda reset to init_lambda at every outer iteration",
    4: "the window's error() summed without its last edge",
    5: "H_ij written as P instead of P^T",
    6: "the fixed flag ignored for every frame but the window's first",
}


def _assemble(fault, Xs, edges, fixed, Hs, bs, mask):
    """np_joint.assemble, with fault 2 or 5"""
    fi, nf = J.free_index(fixed)
    n = 6 * nf
    H, b = np.zeros((n, n)), np.zeros(n)
    for (i, j), He, be in zip(edges, Hs, bs):
        A = J.adjoint(J.edge_pose(Xs[i], Xs[j]))
        a, c = fi[i], fi[j]
        if a >= 0:
            H[6 * a : 6 * a + 6, 6 * a : 6 * a + 6] += He
            b[6 * a : 6 * a + 6] += be
        if c >= 0:
            H[6 * c : 6 * c + 6, 6 * c : 6 * c + 6] += A.T @ He @ A
            b[6 * c : 6 * c + 6] += A.T @ be
        if a >= 0 and c >= 0:
            P = He @ A
            Hij = P.T if fault == 5 else P
            H[6 * a : 6 * a + 6, 6 * c : 6 * c + 6] += Hij
            H[6 * c : 6 * c + 6, 6 * a : 6 * a + 6] += Hij.T
    d = J.dof_term(mask)
    for k in range(1 if fault == 2 else nf):
        H[6 * k : 6 * k + 6, 6 * k : 6 * k + 6] += np.diag(d)
    return H, b


def _faulty_optimize(call, fault, o, X0, fixed, edges, data):
    """np_joint.optimize with the edge reductions of `call` on `data`, and fault `fault` (None: none)"""
    if fault == 6:
        fixed = [fixed[0]] + [0] * (len(fixed) - 1)
    lin = lambda Ts: [call.terms(T, d) + (15.0,) for T, d in zip(Ts, data)]
    err = lambda Ts: [call.terms(T, d)[2] for T, d in zip(Ts, data)]
    r = J.WindowResult(X=[np.array(X, dtype=np.float64) for X in X0])
    _, nf = J.free_index(fixed)
    if o.max_iterations <= 0 or nf == 0 or not edges:
        return r
    lam = o.init_lambda
    for it in range(o.max_iterations):
        if r.converged:
            break
        if fault == 3:
            lam = o.init_lambda
        terms = lin([J.edge_pose(r.X[i], r.X[j]) for i, j in edges])
        H, b = _assemble(fault, r.X, edges, fixed, [t[0] for t in terms], [t[1] for t in terms], o.dof_mask)
        e = float(sum(t[2] for t in terms))
        r.inliers = float(sum(t[3] for t in terms))
        if not o.lm:
            d = J.damped_solve(H, b, o.gn_lambda)
            r.converged = J._all_converged(d, o)
            r.X = J._update(r.X, fixed, d, _exp)
            r.iterations, r.error = it, e
            continue
        success = False
        for _ in range(o.max_inner_iterations):
            d = J.damped_solve(H, b, lam)
            Xn = J._update(r.X, fixed, d, _exp)
            ev = err([J.edge_pose(Xn[i], (r.X if fault == 1 else Xn)[j]) for i, j in edges])
            en = float(sum(ev[:-1] if fault == 4 else ev))
            if en <= e:
                r.converged = J._all_converged(d, o)
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


def _faulty_runs(call, fault, o):
    def model(ok, X0, lf, le, data):
        r = _faulty_optimize(call, fault, ok, X0, lf, le, data)
        return r.X, r.converged, r.iterations, r.inliers, r.error

    return call.runs(model, o, 10)


FAULT_OPTIONS = Options(lm=True, max_iterations=10, dof_mask=(1.0, 1.0, 1.0, 1.0, 1.0, 0.5))
H_SCALE = 0.3  # the edges' H at 0.3 of the curvature: LM rejects trials until lambda makes up the difference


def test_the_unmutated_copy_passes():
    """the copy the faults are planted in, without a fault, is a correct device to the checker (GN and LM), and its LM rejects trials"""
    call = Call(list(SHAPES), 5, H_SCALE)
    for o in (FAULT_OPTIONS, Options(**{**FAULT_OPTIONS.__dict__, "lm": False})):
        st = _replay(call, _faulty_runs(call, None, o), o)
        assert st.rejected > 0 if o.lm else st.trials.sum() == 0


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_the_checker_catches_a_planted_fault(fault):
    call = Call(list(SHAPES), 5, H_SCALE)
    with pytest.raises(AssertionError, match=r"window \d+, iteration \d+: ") as err:
        _replay(call, _faulty_runs(call, fault, FAULT_OPTIONS), FAULT_OPTIONS)
    print(f"fault {fault} ({FAULTS[fault]}): {str(err.value).splitlines()[0]}")
