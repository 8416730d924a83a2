"""np_align.optimize driven by the oracle's own reductions (O.Registration.linearize / .error) against the oracle's align() with a trace:
the replay that judges batched align() on the GPU (test_gpu_align_batch_replay.py) is first pinned to the reference optimiser here,
Gauss-Newton and Levenberg-Marquardt, under every optimiser setting, every outer iteration.

Per linearize the trace holds the pose and H | b | e before the update.  Replay and oracle differ only in the solve (LU here, LDLT there).
Each pose agrees to at most 3.2e-15 relative to its largest entry (POSE_TOL = 1e-14).  H | b | e agree to at most 2.2e-14 on the scales
of np_factors.tight_ratios (SUMS_TOL = 1e-13); b_k is taken relative to sqrt(2 e H_kk) because near convergence b itself is mostly
cancellation.  Prints the worst ratios reached (run with -s to see them)."""
import numpy as np
import pytest

import np_align as NA
import np_factors as NF
import oracle as O
from conftest import noise_poses

POSE_TOL = 1e-14  # pose, relative to its largest entry
SUMS_TOL = 1e-13  # H | b | e on the scales of np_factors.tight_ratios

# name, Registration kwargs, set_optimizer kwargs
CASES = [
    ("GN", {}, dict(type=O.OPT_GN)),
    ("GN_lambda0", {}, dict(type=O.OPT_GN, gn_lambda=0.0)),
    ("GN_lambda_big", {}, dict(type=O.OPT_GN, gn_lambda=300.0)),
    ("LM", {}, dict(type=O.OPT_LM)),
    ("LM_init_small_factor2", {}, dict(type=O.OPT_LM, init_lambda=1e-8, lambda_factor=2.0)),
    ("LM_init_large_factor1e3", {}, dict(type=O.OPT_LM, init_lambda=1e4, lambda_factor=1e3)),
    # a sharp Cauchy knee and almost no damping: trials are rejected, and with 1 or 3 inner iterations the outer loop breaks
    ("LM_inner1_cauchy_break", dict(robust=O.ROBUST_CAUCHY, robust_c=1e-4), dict(type=O.OPT_LM, max_inner_iterations=1, init_lambda=1e-8)),
    ("LM_inner3_cauchy_break", dict(robust=O.ROBUST_CAUCHY, robust_c=1e-4), dict(type=O.OPT_LM, max_inner_iterations=3, init_lambda=1e-8)),
    ("GN_tight_eps", {}, dict(type=O.OPT_GN, rotation_eps=1e-12, translation_eps=1e-12, max_iterations=30)),
    ("GN_loose_eps", {}, dict(type=O.OPT_GN, rotation_eps=10.0, translation_eps=10.0)),
    ("GN_maxit2", {}, dict(type=O.OPT_GN, max_iterations=2)),
    ("LM_rejector_none_ICP", dict(factor=O.FACTOR_ICP, rejector=O.REJECT_NONE), dict(type=O.OPT_LM)),
    ("LM_max_dist_0.05_plane", dict(factor=O.FACTOR_PLANE, max_dist_sq=0.05), dict(type=O.OPT_LM)),
    ("GN_max_dist_25_huber", dict(robust=O.ROBUST_HUBER, robust_c=0.05, max_dist_sq=25.0), dict(type=O.OPT_GN)),
    ("LM_cauchy", dict(robust=O.ROBUST_CAUCHY, robust_c=0.01), dict(type=O.OPT_LM)),
]


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    s = np.abs(b).max()
    return float(np.abs(a - b).max() / s) if s > 0 else float(np.abs(a).max())


def _starts():
    T30 = np.eye(4)
    T30[:3, :3] = O.se3_exp(np.r_[np.deg2rad(30.0) * np.array([0.6, 0.0, 0.8]), 0, 0, 0])[:3, :3]
    T30[:3, 3] = [0.3, -0.2, 0.1]
    return [noise_poses()[1], T30]


@pytest.mark.parametrize("name,reg_kw,opt_kw", CASES, ids=[c[0] for c in CASES])
def test_replay_matches_the_oracle_optimizer(golden_prepared, name, reg_kw, opt_kw):
    g = golden_prepared
    tc, tt, sc = g["target"], g["target_tree"], g["source"]
    reg = O.Registration(num_threads=0, **reg_kw)
    reg.set_optimizer(**opt_kw)
    o = NA.Options(lm=opt_kw["type"] == O.OPT_LM, **{k: v for k, v in opt_kw.items() if k != "type"})
    worst_T = worst = 0.0
    for T0 in _starts():
        ref = reg.align(tc, tt, sc, T0, trace=True)
        rep = NA.optimize(lambda T: reg.linearize(tc, tt, sc, T), lambda T: reg.error(tc, sc, T), O.se3_exp, T0, o)
        assert len(rep.trace) == len(ref.trace), (name, len(rep.trace), len(ref.trace))
        for k, (row, (T, H, b, e)) in enumerate(zip(ref.trace, rep.trace)):
            r = (_rel(T, row[:16].reshape(4, 4)),) + NF.tight_ratios((H, b, e), (row[16:52].reshape(6, 6), row[52:58], row[58]))
            assert r[0] <= POSE_TOL and max(r[1:]) <= SUMS_TOL, (name, k, r)
            worst_T, worst = max(worst_T, r[0]), max(worst, *r[1:])
        r = (_rel(rep.T, ref.T_target_source),) + NF.tight_ratios((rep.H, rep.b, rep.error), (ref.H, ref.b, ref.error))
        assert r[0] <= POSE_TOL and max(r[1:]) <= SUMS_TOL, (name, "result", r)
        worst_T, worst = max(worst_T, r[0]), max(worst, *r[1:])
        assert (rep.converged, rep.iterations) == (ref.converged, ref.iterations), (name, rep.converged, rep.iterations, ref.converged, ref.iterations)
    print(f"{name}: worst pose {worst_T:.2e}, H|b|e {worst:.2e}, iterations {ref.iterations}, linearizes {rep.linearizes}, trials {rep.trials}")


def test_cases_take_every_branch(golden_prepared):
    """the settings above reach what they are there for: a rejected trial, the break when none is accepted, convergence at iteration 0
    and running out of iterations"""
    g = golden_prepared
    tc, tt, sc = g["target"], g["target_tree"], g["source"]
    seen = set()
    for name, reg_kw, opt_kw in CASES:
        reg = O.Registration(num_threads=0, **reg_kw)
        o = NA.Options(lm=opt_kw["type"] == O.OPT_LM, **{k: v for k, v in opt_kw.items() if k != "type"})
        for T0 in _starts():
            rep = NA.optimize(lambda T: reg.linearize(tc, tt, sc, T), lambda T: reg.error(tc, sc, T), O.se3_exp, T0, o)
            if o.lm and rep.trials > rep.linearizes:
                seen.add("rejected trial")
            if o.lm and not rep.converged and rep.iterations + 1 < o.max_iterations:
                seen.add("break")
            if rep.converged and rep.iterations == 0:
                seen.add("converged at 0")
            if not rep.converged and rep.iterations + 1 == o.max_iterations:
                seen.add("out of iterations")
    assert seen == {"rejected trial", "break", "converged at 0", "out of iterations"}, seen


def test_dof_term():
    H = np.arange(36.0).reshape(6, 6)
    out = NA.add_dof(H, [0, 0, 0, 1, 1, 1])
    assert np.array_equal(np.diag(out) - np.diag(H), [1e9, 1e9, 1e9, 0, 0, 0])
    assert np.array_equal(NA.add_dof(H, [1] * 6), H)
    assert np.array_equal(NA.dof_term([0.5, 1, 2, 1, 0, 1]), [5e8, 0, 1e9, 0, 1e9, 0])
    # a locked axis: the step along it is ~b / 1e9
    d = NA.damped_solve(NA.add_dof(np.eye(6), [0, 1, 1, 1, 1, 1]), np.ones(6), 0.0)
    assert abs(d[0]) < 1e-8 and np.allclose(d[1:], -1.0)
