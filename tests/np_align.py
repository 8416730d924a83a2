"""The optimiser of Registration<>::align restated in numpy (FP64): GaussNewtonOptimizer / LevenbergMarquardtOptimizer as optimize() of
oracle/sgicp_oracle.cpp has them (registration/optimizer.hpp:24-63 and :83-149, termination_criteria.hpp:10-20), with the reductions
passed in as callables so the same replay drives the oracle, the GPU's linearize_batch / error_batch, or a model.

  * the damped solve of H + lambda I (an FP64 LU solve here; the reference factors with LDLT, both exact to ~u cond(H + lambda I));
  * criteria_converged: |delta_rot| <= rotation_eps and |delta_trans| <= translation_eps;
  * LM: the `<=` acceptance test, lambda divided on acceptance and multiplied on rejection and carried across outer iterations, the
    break out of the outer loop when no trial is accepted;
  * `iterations` is the index of the last outer iteration run;
  * the RestrictDoFFactor term H(i, i) += 1e9 |mask_i - 1| as batched align() adds it (an all-ones mask adds nothing).

No GPU, no oracle state: linearize(T) -> (H, b, e), error(T) -> e, exp(delta) -> 4x4 (O.se3_exp in the tests)."""
from dataclasses import dataclass, field

import numpy as np


@dataclass
class Options:
    """sgb_align_options' optimiser fields and the reference's defaults (registration.hpp, optimizer.hpp)"""

    lm: bool = True
    max_iterations: int = 20
    gn_lambda: float = 1e-6
    max_inner_iterations: int = 10
    init_lambda: float = 1e-3
    lambda_factor: float = 10.0
    rotation_eps: float = 0.1 * np.pi / 180.0
    translation_eps: float = 1e-3
    dof_mask: tuple = (1.0, 1.0, 1.0, 1.0, 1.0, 1.0)


@dataclass
class Result:
    T: np.ndarray
    converged: bool = False
    iterations: int = 0
    H: np.ndarray = field(default_factory=lambda: np.zeros((6, 6)))
    b: np.ndarray = field(default_factory=lambda: np.zeros(6))
    error: float = 0.0
    linearizes: int = 0  # reductions run: what batched align() launches per member
    trials: int = 0
    trace: list = field(default_factory=list)  # per linearize: (T, H, b, e) before the update, like the oracle's trace


def dof_term(mask):
    """diagonal of the RestrictDoFFactor term: 1e9 |mask_i - 1|"""
    return 1e9 * np.abs(np.asarray(mask, dtype=np.float64) - 1.0)


def add_dof(H, mask):
    out = np.array(H, dtype=np.float64)
    d = dof_term(mask)
    for i in range(6):
        out[i, i] += d[i]
    return out


def damped_solve(H, b, lam):
    """delta = (H + lam I)^-1 (-b); a singular system (an empty member: H = 0, b = 0) gives its minimum-norm solution, 0 there, as the
    reference's zero pivots do"""
    A = np.asarray(H, dtype=np.float64) + lam * np.eye(6)
    try:
        return np.linalg.solve(A, -np.asarray(b, dtype=np.float64))
    except np.linalg.LinAlgError:
        return np.linalg.pinv(A) @ -np.asarray(b, dtype=np.float64)


def criteria_converged(delta, rotation_eps, translation_eps):
    return bool(np.linalg.norm(delta[:3]) <= rotation_eps and np.linalg.norm(delta[3:]) <= translation_eps)


def near_threshold(delta, o, rel=1e-9):
    """True where criteria_converged could go either way between two FP64 evaluations of the same step"""
    return bool(abs(np.linalg.norm(delta[:3]) - o.rotation_eps) <= rel * o.rotation_eps or abs(np.linalg.norm(delta[3:]) - o.translation_eps) <= rel * o.translation_eps)


def optimize(linearize, error, exp, T0, o):
    """optimize() of the oracle: the result of Registration<>::align from T0 with the reductions given"""
    r = Result(T=np.array(T0, dtype=np.float64))
    lam = o.init_lambda
    for i in range(o.max_iterations):
        if r.converged:
            break
        H, b, e = linearize(r.T)
        H = add_dof(H, o.dof_mask)
        r.linearizes += 1
        r.trace.append((r.T.copy(), H.copy(), np.array(b, dtype=np.float64), float(e)))
        if not o.lm:
            d = damped_solve(H, b, o.gn_lambda)
            r.converged = criteria_converged(d, o.rotation_eps, o.translation_eps)
            r.T = r.T @ exp(d)
            r.iterations, r.H, r.b, r.error = i, H, np.array(b), float(e)
            continue
        success = False
        for _ in range(o.max_inner_iterations):
            d = damped_solve(H, b, lam)
            T_new = r.T @ exp(d)
            e_new = error(T_new)
            r.trials += 1
            if e_new <= e:
                r.converged = criteria_converged(d, o.rotation_eps, o.translation_eps)
                r.T = T_new
                lam /= o.lambda_factor
                success = True
                e = e_new
                break
            lam *= o.lambda_factor
        r.iterations, r.H, r.b, r.error = i, H, np.array(b), float(e)
        if not success:
            break
    return r
