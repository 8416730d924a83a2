"""Graduated non-convexity for joint windows (sgb_align_joint_gnc) driven from the host with public Context calls on a context that holds one
window: the model every window of the device call must equal bit for bit.  The weight formulas and the mu schedule are np_gnc's; the edge
poses come from Context.joint_edge_poses, the device's own X_j^-1 X_i (a numpy product differs in the last bits, and so would every row of
the reweighting linearize)."""
import numpy as np

from np_gnc import GM, TLS, binary, mu0, mu_next, r2_max, stage_weights


class Model:
    """the host-driven loop's results for one window: the align_joint fields of its last stage (iterations summed), stages, mu, g"""


def host_joint_gnc(ctx, init_X, c2, fixed=None, kind=TLS, max_stages=64, stage_iterations=3, w=None, **align):
    """the GNC loop of sgb_align_joint_gnc on ctx, whose frames, pairing and target are those of one window: set_source_weights(None),
    joint_edge_poses of the stage's frames, linearize_batch_points at those poses, the formulas, set_source_weights(w * g), align_joint.
    w: the caller's weights (None: none), put back in force at the end."""
    import small_gicp_b200 as sg

    lin = {k: align[k] for k in ("factor", "robust_c", "rejector", "max_dist_sq") if k in align}
    max_iterations = align.pop("max_iterations", 20)
    X = np.asarray(init_X, dtype=np.float64)
    iterations = 0
    mu, ones = 0.0, False
    for s in range(max_stages):
        ctx.set_source_weights(None)
        T = ctx.joint_edge_poses(X)
        terms = ctx.linearize_batch_points(T, robust=sg.ROBUST_NONE, hessians=False, **lin)
        matched = np.concatenate(ctx.correspondences_batch()) != sg.NO_CORRESPONDENCE
        r2 = 2.0 * terms.point_e
        if s == 0:
            mu, ones = mu0(kind, r2_max(r2, matched), c2)
        else:
            mu = mu_next(kind, mu)
        g = stage_weights(kind, r2, matched, mu, ones, c2)
        last = ones or (kind == GM and mu == 1.0) or s == max_stages - 1 or (kind == TLS and binary(g, matched))
        ctx.set_source_weights(g if w is None else w * g)
        res = ctx.align_joint(X, fixed=fixed, max_iterations=max_iterations if last else stage_iterations, **align)
        iterations += int(res.iterations[0])
        X = res.X
        if last:
            break
    ctx.set_source_weights(w)
    m = Model()
    m.X, m.converged, m.num_inliers, m.error = X, bool(res.converged[0]), int(res.num_inliers[0]), float(res.error[0])
    m.iterations, m.stages, m.mu, m.g = iterations, s + 1, mu, g
    return m
