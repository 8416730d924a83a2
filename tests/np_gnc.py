"""Graduated non-convexity (sgb_align_batch_gnc) in numpy: the weight formulas and mu schedules of sgb_math.cuh operation for operation
(every numpy float64 operation is correctly rounded, as the device's explicit _rn intrinsics are, so the results agree bit for bit), and the
GNC loop driven from the host with public Context calls on a context that holds one member: the model every member of the device call
must equal bit for bit."""
import numpy as np

GM, TLS = 0, 1  # sgb_gnc_kind
FACTOR = 1.4


def weight(kind, r2, mu, c2):
    """g of squared residuals r2 (array) under the surrogate of shape mu (scalar or array), noise bound c2; gnc_weight<KIND>"""
    r2, mu, c2 = np.broadcast_arrays(*(np.asarray(x, dtype=np.float64) for x in (r2, mu, c2)))
    if kind == GM:
        a = mu * c2
        q = a / (r2 + a)
        return q * q
    mu1 = mu + 1.0
    lo = (mu / mu1) * c2
    hi = (mu1 / mu) * c2
    with np.errstate(divide="ignore", invalid="ignore"):
        mid = (np.sqrt(c2) / np.sqrt(r2)) * np.sqrt(mu * mu1) - mu
    mid = np.where(mid < 0.0, 0.0, np.where(mid > 1.0, 1.0, mid))
    return np.where(r2 <= lo, 1.0, np.where(r2 >= hi, 0.0, mid))


def mu0(kind, r2max, c2):
    """stage 0's (mu, ones): ones = TLS without outliers (every weight 1, the only stage; mu reported as 0)"""
    t = 2.0 * r2max
    if kind == GM:
        m = t / c2
        return (1.0 if m <= 1.0 else m), False
    if t <= c2:
        return 0.0, True
    return c2 / (t - c2), False


def mu_next(kind, mu):
    return max(mu / FACTOR, 1.0) if kind == GM else FACTOR * mu


def schedule(kind, r2max, c2, max_stages):
    """the mu of every stage until the last that the schedule alone decides (GM: mu = 1; TLS without outliers; max_stages), as
    gnc_stage_begin runs it: TLS's binary-weights end is not part of it"""
    mu, ones = mu0(kind, r2max, c2)
    mus = [mu]
    while not (ones or (kind == GM and mu == 1.0) or len(mus) == max_stages):
        mu = mu_next(kind, mu)
        mus.append(mu)
    return mus


def r2_max(r2, matched):
    """the largest r^2 > 0 over the points with a correspondence, 0 without any"""
    r = r2[matched]
    r = r[r > 0.0]
    return float(r.max()) if r.size else 0.0


def stage_weights(kind, r2, matched, mu, ones, c2):
    """every point's g of a stage: 0 without a correspondence, 1 for TLS without outliers"""
    g = np.zeros(r2.shape)
    g[matched] = 1.0 if ones else weight(kind, r2[matched], mu, c2)
    return g


def binary(g, matched):
    return bool(np.all((g[matched] == 0.0) | (g[matched] == 1.0)))


def run_fixed(kind, r2, c2, max_stages):
    """the stage loop on fixed residuals (every point matched, nothing re-aligned) -> list of (mu, g) per stage"""
    matched = np.ones(r2.shape, dtype=bool)
    mu, ones = mu0(kind, r2_max(r2, matched), c2)
    out = []
    for s in range(max_stages):
        if s:
            mu = mu_next(kind, mu)
        g = stage_weights(kind, r2, matched, mu, ones, c2)
        out.append((mu, g))
        if ones or (kind == GM and mu == 1.0) or (kind == TLS and binary(g, matched)):
            break
    return out


class Model:
    """the host-driven loop's results for one member: the align_batch fields of its last stage (iterations summed), stages, mu, g"""


def host_gnc(ctx, init_T, c2, kind=TLS, max_stages=64, stage_iterations=3, w=None, **align):
    """the GNC loop of sgb_align_batch_gnc driven from the host with public calls on ctx, which holds one member (set_source_batch with one
    cloud, or a pairing of one member): set_source_weights(None), linearize_batch_points at the stage's pose, the formulas above,
    set_source_weights(w * g), align_batch.  w: the caller's weights (None: none), put back in force at the end."""
    import small_gicp_b200 as sg

    lin = {k: align[k] for k in ("factor", "robust_c", "rejector", "max_dist_sq") if k in align}
    max_iterations = align.pop("max_iterations", 20)
    T = np.asarray(init_T, dtype=np.float64)
    iterations = 0
    mu, ones = 0.0, False
    for s in range(max_stages):
        ctx.set_source_weights(None)
        terms = ctx.linearize_batch_points(T[None], robust=sg.ROBUST_NONE, hessians=False, **lin)
        matched = ctx.correspondences_batch()[0] != sg.NO_CORRESPONDENCE
        r2 = 2.0 * terms.point_e
        if s == 0:
            mu, ones = mu0(kind, r2_max(r2, matched), c2)
        else:
            mu = mu_next(kind, mu)
        g = stage_weights(kind, r2, matched, mu, ones, c2)
        last = ones or (kind == GM and mu == 1.0) or s == max_stages - 1 or (kind == TLS and binary(g, matched))
        ctx.set_source_weights(g if w is None else w * g)
        res = ctx.align_batch(T[None], max_iterations=max_iterations if last else stage_iterations, **align)
        iterations += int(res.iterations[0])
        T = res.T_target_source[0]
        if last:
            break
    ctx.set_source_weights(w)
    m = Model()
    m.T_target_source, m.converged, m.num_inliers, m.error = T, bool(res.converged[0]), int(res.num_inliers[0]), float(res.error[0])
    m.H, m.b, m.iterations, m.stages, m.mu, m.g = res.H[0], res.b[0], iterations, s + 1, mu, g
    return m
