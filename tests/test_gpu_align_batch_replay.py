"""Batched align() checked one outer iteration at a time against an FP64 replay of the reference optimiser (np_align, itself pinned to
the oracle's optimize() by test_np_align.py), for every field of sgb_align_options and at the batch-size limits.

A converged pose is a fixed point of any step that vanishes with b, so end results cannot show a wrong damping, a misplaced DoF term or
lambda not carried between outer iterations.  Here the state after k outer iterations is taken from align_batch(..., max_iterations=k),
k = 0 .. K (K = the full run's largest iteration count + 1), and every member's step from T_{k-1} to T_k is recomputed:

  * Linearize.  A second context holding the same batch linearises at T_{k-1} (linearize_batch).  Run k's H must be that H plus the
    RestrictDoF term diag(1e9 |mask - 1|), and b, the inlier count and (GN) the error must be those of the linearize: bit for bit on the
    tie-free random-feature scene of test_gpu_storage_model.Data, to np_factors.TIGHT on the golden pair.
  * GN.  delta_ref = (H_dev + gn_lambda I)^-1 (-b) in FP64 and T_ref = T_{k-1} O.se3_exp(delta_ref) against run k's pose; `converged`
    against the criteria on delta_ref (skipped within 1e-9 relative of a threshold).
  * LM.  The replay carries its own lambda per member and proposes its own trials from T_{k-1}, evaluated by error_batch on the second
    context.  A trial whose error is within 1e-9 relative of e is ambiguous and the replay follows the branch the device's T_k shows;
    any other decision must be the device's.  The accepted candidate must match T_k as in GN, error_batch at the device's T_k must give
    run k's error, and a member that accepts no trial must stop: iterations = k - 1, not converged, pose unchanged.
  * A member that has stopped gives the same results, bit for bit, in every later prefix.

Step tolerance.  The device solves (H + lambda I) delta = -b by LDLT with diagonal pivoting, a backward-stable solve: in the norm
scaled by S = diag(A)^-1/2 its forward error is at most ~n u kappa_s |S^-1 delta| with kappa_s = cond(S A S) (the Jacobi-scaled
condition number, which the 1e9 DoF terms do not inflate), so |delta_dev - delta_ref| <= n u kappa_s max(S) |S^-1 delta_ref|.  The
exponential (CUDA sin / cos within 2 ulp, FMA contraction) and the product T_{k-1} E add a few u per entry, times |t_{k-1}| in the
translation.  So  |T_dev - T_ref|_max <= C u (n kappa_s max(S) |S^-1 delta_ref| + 1 + |t_{k-1}|_max),  and the ratio of the two sides
must stay below STEP_RATIO (C, the constants of the exponential and the product).  Each case prints its worst ratio (run with -s).

Cases put every field of sgb_align_options off its default at least once; for each field two cases differing only in it must give
different results (a swapped or dropped field fails there or in the replay).  The batch-size tests run the replay across the step
kernel's 128-member CTA boundary and at the 65536-member limit."""
import time

import numpy as np
import pytest

import np_align as NA
import np_factors as NF
import oracle as O
from conftest import noise_poses, pose_error
from test_gpu_storage_model import Data, about

pytestmark = pytest.mark.gpu

U = 2.0**-53
STEP_RATIO = 16.0  # the worst ratio observed on an H100 is 1.3 (LM_factor1e3)
AMBIGUOUS = 1e-9  # |e_trial - e| <= AMBIGUOUS e: either LM branch is right

DEFAULTS = dict(factor=2, robust=0, robust_c=1.0, rejector=1, max_dist_sq=1.0, optimizer=1, max_iterations=20, gn_lambda=1e-6,
                max_inner_iterations=10, init_lambda=1e-3, lambda_factor=10.0, rotation_eps=0.1 * np.pi / 180.0, translation_eps=1e-3,
                dof_mask=None)


def _sg():
    import small_gicp_b200 as sg

    return sg


def _options(kw):
    return NA.Options(lm=kw["optimizer"] == 1, max_iterations=kw["max_iterations"], gn_lambda=kw["gn_lambda"],
                      max_inner_iterations=kw["max_inner_iterations"], init_lambda=kw["init_lambda"], lambda_factor=kw["lambda_factor"],
                      rotation_eps=kw["rotation_eps"], translation_eps=kw["translation_eps"],
                      dof_mask=tuple([1.0] * 6 if kw["dof_mask"] is None else kw["dof_mask"]))


class Sub:
    """the per-member arrays of a BatchAlignResult restricted to some members"""

    def __init__(self, r, idx):
        for f in ("T_target_source", "converged", "iterations", "num_inliers", "error", "H", "b"):
            setattr(self, f, getattr(r, f)[idx])


FIELDS = ("T_target_source", "converged", "iterations", "num_inliers", "error", "H", "b")


def _same_member(r1, m1, r2, m2):
    return all(np.array_equal(getattr(r1, f)[m1], getattr(r2, f)[m2]) for f in FIELDS)


def step_ratio(A, delta, T_prev, T_dev, T_ref):
    """|T_dev - T_ref|_max over the bound of the module docstring (without C)"""
    err = float(np.abs(T_dev - T_ref).max())
    if err == 0.0:
        return 0.0
    d = np.diag(A)
    s = np.where(d > 0, 1.0 / np.sqrt(np.where(d > 0, d, 1.0)), 1.0)
    kappa = np.linalg.cond(A * s[:, None] * s[None, :])
    if not np.isfinite(kappa):
        return 0.0  # a singular system (no inliers, no damping): the solve's zero pivots are checked by the host tests
    bound = U * (6.0 * kappa * s.max() * np.linalg.norm(delta / s) + 1.0 + np.abs(T_prev[:3, 3]).max())
    return err / bound


class Stats:
    def __init__(self):
        self.gn = 0.0
        self.lm = 0.0
        self.damping = 0.0  # largest |delta(lambda) - delta(0)| / |delta(0)| of a GN step
        self.ambiguous = 0
        self.linearizes = None
        self.trials = None


def replay(runs, kw, ctx_rep, exact, stats):
    """Check runs[k] (align_batch with max_iterations = k, k = 0 .. K, restricted to the members ctx_rep holds, in its order) step by
    step.  Returns per-member (linearizes, trials) as the replay counts them."""
    o = _options(kw)
    B = len(runs[0].iterations)
    I = runs[-1].iterations
    lam = np.full(B, o.init_lambda)
    lin_count = np.zeros(B, dtype=np.int64)
    trial_count = np.zeros(B, dtype=np.int64)
    dof = NA.dof_term(o.dof_mask)
    lin_kw = dict(factor=kw["factor"], robust=kw["robust"], robust_c=kw["robust_c"], rejector=kw["rejector"], max_dist_sq=kw["max_dist_sq"])

    def close(a, b, tag):
        if exact:
            assert np.array_equal(a, b), tag
        else:
            a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
            s = np.abs(b).max()
            assert np.abs(a - b).max() <= NF.TIGHT * max(s, 1e-300) or (s == 0 and not a.any()), tag

    for k in range(1, len(runs)):
        prev, cur = runs[k - 1], runs[k]
        Tp, Tc = prev.T_target_source, cur.T_target_source
        iterating = np.array([k - 1 <= I[m] for m in range(B)])
        for m in np.nonzero(~iterating)[0]:  # stopped: unchanged from now on
            assert _same_member(cur, m, prev, m), (k, m, "a stopped member changed")
        if not iterating.any():
            continue
        H_l, b_l, e_l, n_l = ctx_rep.linearize_batch(Tp, active=iterating, **lin_kw)
        members = np.nonzero(iterating)[0]
        for m in members:
            lin_count[m] += 1
            tag = (k, m)
            if exact:
                close(cur.H[m], NA.add_dof(H_l[m], o.dof_mask), tag + ("H",))
                close(cur.b[m], b_l[m], tag + ("b",))
            elif n_l[m] == 0:
                assert np.array_equal(cur.H[m], np.diag(dof)) and not cur.b[m].any(), tag
            else:
                r = NF.tight_ratios((cur.H[m] - np.diag(dof), cur.b[m], e_l[m]), (H_l[m], b_l[m], e_l[m]))
                assert max(r) <= NF.TIGHT, tag + r
            if exact:
                assert cur.num_inliers[m] == n_l[m], tag
            else:
                assert abs(int(cur.num_inliers[m]) - int(n_l[m])) <= 2, tag
            assert cur.iterations[m] == k - 1, tag
            if not o.lm:
                close(cur.error[m], e_l[m], tag + ("GN error",))
                A = cur.H[m] + o.gn_lambda * np.eye(6)
                d = NA.damped_solve(cur.H[m], cur.b[m], o.gn_lambda)
                T_ref = Tp[m] @ O.se3_exp(d)
                ratio = step_ratio(A, d, Tp[m], Tc[m], T_ref)
                stats.gn = max(stats.gn, ratio)
                assert ratio <= STEP_RATIO, tag + ("GN step", ratio)
                if not NA.near_threshold(d, o):
                    assert bool(cur.converged[m]) == NA.criteria_converged(d, o.rotation_eps, o.translation_eps), tag
                if o.gn_lambda > 0 and np.linalg.norm(d) > 0:
                    d0 = NA.damped_solve(cur.H[m], cur.b[m], 0.0)
                    stats.damping = max(stats.damping, float(np.linalg.norm(d - d0) / np.linalg.norm(d0)))
        if not o.lm:
            continue
        # LM: the device's branch is visible in run k: it went on (accepted), converged (accepted), or moved (accepted)
        dev_acc = {m: bool(k - 1 < I[m] or cur.converged[m] or not np.array_equal(Tc[m], Tp[m])) for m in members}
        accepted = {}
        trialing = list(members)
        for _ in range(o.max_inner_iterations):
            if not trialing:
                break
            cands = Tp.copy()
            deltas = {}
            for m in trialing:
                deltas[m] = NA.damped_solve(cur.H[m], cur.b[m], lam[m])
                cands[m] = Tp[m] @ O.se3_exp(deltas[m])
            act = np.zeros(B, dtype=bool)
            act[trialing] = True
            et = ctx_rep.error_batch(cands, active=act)
            still = []
            for m in trialing:
                trial_count[m] += 1
                diff = et[m] - e_l[m]
                if abs(diff) <= AMBIGUOUS * e_l[m]:
                    stats.ambiguous += 1
                    A = cur.H[m] + lam[m] * np.eye(6)
                    acc = dev_acc[m] and step_ratio(A, deltas[m], Tp[m], Tc[m], cands[m]) <= STEP_RATIO
                else:
                    acc = diff <= 0
                if acc:
                    accepted[m] = (deltas[m], cands[m], lam[m])
                    lam[m] /= o.lambda_factor
                else:
                    lam[m] *= o.lambda_factor
                    still.append(m)
            trialing = still
        act = np.zeros(B, dtype=bool)
        act[list(accepted)] = True
        e_at_dev = ctx_rep.error_batch(Tc, active=act) if act.any() else None
        for m in members:
            tag = (k, m)
            assert (m in accepted) == dev_acc[m], tag + ("LM decision: replay", m in accepted, "device", dev_acc[m])
            if m in accepted:
                d, cand, lm_lambda = accepted[m]
                ratio = step_ratio(cur.H[m] + lm_lambda * np.eye(6), d, Tp[m], Tc[m], cand)
                stats.lm = max(stats.lm, ratio)
                assert ratio <= STEP_RATIO, tag + ("LM step", ratio)
                if not NA.near_threshold(d, o):
                    assert bool(cur.converged[m]) == NA.criteria_converged(d, o.rotation_eps, o.translation_eps), tag
                close(cur.error[m], e_at_dev[m], tag + ("error at T_k",))
            else:  # no trial accepted: the member stops where it is
                assert np.array_equal(Tc[m], Tp[m]) and not cur.converged[m] and I[m] == k - 1, tag
                close(cur.error[m], e_l[m], tag + ("error of the linearize",))
    stats.linearizes, stats.trials = lin_count, trial_count
    return lin_count, trial_count


def prefix_runs(ctx, starts, kw):
    """align_batch with max_iterations = 0 .. K; the full run's launches"""
    k0 = ctx.kernel_launches
    full = ctx.align_batch(starts, **kw)
    launches = ctx.kernel_launches - k0
    K = min(int(full.iterations.max()) + 1, kw["max_iterations"])
    runs = [ctx.align_batch(starts, **{**kw, "max_iterations": k}) for k in range(K)] + [full]
    if K < kw["max_iterations"]:
        again = ctx.align_batch(starts, **{**kw, "max_iterations": K})
        assert all(_same_member(again, m, full, m) for m in range(len(starts)))
    return full, runs, launches


# ---- scenes: the golden pair (kd-tree, voxel maps) and the tie-free random-feature scene ----
def _rot_start(centre, deg, axis, t):
    ax = np.asarray(axis, dtype=float)
    ax /= np.linalg.norm(ax)
    return about(centre, np.r_[np.deg2rad(deg) * ax, t])


class Scene:
    def __init__(self, target_fn, pts, covs, starts, exact):
        self.target_fn = target_fn
        self.ctx, self.rep = target_fn(), target_fn()
        self.pts, self.covs, self.starts, self.exact = pts, covs, np.array(starts), exact
        for c in (self.ctx, self.rep):
            c.set_source_batch(pts, covs)

    def close(self):
        self.ctx.close()
        self.rep.close()


@pytest.fixture(scope="module")
def golden_members(golden_prepared):
    g = golden_prepared
    sc = g["source"]
    P, C = sc.points, sc.covs
    c = NF.box_centre(P)
    starts = list(noise_poses()) + [_rot_start(c, 30, [0.6, 0, 0.8], [0.3, -0.2, 0.1]), _rot_start(c, 60, [0, 1, 0.2], [0, 0.2, 0]),
                                    _rot_start(c, 178, [0.3, -0.5, 1.0], [0.1, 0, 0])]
    pts = [P] * len(starts) + [P[:0], P + np.array([1000.0, 0, 0, 0])]
    covs = [C] * len(starts) + [C[:0], C]
    return pts, covs, starts + [np.eye(4), np.eye(4)]  # ... + "empty", "none" (no inliers)


@pytest.fixture(scope="module")
def robust_cs(golden_prepared):
    """Huber (ICP) and Cauchy (point-to-plane) c at the median cost of the identity start: Huber compares c with sqrt(e), Cauchy with e"""
    g = golden_prepared
    tc, tt, sc = g["target"], g["target_tree"], g["source"]
    idx, d2, _ = tt.knn(sc.points, 1)
    ok = d2[:, 0] <= 1.0
    r = tc.points[idx[ok, 0].astype(np.int64), :3] - sc.points[ok, :3]
    n = tc.normals[idx[ok, 0].astype(np.int64), :3]
    return float(np.sqrt(np.median(0.5 * d2[ok, 0]))), float(np.median(0.5 * ((n * r) ** 2).sum(1)))


@pytest.fixture(scope="module")
def data():
    return Data()


def _data_members(d):
    sl = lambda s, n: (d.sp[s : s + n], d.scv[s : s + n])
    out = []
    for (s, n), delta in (((0, 20000), [0.002, -0.001, 0.0015, 0.03, 0.0, -0.02]), ((20000, 5000), [0.01, -0.012, 0.008, 0.25, -0.2, 0.15]),
                          ((25000, 12000), [0.02, -0.015, 0.01, 0.25, -0.2, 0.15])):
        p, cv = sl(s, n)
        out.append((p, cv, d.aligned @ about(NF.box_centre(p), delta)))
    for (s, n), deg in (((40000, 3000), 30), ((45000, 3000), 170)):
        p, cv = sl(s, n)
        out.append((p, cv, d.aligned @ _rot_start(NF.box_centre(p), deg, [1, 0.4, -0.3], [0.1, 0, 0.05])))
    out.append((d.sp[:0], d.scv[:0], d.aligned))
    p, cv = sl(50000, 2000)
    out.append((p + np.array([1000.0, 0, 0, 0]), cv, d.aligned))
    return out


_SCENES = {}


@pytest.fixture(scope="module")
def scenes(golden_prepared, golden_members, data):
    sg = _sg()
    g = golden_prepared
    tc = g["target"]

    def kd(tp, tn, tcv):
        def f():
            ctx = sg.Context(0)
            ctx.set_target(tp, tn, tcv)
            ctx.build_target_kdtree()
            return ctx

        return f

    def vox(tp, tcv, offsets):
        def f():
            ctx = sg.Context(0)
            ctx.build_target_voxelmap(tp, tcv, 1.0, offsets)
            return ctx

        return f

    def get(name):
        if name not in _SCENES:
            if name.startswith("golden"):
                pts, covs, starts = golden_members
                fn = kd(tc.points, tc.normals, tc.covs) if name == "golden" else vox(tc.points, tc.covs, int(name[len("golden_vox"):]))
                _SCENES[name] = Scene(fn, pts, covs, starts, exact=False)
            else:
                M = _data_members(data)
                fn = kd(data.tp, data.tn, data.tcv) if name == "data" else vox(data.tp, data.tcv, 7)
                _SCENES[name] = Scene(fn, [m[0] for m in M], [m[1] for m in M], [m[2] for m in M], exact=True)
        return _SCENES[name]

    yield get
    for s in _SCENES.values():
        s.close()
    _SCENES.clear()


GN, LM = dict(optimizer=0), dict(optimizer=1)
CAUCHY_KNEE = dict(robust=2, robust_c=1e-4, init_lambda=1e-8)
CASES = {  # name -> (scene, options off the defaults); "H": gn_lambda from the members' H diagonal; "huber" / "cauchy": c at the median cost
    "GN": ("golden", GN),
    "GN_lambda0": ("golden", {**GN, "gn_lambda": 0.0}),
    "GN_lambda_H": ("golden", {**GN, "gn_lambda": "H"}),
    "LM": ("golden", LM),
    "LM_init_small": ("golden", {**LM, "init_lambda": 1e-8}),
    "LM_init_large": ("golden", {**LM, "init_lambda": 1e4}),
    "LM_factor2": ("golden", {**LM, "lambda_factor": 2.0}),
    "LM_factor1e3": ("golden", {**LM, "lambda_factor": 1e3}),
    "LM_inner1_cauchy": ("golden", {**LM, **CAUCHY_KNEE, "max_inner_iterations": 1}),
    "LM_inner3_cauchy": ("golden", {**LM, **CAUCHY_KNEE, "max_inner_iterations": 3}),
    "LM_inner0_cauchy": ("golden", {**LM, **CAUCHY_KNEE, "max_inner_iterations": 0}),  # no trial at all: every member stops at once
    "GN_eps_loose": ("golden", {**GN, "rotation_eps": 10.0, "translation_eps": 10.0}),
    "LM_eps_loose": ("golden", {**LM, "rotation_eps": 10.0, "translation_eps": 10.0}),
    "GN_rot_eps_tight": ("golden", {**GN, "rotation_eps": 1e-12}),
    "GN_trans_eps_tight": ("golden", {**GN, "translation_eps": 1e-12}),
    "GN_eps_tight_50": ("golden", {**GN, "rotation_eps": 1e-12, "translation_eps": 1e-12, "max_iterations": 50}),
    "LM_eps_tight_50": ("golden", {**LM, "rotation_eps": 1e-12, "translation_eps": 1e-12, "max_iterations": 50}),
    "LM_maxit1": ("golden", {**LM, "max_iterations": 1}),
    "GN_maxit2": ("golden", {**GN, "max_iterations": 2}),
    "LM_maxit50": ("golden", {**LM, "max_iterations": 50}),
    "LM_reject_none": ("golden", {**LM, "rejector": 0}),
    "LM_dist_0.05": ("golden", {**LM, "max_dist_sq": 0.05}),
    "LM_dist_25": ("golden", {**LM, "max_dist_sq": 25.0}),
    "LM_ICP": ("golden", {**LM, "factor": 0, "robust_c": "huber"}),
    "LM_ICP_huber": ("golden", {**LM, "factor": 0, "robust": 1, "robust_c": "huber"}),
    "LM_ICP_huber_2c": ("golden", {**LM, "factor": 0, "robust": 1, "robust_c": "huber2"}),
    "GN_plane": ("golden", {**GN, "factor": 1}),
    "GN_plane_cauchy": ("golden", {**GN, "factor": 1, "robust": 2, "robust_c": "cauchy"}),
    "GN_dof_rot_locked": ("golden", {**GN, "dof_mask": [0, 0, 0, 1, 1, 1]}),
    "LM_dof_rot_locked": ("golden", {**LM, "dof_mask": [0, 0, 0, 1, 1, 1]}),
    "LM_dof_trans_locked": ("golden", {**LM, "dof_mask": [1, 1, 1, 0, 0, 0]}),
    "GN_dof_mixed": ("golden", {**GN, "dof_mask": [0.5, 1, 2, 1, 0, 1]}),
    "LM_vox1": ("golden_vox1", LM),
    "GN_vox7": ("golden_vox7", GN),
    "LM_vox27_dof": ("golden_vox27", {**LM, "dof_mask": [0.5, 1, 2, 1, 0, 1]}),
    "data_GN": ("data", GN),
    "data_LM": ("data", LM),
    "data_LM_dof_mixed": ("data", {**LM, "dof_mask": [0.5, 1, 2, 1, 0, 1]}),
    "data_GN_plane_cauchy": ("data", {**GN, "factor": 1, "robust": 2, "robust_c": 0.5}),
    "data_LM_vox7": ("data_vox7", LM),
}

# field -> two cases that differ only in it
SENSITIVITY = {
    "optimizer_kind": ("GN", "LM"),
    "gn_lambda": ("GN", "GN_lambda_H"),
    "init_lambda": ("LM", "LM_init_large"),
    "lambda_factor": ("LM", "LM_factor2"),
    "max_inner_iterations": ("LM_inner0_cauchy", "LM_inner1_cauchy"),  # past this knee 3 trials are rejected wherever 1 is
    "rotation_eps": ("GN", "GN_rot_eps_tight"),
    "translation_eps": ("GN", "GN_trans_eps_tight"),
    "max_iterations": ("LM", "LM_maxit1"),
    "rejector_kind": ("LM", "LM_reject_none"),
    "max_dist_sq": ("LM", "LM_dist_25"),
    "factor_kind": ("LM", "LM_ICP"),
    "robust_kind": ("LM_ICP", "LM_ICP_huber"),
    "robust_c": ("LM_ICP_huber", "LM_ICP_huber_2c"),
    "dof_mask": ("LM", "LM_dof_trans_locked"),
}

_FULL = {}
_GN_LAMBDA = {}


def _resolve(name, scene, robust_cs):
    kw = {**DEFAULTS, **CASES[name][1]}
    huber, cauchy = robust_cs
    kw["robust_c"] = {"huber": huber, "huber2": 2.0 * huber, "cauchy": cauchy}.get(kw["robust_c"], kw["robust_c"])
    if kw["gn_lambda"] == "H":
        if "H" not in _GN_LAMBDA:  # the median diagonal entry of the members' H at their starts: damping changes delta by >= 10 %
            H, _, _, n = scene.rep.linearize_batch(scene.starts, factor=kw["factor"])
            _GN_LAMBDA["H"] = float(np.median(np.concatenate([np.diag(h) for h, c in zip(H, n) if c > 0])))
        kw["gn_lambda"] = _GN_LAMBDA["H"]
    return kw


@pytest.mark.parametrize("name", list(CASES))
def test_step_by_step(scenes, robust_cs, golden_prepared, name):
    scene = scenes(CASES[name][0])
    kw = _resolve(name, scene, robust_cs)
    full, runs, _ = prefix_runs(scene.ctx, scene.starts, kw)
    _FULL[name] = full
    st = Stats()
    replay(runs, kw, scene.rep, scene.exact, st)
    if name == "GN_lambda_H":
        assert st.damping >= 0.1, st.damping
    msg = f"{name}: worst step ratio GN {st.gn:.2f} / LM {st.lm:.2f}, ambiguous trials {st.ambiguous}, iterations {full.iterations.tolist()}"
    # the oracle supports every option but the DoF mask: the final results of the moderate starts (noise_poses) must match it
    if kw["dof_mask"] is None and CASES[name][0].startswith("golden"):
        g = golden_prepared
        tc, sc = g["target"], g["source"]
        reg = O.Registration(factor=kw["factor"], robust=kw["robust"], robust_c=kw["robust_c"], rejector=kw["rejector"], max_dist_sq=kw["max_dist_sq"],
                             num_threads=0)
        reg.set_optimizer(type=kw["optimizer"], max_iterations=kw["max_iterations"], gn_lambda=kw["gn_lambda"], max_inner_iterations=kw["max_inner_iterations"],
                          init_lambda=kw["init_lambda"], lambda_factor=kw["lambda_factor"], rotation_eps=kw["rotation_eps"], translation_eps=kw["translation_eps"])
        voxel = CASES[name][0] != "golden"
        vm = O.GaussianVoxelMap(tc, 1.0, int(CASES[name][0][len("golden_vox"):])) if voxel else None
        worst = (0.0, 0.0)
        # with eps below what FP64 can resolve, LM ends on a break decided by the last bits of two nearly equal errors: pose only
        chaotic = kw["optimizer"] == 1 and kw["rotation_eps"] < 1e-9
        for m in range(len(noise_poses())):
            ref = reg.align(vm, None, sc, scene.starts[m]) if voxel else reg.align(tc, g["target_tree"], sc, scene.starts[m])
            rot, trans = pose_error(ref.T_target_source, full.T_target_source[m])
            worst = (max(worst[0], rot), max(worst[1], trans))
            assert rot < 1e-4 and trans < 1e-3, (name, m, rot, trans)
            assert chaotic or full.iterations[m] == ref.iterations, (name, m, full.iterations[m], ref.iterations)
            assert abs(full.num_inliers[m] - ref.num_inliers) <= 2, (name, m, full.num_inliers[m], ref.num_inliers)
        msg += f", vs oracle {worst[0]:.1e} rad / {worst[1]:.1e} m"
    print(msg)


@pytest.mark.parametrize("field", list(SENSITIVITY))
def test_each_option_changes_the_result(scenes, robust_cs, field):
    """two runs that differ only in `field` differ for at least one member (each also passes test_step_by_step)"""
    a, b = SENSITIVITY[field]
    kws = []
    for name in (a, b):
        kw = _resolve(name, scenes(CASES[name][0]), robust_cs)
        kws.append(kw)
        if name not in _FULL:
            scene = scenes(CASES[name][0])
            _FULL[name] = scene.ctx.align_batch(scene.starts, **kw)
    diff = {k for k in DEFAULTS if not np.array_equal(np.asarray(kws[0][k], dtype=object), np.asarray(kws[1][k], dtype=object))}
    if kws[0]["robust"] == kws[1]["robust"] == 0:
        diff.discard("robust_c")  # read by no factor without a robust kernel
    assert diff == {{"optimizer_kind": "optimizer", "factor_kind": "factor", "robust_kind": "robust", "rejector_kind": "rejector"}.get(field, field)}, diff
    ra, rb = _FULL[a], _FULL[b]
    assert not all(_same_member(ra, m, rb, m) for m in range(len(ra.iterations))), field


@pytest.mark.parametrize("name", ["LM", "LM_inner3_cauchy", "LM_factor1e3", "GN", "LM_vox1"])
def test_launches_follow_the_rounds(scenes, robust_cs, golden_members, name):
    """B = 1: 6 launches per kd-tree linearize round (3 per voxel-map one) and 3 per error round, as many as the replay counts"""
    pts, covs, starts = golden_members
    scene = scenes(CASES[name][0])
    voxel = CASES[name][0] != "golden"
    kw = _resolve(name, scene, robust_cs)
    for m in (1, 6):  # a moderate and a near-pi start
        one = Scene(scene.target_fn, [pts[m]], [covs[m]], [starts[m]], exact=False)
        full, runs, launches = prefix_runs(one.ctx, one.starts, kw)
        lin, trials = replay(runs, kw, one.rep, False, Stats())
        assert launches == (3 if voxel else 6) * int(lin[0]) + 3 * int(trials[0]), (name, m, launches, lin, trials)
        one.close()


# ---- batch-size edges, on the tie-free scene (bit-exact linearize checks) ----
def _small_members(d, rng, B, lo, hi, empty_every=0):
    """B members of lo .. hi - 1 random consecutive source points (every `empty_every`-th empty), each from its own start near the
    truth (<= 3 deg / 0.2 m about its centre)"""
    sizes = rng.integers(lo, hi, B)
    if empty_every:
        sizes[empty_every // 2 :: empty_every] = 0
    first = rng.integers(0, len(d.sp) - hi, B)
    pts = [d.sp[f : f + n] for f, n in zip(first, sizes)]
    covs = [d.scv[f : f + n] for f, n in zip(first, sizes)]
    starts = []
    for p in pts:
        ax = rng.normal(size=3)
        ax /= np.linalg.norm(ax)
        starts.append(d.aligned @ about(NF.box_centre(p), np.r_[ax * np.deg2rad(rng.uniform(0, 3)), rng.uniform(-0.2, 0.2, 3)]))
    return pts, covs, np.array(starts)


def _kd(d):
    def f():
        ctx = _sg().Context(0)
        ctx.set_target(d.tp, d.tn, d.tcv)
        ctx.build_target_kdtree()
        return ctx

    return f


@pytest.mark.parametrize("B", [127, 128, 129, 257])
def test_step_kernel_cta_boundary(data, B):
    """the step kernel runs 128 members per CTA: the replay on every member of batches that end just before, at and after a CTA"""
    rng = np.random.default_rng(B)
    pts, covs, starts = _small_members(data, rng, B, 50, 2000, empty_every=64)
    scene = Scene(_kd(data), pts, covs, starts, exact=True)
    for optimizer in (0, 1):
        kw = {**DEFAULTS, "optimizer": optimizer}
        full, runs, _ = prefix_runs(scene.ctx, scene.starts, kw)
        st = Stats()
        replay(runs, kw, scene.rep, True, st)
        assert int(full.iterations[B - 1]) >= 1 and full.num_inliers[B - 1] > 0
        print(f"B = {B}, {'LM' if optimizer else 'GN'}: worst step ratio GN {st.gn:.2f} / LM {st.lm:.2f}, iterations up to {int(full.iterations.max())}")
    scene.close()


def test_member_limit(data):
    """SGB_BATCH_MAX_MEMBERS = 65536 members of 0 - 39 points: sampled members bit-identical to the same member aligned alone, the replay
    on them, and their linearize against the storage model.  On one H100 80GB HBM3 this test takes about 6 s, of which the 65536-member
    upload (one store_source per member) is 4.8 s."""
    t0 = time.perf_counter()
    B = 65536  # SGB_BATCH_MAX_MEMBERS
    rng = np.random.default_rng(65536)
    pts, covs, starts = _small_members(data, rng, B, 3, 40, empty_every=97)
    sample = np.unique(np.r_[[0, 127, 128, 129, B - 1], rng.choice(B, 11, replace=False)])
    ctx = _kd(data)()
    ctx.set_source_batch(pts, covs)
    t_upload = time.perf_counter() - t0
    rep = _kd(data)()
    rep.set_source_batch([pts[m] for m in sample], [covs[m] for m in sample])
    for optimizer in (0, 1):
        kw = {**DEFAULTS, "optimizer": optimizer, "max_iterations": 3}
        full, runs, _ = prefix_runs(ctx, starts, kw)
        assert (full.num_inliers > 0).sum() > B // 2
        for m in sample:
            one = _kd(data)()
            one.set_source_batch([pts[m]], [covs[m]])
            alone = one.align_batch(starts[m : m + 1], **kw)
            assert _same_member(full, m, alone, 0), (optimizer, m)
            one.close()
        st = Stats()
        replay([Sub(r, sample) for r in runs], kw, rep, True, st)
        print(f"B = {B}, {'LM' if optimizer else 'GN'}: worst step ratio on the sample GN {st.gn:.2f} / LM {st.lm:.2f}")
    # linearize of the sampled members at their starts against the storage model of each
    H, b, e, n = rep.linearize_batch(starts[sample])
    corrs = rep.correspondences_batch()
    for j, m in enumerate(sample):
        if n[j] == 0:
            assert not H[j].any() and e[j] == 0.0
            continue
        model = (NF.stored_points(pts[m]), NF.stored_covs(covs[m])) + data.tgt_model
        r = NF.tight_ratios((H[j], b[j], e[j]), NF.linearize(starts[m], corrs[j], 2, 0, 1.0, *model))
        assert max(r) <= NF.TIGHT, (m, r)
    ctx.close()
    rep.close()
    print(f"B = {B}: upload {t_upload:.1f} s, whole test {time.perf_counter() - t0:.1f} s")
