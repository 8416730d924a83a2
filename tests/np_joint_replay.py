"""Joint window registration (sgb_align_joint) checked one outer iteration at a time against an FP64 replay of np_joint, for every window
of a call.  No GPU: the edge reductions are callables, so the same checker runs on the device's results (tests/test_gpu_align_joint_replay.py,
the edges relinearised on a second context) and on the host build of the step (tests/test_joint_replay_on_host.py, numpy edge terms).

A converged window is a fixed point of any step that vanishes with b, so end results cannot show an H_ij block on the wrong frame, a DoF
term on one frame only, a trial pose built from the wrong frame or lambda not carried between outer iterations.  Here runs[k] is the
result of align_joint with max_iterations = k, k = 0 .. K, and every window's step from X_{k-1} to X_k is recomputed:

  * Linearize.  The window's active edges are linearised at the edge poses X_j^-1 X_i of X_{k-1} and assembled with np_joint.assemble
    (the DoF mask included).  num_inliers must be the summed inliers exactly, and (GN) the window's error the sum of the edges' e in member
    order to ERROR_RTOL: the device forms the edge poses with its own pose_inverse / pose_mul, the replay in numpy, a few ulp apart.
  * GN.  delta_ref = (H + gn_lambda I)^-1 (-b) and X_{k-1} exp(delta_f) for every free frame f against run k's frames; fixed frames bit
    for bit; `converged` against the criteria over every free frame (skipped within np_align.near_threshold of a threshold).
  * LM.  The replay carries its own lambda per window and proposes its own trials from X_{k-1}, each evaluated by `error` at the
    candidate edge poses.  A trial whose error is within AMBIGUOUS of e (relative) may go either way and the replay follows the branch the
    device took; any other decision must be the device's.  An accepted candidate must match X_k as in GN and the error at X_k must be run
    k's error; a window that accepts no trial must stop: iterations = k - 1, not converged, frames unchanged, the linearize's error.
  * A window that has stopped gives the same frames and results, bit for bit, in every later prefix.

Step tolerance.  The device solves (H + lambda I) delta = -b, n = 6 n_free, by LDLT with diagonal pivoting (solve_ldlt_n), a backward
stable solve: in the norm scaled by S = diag(A)^-1/2 its forward error is at most ~n u kappa_s |S^-1 delta| with kappa_s = cond(S A S)
(the Jacobi-scaled condition number, which the 1e9 DoF terms do not inflate), so |delta_dev - delta_ref| <= n u kappa_s max(S)
|S^-1 delta_ref|.  The exponential of each frame's 6-vector (CUDA sin / cos within 2 ulp, FMA contraction) and the product
X_{k-1} E add a few u per entry, times |t_{k-1}| in the translation.  The edge poses of the device and of the replay differ by a few
ulp, which moves every residual by ~u |p| (p: a source point in its frame's coordinates, `lever` = the largest |p|) and so b by ~u |p|
times H: the step moves by ~u |p| however small it is, which near convergence is the whole difference.  So over the window's free frames

    max_f |X_dev,f - X_ref,f|_max <= C u (n kappa_s max(S) |S^-1 delta_ref| + 1 + max_f |t_{k-1},f|_max + lever),

the batch replay's bound at n = 6 n_free plus the lever term (the batch replay linearises at the device's own pose: lever 0 there).
step_ratio is the ratio of the two sides without C; it must stay below STEP_RATIO.

Rounds.  sgb_align_joint runs rounds in lockstep over the windows: an error() round of every window with a pending trial while any has one,
else a linearize of every window still iterating.  replay_joint returns each window's linearize and trial counts and the round sequence
that rule gives, which fixes the launch count of the call."""
from dataclasses import dataclass, field

import numpy as np

import np_align as NA
import np_joint as J

U = 2.0**-53
STEP_RATIO = 16.0  # the batch replay's limit; the worst ratios observed on an H100 are 1.72 (GN) and 1.39 (LM)
AMBIGUOUS = 1e-9  # |e_trial - e| <= AMBIGUOUS e: either LM branch is right
ERROR_RTOL = 1e-12  # GN error against the edges' sum (edge poses formed in numpy and on the device)


def options(kw):
    """np_align.Options from the keywords of align_joint"""
    return NA.Options(lm=kw["optimizer"] == 1, max_iterations=kw["max_iterations"], gn_lambda=kw["gn_lambda"],
                      max_inner_iterations=kw["max_inner_iterations"], init_lambda=kw["init_lambda"], lambda_factor=kw["lambda_factor"],
                      rotation_eps=kw["rotation_eps"], translation_eps=kw["translation_eps"],
                      dof_mask=tuple([1.0] * 6 if kw.get("dof_mask") is None else kw["dof_mask"]))


def step_ratio(A, delta, X_prev, X_dev, X_ref, lever=0.0):
    """max over the frames of |X_dev - X_ref|_max over the bound of the module docstring (without C); A = H + lambda I (n x n), X_*: the
    window's free frames, lever: the largest |p| of the source points"""
    err = max(float(np.abs(a - b).max()) for a, b in zip(X_dev, X_ref)) if len(X_dev) else 0.0
    if err == 0.0:
        return 0.0
    d = np.diag(A)
    s = np.where(d > 0, 1.0 / np.sqrt(np.where(d > 0, d, 1.0)), 1.0)
    kappa = np.linalg.cond(A * s[:, None] * s[None, :])
    if not np.isfinite(kappa):
        return 0.0  # a singular system (no inliers, no damping): the solve's zero pivots are checked by the host tests
    t = max(float(np.abs(X[:3, 3]).max()) for X in X_prev)
    bound = U * (A.shape[0] * kappa * s.max() * np.linalg.norm(delta / s) + 1.0 + t + lever)
    return err / bound


@dataclass
class ReplayStats:
    gn: float = 0.0  # worst GN step ratio
    lm: float = 0.0  # worst LM step ratio
    ambiguous: int = 0  # trials within AMBIGUOUS of e
    rejected: int = 0  # rejected trials
    all_rejected: int = 0  # windows stopped because every trial of an iteration was rejected
    converged: int = 0  # windows that ended converged by the epsilons
    linearizes: np.ndarray = None  # per window
    trials: np.ndarray = None  # per window
    rounds: list = field(default_factory=list)  # "lin" / "err", in the order sgb_align_joint runs them


def _fail(cond, w, k, what, *detail):
    assert cond, f"window {w}, iteration {k}: {what}" + (" " + repr(detail) if detail else "")


def round_sequence(events):
    """the rounds of sgb_align_joint from each window's events ("lin" / "err" in its own order): an error() round of every window whose next
    event is a trial while any is, else a linearize of every window whose next event is one"""
    pos = [0] * len(events)
    out = []
    while True:
        nxt = [ev[p] if p < len(ev) else None for ev, p in zip(events, pos)]
        kind = "err" if "err" in nxt else ("lin" if "lin" in nxt else None)
        if kind is None:
            return out
        out.append(kind)
        for w, n in enumerate(nxt):
            if n == kind:
                pos[w] += 1


def replay_joint(runs, windows, edges, fixed, kw, linearize, error, exp=None, lever=0.0):
    """Check runs[k] (align_joint with max_iterations = k, k = 0 .. K; attributes X (F,4,4), converged, iterations, num_inliers, error per
    window) step by step.  windows: offsets (W + 1,); edges: [(i, j)] global frame indices in member order; fixed (F,) flags;
    kw: align_joint's option keywords; linearize(Xs, active) -> (H (E,6,6), b (E,6), e (E,), inliers (E,)) and error(Xs, active) -> e (E,)
    of the edges at X_j^-1 X_i of the frame poses Xs (F,4,4), active (E,) bool; lever: the largest |p| of the source points (step
    tolerance).  Returns a ReplayStats."""
    if exp is None:
        from test_np_joint import _exp as exp
    o = options(kw)
    off = list(windows)
    W, E = len(off) - 1, len(edges)
    fixed = [bool(f) for f in fixed]
    win_of = np.searchsorted(off, np.arange(off[-1]), side="right") - 1
    wedges = [[q for q, (i, _) in enumerate(edges) if win_of[i] == w] for w in range(W)]
    local = []  # per window: frames, local edges, local fixed
    for w in range(W):
        fr = list(range(off[w], off[w + 1]))
        local.append((fr, [(edges[q][0] - off[w], edges[q][1] - off[w]) for q in wedges[w]], [fixed[f] for f in fr]))
    nfree = [sum(not f for f in lf) for _, _, lf in local]
    starts = [o.max_iterations > 0 and nfree[w] > 0 and len(wedges[w]) > 0 for w in range(W)]
    I = np.asarray(runs[-1].iterations)
    lam = np.full(W, o.init_lambda)
    st = ReplayStats(linearizes=np.zeros(W, dtype=np.int64), trials=np.zeros(W, dtype=np.int64))
    events = [[] for _ in range(W)]
    X0 = np.asarray(runs[0].X)
    for w in range(W):
        _fail(not runs[0].converged[w] and runs[0].iterations[w] == 0 and runs[0].error[w] == 0 and runs[0].num_inliers[w] == 0, w, 0,
              "max_iterations = 0 left results")

    def same(a, b):
        return np.array_equal(np.asarray(a, dtype=np.float64).view(np.uint64), np.asarray(b, dtype=np.float64).view(np.uint64))

    def unchanged(cur, prev, w):
        fr = local[w][0]
        return same(cur.X[fr], prev.X[fr]) and all(same(getattr(cur, f)[w], getattr(prev, f)[w])
                                                   for f in ("converged", "iterations", "num_inliers", "error"))

    def edge_mask(ws):
        a = np.zeros(E, dtype=bool)
        for w in ws:
            a[wedges[w]] = True
        return a

    for k in range(1, len(runs)):
        prev, cur = runs[k - 1], runs[k]
        Xp, Xc = np.asarray(prev.X), np.asarray(cur.X)
        iterating = [starts[w] and k - 1 <= I[w] for w in range(W)]
        for w in range(W):
            _fail(all(same(Xc[f], X0[f]) for f in local[w][0] if fixed[f]), w, k, "a fixed frame moved")
            if not iterating[w]:
                _fail(unchanged(cur, prev, w), w, k, "a stopped window changed")
        members = [w for w in range(W) if iterating[w]]
        if not members:
            continue
        H_l, b_l, e_l, n_l = linearize(Xp, edge_mask(members))
        sys = {}
        for w in members:
            fr, le, lf = local[w]
            q = wedges[w]
            H, b = J.assemble(list(Xp[fr]), le, lf, list(H_l[q]), list(b_l[q]), o.dof_mask)
            e = 0.0
            for x in e_l[q]:  # member order, as the device sums
                e += float(x)
            sys[w] = (H, b, e)
            st.linearizes[w] += 1
            events[w].append("lin")
            _fail(cur.iterations[w] == k - 1, w, k, "iterations", int(cur.iterations[w]))
            _fail(int(cur.num_inliers[w]) == int(np.sum(n_l[q])), w, k, "num_inliers: device, replay", int(cur.num_inliers[w]), int(np.sum(n_l[q])))

        def free_frames(w):
            return [f for f in local[w][0] if not fixed[f]]

        def candidate(w, d):
            """X_{k-1} exp(delta_f) for the free frames of window w"""
            return [Xp[f] @ exp(d[6 * m : 6 * m + 6]) for m, f in enumerate(free_frames(w))]

        def check_step(w, A, d, cand, which):
            ff = free_frames(w)
            r = step_ratio(A, d, [Xp[f] for f in ff], [Xc[f] for f in ff], cand, lever)
            _fail(r <= STEP_RATIO, w, k, f"{which} step ratio", r)
            if which == "GN":
                st.gn = max(st.gn, r)
            else:
                st.lm = max(st.lm, r)
            dd = [d[6 * m : 6 * m + 6] for m in range(len(ff))]
            if not any(NA.near_threshold(x, o) for x in dd):
                conv = all(NA.criteria_converged(x, o.rotation_eps, o.translation_eps) for x in dd)
                _fail(bool(cur.converged[w]) == conv, w, k, "converged: device, replay", bool(cur.converged[w]), conv)

        if not o.lm:
            for w in members:
                H, b, e = sys[w]
                _fail(abs(cur.error[w] - e) <= ERROR_RTOL * abs(e), w, k, "GN error: device, sum of the edges", float(cur.error[w]), e)
                d = J.damped_solve(H, b, o.gn_lambda)
                check_step(w, H + o.gn_lambda * np.eye(H.shape[0]), d, candidate(w, d), "GN")
            continue
        # LM: the device's branch is visible in run k: it went on, converged or moved (accepted), else it stopped where it was
        dev_acc = {w: bool(k - 1 < I[w] or cur.converged[w] or not same(Xc[local[w][0]], Xp[local[w][0]])) for w in members}
        accepted = {}
        trialing = list(members)
        for _ in range(o.max_inner_iterations):
            if not trialing:
                break
            Xt = Xp.copy()
            props = {}
            for w in trialing:
                H, b, _ = sys[w]
                d = J.damped_solve(H, b, lam[w])
                cand = candidate(w, d)
                for f, Xf in zip(free_frames(w), cand):
                    Xt[f] = Xf
                props[w] = (d, cand, lam[w])
            et = error(Xt, edge_mask(trialing))
            still = []
            for w in trialing:
                st.trials[w] += 1
                events[w].append("err")
                e = sys[w][2]
                en = 0.0
                for x in et[wedges[w]]:
                    en += float(x)
                d, cand, lw = props[w]
                if abs(en - e) <= AMBIGUOUS * abs(e):
                    st.ambiguous += 1
                    H = sys[w][0]
                    ff = free_frames(w)
                    r = step_ratio(H + lw * np.eye(H.shape[0]), d, [Xp[f] for f in ff], [Xc[f] for f in ff], cand, lever)
                    acc = dev_acc[w] and r <= STEP_RATIO
                else:
                    acc = en <= e
                if acc:
                    accepted[w] = props[w]
                    lam[w] /= o.lambda_factor
                else:
                    st.rejected += 1
                    lam[w] *= o.lambda_factor
                    still.append(w)
            trialing = still
        e_at_dev = error(Xc, edge_mask(accepted)) if accepted else None
        for w in members:
            _fail((w in accepted) == dev_acc[w], w, k, "LM decision: replay accepted, device accepted", w in accepted, dev_acc[w])
            if w in accepted:
                d, cand, lw = accepted[w]
                H = sys[w][0]
                check_step(w, H + lw * np.eye(H.shape[0]), d, cand, "LM")
                e = 0.0
                for x in e_at_dev[wedges[w]]:
                    e += float(x)
                _fail(abs(cur.error[w] - e) <= ERROR_RTOL * abs(e), w, k, "LM error at X_k: device, replay", float(cur.error[w]), e)
            else:  # no trial accepted: the window stops where it is
                st.all_rejected += 1
                fr = local[w][0]
                _fail(same(Xc[fr], Xp[fr]) and not cur.converged[w] and I[w] == k - 1, w, k, "all trials rejected but the window went on")
                e = sys[w][2]
                _fail(abs(cur.error[w] - e) <= ERROR_RTOL * abs(e), w, k, "error after all trials rejected: device, linearize",
                      float(cur.error[w]), e)
    st.converged = int(np.sum(np.asarray(runs[-1].converged)))
    st.rounds = round_sequence(events)
    return st
