"""Joint window registration (sgb_align_joint) checked one outer iteration at a time against the FP64 replay of np_joint_replay, for every
field of sgb_align_options, on many kd-trees and many voxel maps, and on window shapes the other tests never build.

Each case runs align_joint with max_iterations = k, k = 0 .. K (K = the full run's largest iteration count + 1) on one context, and
replays every window's step on a second context holding the same frames and edges, whose linearize_batch / error_batch (with the `active`
masks of the windows in the round) give the edges' H_e | b_e | e_e at the edge poses X_j^-1 X_i formed in numpy.  This checks what only
the device has: the 256-thread CTA assembly, solve_ldlt_n and update, the copy of each edge's sums through edge_member, the window's
error() summed in member order, the edge poses written from X or from the candidate after a trial, the host loop's ordering of trial and
linearize rounds across windows, and shared memory sized for the largest window of the call.  Per case:

  * the replay (module docstring of np_joint_replay: decisions, steps to STEP_RATIO, stopped windows bit for bit); the worst GN and LM
    step ratios, the ambiguous trials and the rejected trials are printed (run with -s);
  * the full run's kernel launches: 1 set-up launch, per linearize round the pairs round's launches (3 on kd-trees, 2 on voxel maps) plus
    the step, per error() round 2 plus the step, over the round sequence the replay derives (this counts the rejected trials, which the
    poses cannot show);
  * align_joint_async from the same poses gives X and every info field bit for bit.

The cases put every field of sgb_align_options off its default at least once; for each field two cases that differ only in it give
different frames.  The calls: "mix" holds four windows of different sizes -- a 3-frame chain; a 6-frame window with its fixed frames not
first, edges both ways between one pair, a duplicate edge and a free frame without an edge; an 8-frame chain with skips and a loop edge;
a pair one of whose frames is 1000 m away (no correspondence) -- with their edges interleaved across windows and shuffled within each, so
that windows in a trial round and windows waiting to linearize share rounds.  "w32" is one window of 32 frames (n = 186)."""
import time

import numpy as np
import pytest

import np_joint as J
import np_joint_replay as R
from test_gpu_align_joint import Frames, _context, _perturbed, _window_edges

pytestmark = pytest.mark.gpu

DEFAULTS = dict(factor=2, robust=0, robust_c=1.0, rejector=1, max_dist_sq=1.0, optimizer=1, max_iterations=20, gn_lambda=1e-6,
                max_inner_iterations=10, init_lambda=1e-3, lambda_factor=10.0, rotation_eps=0.1 * np.pi / 180.0, translation_eps=1e-3,
                dof_mask=None)
LAUNCHES_PER_LIN = {"kdtree": 3, "voxelmap": 2}


class Call:
    """windows of Frames: per window (frame indices, local edges, local fixed flags, seed); `far`: local frames moved 1000 m"""

    def __init__(self, wins, far=(), rot=0.02, trans=0.2):
        self.idx, self.off, self.fixed, per_win, X = [], [0], [], [], []
        for w, (fidx, edges, fixed, seed) in enumerate(wins):
            base = len(self.idx)
            self.idx += fidx
            self.fixed += fixed
            per_win.append([(base + i, base + j) for i, j in edges])
            Xw = _perturbed(FRAMES[0], fidx, seed, rot, trans)
            for f in far:
                if f[0] == w:
                    Xw[f[1]][:3, 3] += 1000.0
            X.append(Xw)
            self.off.append(len(self.idx))
        self.X0 = np.concatenate(X)
        # member order: the windows' edges interleaved, each window's shuffled
        rng = np.random.default_rng(len(self.idx))
        queues = [list(rng.permutation(len(e))) for e in per_win]
        self.edges = []
        while any(queues):
            for w, q in enumerate(queues):
                if q:
                    self.edges.append(per_win[w][q.pop()])


FRAMES = []  # the module's Frames, set by the fixture


def _calls():
    odd = [(1, 0), (0, 1), (2, 1), (2, 1), (3, 2), (4, 3), (3, 1)]  # both ways, a duplicate; local frame 5 has no edge
    return {
        "mix": Call([(list(range(0, 3)), _window_edges(3), [1, 0, 0], 21), (list(range(20, 26)), odd, [0, 0, 1, 0, 1, 0], 22),
                     (list(range(10, 18)), _window_edges(8), [1] + [0] * 7, 23), ([30, 31], [(1, 0)], [1, 0], 24)], far=[(3, 1)]),
        "w32": Call([(list(range(4, 36)), _window_edges(32), [1] + [0] * 31, 25)]),
    }


GN, LM = dict(optimizer=0), dict(optimizer=1)
CAUCHY_KNEE = dict(robust=2, robust_c=1e-4, init_lambda=1e-8)
CASES = {  # name -> (kind, call, options off the defaults); "H": gn_lambda at the median H diagonal; "huber" / "cauchy": c at the median cost
    "GN": ("kdtree", "mix", GN),
    "LM": ("kdtree", "mix", LM),
    "GN_w32": ("kdtree", "w32", GN),
    "LM_w32": ("kdtree", "w32", LM),
    "GN_lambda_H": ("kdtree", "mix", {**GN, "gn_lambda": "H"}),
    "LM_init_large": ("kdtree", "mix", {**LM, "init_lambda": 1e3}),
    "LM_factor2": ("kdtree", "mix", {**LM, "lambda_factor": 2.0}),
    "LM_factor1e3": ("kdtree", "mix", {**LM, "lambda_factor": 1e3}),
    "LM_inner0_cauchy": ("kdtree", "mix", {**LM, **CAUCHY_KNEE, "max_inner_iterations": 0}),
    "LM_inner1_cauchy": ("kdtree", "mix", {**LM, **CAUCHY_KNEE, "max_inner_iterations": 1}),
    "LM_inner3_cauchy": ("kdtree", "mix", {**LM, **CAUCHY_KNEE, "max_inner_iterations": 3}),
    "GN_eps_loose": ("kdtree", "mix", {**GN, "rotation_eps": 10.0, "translation_eps": 10.0}),
    "LM_eps_loose": ("kdtree", "mix", {**LM, "rotation_eps": 10.0, "translation_eps": 10.0}),
    "GN_rot_eps_tight": ("kdtree", "mix", {**GN, "rotation_eps": 1e-12}),
    "GN_trans_eps_tight": ("kdtree", "mix", {**GN, "translation_eps": 1e-12}),
    "LM_maxit1": ("kdtree", "mix", {**LM, "max_iterations": 1}),
    "GN_maxit2": ("kdtree", "mix", {**GN, "max_iterations": 2}),
    "LM_maxit50": ("kdtree", "mix", {**LM, "max_iterations": 50}),
    "LM_reject_none": ("kdtree", "mix", {**LM, "rejector": 0}),
    "LM_dist_0.05": ("kdtree", "mix", {**LM, "max_dist_sq": 0.05}),
    "LM_dist_25": ("kdtree", "mix", {**LM, "max_dist_sq": 25.0}),
    "LM_ICP": ("kdtree", "mix", {**LM, "factor": 0, "robust_c": "huber"}),
    "LM_ICP_huber": ("kdtree", "mix", {**LM, "factor": 0, "robust": 1, "robust_c": "huber"}),
    "LM_ICP_huber_2c": ("kdtree", "mix", {**LM, "factor": 0, "robust": 1, "robust_c": "huber2"}),
    "GN_plane": ("kdtree", "mix", {**GN, "factor": 1}),
    "GN_plane_cauchy": ("kdtree", "mix", {**GN, "factor": 1, "robust": 2, "robust_c": "cauchy"}),
    "GN_dof_planar": ("kdtree", "mix", {**GN, "dof_mask": [0, 0, 1, 1, 1, 0]}),
    "LM_dof_planar": ("kdtree", "mix", {**LM, "dof_mask": [0, 0, 1, 1, 1, 0]}),
    "LM_dof_frac": ("kdtree", "mix", {**LM, "dof_mask": [0.5, 1, 2, 1, 0, 1]}),
    "LM_weights_cauchy": ("kdtree", "mix", {**LM, "robust": 2, "robust_c": "cauchy", "weights": True}),
    "GN_vox": ("voxelmap", "mix", GN),
    "LM_vox": ("voxelmap", "mix", LM),
    "LM_vox_w32": ("voxelmap", "w32", LM),
    "LM_vox_ICP_huber": ("voxelmap", "mix", {**LM, "factor": 0, "robust": 1, "robust_c": "huber"}),
    "LM_vox_inner3_cauchy": ("voxelmap", "mix", {**LM, **CAUCHY_KNEE, "max_inner_iterations": 3}),
    "GN_vox_dof_frac": ("voxelmap", "mix", {**GN, "dof_mask": [0.5, 1, 2, 1, 0, 1]}),
    "LM_vox_weights_cauchy": ("voxelmap", "mix", {**LM, "robust": 2, "robust_c": "cauchy", "weights": True}),
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
    "dof_mask": ("LM", "LM_dof_planar"),
}


class Scene:
    """one call on one kind of target: the run context, the replay context, the per-point weights"""

    def __init__(self, kind, call):
        import torch

        self.kind, self.call = kind, call
        cl, mp = [e[0] for e in call.edges], [e[1] for e in call.edges]
        self.ctx = _context(FRAMES[0], call.idx, kind, cl, mp)
        self.stream = torch.cuda.Stream()  # the run context's stream (align_joint_async needs a torch stream), alive as long as it
        self.ctx.set_stream(self.stream.cuda_stream)
        self.rep = _context(FRAMES[0], call.idx, kind, cl, mp)
        n = sum(len(FRAMES[0].pts[call.idx[i]]) for i in cl)
        self.weights = np.random.default_rng(n).uniform(0.2, 1.5, n)
        self.c = {}

    def edge_poses(self, Xs):
        return np.array([J.edge_pose(Xs[i], Xs[j]) for i, j in self.call.edges])

    def robust_c(self, factor):
        """(Huber c, Cauchy c) at the median cost of the start's inlier points: Huber compares c with sqrt(e), Cauchy with e"""
        if factor not in self.c:
            t = self.rep.linearize_batch_points(self.edge_poses(self.call.X0), factor=factor, hessians=False)
            e = t.point_e[t.point_e > 0]
            self.c[factor] = (float(np.sqrt(np.median(e))), float(np.median(e)))
        return self.c[factor]

    def close(self):
        self.stream.synchronize()
        self.ctx.close()
        self.rep.close()


_SCENES, _RESULTS = {}, {}


@pytest.fixture(scope="module")
def scenes():
    FRAMES.append(Frames(40))
    calls = _calls()

    def get(kind, call):
        if (kind, call) not in _SCENES:
            _SCENES[(kind, call)] = Scene(kind, calls[call])
        return _SCENES[(kind, call)]

    yield get
    for s in _SCENES.values():
        s.close()
    _SCENES.clear()
    _RESULTS.clear()
    FRAMES.clear()


def _resolve(name, scene):
    kw = {**DEFAULTS, **CASES[name][2]}
    kw.pop("weights", None)
    huber, cauchy = scene.robust_c(kw["factor"])
    kw["robust_c"] = {"huber": huber, "huber2": 2.0 * huber, "cauchy": cauchy}.get(kw["robust_c"], kw["robust_c"])
    if kw["gn_lambda"] == "H":  # the median diagonal entry of the edges' H at the start
        H, _, _, n = scene.rep.linearize_batch(scene.edge_poses(scene.call.X0), factor=kw["factor"])
        kw["gn_lambda"] = float(np.median(np.concatenate([np.diag(h) for h, c in zip(H, n) if c > 0])))
    return kw


def _run_case(scenes, name):
    """the replay of case `name` (cached): (full run, ReplayStats, kw)"""
    if name in _RESULTS:
        return _RESULTS[name]
    t0 = time.perf_counter()
    kind, call_name, opts = CASES[name]
    scene = scenes(kind, call_name)
    call, ctx, rep = scene.call, scene.ctx, scene.rep
    kw = _resolve(name, scene)
    weights = scene.weights if opts.get("weights") else None
    for c in (ctx, rep):
        c.set_source_weights(weights)
    args = dict(windows=call.off, fixed=call.fixed)
    ctx.align_joint(call.X0, **args, **{**kw, "max_iterations": 1})  # the pairing's view of the target is built here
    k0 = ctx.kernel_launches
    full = ctx.align_joint(call.X0, **args, **kw)
    launches = ctx.kernel_launches - k0
    K = min(int(full.iterations.max()) + 1, kw["max_iterations"])
    runs = [ctx.align_joint(call.X0, **args, **{**kw, "max_iterations": k}) for k in range(K)] + [full]
    lin_kw = {f: kw[f] for f in ("factor", "robust", "robust_c", "rejector", "max_dist_sq")}
    linearize = lambda Xs, active: rep.linearize_batch(scene.edge_poses(Xs), active=active, **lin_kw)
    error = lambda Xs, active: rep.error_batch(scene.edge_poses(Xs), active=active)
    lever = max(float(np.abs(FRAMES[0].pts[i][:, :3]).max()) for i in call.idx)
    st = R.replay_joint(runs, call.off, call.edges, call.fixed, kw, linearize, error, lever=lever)
    # launches: 1 set-up, then per round the pairs round's launches and the step
    n_lin, n_err = st.rounds.count("lin"), st.rounds.count("err")
    assert launches == 1 + n_lin * (LAUNCHES_PER_LIN[kind] + 1) + n_err * 3, (name, launches, n_lin, n_err)
    # align_joint_async from the same poses: the same results, bit for bit
    import torch

    with torch.cuda.stream(scene.stream):
        a = ctx.align_joint_async(torch.from_numpy(np.ascontiguousarray(call.X0)).cuda(), **args, **kw)
        ctx.synchronize()
        aX, ainfo = a.X.cpu().numpy(), a.info4.cpu().numpy()
    scene.stream.synchronize()
    assert np.ascontiguousarray(aX).tobytes() == full.X.tobytes(), (name, "async X")
    info = np.stack([full.converged.astype(np.float64), full.iterations, full.num_inliers, full.error], 1)
    assert np.array_equal(np.ascontiguousarray(ainfo).view(np.uint64), info.view(np.uint64)), (name, "async info")
    for c in (ctx, rep):
        c.set_source_weights(None)
    print(f"{name}: worst step ratio GN {st.gn:.3g} / LM {st.lm:.3g}, ambiguous trials {st.ambiguous}, rejected trials {st.rejected}, "
          f"all-rejected stops {st.all_rejected}, rounds {n_lin} lin + {n_err} error(), iterations {full.iterations.tolist()}, "
          f"converged {full.converged.astype(int).tolist()}, {time.perf_counter() - t0:.1f} s")
    _RESULTS[name] = (full, st, kw)
    return _RESULTS[name]


@pytest.mark.parametrize("name", list(CASES))
def test_step_by_step(scenes, name):
    full, st, kw = _run_case(scenes, name)
    if kw["optimizer"] == 1:
        assert st.trials.sum() == st.linearizes.sum() + st.rejected - st.all_rejected
    else:
        assert st.trials.sum() == 0


def test_cases_reach_every_branch(scenes):
    """over the cases: rejected trials, windows stopped with every trial rejected, windows converged by the epsilons, GN and LM steps"""
    stats = [_run_case(scenes, n)[1] for n in CASES]
    worst_gn, worst_lm = max(s.gn for s in stats), max(s.lm for s in stats)
    print(f"all cases: worst step ratio GN {worst_gn:.3g} / LM {worst_lm:.3g}, ambiguous trials {sum(s.ambiguous for s in stats)}, "
          f"rejected trials {sum(s.rejected for s in stats)}, all-rejected stops {sum(s.all_rejected for s in stats)}")
    assert sum(s.rejected for s in stats) > 0
    assert sum(s.all_rejected for s in stats) > 0
    assert sum(s.converged for s in stats) > 0
    assert worst_gn > 0 and worst_lm > 0


@pytest.mark.parametrize("field", list(SENSITIVITY))
def test_each_option_changes_the_result(scenes, field):
    """two runs that differ only in `field` differ in some frame (each also passes test_step_by_step)"""
    a, b = SENSITIVITY[field]
    (ra, _, ka), (rb, _, kb) = _run_case(scenes, a), _run_case(scenes, b)
    diff = {k for k in DEFAULTS if not np.array_equal(np.asarray(ka[k], dtype=object), np.asarray(kb[k], dtype=object))}
    if ka["robust"] == kb["robust"] == 0:
        diff.discard("robust_c")  # read by no factor without a robust kernel
    assert diff == {{"optimizer_kind": "optimizer", "factor_kind": "factor", "robust_kind": "robust", "rejector_kind": "rejector"}.get(field, field)}, diff
    assert not np.array_equal(ra.X, rb.X), field
