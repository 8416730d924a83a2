"""Stream-ordered graduated non-convexity for joint windows (sgb_align_joint_gnc_async, Context.align_joint_gnc_async): every stage and
joint round on the device.

  1. model equality: every window's X, info, stages, mu and per-point g, and the correspondences and error_batch afterwards, are
     bit-identical to the loop driven from the host with public calls on a context holding that window alone (np_joint_gnc.host_joint_gnc),
     over many kd-trees and many voxel maps (1 and 7 offsets), ICP / point-to-plane / GICP, GN and LM, GM and TLS, with and without caller
     weights, stage_iterations 1 and 3, max_iterations 0, 1 and 20, a DoF mask, and windows of 3, 8 and 32 frames with a fixed frame that
     is not the first, edges both ways and a duplicate edge;
  2. window counts 1, 17 and 1024 (permuted), windows finishing at different stages in one call, against the same model;
  3. degenerate windows: no edge, no free frame, an edge-less free frame, every window done from the start, a call with no edge at all:
     the same model for a window with an edge, the stated result for one without;
  4. no host wait; capture in torch.cuda.graph and replay from new poses and new weights, refusals inside a capture, and calls in sequence,
     each bit-identical to align_joint_gnc on a second context prepared alike; calls in sequence (options, windows, fixed flags, pairing,
     target, interleaved align_joint_async and align_batch_gnc_async) never replay a stale graph; the launch counter does not depend on
     the stage count;
  5. misuse fails with a message, enqueues nothing and leaves the weights in force."""
import ctypes
import itertools
from types import SimpleNamespace

import numpy as np
import pytest

import np_gnc as G
from test_gpu_align_joint import _perturbed
from np_joint_gnc import host_joint_gnc
from test_gpu_align_joint_gnc import C2, KINDS, MASK, WA, WB, WC, Scene, Window, _rows, check_window, multi
from test_gpu_batch_weights import random_weights

pytestmark = pytest.mark.gpu

GN, LM = 0, 1
ICP, PLANE, GICP = 0, 1, 2


def _torch():
    return pytest.importorskip("torch")


def _sg():
    import small_gicp_b200 as sg

    return sg


@pytest.fixture(scope="module")
def scene():
    return Scene()


@pytest.fixture(autouse=True)
def _side_stream():
    """every test runs on a torch stream of its own (the default stream is the null stream, which set_stream cannot name)"""
    torch = _torch()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        yield
    side.synchronize()


def _bind(ctx):
    ctx.set_stream(_torch().cuda.current_stream().cuda_stream)
    return ctx


def _bits(a, b, tag):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64)), (tag, a.shape, b.shape)


def _dev(X):
    return _torch().from_numpy(np.ascontiguousarray(X)).cuda()


def compare(r, a, tag):
    """a JointGncAlignResult against an AsyncJointGncAlignResult, bit for bit"""
    for f in ("X", "error", "mu"):
        _bits(getattr(r, f), getattr(a, f).cpu().numpy(), (tag, f))
    for f in ("converged", "iterations", "num_inliers", "stages"):
        _bits(np.asarray(getattr(r, f), dtype=np.float64), getattr(a, f).cpu().numpy(), (tag, f))
    _bits(r.point_w, a.point_w.cpu().numpy(), (tag, "point_w"))


def check(c1, c2, X, c2_, off, fixed, tag, **kw):
    """align_joint_gnc on c1, align_joint_gnc_async on c2 (prepared alike) from the same frames: every output bitwise equal, and the
    correspondences and error_batch at other edge poses each leaves behind"""
    r = c1.align_joint_gnc(X, c2_, windows=off, fixed=fixed, point_weights=True, **kw)
    a = c2.align_joint_gnc_async(_dev(X), c2_, windows=off, fixed=fixed, point_weights=True, **kw)
    c2.synchronize()
    compare(r, a, tag)
    for m, (x, y) in enumerate(zip(c1.correspondences_batch(), c2.correspondences_batch())):
        assert np.array_equal(x, y), (tag, "correspondences", m)
    if c1._batch_offsets.size > 1:
        T1 = c1.joint_edge_poses(r.X, windows=off)
        _bits(c1.error_batch(T1), c2.error_batch(T1), (tag, "error_batch"))
    return r, a


def check_model(ctx, X, c2, off, fixed, er, solo, tag, w=None, **kw):
    """align_joint_gnc_async on ctx with the weights w in force against np_joint_gnc.host_joint_gnc, once per distinct window: solo(k) is a
    context holding window k alone and that window's name, or None for a window without an edge (no context can hold it alone: its result
    is the stated one, X as given, no iteration, one stage at the first mu).  er: each window's edge range.  Every window's outputs bit for
    bit, and the correspondences and error_batch at other edge poses each leaves behind."""
    ctx.set_source_weights(w)
    a = ctx.align_joint_gnc_async(_dev(X), c2, windows=off, fixed=fixed, point_weights=True, **kw)
    ctx.synchronize()
    r = SimpleNamespace(**{f: getattr(a, f).cpu().numpy() for f in ("X", "converged", "iterations", "num_inliers", "error", "stages", "mu", "point_w")})
    corr = ctx.correspondences_batch()
    E = ctx._batch_offsets.size - 1
    T1 = ctx.joint_edge_poses(r.X, windows=off) if E else None
    e1 = ctx.error_batch(T1) if E else None
    model = dict(kw)
    gnc = model.pop("gnc", G.TLS)
    models = {}
    for k, (e0, e1_) in enumerate(er):
        f0, f1 = off[k], off[k + 1]
        if e0 == e1_:
            _bits(r.X[f0:f1], X[f0:f1], (tag, k, "X of a window without an edge"))
            assert not r.converged[k] and r.iterations[k] == 0 and r.error[k] == 0 and r.num_inliers[k] == 0, (tag, k)
            assert r.stages[k] == 1 and r.mu[k] == (1.0 if gnc == G.GM else 0.0), (tag, k)
            continue
        solo_ctx, name = solo(k)
        rows = _rows(ctx, e0, e1_)
        ws = None if w is None else w[rows].copy()
        key = (name, X[f0:f1].tobytes(), T1[e0:e1_].tobytes(), None if ws is None else ws.tobytes())
        if key not in models:
            m = host_joint_gnc(solo_ctx, X[f0:f1], c2, fixed=list(fixed[f0:f1]), kind=gnc, w=ws, **model)
            models[key] = m, solo_ctx.correspondences_batch(), solo_ctx.error_batch(T1[e0:e1_])
        m, m_corr, m_e1 = models[key]
        check_window(r, k, off, m, rows, tag)
        for q, (x, y) in enumerate(zip(corr[e0:e1_], m_corr)):
            assert np.array_equal(x, y), (tag, "correspondences", k, q)
        _bits(e1[e0:e1_], m_e1, (tag, "error_batch", k))
    return r


def solos(s, wins, kind):
    """solo(k) of check_model for the windows wins of multi(s, wins, kind): one context per distinct window"""
    ctxs = {}

    def solo(k):
        w = wins[k]
        if id(w) not in ctxs:
            ctxs[id(w)] = s.context(w.idx, kind, w.edges)
        return ctxs[id(w)], id(w)

    return solo


def twins(s, wins, kind):
    """two contexts holding the windows' frames and edges, the second bound to the current stream; the call's offsets, X and fixed flags"""
    c1, off, X, fixed, er = multi(s, wins, kind)
    c2 = _bind(multi(s, wins, kind)[0])
    return c1, c2, off, X, fixed, er


# ---- 1. equality with the host loop ----
COMBOS = list(itertools.product((GN, LM), (G.GM, G.TLS), (False, True), (1, 3), (20, 1, 0), (None, MASK)))


@pytest.mark.parametrize("kind", KINDS)
def test_equals_the_host_loop(scene, kind):
    s = scene
    wins = (WA, WB, WC)
    ctx, off, X, fixed, er = multi(s, wins, kind)
    _bind(ctx)
    solo = solos(s, wins, kind)
    n = int(ctx._batch_offsets[-1])
    factors = (ICP, PLANE, GICP) if kind == "kdtree" else (ICP, GICP)
    stages = []
    for fi, factor in enumerate(factors):
        for ci in range(4):
            opt, gnc, weighted, si, it, mask = COMBOS[(13 * fi + 29 * ci + 7 * KINDS.index(kind)) % len(COMBOS)]
            tag = (kind, factor, opt, gnc, weighted, si, it, mask)
            w = random_weights(n, 5 + ci) if weighted else None
            r = check_model(ctx, X, C2[factor], off, fixed, er, solo, tag, w=w, gnc=gnc, stage_iterations=si, factor=factor, optimizer=opt,
                            max_dist_sq=1.0, max_iterations=it, dof_mask=mask)
            stages += list(r.stages)
    print(kind, "stages: min", min(stages), "max", max(stages))
    assert max(stages) > 10  # the schedules ran many stages


def test_max_iterations_zero_and_one_stage(scene):
    s = scene
    wins = (WA, WB)
    ctx, off, X, fixed, er = multi(s, wins, "kdtree")
    _bind(ctx)
    solo = solos(s, wins, "kdtree")
    for gnc in (G.GM, G.TLS):
        for kw in (dict(max_iterations=0), dict(max_stages=1), dict(max_stages=1, max_iterations=0), dict(stage_iterations=1, max_iterations=0)):
            r = check_model(ctx, X, C2[GICP], off, fixed, er, solo, ("schedule", gnc, kw), gnc=gnc, factor=GICP, max_dist_sq=1.0, **kw)
            if kw.get("max_stages") == 1:
                assert np.all(r.stages == 1)
    # TLS without outliers: one stage of weights 1
    r = check_model(ctx, X, 1e30, off, fixed, er, solo, "tls without outliers", gnc=G.TLS, factor=GICP, max_dist_sq=1e6, max_iterations=10)
    assert np.all(r.stages == 1) and np.all(r.mu == 0.0)


# ---- 2. window counts ----
@pytest.mark.parametrize("count,pool", [(1, "B"), (17, "ABD"), (1024, "D")])
def test_window_counts(scene, count, pool):
    """every window of a shape with that shape's weights: one host loop per shape is the model of all its windows"""
    s = scene
    shapes = {"A": WA, "B": WB, "D": Window([20, 21], [(1, 0)], [1, 0], 24)}
    names = [pool[i] for i in np.random.default_rng(count).integers(len(pool), size=count)]  # a permuted pairing of window shapes
    wins = [shapes[k] for k in names]
    ctx, off, X, fixed, er = multi(s, wins, "kdtree")
    _bind(ctx)
    rows = {k: _rows(ctx, *r) for k, r in zip(names, er)}
    sw = {k: random_weights(rows[k].stop - rows[k].start, 3 + i) for i, k in enumerate(shapes) if k in rows}
    w = np.concatenate([sw[k] for k in names])
    for gnc, weights in ((G.TLS, None), (G.GM, w)):
        r = check_model(ctx, X, C2[GICP], off, fixed, er, solos(s, wins, "kdtree"), (count, gnc), w=weights, gnc=gnc, factor=GICP, max_dist_sq=1.0)
        if count == 17:
            assert len(set(r.stages)) > 1  # windows finished at different stages in one call


# ---- 3. degenerate windows ----
def test_degenerate_windows(scene):
    s = scene
    idx = [5, 6, 7, 8, 9, 10]
    X = _perturbed(s.fr, idx, 4)
    ctx = _bind(s.context(idx, "kdtree", [(1, 0), (4, 3)]))
    # each window with an edge alone, by its first frame: frames 0 .. 2 or 3 .. 4 of idx and its one edge 1 -> 0 (local)
    alone = {f0: s.context(idx[f0:f1], "kdtree", [(1, 0)]) for f0, f1 in ((0, 3), (3, 5))}

    def solo(off):
        return lambda k: (alone[off[k]], off[k])

    for gnc in (G.GM, G.TLS):
        # windows: [] (empty) | [0, 1, 2] with edge 1 -> 0 and the edge-less free frame 2 | [3, 4] all fixed with an edge | [5] alone
        off = [0, 0, 3, 5, 6]
        check_model(ctx, X, C2[GICP], off, [1, 0, 0, 1, 1, 0], [(0, 0), (0, 1), (1, 2), (2, 2)], solo(off), ("degenerate", gnc), gnc=gnc, factor=GICP,
                    max_dist_sq=1.0)
        # every window done from the start
        off = [0, 3, 5, 6]
        r = check_model(ctx, X, C2[GICP], off, [1, 1, 1, 1, 1, 0], [(0, 1), (1, 2), (2, 2)], solo(off), ("all done", gnc), gnc=gnc, factor=GICP,
                        max_dist_sq=1.0)
        assert np.all(r.iterations == 0)


def test_call_without_edges(scene):
    """a pairing of no member: no edge and no point at all, the stated result for every window"""
    s = scene
    idx = [11, 12, 13]
    X = _perturbed(s.fr, idx, 5)
    none = np.zeros(0, dtype=np.uint32)
    ctx = _bind(s.context(idx, "voxelmap1", [(1, 0)]))
    ctx.set_source_pairs(none, none)
    for gnc, mu in ((G.GM, 1.0), (G.TLS, 0.0)):
        n0 = ctx.kernel_launches
        r = check_model(ctx, X, C2[GICP], [0, 2, 3], [1, 0, 0], [(0, 0), (0, 0)], None, ("no edge", gnc), gnc=gnc, factor=GICP, max_dist_sq=1.0)
        assert ctx.kernel_launches - n0 == 4
        _bits(r.X, X, "initial poses")
        assert np.all(r.stages == 1) and np.all(r.mu == mu) and np.all(r.iterations == 0) and not np.any(r.converged)


# ---- 4. behaviour around the call ----
def test_no_host_synchronisation(scene):
    torch = _torch()
    s = scene
    c1, c2, off, X, fixed, er = twins(s, (WA, WB), "kdtree")
    kw = dict(windows=off, fixed=fixed, gnc=G.TLS, factor=GICP, max_dist_sq=1.0)
    ref = c1.align_joint_gnc(X, C2[GICP], **kw)
    Xd = _dev(X)
    c2.align_joint_gnc_async(Xd, C2[GICP], **kw)  # warm: the tables are uploaded and the graph is built and cached
    c2.synchronize()
    torch.cuda._sleep(2_000_000_000)  # about a second of spinning on the context's stream
    a = c2.align_joint_gnc_async(Xd, C2[GICP], **kw)
    done = torch.cuda.Event()
    done.record()
    assert not done.query(), "the call waited for the stream"
    moved = (a.X @ torch.eye(4, dtype=torch.float64, device="cuda")).clone()  # a torch op consuming the frames, no synchronisation
    c2.synchronize()
    _bits(ref.X, a.X.cpu().numpy(), "after synchronize")
    _bits(ref.X, moved.cpu().numpy(), "stream-ordered consumer")


def test_graph_capture_and_replay(scene):
    torch = _torch()
    sg = _sg()
    s = scene
    c1, c2, off, X, fixed, er = twins(s, (WA, WB), "voxelmap7")
    n = int(c1._batch_offsets[-1])
    kw = dict(windows=off, fixed=fixed, gnc=G.TLS, factor=GICP, max_dist_sq=1.0, stage_iterations=2)
    Xd = _dev(X)
    side = torch.cuda.Stream()
    # a first call inside a capture is refused: it would allocate and upload its tables
    fresh = multi(s, (WA, WB), "voxelmap7")[0]
    fresh.set_stream(side.cuda_stream)
    g = torch.cuda.CUDAGraph()
    n0 = fresh.kernel_launches
    with pytest.raises(sg.SgbError, match="call it once outside the capture first"):
        with torch.cuda.graph(g, stream=side):
            fresh.align_joint_gnc_async(Xd, C2[GICP], point_weights=True, **kw)
    assert fresh.kernel_launches == n0
    torch.cuda.synchronize()
    c2.set_stream(side.cuda_stream)
    ws = [random_weights(n, 11 + k) for k in range(3)]
    c2.set_source_weights(ws[0])  # a capture reads the weights in force through their buffer: set again, they are read at each replay
    with torch.cuda.stream(side):
        out = c2.align_joint_gnc_async(Xd, C2[GICP], point_weights=True, **kw)  # warm-up outside the capture
    side.synchronize()
    # a call whose window tables changed is refused inside the capture
    g = torch.cuda.CUDAGraph()
    n0 = c2.kernel_launches
    with pytest.raises(sg.SgbError, match="call it once outside the capture first"):
        with torch.cuda.graph(g, stream=side):
            c2.align_joint_gnc_async(Xd, C2[GICP], point_weights=True, out=out, **dict(kw, fixed=[1] + list(fixed[1:3]) + [1] + list(fixed[4:])))
    assert c2.kernel_launches == n0
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        c2.align_joint_gnc_async(Xd, C2[GICP], point_weights=True, out=out, **kw)
    c2.synchronize()
    for k, w in ((31, ws[0]), (32, ws[1]), (33, ws[2]), (32, ws[1])):
        Xk = np.concatenate([_perturbed(s.fr, win.idx, k) for win in (WA, WB)])
        c1.set_source_weights(w)
        c2.set_source_weights(w)
        with torch.cuda.stream(side):
            Xd.copy_(torch.from_numpy(Xk))
            g.replay()
        side.synchronize()
        compare(c1.align_joint_gnc(Xk, C2[GICP], point_weights=True, **kw), out, ("replay", k))
    c2.set_stream(None)


def test_calls_in_sequence_never_replay_a_stale_graph(scene):
    s = scene
    c1, c2, off, X, fixed, er = twins(s, (WA, WB), "kdtree")
    base = dict(gnc=G.TLS, max_stages=40, stage_iterations=3, factor=GICP, max_dist_sq=1.0, max_iterations=20)

    def call(tag, X_=None, c2_=C2[GICP], off_=off, fixed_=fixed, **change):
        check(c1, c2, X if X_ is None else X_, c2_, off_, fixed_, tag, **dict(base, **change))

    call("first")
    call("new poses", X_=np.concatenate([_perturbed(s.fr, w.idx, 40) for w in (WA, WB)]))
    for change in (dict(gnc=G.GM), dict(max_stages=3), dict(stage_iterations=1), dict(optimizer=GN), dict(factor=ICP), dict(max_iterations=1),
                   dict(max_dist_sq=0.5), dict(dof_mask=MASK)):
        call(("options", change), **change)
    call("noise bound", c2_=0.1)
    call("new windows", off_=[0, 11], fixed_=[1, 0, 0, 1, 0, 0, 0, 0, 0, 0, 0])  # the same frames as one window
    call("new fixed flags", fixed_=[1, 0, 0, 1, 0, 0, 1, 0, 0, 0, 0])
    # interleaved calls that share the member phases, the GNC buffers and the asynchronous window tables
    fx2 = [1, 0, 1, 0, 0, 0, 1, 0, 0, 0, 0]
    rj = c1.align_joint(X, windows=off, fixed=fx2, factor=GICP, max_dist_sq=1.0)
    aj = c2.align_joint_async(_dev(X), windows=off, fixed=fx2, factor=GICP, max_dist_sq=1.0)  # other window tables in the shared cache
    c2.synchronize()
    _bits(rj.X, aj.X.cpu().numpy(), "align_joint_async between")
    call("after align_joint_async")
    E = c1._batch_offsets.size - 1
    T = c1.joint_edge_poses(X, windows=off)
    rb = c1.align_batch_gnc(T, C2[GICP], gnc=G.GM, factor=GICP, max_dist_sq=1.0, point_weights=True)
    ab = c2.align_batch_gnc_async(_dev(T), C2[GICP], gnc=G.GM, factor=GICP, max_dist_sq=1.0, point_weights=True)
    c2.synchronize()
    _bits(rb.T_target_source, ab.T_target_source.cpu().numpy(), "align_batch_gnc_async between")
    assert E == ab.T16.shape[0]
    call("after align_batch_gnc_async")
    # a re-pairing, then a target rebuild under it
    edges = [(1, 0), (2, 0), (4, 3), (5, 4), (7, 6), (10, 9), (9, 8)]
    for c in (c1, c2):
        c.set_source_pairs(np.array([i for i, _ in edges], dtype=np.uint32), np.array([j for _, j in edges], dtype=np.uint32))
    call("re-paired")
    idx = WA.idx + WB.idx
    for c in (c1, c2):
        c.build_target_voxelmaps([s.pts[i] for i in idx], [s.covs[i] for i in idx], 1.0, 1)
    call("new target")
    call("new target, again", gnc=G.GM)


def test_launch_count_is_constant(scene):
    torch = _torch()
    s = scene
    ctx, off, X, fixed, er = multi(s, (WA, WB), "kdtree")
    _bind(ctx)
    Xd = _dev(X)
    kw = dict(windows=off, fixed=fixed, factor=GICP, max_dist_sq=1.0)
    ctx.align_joint_gnc_async(Xd, C2[GICP], **kw)  # warm: the first call builds the pairing's view
    seen = set()
    for max_stages in (1, 2, 5, 12, 64):
        for gnc, c2 in ((G.GM, C2[GICP]), (G.TLS, C2[GICP]), (G.GM, 1e-4), (G.TLS, 1e-3)):
            n0 = ctx.kernel_launches
            a = ctx.align_joint_gnc_async(Xd, c2, gnc=gnc, max_stages=max_stages, **kw)
            assert ctx.kernel_launches - n0 == 3, (max_stages, gnc, ctx.kernel_launches - n0)
            ctx.synchronize()
            seen.add((gnc, int(a.stages.max().item())))
    print("stage counts", sorted(seen))
    for gnc in (G.GM, G.TLS):
        st = [k for g, k in seen if g == gnc]
        assert min(st) == 1 and max(st) >= 10, (gnc, st)
    torch.cuda.synchronize()


def _managed(nbytes):
    """a managed allocation (cudaMallocManaged) as a ctypes pointer, or None where the runtime library cannot be loaded"""
    try:
        rt = ctypes.CDLL("libcudart.so.12")
    except OSError:
        return None, None
    p = ctypes.c_void_p()
    assert rt.cudaMallocManaged(ctypes.byref(p), ctypes.c_size_t(nbytes), ctypes.c_uint(1)) == 0
    return rt, p


def test_misuse_fails_with_a_message(scene):
    torch = _torch()
    sg = _sg()
    s = scene
    c1, ctx, off, X, fixed, er = twins(s, (WA, WB), "kdtree")
    Xd = _dev(X)
    ctx.set_stream(None)
    with pytest.raises(sg.SgbError, match="set the context's stream"):
        ctx.align_joint_gnc_async(Xd, C2[GICP], windows=off, fixed=fixed)
    _bind(ctx)
    n = int(ctx._batch_offsets[-1])
    w = random_weights(n, 31)
    ctx.set_source_weights(w)
    c1.set_source_weights(w)
    kw0 = dict(windows=off, fixed=fixed, max_dist_sq=1.0, point_weights=True)
    ref = c1.align_joint_gnc(X, C2[GICP], **kw0)

    def usable():
        a = ctx.align_joint_gnc_async(Xd, C2[GICP], **kw0)
        ctx.synchronize()
        compare(ref, a, "usable")

    usable()
    # every refusal of the synchronous call but the capture's
    for kw, msg in ((dict(robust=sg.ROBUST_HUBER), "robust_kind must be SGB_ROBUST_NONE"), (dict(gnc=2), "invalid GNC kind"),
                    (dict(gnc=-1), "invalid GNC kind"), (dict(c2=0.0), "noise_bound_sq must be finite and > 0"), (dict(c2=-1.0), "noise_bound_sq"),
                    (dict(c2=np.inf), "noise_bound_sq"), (dict(c2=np.nan), "noise_bound_sq"), (dict(max_stages=0), "max_stages must be >= 1"),
                    (dict(stage_iterations=0), "stage_iterations must be >= 1"), (dict(factor=7), "invalid factor"),
                    (dict(windows=[0, 3]), "must run from 0"), (dict(windows=[0, 3, 2, 11]), "ascending"),
                    (dict(windows=[0, 2, 11]), "both frames of an edge"), (dict(fixed=[0] * 11), "no fixed frame")):
        c2 = kw.pop("c2", C2[GICP])
        n0 = ctx.kernel_launches
        with pytest.raises(sg.SgbError, match="sgb_align_joint_gnc_async: .*" + msg):
            ctx.align_joint_gnc_async(Xd, c2, **dict(kw0, **kw))
        assert ctx.kernel_launches == n0, msg
    usable()
    # host, page-locked and managed pointers
    L, h = ctx._L, ctx._h
    o = sg.capi._align_options(max_dist_sq=1.0)
    g = sg.capi.GncOptions(G.TLS, C2[GICP], 64, 3)
    K, W = X.shape[0], len(off) - 1
    offs = np.ascontiguousarray(np.array(off, dtype=np.uintp))
    fx = np.ascontiguousarray(np.array(fixed, dtype=np.uint8))
    host = np.zeros((K, 16))
    pinned = torch.zeros((K, 16), dtype=torch.float64).pin_memory()
    dev = [torch.zeros((r, k), dtype=torch.float64, device="cuda") for r, k in ((K, 16), (W, 4), (W, 2))]
    pw = torch.zeros(n, dtype=torch.float64, device="cuda")
    Xc = Xd.transpose(1, 2).contiguous()
    p = sg.capi._d
    hp = host.ctypes.data_as(sg.capi._dp)
    rt, managed = _managed(n * 8)
    mp = ctypes.cast(managed, sg.capi._dp) if managed is not None else None
    full = [p(Xc), p(dev[0]), p(dev[1]), p(dev[2]), p(pw)]

    def with_(i, v):
        a = list(full)
        a[i] = v
        return a

    cases = [((o, None, full), "null GNC options"), ((None, g, full), "null options"), ((o, g, with_(1, None)), "null output"),
             ((o, g, with_(2, None)), "null output"), ((o, g, with_(0, None)), "null poses")]
    for i, what in enumerate(("init_X16xK", "out_X16xK", "out_info4xW", "out_gnc2xW", "out_point_w")):
        cases.append(((o, g, with_(i, hp)), what + " must be device memory"))
    cases.append(((o, g, with_(1, p(pinned))), "out_X16xK must be device memory"))
    if mp is not None:
        cases.append(((o, g, with_(4, mp)), "out_point_w must be device memory"))
        cases.append(((o, g, with_(0, mp)), "init_X16xK must be device memory"))
    for (oo, gg, args), msg in cases:
        n0 = ctx.kernel_launches
        rc = L.sgb_align_joint_gnc_async(h, None if oo is None else ctypes.byref(oo), None if gg is None else ctypes.byref(gg), W,
                                         offs.ctypes.data_as(ctypes.POINTER(ctypes.c_size_t)), fx.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), *args)
        assert rc != 0, msg
        assert msg in L.sgb_last_error(h).decode(), (msg, L.sgb_last_error(h))
        assert ctx.kernel_launches == n0, msg
    if managed is not None:
        rt.cudaFree(managed)
    usable()
    # what align_joint refuses: no pairing with a maps table, a self-edge
    T = c1.joint_edge_poses(X, windows=off)
    before = c1.linearize_batch_points(T, factor=GICP)
    after = ctx.linearize_batch_points(T, factor=GICP)
    _bits(before.point_e, after.point_e, "weights in force")  # the weights in force are those set before the refusals
    _bits(before.H, after.H, "weights in force")
    ctx.set_source_pairs(np.array([1, 2], dtype=np.uint32), None)
    with pytest.raises(sg.SgbError, match="pairing with a maps table"):
        ctx.align_joint_gnc_async(Xd, C2[GICP], windows=off)
    ctx.set_source_pairs(np.array([1, 2], dtype=np.uint32), np.array([0, 2], dtype=np.uint32))
    with pytest.raises(sg.SgbError, match="of its own frame"):
        ctx.align_joint_gnc_async(Xd, C2[GICP], windows=off)
