"""Stream-ordered graduated non-convexity (sgb_align_batch_gnc_async, Context.align_batch_gnc_async): every stage and round on the device.

  1. model equality: every member's T, info, H | b, stages, mu and per-point g, and the correspondences and error_batch afterwards, are
     bit-identical to the loop driven from the host with public calls on a context holding that member alone (np_gnc.host_gnc), over every
     target kind, factor, optimiser, GNC kind, with and without caller weights, stage_iterations 1 and 3, max_iterations 0, 1 and 20;
  2. degenerate schedules: TLS without outliers, max_stages = 1, an empty target, against the same model;
  3. batch sizes 1, 17 and 1024, and a permuted batch, against the same model;
  4. no host wait; capture in torch.cuda.graph and replay from new poses and new weights, and calls in sequence, each bit-identical to
     align_batch_gnc on a second context prepared alike; calls in sequence never replay a stale graph; the launch counter does not
     depend on the stage count;
  5. misuse fails with a message, enqueues nothing and leaves the weights in force."""
import ctypes
import itertools
from types import SimpleNamespace

import numpy as np
import pytest

import np_gnc as G
from test_gpu_align_gnc import C2, FIELDS, KINDS, PLANE_KINDS, _rows, check_member, members, pair, poses, target
from test_gpu_batch_points import LEAF, Scene
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


def _dev(T):
    return _torch().from_numpy(np.ascontiguousarray(T)).cuda()


def check(sync_ctx, async_ctx, T0, T1, c2, tag, **kw):
    """align_batch_gnc on sync_ctx, align_batch_gnc_async on async_ctx (prepared alike) from the same poses: every output bitwise equal,
    and the correspondences and error_batch each leaves behind"""
    r = sync_ctx.align_batch_gnc(T0, c2, point_weights=True, **kw)
    a = async_ctx.align_batch_gnc_async(_dev(T0), c2, point_weights=True, **kw)
    async_ctx.synchronize()
    compare(r, a, tag)
    for m, (x, y) in enumerate(zip(sync_ctx.correspondences_batch(), async_ctx.correspondences_batch())):
        assert np.array_equal(x, y), (tag, "correspondences", m)
    _bits(sync_ctx.error_batch(T1), async_ctx.error_batch(T1), (tag, "error_batch"))
    return r, a


def check_model(ctx, solo, member, T0, T1, c2, tag, w=None, **kw):
    """align_batch_gnc_async on ctx with the weights w in force against np_gnc.host_gnc on solo, once per distinct member (member(p) pairs
    solo with member p alone and names its cloud; a member without points is skipped, as the host loop has none to run): every member's
    outputs bit for bit, and the correspondences and error_batch each leaves behind"""
    ctx.set_source_weights(w)
    a = ctx.align_batch_gnc_async(_dev(T0), c2, point_weights=True, **kw)
    ctx.synchronize()
    r = SimpleNamespace(**{f: getattr(a, f).cpu().numpy() for f in FIELDS + ("stages", "mu", "point_w")})
    corr, e1 = ctx.correspondences_batch(), ctx.error_batch(T1)
    model = dict(kw)
    gnc = model.pop("gnc", G.TLS)
    models = {}
    for p in range(len(T0)):
        rows = _rows(ctx, p)
        if rows.start == rows.stop:
            continue
        ws = None if w is None else w[rows].copy()
        cloud = member(p)
        key = (cloud, T0[p].tobytes(), T1[p].tobytes(), None if ws is None else ws.tobytes())
        if key not in models:
            m = G.host_gnc(solo, T0[p], c2, kind=gnc, w=ws, **model)
            models[key] = m, solo.correspondences_batch()[0], solo.error_batch(T1[p : p + 1])[0]
        m, m_corr, m_e1 = models[key]
        check_member(r, p, m, rows, tag)
        assert np.array_equal(corr[p], m_corr), (tag, "correspondences", p)
        _bits(e1[p], m_e1, (tag, "error_batch", p))
    return r


def compare(r, a, tag):
    """a GncAlignResult against an AsyncGncAlignResult, bit for bit"""
    for f in ("T_target_source", "H", "b", "error", "mu"):
        _bits(getattr(r, f), getattr(a, f).cpu().numpy(), (tag, f))
    for f in ("converged", "iterations", "num_inliers", "stages"):
        _bits(np.asarray(getattr(r, f), dtype=np.float64), getattr(a, f).cpu().numpy(), (tag, f))
    _bits(r.point_w, a.point_w.cpu().numpy(), (tag, "point_w"))


def twins(s, kind):
    """two contexts holding the kind's target and members, the second bound to the current stream"""
    c1, c2 = target(s, kind), _bind(target(s, kind))
    pair(c1, s, kind)
    pair(c2, s, kind)
    return c1, c2


def solo_of(s, kind):
    """a context holding the kind's target, and the member(p) of check_model that pairs it with member p of the kind's batch"""
    solo = target(s, kind)

    def member(p):
        pair(solo, s, kind, p)
        return p

    return solo, member


# ---- 1. equality with the host loop ----
COMBOS = list(itertools.product((GN, LM), (G.GM, G.TLS), (False, True), (1, 3), (20, 1, 0)))


@pytest.mark.parametrize("kind", KINDS)
def test_equals_the_host_loop(scene, kind):
    s = scene
    ctx = _bind(target(s, kind))
    pair(ctx, s, kind)
    solo, member = solo_of(s, kind)
    cl = members(kind)
    T0, T1 = poses(s, cl), poses(s, cl, 1)
    n = int(ctx._batch_offsets[-1])
    factors = (ICP, PLANE, GICP) if kind in PLANE_KINDS else (ICP, GICP)
    stages = []
    for fi, factor in enumerate(factors):
        for ci in range(4):
            opt, gnc, weighted, si, it = COMBOS[(7 * fi + 11 * ci + 3 * len(kind)) % len(COMBOS)]
            tag = (kind, factor, opt, gnc, weighted, si, it)
            w = random_weights(n, 5 + ci) if weighted else None
            r = check_model(ctx, solo, member, T0, T1, C2[factor], tag, w=w, gnc=gnc, max_stages=40, stage_iterations=si, factor=factor,
                            optimizer=opt, max_dist_sq=0.25, max_iterations=it)
            stages.append(r.stages)
    st = np.concatenate(stages)
    print(kind, "stages: min", st.min(), "max", st.max())
    assert st.max() > 2  # the schedules ran several stages


# ---- 2. degenerate schedules ----
def test_degenerate_schedules(scene):
    s = scene
    ctx = _bind(target(s, "kdtree"))
    solo, member = solo_of(s, "kdtree")
    cl = members("kdtree")
    T0, T1 = poses(s, cl), poses(s, cl, 1)
    # TLS without outliers: one stage of weights 1
    for factor, opt in ((ICP, GN), (GICP, LM), (PLANE, LM)):
        r = check_model(ctx, solo, member, T0, T1, 1e30, ("tls without outliers", factor), gnc=G.TLS, factor=factor, optimizer=opt, max_dist_sq=1e6,
                        max_iterations=10)
        assert np.all(r.stages == 1) and np.all(r.mu == 0.0)
    # one stage
    for gnc in (G.GM, G.TLS):
        r = check_model(ctx, solo, member, T0, T1, C2[GICP], ("one stage", gnc), gnc=gnc, max_stages=1, factor=GICP, max_dist_sq=0.25)
        assert np.all(r.stages == 1)


def test_empty_target(scene):
    s = scene
    ctxs = []
    for _ in range(2):
        ctx = _sg().Context(0)
        ctx.set_target(np.zeros((0, 4)), None, np.zeros((0, 4, 4)))
        ctx.build_target_kdtree()
        ctx.set_source_batch(s.srcs, s.scovs)
        ctxs.append(ctx)
    ctx, solo = _bind(ctxs[0]), ctxs[1]

    def member(p):
        solo.set_source_pairs([p])
        return p

    cl = list(range(len(s.srcs)))
    for gnc in (G.GM, G.TLS):
        check_model(ctx, solo, member, poses(s, cl), poses(s, cl, 1), C2[GICP], ("empty target", gnc), gnc=gnc, factor=GICP, max_dist_sq=0.25)


# ---- 3. batch sizes ----
@pytest.mark.parametrize("B", [1, 17, 1024])
def test_batch_sizes(scene, B):
    """every replica of a cloud at the cloud's poses and weights: one host loop per cloud is the model of all its replicas"""
    s = scene
    ctx = _bind(target(s, "kdtree"))
    solo = target(s, "kdtree")
    rng = np.random.default_rng(B)
    clouds = [0, 1, 2, 4]
    cl = clouds[:B] if B == 1 else list(rng.permutation(np.resize(clouds, B)))  # a permuted batch
    ctx.set_source_pairs(cl)

    def member(p):
        pair(solo, s, "kdtree", cl[p])
        return cl[p]

    T0, T1 = (dict(zip(clouds, poses(s, clouds, k))) for k in (0, 1))
    cw = {c: random_weights(len(s.srcs[c]), 3 + c) for c in clouds}
    w = np.concatenate([cw[c] for c in cl])
    for gnc, weights in ((G.TLS, None), (G.GM, w)):
        check_model(ctx, solo, member, np.array([T0[c] for c in cl]), np.array([T1[c] for c in cl]), C2[GICP], ("B", B, gnc), w=weights, gnc=gnc,
                    factor=GICP, max_dist_sq=0.25)


# ---- 4. behaviour around the call ----
def test_no_host_wait(scene):
    torch = _torch()
    s = scene
    c1, c2 = twins(s, "kdtree")
    cl = members("kdtree")
    T0 = poses(s, cl)
    ref = c1.align_batch_gnc(T0, C2[GICP], gnc=G.TLS, factor=GICP, max_dist_sq=0.25)
    Td = _dev(T0)
    c2.align_batch_gnc_async(Td, C2[GICP], gnc=G.TLS, factor=GICP, max_dist_sq=0.25)  # warm: the graph is built and cached
    c2.synchronize()
    torch.cuda._sleep(2_000_000_000)  # about a second of spinning on the context's stream
    a = c2.align_batch_gnc_async(Td, C2[GICP], gnc=G.TLS, factor=GICP, max_dist_sq=0.25)
    done = torch.cuda.Event()
    done.record()
    assert not done.query(), "the call waited for the stream"
    moved = (a.T_target_source @ torch.eye(4, dtype=torch.float64, device="cuda")).clone()  # a torch op consuming the poses, no synchronisation
    c2.synchronize()
    _bits(ref.T_target_source, a.T_target_source.cpu().numpy(), "after synchronize")
    _bits(ref.T_target_source, moved.cpu().numpy(), "stream-ordered consumer")


def test_graph_capture_and_replay(scene):
    torch = _torch()
    sg = _sg()
    s = scene
    c1, c2 = target(s, "kdtrees"), target(s, "kdtrees")
    cl = members("kdtrees")
    n = int(c1._batch_offsets[-1])
    kw = dict(gnc=G.TLS, factor=GICP, max_dist_sq=0.25, stage_iterations=2)
    T0 = _dev(poses(s, cl))
    side = torch.cuda.Stream()
    # a first call inside a capture is refused: it would allocate
    fresh = target(s, "kdtrees")
    fresh.set_stream(side.cuda_stream)
    g = torch.cuda.CUDAGraph()
    with pytest.raises(sg.SgbError, match="call it once outside the capture first"):
        with torch.cuda.graph(g, stream=side):
            fresh.align_batch_gnc_async(T0, C2[GICP], point_weights=True, **kw)
    torch.cuda.synchronize()
    c2.set_stream(side.cuda_stream)
    ws = [random_weights(n, 11 + k) for k in range(3)]
    c2.set_source_weights(ws[0])  # a capture reads the weights in force through their buffer: set again, they are read at each replay
    with torch.cuda.stream(side):
        out = c2.align_batch_gnc_async(T0, C2[GICP], point_weights=True, **kw)  # warm-up outside the capture
    side.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        c2.align_batch_gnc_async(T0, C2[GICP], point_weights=True, out=out, **kw)
    c2.synchronize()
    for k, w in ((1, ws[0]), (2, ws[1]), (3, ws[2]), (2, ws[1])):
        Tk = poses(s, cl, k)
        c1.set_source_weights(w)
        c2.set_source_weights(w)
        with torch.cuda.stream(side):
            T0.copy_(torch.from_numpy(Tk))
            g.replay()
        side.synchronize()
        compare(c1.align_batch_gnc(Tk, C2[GICP], point_weights=True, **kw), out, ("replay", k))
    c2.set_stream(None)


def test_calls_in_sequence_never_replay_a_stale_graph(scene):
    s = scene
    c1, c2 = twins(s, "kdtrees")
    cl = members("kdtrees")
    base = dict(gnc=G.TLS, max_stages=40, stage_iterations=3, factor=GICP, max_dist_sq=0.25, max_iterations=20)

    def call(tag, k=0, c2_=C2[GICP], cl_=cl, **change):
        kw = dict(base, **change)
        check(c1, c2, poses(s, cl_, k), poses(s, cl_, k + 1), c2_, tag, **kw)

    call("first")
    call("same again", k=1)
    for change in (dict(gnc=G.GM), dict(max_stages=3), dict(stage_iterations=1), dict(optimizer=GN), dict(factor=ICP), dict(max_iterations=1),
                   dict(max_dist_sq=1.0)):
        call(("options", change), **change)
    call("noise bound", c2_=0.1)
    c1.set_source_batch(s.srcs[1:] + s.srcs[:1], s.scovs[1:] + s.scovs[:1])  # other clouds
    c2.set_source_batch(s.srcs[1:] + s.srcs[:1], s.scovs[1:] + s.scovs[:1])
    call("new batch", cl_=[1, 2, 3, 4, 0])
    for c in (c1, c2):
        c.set_source_pairs([0, 2, 2, 3], [4, 3, 0, 1])
    call("re-paired", cl_=[1, 3, 3, 4])
    for c in (c1, c2):
        c.build_target_voxelmaps(s.maps, s.mcovs, LEAF, 7)  # a target rebuild under the same pairing
    call("new target", cl_=[1, 3, 3, 4])
    for c in (c1, c2):
        c.set_target(s.tp, s.tn, s.tcv)
        c.build_target_kdtree()
        c.set_source_batch(s.srcs, s.scovs)
    call("single tree", cl_=list(range(5)), factor=PLANE)


def test_launch_count_is_constant(scene):
    torch = _torch()
    s = scene
    ctx = _bind(target(s, "kdtree"))
    cl = members("kdtree")
    Td = _dev(poses(s, cl))
    ctx.align_batch_gnc_async(Td, C2[GICP])  # warm: the first call builds the pairing's view
    seen = set()
    for max_stages in (1, 2, 5, 12, 40):
        for gnc, c2 in ((G.GM, C2[GICP]), (G.TLS, C2[GICP]), (G.TLS, 1e-3)):
            n0 = ctx.kernel_launches
            a = ctx.align_batch_gnc_async(Td, c2, gnc=gnc, max_stages=max_stages, factor=GICP, max_dist_sq=0.25)
            assert ctx.kernel_launches - n0 == 4, (max_stages, gnc, ctx.kernel_launches - n0)
            ctx.synchronize()
            seen.add(int(a.stages.max().item()))
    print("stage counts", sorted(seen))
    assert min(seen) == 1 and max(seen) >= 10
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
    ctx = sg.Context(0)
    c1 = target(s, "kdtree")
    ctx.set_target(s.tp, s.tn, s.tcv)
    ctx.build_target_kdtree()
    cl = members("kdtree")
    T0 = poses(s, cl)
    Td = _dev(T0)
    with pytest.raises(sg.SgbError, match="set the context's stream"):
        ctx.align_batch_gnc_async(Td, C2[GICP])
    _bind(ctx)
    with pytest.raises(sg.SgbError, match="no batch"):
        ctx.align_batch_gnc_async(Td, C2[GICP])
    ctx.set_source_batch(s.srcs, s.scovs)
    n = int(ctx._batch_offsets[-1])
    w = random_weights(n, 31)
    ctx.set_source_weights(w)
    c1.set_source_weights(w)
    ref = c1.align_batch_gnc(T0, C2[GICP], max_dist_sq=0.25, point_weights=True)

    def usable():
        a = ctx.align_batch_gnc_async(Td, C2[GICP], max_dist_sq=0.25, point_weights=True)
        ctx.synchronize()
        compare(ref, a, "usable")

    # every refusal of the synchronous call
    for kw, msg in ((dict(robust=sg.ROBUST_HUBER), "robust_kind must be SGB_ROBUST_NONE"), (dict(gnc=2), "invalid GNC kind"),
                    (dict(gnc=-1), "invalid GNC kind"), (dict(c2=0.0), "noise_bound_sq must be finite and > 0"),
                    (dict(c2=-1.0), "noise_bound_sq"), (dict(c2=np.inf), "noise_bound_sq"), (dict(c2=np.nan), "noise_bound_sq"),
                    (dict(max_stages=0), "max_stages must be >= 1"), (dict(stage_iterations=0), "stage_iterations must be >= 1"),
                    (dict(factor=7), "invalid factor")):
        c2 = kw.pop("c2", C2[GICP])
        n0 = ctx.kernel_launches
        with pytest.raises(sg.SgbError, match="sgb_align_batch_gnc_async: " + msg):
            ctx.align_batch_gnc_async(Td, c2, max_dist_sq=0.25, **kw)
        assert ctx.kernel_launches == n0, msg
    usable()
    # host, page-locked and managed pointers
    L, h = ctx._L, ctx._h
    o = sg.capi._align_options(max_dist_sq=0.25)
    g = sg.capi.GncOptions(G.TLS, C2[GICP], 64, 3)
    B = len(cl)
    host = np.zeros((B, 42))
    pinned = torch.zeros((B, 16), dtype=torch.float64).pin_memory()
    dev = [torch.zeros((B, k), dtype=torch.float64, device="cuda") for k in (16, 4, 42, 2)]
    pw = torch.zeros(n, dtype=torch.float64, device="cuda")
    Tc = Td.transpose(1, 2).contiguous()
    p = sg.capi._d
    hp = host.ctypes.data_as(sg.capi._dp)
    rt, managed = _managed(n * 8)
    mp = ctypes.cast(managed, sg.capi._dp) if managed is not None else None
    full = [p(Tc), p(dev[0]), p(dev[1]), p(dev[2]), p(dev[3]), p(pw)]

    def with_(i, v):
        a = list(full)
        a[i] = v
        return a

    cases = [((o, None, full), "null GNC options"), ((None, g, full), "null options"), ((o, g, with_(1, None)), "null output"),
             ((o, g, with_(2, None)), "null output"), ((o, g, with_(0, None)), "null poses")]
    for i, what in enumerate(("init_T16xB", "out_T16xB", "out_info4xB", "out_Hb42xB", "out_gnc2xB", "out_point_w")):
        cases.append(((o, g, with_(i, hp)), what + " must be device memory"))
    cases.append(((o, g, with_(1, p(pinned))), "out_T16xB must be device memory"))
    if mp is not None:
        cases.append(((o, g, with_(5, mp)), "out_point_w must be device memory"))
        cases.append(((o, g, with_(0, mp)), "init_T16xB must be device memory"))
    for (oo, gg, args), msg in cases:
        n0 = ctx.kernel_launches
        assert L.sgb_align_batch_gnc_async(h, None if oo is None else ctypes.byref(oo), None if gg is None else ctypes.byref(gg), *args) != 0
        assert msg in L.sgb_last_error(h).decode(), (msg, L.sgb_last_error(h))
        assert ctx.kernel_launches == n0, msg
    if managed is not None:
        rt.cudaFree(managed)
    usable()
    # what align_batch refuses: point-to-plane against submaps
    sub = _bind(target(s, "submaps"))
    pair(sub, s, "submaps")
    with pytest.raises(sg.SgbError, match="SGB_FACTOR_PLANE_ICP is not available against submaps"):
        sub.align_batch_gnc_async(_dev(poses(s, members("submaps"))), C2[PLANE], factor=PLANE)
    # the weights in force are those set before the refusals
    before = c1.linearize_batch_points(T0, factor=GICP)
    after = ctx.linearize_batch_points(T0, factor=GICP)
    _bits(before.point_e, after.point_e, "weights in force")
    _bits(before.H, after.H, "weights in force")
