"""Stream-ordered joint window registration (sgb_align_joint_async, Context.align_joint_async) on the GPU, against sgb_align_joint bit for
bit:
  1. X, info and, afterwards, correspondences_batch and error_batch on the edges equal align_joint's on kd-tree and voxel-map frames, over
     ICP / point-to-plane / GICP, none / Huber / Cauchy, GN / LM, a DoF mask, max_iterations 0 / 1 / 20, custom fixed flags, windows of 3,
     8 and 32 frames, 1, 17 and 1024 windows, and degenerate windows (no edge, no free frame, a free frame without an edge); the state
     left behind also on two fresh contexts built alike (error_batch refused alike over an edge that was never linearised), and when no
     window starts with a round to go;
  2. calls in sequence across option, window and fixed-flag changes, a synchronous align_joint, a re-pairing and a target rebuild;
  3. no host synchronisation, and a torch consumer of the poses queued after the call;
  4. capture in torch.cuda.graph replayed from new poses, and a capture that would need an upload of the window tables;
  5. the launch counter at several round counts;
  6. misuse fails with a message, enqueues nothing and leaves the context usable."""
import ctypes
import numpy as np
import pytest

from test_gpu_align_joint import Frames, _context, _perturbed, _window_edges

pytestmark = pytest.mark.gpu

GN, LM = 0, 1
# factor, robust, robust_c, optimizer, dof_mask, max_iterations
OPTIONS = [
    (2, 0, 1.0, LM, None, 20),
    (2, 1, 0.5, GN, None, 20),
    (0, 2, 0.5, LM, [1, 1, 0, 1, 1, 1], 20),
    (1, 0, 1.0, GN, None, 20),
    (0, 1, 0.5, GN, None, 1),
    (2, 2, 0.5, LM, None, 1),
    (2, 0, 1.0, LM, None, 0),
]


def _torch():
    return pytest.importorskip("torch")


def _sg():
    import small_gicp_b200 as sg

    return sg


@pytest.fixture(scope="module")
def frames():
    return Frames(40)


@pytest.fixture(autouse=True)
def _side_stream():
    """every test runs on a torch stream of its own (the default stream is the null stream, which set_stream cannot name)"""
    torch = _torch()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        yield
    side.synchronize()


def _bind(ctx):
    torch = _torch()
    ctx.set_stream(torch.cuda.current_stream().cuda_stream)
    return ctx


def _kw(opt):
    f, r, c, o, dof, it = opt
    return dict(factor=f, robust=r, robust_c=c, optimizer=o, dof_mask=dof, max_iterations=it)


def _same(a, b, tag):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes(), (tag, a, b)


class Call:
    """one call's frames and edges: frame k = frames idx[k]; edges (i, j) global; windows offsets; fixed flags (None: first of each window)"""

    def __init__(self, idx, edges, windows, fixed=None, seed=3):
        self.idx, self.edges, self.windows, self.fixed = list(idx), list(edges), list(windows), fixed
        self.seed = seed

    def context(self, fr, kind):
        return _bind(_context(fr, self.idx, kind, [e[0] for e in self.edges], [e[1] for e in self.edges]))

    def poses(self, fr, seed=None):
        X = []
        for w in range(len(self.windows) - 1):
            part = self.idx[self.windows[w] : self.windows[w + 1]]
            if part:
                X.append(_perturbed(fr, part, (self.seed if seed is None else seed) + w))
        return np.concatenate(X) if X else np.zeros((0, 4, 4))

    def linearised(self, max_it):
        """the edges sgb_align_joint linearises: those of windows with a free frame (max_iterations > 0)"""
        K = len(self.idx)
        off = self.windows
        fixed = self.fixed if self.fixed is not None else [int(k in off[:-1]) for k in range(K)]
        win = np.searchsorted(off, np.arange(K), side="right") - 1
        free = {w: any(not fixed[k] for k in range(off[w], off[w + 1])) for w in range(len(off) - 1)}
        return np.array([max_it > 0 and free[win[i]] for i, _ in self.edges], dtype=bool)


def _check(ctx, call, X, opt, tag):
    """align_joint, then align_joint_async from the same poses on the same context: results and the state each leaves bitwise equal"""
    torch = _torch()
    kw = _kw(opt)
    r = ctx.align_joint(X, windows=call.windows, fixed=call.fixed, **kw)
    corr = ctx.correspondences_batch()
    act = call.linearised(opt[5])
    T1 = np.array([np.linalg.inv(r.X[j]) @ r.X[i] for i, j in call.edges]).reshape(-1, 4, 4)  # the edges' final poses, nudged
    T1[:, :3, 3] += 0.01
    e1 = ctx.error_batch(T1, active=act) if act.any() else None
    a = ctx.align_joint_async(torch.from_numpy(np.ascontiguousarray(X)).cuda(), windows=call.windows, fixed=call.fixed, **kw)
    ctx.synchronize()
    _same(r.X, a.X.cpu().numpy(), (tag, "X"))
    _same(r.converged, a.converged.cpu().numpy() != 0, (tag, "converged"))
    for name in ("iterations", "num_inliers"):
        _same(getattr(r, name), getattr(a, name).cpu().numpy().astype(np.int64), (tag, name))
    _same(r.error, a.error.cpu().numpy(), (tag, "error"))
    for m, (x, y) in enumerate(zip(corr, ctx.correspondences_batch())):
        _same(x, y, (tag, "correspondences", m))
    if e1 is not None:
        _same(e1, ctx.error_batch(T1, active=act), (tag, "error_batch"))
    return r, a


def _state_after(ctx, call, X, opt):
    """what a context leaves behind: the edges' correspondences, and error_batch at the edges' poses from X (nudged) over every edge and
    over the edges the align linearised -- each result's bits, or the message of its refusal"""
    sg = _sg()
    T1 = np.array([np.linalg.inv(X[j]) @ X[i] for i, j in call.edges]).reshape(-1, 4, 4)
    T1[:, :3, 3] += 0.01
    errs = []
    for act in (None, call.linearised(opt[5])):
        try:
            errs.append(ctx.error_batch(T1, active=act).tobytes())
        except sg.SgbError as e:
            errs.append(str(e))
    return ctx.correspondences_batch(), errs


def _check_fresh(frames, call, kind, X, opt, tag):
    """align_joint and align_joint_async on two fresh contexts built alike: results and the state each leaves equal; returns the async
    call's launch count"""
    torch = _torch()
    kw = _kw(opt)
    s, c = call.context(frames, kind), call.context(frames, kind)
    r = s.align_joint(X, windows=call.windows, fixed=call.fixed, **kw)
    n0 = c.kernel_launches
    a = c.align_joint_async(torch.from_numpy(np.ascontiguousarray(X)).cuda(), windows=call.windows, fixed=call.fixed, **kw)
    launches = c.kernel_launches - n0
    c.synchronize()
    _same(r.X, a.X.cpu().numpy(), (tag, "X"))
    _same(np.c_[r.converged, r.iterations, r.num_inliers, r.error], a.info4.cpu().numpy(), (tag, "info"))
    (cs, es), (ca, ea) = _state_after(s, call, r.X, opt), _state_after(c, call, r.X, opt)
    for m, (x, y) in enumerate(zip(cs, ca)):
        _same(x, y, (tag, "correspondences", m))
    assert es == ea, (tag, "error_batch", es, ea)
    s.close()
    c.close()
    return launches


def _two_windows():
    """a window of 8 frames (chains and a loop edge) and one of 3"""
    e8 = _window_edges(8)
    e3 = [(9, 8), (10, 9), (10, 8)]
    return Call(list(range(8)) + [20, 21, 22], e8 + e3, [0, 8, 11])


@pytest.mark.parametrize("kind", ["kdtree", "voxelmap"])
def test_equals_align_joint_over_the_options(frames, kind):
    call = _two_windows()
    ctx = call.context(frames, kind)
    X = call.poses(frames)
    for opt in OPTIONS:
        if opt[0] == 1 and kind == "voxelmap":
            continue  # no normals in a voxel map
        _check(ctx, call, X, opt, (kind, opt))
    call.fixed = [1, 0, 0, 1, 0, 0, 0, 1, 0, 1, 0]  # custom fixed frames
    for opt in (OPTIONS[0], OPTIONS[1]):
        r, a = _check(ctx, call, X, opt, (kind, "fixed", opt))
        fixed = np.array(call.fixed, dtype=bool)
        _same(X[fixed], a.X.cpu().numpy()[fixed], (kind, "fixed frames"))


@pytest.mark.parametrize("F", [3, 8, 32])
def test_window_sizes(frames, F):
    call = Call(list(range(F)), _window_edges(F), [0, F])
    ctx = call.context(frames, "kdtree")
    for opt in (OPTIONS[0], OPTIONS[1]):
        _check(ctx, call, call.poses(frames), opt, ("F", F, opt))


@pytest.mark.parametrize("count", [1, 17, 1024])
def test_window_counts(frames, count):
    small = ([1, 2, 3], [(1, 0), (2, 1), (2, 0)])
    idx, edges, off = [], [], [0]
    for w in range(count):
        base = len(idx)
        idx += small[0]
        edges += [(base + i, base + j) for i, j in small[1]]
        off.append(len(idx))
    call = Call(idx, edges, off)
    ctx = call.context(frames, "kdtree")
    _check(ctx, call, call.poses(frames), OPTIONS[0], ("count", count))


@pytest.mark.parametrize("kind", ["kdtree", "voxelmap"])
def test_degenerate_windows(frames, kind):
    # windows: [] (empty) | [0, 1, 2] with edge 1 -> 0 and edge-less frame 2 | [3, 4] all fixed with an edge | [5] alone
    call = Call([5, 6, 7, 8, 9, 10], [(1, 0), (4, 3)], [0, 0, 3, 5, 6], fixed=[1, 0, 0, 1, 1, 0])
    ctx = call.context(frames, kind)
    X = _perturbed(frames, call.idx, 4)
    for opt in (OPTIONS[0], OPTIONS[4], OPTIONS[6]):
        _check(ctx, call, X, opt, ("degenerate", kind, opt))
    # no edge at all: nothing but the set-up and the outputs
    ctx.set_source_pairs(np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint32))
    call.edges = []
    _check(ctx, call, X, OPTIONS[0], ("no edge", kind))


@pytest.mark.parametrize("kind", ["kdtree", "voxelmap"])
def test_fresh_contexts_are_left_alike(frames, kind):
    """the linearisation flags the async call sets on a fresh context are the synchronous call's: error_batch over every edge is refused
    on both while an edge of a window without a free frame was never linearised, and equal over the linearised edges"""
    # windows: [] | [0, 1, 2] with edge 1 -> 0 | [3, 4] all fixed with an edge | [5] alone
    call = Call([5, 6, 7, 8, 9, 10], [(1, 0), (4, 3)], [0, 0, 3, 5, 6], fixed=[1, 0, 0, 1, 1, 0])
    X = _perturbed(frames, call.idx, 4)
    for opt in OPTIONS:
        if opt[0] == 1 and kind == "voxelmap":
            continue
        _check_fresh(frames, call, kind, X, opt, ("fresh", kind, opt))
    call = _two_windows()
    call.fixed = [1, 0, 0, 1, 0, 0, 0, 1, 1, 1, 1]  # the second window all fixed
    _check_fresh(frames, call, kind, call.poses(frames), OPTIONS[0], ("fresh", kind, "fixed window"))


@pytest.mark.parametrize("kind", ["kdtree", "voxelmap"])
def test_windows_done_from_the_start(frames, kind):
    """edges, iterations, but no window with both a free frame and an edge: the device loop runs one round without tiles, where
    sgb_align_joint runs none; the poses come back as they went in, no window iterates, no edge is linearised, 3 launches"""
    torch = _torch()
    call = Call([5, 6, 7, 8, 9, 10], [(1, 0), (2, 1), (4, 3)], [0, 3, 5, 6], fixed=[1, 1, 1, 1, 1, 0])
    X = _perturbed(frames, call.idx, 4)
    for opt in (OPTIONS[0], OPTIONS[1]):
        assert _check_fresh(frames, call, kind, X, opt, ("done", kind, opt)) == 4  # + the pairing's view of the target
    ctx = call.context(frames, kind)
    Xd = torch.from_numpy(X).cuda()
    ctx.align_joint_async(Xd, windows=call.windows, fixed=call.fixed)
    n0 = ctx.kernel_launches
    a = ctx.align_joint_async(Xd, windows=call.windows, fixed=call.fixed)
    assert ctx.kernel_launches - n0 == 3
    ctx.synchronize()
    _same(X, a.X.cpu().numpy(), "initial poses")
    _same(np.zeros((3, 4)), a.info4.cpu().numpy(), "no window iterated")
    assert all(np.all(c == np.iinfo(np.uint64).max) for c in ctx.correspondences_batch())


def test_calls_in_sequence_never_replay_a_stale_loop(frames):
    """options, windows and fixed flags change back to back, with a synchronous align_joint, a re-pairing and a target rebuild between:
    each call equals align_joint"""
    torch = _torch()
    call = _two_windows()
    ctx = call.context(frames, "kdtree")
    X = call.poses(frames)
    for k, opt in enumerate((OPTIONS[0], OPTIONS[1], OPTIONS[0], OPTIONS[5])):
        _check(ctx, call, call.poses(frames, 10 * k), opt, ("sequence", k))
    call.fixed = [1, 1, 0, 0, 0, 0, 0, 0, 1, 0, 0]
    _check(ctx, call, X, OPTIONS[0], "fixed flags")
    one = Call(call.idx, call.edges, [0, 11], fixed=[1] + [0] * 7 + [1, 0, 0])  # one window of both
    _check(ctx, one, X, OPTIONS[0], "windows")
    # a synchronous call with other windows, then the async call with the previous ones, compared against a fresh context
    ctx.align_joint(X, windows=[0, 11], fixed=one.fixed, **_kw(OPTIONS[1]))
    a = ctx.align_joint_async(torch.from_numpy(X).cuda(), windows=call.windows, fixed=call.fixed, **_kw(OPTIONS[0]))
    ref = call.context(frames, "kdtree").align_joint(X, windows=call.windows, fixed=call.fixed, **_kw(OPTIONS[0]))
    ctx.synchronize()
    _same(ref.X, a.X.cpu().numpy(), "after a synchronous call")
    # a re-pairing: other edges over the same frames
    call.edges = [(1, 0), (2, 1), (3, 2), (7, 0), (9, 8), (10, 8)]
    ctx.set_source_pairs(np.array([e[0] for e in call.edges], dtype=np.uint32), np.array([e[1] for e in call.edges], dtype=np.uint32))
    _check(ctx, call, X, OPTIONS[0], "re-paired")
    # a target rebuild under the same pairing
    pts = [frames.pts[i] for i in call.idx]
    ctx.build_target_voxelmaps(pts, [frames.covs[i] for i in call.idx], 1.0, 1)
    _check(ctx, call, X, OPTIONS[0], "new target")
    ctx.build_target_kdtrees(pts, [frames.normals[i] for i in call.idx], [frames.covs[i] for i in call.idx])
    _check(ctx, call, X, OPTIONS[3], "kd-trees again")


def test_no_host_synchronisation(frames):
    torch = _torch()
    call = _two_windows()
    ctx = call.context(frames, "kdtree")
    X = call.poses(frames)
    ref = ctx.align_joint(X, windows=call.windows)
    Xd = torch.from_numpy(X).cuda()
    ctx.align_joint_async(Xd, windows=call.windows)  # warm: the tables are uploaded, the loop graph is built and cached
    ctx.synchronize()
    torch.cuda._sleep(2_000_000_000)  # about a second of spinning on the context's stream
    a = ctx.align_joint_async(Xd, windows=call.windows)
    done = torch.cuda.Event()
    done.record()
    assert not done.query(), "the call waited for the stream"
    moved = (a.X @ torch.eye(4, dtype=torch.float64, device="cuda")).clone()  # a torch op consuming the poses, no synchronisation
    ctx.synchronize()
    _same(ref.X, a.X.cpu().numpy(), "after synchronize")
    _same(ref.X, moved.cpu().numpy(), "stream-ordered consumer")


def test_graph_capture_and_replay(frames):
    torch = _torch()
    sg = _sg()
    call = _two_windows()
    ctx = _context(frames, call.idx, "kdtree", [e[0] for e in call.edges], [e[1] for e in call.edges])
    X0 = torch.from_numpy(call.poses(frames)).cuda()
    side = torch.cuda.Stream()
    ctx.set_stream(side.cuda_stream)
    with torch.cuda.stream(side):
        out = ctx.align_joint_async(X0, windows=call.windows)  # warm-up outside the capture
    side.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        ctx.align_joint_async(X0, windows=call.windows, out=out)
    ctx.synchronize()
    for k in (1, 2):
        Xk = call.poses(frames, 100 + k)
        X0.copy_(torch.from_numpy(Xk))
        g.replay()
        torch.cuda.synchronize()
        ref = ctx.align_joint(Xk, windows=call.windows)
        _same(ref.X, out.X.cpu().numpy(), ("replay", k))
        _same(ref.iterations, out.iterations.cpu().numpy().astype(np.int64), ("replay", k))
        _same(ref.error, out.error.cpu().numpy(), ("replay", k))
    # other fixed flags: other window tables, which a capture cannot upload
    g2 = torch.cuda.CUDAGraph()
    with pytest.raises(sg.SgbError, match="call it once outside the capture first"):
        with torch.cuda.graph(g2, stream=side):
            ctx.align_joint_async(X0, windows=call.windows, fixed=[1, 1, 0, 0, 0, 0, 0, 0, 1, 0, 0], out=out)
    torch.cuda.synchronize()
    Xk = call.poses(frames, 7)
    with torch.cuda.stream(side):
        a = ctx.align_joint_async(torch.from_numpy(Xk).cuda(), windows=call.windows)
    ctx.synchronize()
    _same(ctx.align_joint(Xk, windows=call.windows).X, a.X.cpu().numpy(), "usable after the refused capture")


@pytest.mark.parametrize("kind", ["kdtree", "voxelmap"])
def test_launch_counter_is_independent_of_the_rounds(frames, kind):
    torch = _torch()
    call = _two_windows()
    ctx = call.context(frames, kind)
    Xd = torch.from_numpy(call.poses(frames)).cuda()
    n0 = ctx.kernel_launches
    ctx.align_joint_async(Xd, windows=call.windows, max_iterations=2)
    assert ctx.kernel_launches - n0 == 4  # + the pairing's view of the target
    for opt, expect in ((OPTIONS[4], 3), (OPTIONS[1], 3), (OPTIONS[0], 3), (OPTIONS[6], 2)):
        n0 = ctx.kernel_launches
        a = ctx.align_joint_async(Xd, windows=call.windows, **_kw(opt))
        assert ctx.kernel_launches - n0 == expect, (kind, opt, ctx.kernel_launches - n0)
    ctx.synchronize()
    assert a.iterations.cpu().numpy().max() == 0
    # rounds differ, launches do not
    its = set()
    for max_it in (1, 3, 20):
        n0 = ctx.kernel_launches
        a = ctx.align_joint_async(Xd, windows=call.windows, optimizer=GN, max_iterations=max_it)
        assert ctx.kernel_launches - n0 == 3
        ctx.synchronize()
        its.add(int(a.iterations.cpu().numpy().max()))
    assert len(its) > 1
    # no edge: set-up and outputs only
    ctx.set_source_pairs(np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint32))
    n0 = ctx.kernel_launches
    ctx.align_joint_async(Xd, windows=call.windows)
    assert ctx.kernel_launches - n0 == 2
    ctx.synchronize()


def _managed(nbytes):
    """a managed allocation (cudaMallocManaged) as a ctypes pointer, or None where the runtime library cannot be loaded"""
    try:
        rt = ctypes.CDLL("libcudart.so.12")
    except OSError:
        return None, None
    p = ctypes.c_void_p()
    assert rt.cudaMallocManaged(ctypes.byref(p), ctypes.c_size_t(nbytes), ctypes.c_uint(1)) == 0
    return rt, p


def test_misuse_fails_with_a_message(frames):
    torch = _torch()
    sg = _sg()
    call = _two_windows()
    ctx = sg.Context(0)
    Xn = call.poses(frames)
    X = torch.from_numpy(Xn).cuda()
    with pytest.raises(sg.SgbError, match="set the context's stream"):
        ctx.align_joint_async(X)
    _bind(ctx)
    with pytest.raises(sg.SgbError):
        ctx.align_joint_async(X)  # no batch
    pts = [frames.pts[i] for i in call.idx]
    cv = [frames.covs[i] for i in call.idx]
    ctx.build_target_kdtrees(pts, None, cv)
    ctx.set_source_batch(pts, cv)
    with pytest.raises(sg.SgbError, match="pairing with a maps table"):
        ctx.align_joint_async(X, windows=call.windows)
    ctx.set_source_pairs(np.array([e[0] for e in call.edges], dtype=np.uint32), np.array([e[1] for e in call.edges], dtype=np.uint32))
    for kw, msg in ((dict(windows=[0, 8]), "must run from 0"), (dict(windows=[0, 8, 4, 11]), "ascending"), (dict(windows=[0, 4, 11]), "both frames of an edge"),
                    (dict(windows=call.windows, fixed=[0] * 11), "no fixed frame"), (dict(windows=call.windows, factor=7), "invalid"),
                    (dict(windows=call.windows, factor=1), "normals")):
        n0 = ctx.kernel_launches
        with pytest.raises(sg.SgbError, match=msg):
            ctx.align_joint_async(X, **kw)
        assert ctx.kernel_launches == n0, msg
    # host, page-locked and managed pointers
    L, h = ctx._L, ctx._h
    o = sg.capi.AlignOptions(2, 0, 1.0, 1, 1.0, 1, 20, 1e-6, 10, 1e-3, 10.0, 1e-3, 1e-3)
    o.dof_mask[:] = [1.0] * 6
    K, W = 11, 2
    off = np.array(call.windows, dtype=np.uintp)
    offp = off.ctypes.data_as(ctypes.POINTER(ctypes.c_size_t))
    Xc = X.transpose(1, 2).contiguous()
    host = np.zeros((K, 16))
    pinned = torch.zeros((K, 16), dtype=torch.float64).pin_memory()
    dev = [torch.zeros((K, 16), dtype=torch.float64, device="cuda"), torch.zeros((W, 4), dtype=torch.float64, device="cuda")]
    p = sg.capi._d
    rt, managed = _managed(K * 16 * 8)
    cases = [
        ((None, p(Xc), p(dev[0]), p(dev[1])), "null options"),
        ((o, p(Xc), None, p(dev[1])), "null output"),
        ((o, host.ctypes.data_as(sg.capi._dp), p(dev[0]), p(dev[1])), "device memory"),
        ((o, p(Xc), p(pinned), p(dev[1])), "device memory"),
        ((o, p(Xc), p(dev[0]), host.ctypes.data_as(sg.capi._dp)), "device memory"),
    ]
    if managed is not None:
        cases.append(((o, p(Xc), ctypes.cast(managed, sg.capi._dp), p(dev[1])), "device memory"))
    for args, msg in cases:
        n0 = ctx.kernel_launches
        opt = ctypes.byref(args[0]) if args[0] is not None else None
        assert L.sgb_align_joint_async(h, opt, W, offp, None, *args[1:]) != 0
        assert msg in L.sgb_last_error(h).decode(), (msg, L.sgb_last_error(h))
        assert ctx.kernel_launches == n0
    if managed is not None:
        rt.cudaFree(managed)
    # the context is still usable
    r = ctx.align_joint(Xn, windows=call.windows, factor=2)
    a = ctx.align_joint_async(X, windows=call.windows, factor=2)
    ctx.synchronize()
    _same(r.X, a.X.cpu().numpy(), "usable after misuse")
