"""Stream-ordered batched align (sgb_align_batch_async, Context.align_batch_async): the device-driven loop against sgb_align_batch, bit for
bit, on every target kind, with the state it leaves behind; calls in sequence across batch, pairing, submap and target changes; no host
synchronisation; capture in torch.cuda.graph; the launch counter; misuse."""
import numpy as np
import pytest

from test_gpu_batch_pairs import Scene as PairScene
from test_gpu_batch_pairs import _target
from test_gpu_submaps import CL as SUB_CL
from test_gpu_submaps import Scene as SubScene
from test_gpu_submaps import _poses_of

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
def pairs():
    return PairScene()


@pytest.fixture(scope="module")
def subs():
    return SubScene()


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
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and np.array_equal(a, b), (tag, np.nanmax(np.abs(a.astype(float) - b.astype(float))) if a.shape == b.shape else a.shape)


def _check(ctx, T, T1, opt, tag):
    """align_batch, then align_batch_async from the same poses on the same context: results and the state each leaves bitwise equal"""
    torch = _torch()
    kw = _kw(opt)
    r = ctx.align_batch(T, **kw)
    corr = ctx.correspondences_batch()
    e1 = ctx.error_batch(T1) if opt[5] > 0 else None
    a = ctx.align_batch_async(torch.from_numpy(np.ascontiguousarray(T)).cuda(), **kw)
    ctx.synchronize()
    for name in ("T_target_source", "H", "b"):
        _same(getattr(r, name), getattr(a, name).cpu().numpy(), (tag, name))
    _same(r.converged, a.converged.cpu().numpy() != 0, (tag, "converged"))
    for name in ("iterations", "num_inliers"):
        _same(getattr(r, name), getattr(a, name).cpu().numpy().astype(np.int64), (tag, name))
    _same(r.error, a.error.cpu().numpy(), (tag, "error"))
    for m, (x, y) in enumerate(zip(corr, ctx.correspondences_batch())):
        _same(x, y, (tag, "correspondences", m))
    if e1 is not None:
        _same(e1, ctx.error_batch(T1), (tag, "error_batch"))
    return a


@pytest.mark.parametrize("kind", ["tree", "voxelmap", "voxelmaps", "trees"])
def test_equals_align_batch_on_every_target(pairs, kind):
    """one kd-tree (tie-free random target), one voxel map, many voxel maps and many kd-trees (member m against map m), over the options"""
    s = pairs
    sg = _sg()
    ctx = _bind(sg.Context(0))
    _target(ctx, s, kind)
    if kind in ("voxelmaps", "trees"):
        ctx.set_source_batch(s.clouds[: len(s.maps)], s.scovs[: len(s.maps)])
        cl = list(range(len(s.maps)))
    else:
        ctx.set_source_batch(s.clouds, s.scovs)
        cl = list(range(len(s.clouds)))
    T, T1 = s.poses(cl), s.poses(cl, 1)
    for opt in OPTIONS:
        if opt[0] == 1 and kind in ("voxelmap", "voxelmaps"):
            continue  # no normals in a voxel map
        _check(ctx, T, T1, opt, (kind, opt))


@pytest.mark.parametrize("kind", ["trees", "voxelmaps", "tree"])
def test_equals_align_batch_on_pairs(pairs, kind):
    """(cloud, map) pairs with a maps table (many maps) or without (multi-start on one target), empty members included"""
    s = pairs
    ctx = _bind(_sg().Context(0))
    _target(ctx, s, kind)
    ctx.set_source_batch(s.clouds, s.scovs)
    pairs_ = [(0, 0), (0, 2), (2, 2), (3, 2), (5, 4), (1, 3), (0, 1)]
    cl, mp = [p[0] for p in pairs_], [p[1] for p in pairs_]
    ctx.set_source_pairs(cl, mp if kind != "tree" else None)
    T, T1 = s.poses(cl), s.poses(cl, 1)
    for opt in OPTIONS[:3] + OPTIONS[5:]:
        _check(ctx, T, T1, opt, (kind, opt))


@pytest.mark.parametrize("n_entries", [1, 5, 33])
def test_equals_align_batch_on_submaps(subs, n_entries):
    s = subs
    ctx = _bind(s.context())
    lists = [[0], [2, 0], [4, 1, 0, 3, 2], [0, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11] * 3, [0, 2], [], [11, 5, 1]]
    lists = [l[:n_entries] for l in lists]
    poses = [p[:n_entries] for p in _poses_of(s, [[0], [2, 0], [4, 1, 0, 3, 2], [0, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11] * 3, [0, 2], [], [11, 5, 1]])]
    ctx.set_source_submaps(lists, poses, SUB_CL)
    T, T1 = s.poses(SUB_CL), s.poses(SUB_CL, 1)
    for opt in (OPTIONS[0], OPTIONS[1], OPTIONS[2], OPTIONS[6]):
        _check(ctx, T, T1, opt, ("submaps", n_entries, opt))


@pytest.mark.parametrize("B", [1, 17, 4096])
def test_batch_sizes(pairs, B):
    """B copies of the clouds as pairs against the one kd-tree, every member from its own pose"""
    s = pairs
    ctx = _bind(_sg().Context(0))
    _target(ctx, s, "tree")
    ctx.set_source_batch(s.clouds, s.scovs)
    cl = [(p * 7) % len(s.clouds) for p in range(B)]
    ctx.set_source_pairs(cl)
    T, T1 = s.poses(cl), s.poses(cl, 1)
    for opt in (OPTIONS[0], OPTIONS[1]):
        _check(ctx, T, T1, opt, ("B", B, opt))


def test_calls_in_sequence_never_replay_a_stale_loop(pairs):
    """different options and poses back to back, then new batches, re-pairings and target rebuilds: each call equals align_batch"""
    s = pairs
    ctx = _bind(_sg().Context(0))
    _target(ctx, s, "trees")
    ctx.set_source_batch(s.clouds[:5], s.scovs[:5])
    cl = list(range(5))
    for k, opt in enumerate((OPTIONS[0], OPTIONS[1], OPTIONS[0])):
        _check(ctx, s.poses(cl, k), s.poses(cl, k + 1), opt, ("sequence", k))
    ctx.set_source_batch(s.clouds[1:5] + s.clouds[:1], s.scovs[1:5] + s.scovs[:1])  # other clouds
    _check(ctx, s.poses(cl), s.poses(cl, 1), OPTIONS[0], "new batch")
    ctx.set_source_pairs([0, 2, 2, 3], [4, 2, 0, 0])
    _check(ctx, s.poses([0, 2, 2, 3]), s.poses([0, 2, 2, 3], 1), OPTIONS[0], "re-paired")
    _target(ctx, s, "voxelmaps")  # a target rebuild under the same pairing
    _check(ctx, s.poses([0, 2, 2, 3]), s.poses([0, 2, 2, 3], 1), OPTIONS[0], "new target")
    _target(ctx, s, "tree")
    ctx.set_source_batch(s.clouds, s.scovs)
    _check(ctx, s.poses(list(range(6))), s.poses(list(range(6)), 1), OPTIONS[1], "single tree")


def test_no_host_synchronisation(pairs):
    torch = _torch()
    s = pairs
    ctx = _bind(_sg().Context(0))
    _target(ctx, s, "tree")
    ctx.set_source_batch(s.clouds, s.scovs)
    cl = list(range(len(s.clouds)))
    T = s.poses(cl)
    ref = ctx.align_batch(T)
    Td = torch.from_numpy(T).cuda()
    ctx.align_batch_async(Td)  # warm: the loop graph is built and cached
    ctx.synchronize()
    torch.cuda._sleep(2_000_000_000)  # about a second of spinning on the context's stream
    a = ctx.align_batch_async(Td)
    done = torch.cuda.Event()
    done.record()
    assert not done.query(), "the call waited for the stream"
    moved = (a.T_target_source @ torch.eye(4, dtype=torch.float64, device="cuda")).clone()  # a torch op consuming the poses, no synchronisation
    ctx.synchronize()
    _same(ref.T_target_source, a.T_target_source.cpu().numpy(), "after synchronize")
    _same(ref.T_target_source, moved.cpu().numpy(), "stream-ordered consumer")


def test_graph_capture_and_replay(pairs):
    torch = _torch()
    s = pairs
    ctx = _sg().Context(0)
    _target(ctx, s, "tree")
    ctx.set_source_batch(s.clouds, s.scovs)
    cl = list(range(len(s.clouds)))
    T0 = torch.from_numpy(s.poses(cl)).cuda()
    side = torch.cuda.Stream()
    ctx.set_stream(side.cuda_stream)
    with torch.cuda.stream(side):
        out = ctx.align_batch_async(T0)  # warm-up outside the capture
    side.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        ctx.align_batch_async(T0, out=out)
    ctx.synchronize()
    for k in (1, 2):
        Tk = s.poses(cl, k)
        T0.copy_(torch.from_numpy(Tk))
        g.replay()
        torch.cuda.synchronize()
        ref = ctx.align_batch(Tk)
        _same(ref.T_target_source, out.T_target_source.cpu().numpy(), ("replay", k))
        _same(ref.num_inliers, out.num_inliers.cpu().numpy().astype(np.int64), ("replay", k))
        _same(ref.H, out.H.cpu().numpy(), ("replay", k))


@pytest.mark.parametrize("B", [1, 4096])
def test_launch_counter_is_independent_of_the_rounds(pairs, B):
    torch = _torch()
    s = pairs
    ctx = _bind(_sg().Context(0))
    _target(ctx, s, "tree")
    ctx.set_source_batch(s.clouds, s.scovs)
    cl = [(p * 7) % len(s.clouds) for p in range(B)]
    ctx.set_source_pairs(cl)
    Td = torch.from_numpy(s.poses(cl)).cuda()
    for it, expect in ((1, 3), (20, 3), (0, 2)):
        n0 = ctx.kernel_launches
        ctx.align_batch_async(Td, max_iterations=it)
        assert ctx.kernel_launches - n0 == expect, (B, it, ctx.kernel_launches - n0)
    ctx.synchronize()


def test_misuse_fails_with_a_message(pairs):
    torch = _torch()
    sg = _sg()
    s = pairs
    ctx = sg.Context(0)
    _target(ctx, s, "tree")
    T = torch.from_numpy(s.poses(list(range(len(s.clouds))))).cuda()
    with pytest.raises(sg.SgbError, match="set the context's stream"):
        ctx.align_batch_async(T)
    _bind(ctx)
    with pytest.raises(sg.SgbError):
        ctx.align_batch_async(T)  # no batch
    ctx.set_source_batch(s.clouds, s.scovs)
    L, h = ctx._L, ctx._h
    o = sg.capi.AlignOptions(2, 0, 1.0, 1, 1.0, 1, 20, 1e-6, 10, 1e-3, 10.0, 1e-3, 1e-3)
    o.dof_mask[:] = [1.0] * 6
    B = len(s.clouds)
    host = np.zeros((B, 42))
    pinned = torch.zeros((B, 16), dtype=torch.float64).pin_memory()
    dev = [torch.zeros((B, n), dtype=torch.float64, device="cuda") for n in (16, 4, 42)]
    Tc = T.transpose(1, 2).contiguous()
    p = lambda t: sg.capi._d(t)
    cases = [
        ((None, p(Tc), p(dev[0]), p(dev[1]), p(dev[2])), "null options"),
        ((o, p(Tc), None, p(dev[1]), p(dev[2])), "null output"),
        ((o, p(Tc), p(dev[0]), None, None), "null output"),
        ((o, host.ctypes.data_as(sg.capi._dp), p(dev[0]), p(dev[1]), None), "device memory"),
        ((o, p(Tc), p(pinned), p(dev[1]), None), "device memory"),
        ((o, p(Tc), p(dev[0]), p(dev[1]), host.ctypes.data_as(sg.capi._dp)), "device memory"),
    ]
    import ctypes as C

    for args, msg in cases:
        n0 = ctx.kernel_launches
        opt = C.byref(args[0]) if args[0] is not None else None
        assert L.sgb_align_batch_async(h, opt, *args[1:]) != 0
        assert msg in L.sgb_last_error(h).decode(), (msg, L.sgb_last_error(h))
        assert ctx.kernel_launches == n0
    # point-to-plane against submaps
    ctx2 = _bind(_sg().Context(0))
    ctx2.build_target_kdtrees([s.maps[0], s.maps[2]], [s.normals[0], s.normals[2]], [s.covs[0], s.covs[2]])
    ctx2.set_source_batch(s.clouds[:2], s.scovs[:2])
    ctx2.set_source_submaps([[0], [1, 0]], None, [0, 0])
    with pytest.raises(sg.SgbError, match="PLANE_ICP"):
        ctx2.align_batch_async(T[:2], factor=1)
    # the context is still usable
    r = ctx.align_batch(T.cpu().numpy())
    a = ctx.align_batch_async(T)
    ctx.synchronize()
    _same(r.T_target_source, a.T_target_source.cpu().numpy(), "usable after misuse")
