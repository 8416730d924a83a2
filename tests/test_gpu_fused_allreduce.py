"""The multi-GPU exchange fused into the reduction kernel (include/sgicp_b200.h sgb_comm_*, SURVEY.md §8e), exercised on
ONE GPU: several contexts of one process, each holding a shard of the source on its own stream, wired mailbox to mailbox
by raw device pointers (the multi-process wiring over CUDA IPC differs only in how the pointers are obtained; bench.py
--gpus N runs that one).  Every context must end up with the sums of the un-sharded source."""
import numpy as np
import pytest

import np_factors as NF

pytestmark = pytest.mark.gpu


def _sg():
    import small_gicp_b200 as sg

    return sg


def _pair(n=60_000):
    from small_gicp_b200.synthetic import make_pair

    tgt, src, T = make_pair(n)
    scratch = _sg().Context(0)
    tcov = scratch.estimate_features(tgt, 20, normals=False)[1]
    scov = scratch.estimate_features(src, 20, normals=False)[1]
    scratch.close()
    return tgt, tcov, src, scov, T


def _contexts(world, tgt, tcov, src, scov, shards):
    sg = _sg()
    ctxs = []
    for r in range(world):
        c = sg.Context(0)
        c.set_target(tgt, None, tcov)
        c.build_target_kdtree(0)
        lo, hi = shards[r]
        c.set_source(src[lo:hi], scov[lo:hi])
        ctxs.append(c)
    boxes = [c.comm_mailbox() for c in ctxs]
    for r, c in enumerate(ctxs):
        c.comm_connect_ptrs(r, world, boxes)
    return ctxs


@pytest.mark.parametrize("world", [2, 3, 8])
def test_sharded_contexts_exchange_inside_the_kernel(world):
    import torch

    from small_gicp_b200.distributed import shard_range

    sg = _sg()
    tgt, tcov, src, scov, T = _pair()
    n = src.shape[0]
    full = sg.Context(0)
    full.set_target(tgt, None, tcov)
    full.build_target_kdtree(0)
    full.set_source(src, scov)
    shards = [shard_range(n, r, world) for r in range(world)]
    if world == 3:
        shards = [(0, 0), (0, n // 3), (n // 3, n)]  # an empty shard still takes part in the exchange
    ctxs = _contexts(world, tgt, tcov, src, scov, shards)
    outs = [torch.zeros(64, dtype=torch.float64, device="cuda") for _ in range(world)]
    errs = [torch.zeros(1, dtype=torch.float64, device="cuda") for _ in range(world)]
    poses = [np.eye(4), T, T]
    for it, pose in enumerate(poses):
        H0, b0, e0 = full.linearize(pose)
        n0 = full.num_inliers()
        err0 = full.error(pose)
        # every launch is asynchronous: rank r's finishing CTA waits (on the device) for the ranks launched after it
        order = range(world) if it % 2 == 0 else reversed(range(world))
        for r in order:
            ctxs[r].linearize_device(pose, outs[r].data_ptr())
        for r in range(world):
            ctxs[r].error_device(pose, errs[r].data_ptr())
        for c in ctxs:
            c.synchronize()
        ref = outs[0].cpu().numpy()[:44]
        assert np.isfinite(ref).all()
        for r in range(world):
            h = outs[r].cpu().numpy()[:44]
            np.testing.assert_array_equal(h, ref)  # summed in rank order on every rank: bit-identical
            assert float(errs[r].cpu()[0]) == float(errs[0].cpu()[0])
        H, b, e, ninl = ref[:36].reshape(6, 6), ref[36:42], ref[42], ref[43]
        # every shard re-centres its own source box: the exchanged sum is the sum of the per-shard storage models
        Hm, bm, em, err_m = np.zeros((6, 6)), np.zeros(6), 0.0, 0.0
        for r, (lo, hi) in enumerate(shards):
            model = NF.storage_model(src[lo:hi], scov[lo:hi], tgt, None, tcov)
            corr = ctxs[r].correspondences()
            Hr, br, er = NF.linearize(pose, corr, 2, 0, 1.0, *model)
            Hm, bm, em = Hm + Hr, bm + br, em + er
            err_m += NF.error(pose, pose, corr, 2, 0, 1.0, *model)
        ratios = NF.tight_ratios((H, b, e), (Hm, bm, em)) + (abs(float(errs[0].cpu()[0]) - err_m) / err_m,)
        print(f"worst ratio to the per-shard storage models (world {world}, pose {it}): {max(ratios):.2e}")
        assert max(ratios) <= NF.TIGHT, ("H, b, e, error:", ratios)
        assert int(ninl) == sum(int((ctxs[r].correspondences() != NF.NO).sum()) for r in range(world))
        # ... so FP32 roundings differ slightly from the un-sharded run
        assert np.linalg.norm(H - H0) <= 1e-5 * np.linalg.norm(H0)
        assert abs(e - e0) <= 1e-5 * e0 and abs(float(errs[0].cpu()[0]) - err0) <= 1e-5 * err0
        assert abs(ninl - n0) <= 3
        scale = np.sqrt(2.0 * e0 * np.diag(H0))
        assert np.all(np.abs(b - b0) <= 1e-5 * scale)
    # after disconnect a context is single-GPU again
    ctxs[-1].comm_disconnect()
    lo, hi = shards[-1]
    Hs, bs, es = ctxs[-1].linearize(T)
    solo = sg.Context(0)
    solo.set_target(tgt, None, tcov)
    solo.build_target_kdtree(0)
    solo.set_source(src[lo:hi], scov[lo:hi])
    H1, b1, e1 = solo.linearize(T)
    assert np.array_equal(Hs, H1) and es == e1
    for c in ctxs + [full, solo]:
        c.close()


def test_missing_peer_times_out_instead_of_hanging(monkeypatch):
    """A collective whose peer never arrives must not hang the GPU: the waiting CTA gives up (here after 300 ms) and returns NaN."""
    import torch

    sg = _sg()
    tgt, tcov, src, scov, T = _pair(20_000)
    n = src.shape[0]
    ctxs = _contexts(2, tgt, tcov, src, scov, [(0, n // 2), (n // 2, n)])
    ctxs[0].comm_set_timeout_ms(300)
    out = torch.zeros(64, dtype=torch.float64, device="cuda")
    ctxs[0].linearize_device(T, out.data_ptr())  # rank 1 never calls
    ctxs[0].synchronize()
    assert np.isnan(out.cpu().numpy()[:44]).all()
    assert ctxs[0].comm_status() & 1  # ... and it is not a silent NaN: the sticky status word says "timeout"
    with pytest.raises(sg.SgbError):  # the context refuses further collective work until it is reconnected
        ctxs[0].linearize(T)
    for c in ctxs:
        c.close()


def test_host_call_reports_peer_timeout_as_error():
    """sgb_linearize (host-returning) turns a timed-out exchange into a non-zero return code instead of NaN sums with rc == 0."""
    sg = _sg()
    tgt, tcov, src, scov, T = _pair(20_000)
    n = src.shape[0]
    ctxs = _contexts(2, tgt, tcov, src, scov, [(0, n // 2), (n // 2, n)])
    ctxs[0].comm_set_timeout_ms(200)
    with pytest.raises(sg.SgbError, match="peer"):
        ctxs[0].linearize(T)
    for c in ctxs:
        c.close()


def test_failed_call_on_one_rank_tells_the_peers():
    """A call that fails on the HOST of one rank (here: GICP without source covariances) still takes its sequence number and tells the
    peers: they get an error at once (status bit 1), not a 5 s timeout, and after a re-connect the group works again."""
    import time

    import torch

    sg = _sg()
    tgt, tcov, src, scov, T = _pair(20_000)
    n = src.shape[0]
    ctxs = _contexts(2, tgt, tcov, src, scov, [(0, n // 2), (n // 2, n)])
    ctxs[1].set_source(src[n // 2 :], None)  # rank 1 loses its covariances: its GICP linearize fails validation
    out = torch.zeros(64, dtype=torch.float64, device="cuda")
    with pytest.raises(sg.SgbError):
        ctxs[1].linearize_device(T, out.data_ptr())
    t0 = time.perf_counter()
    with pytest.raises(sg.SgbError, match="peer"):
        ctxs[0].linearize(T)
    assert time.perf_counter() - t0 < 2.0  # far below the 5 s timeout: the peer said so
    assert ctxs[0].comm_status() & 2
    # re-connect and carry on
    ctxs[1].set_source(src[n // 2 :], scov[n // 2 :])
    boxes = [c.comm_mailbox() for c in ctxs]
    for r, c in enumerate(ctxs):
        c.comm_connect_ptrs(r, 2, boxes)
    ctxs[1].linearize_device(T, out.data_ptr())
    H, b, e = ctxs[0].linearize(T)
    assert np.isfinite(H).all() and e > 0
    for c in ctxs:
        c.close()


def _lm(linearize, error, max_iterations=20, max_inner=10, lam=1e-3, lam_factor=10.0):
    """LevenbergMarquardtOptimizer::optimize (registration/optimizer.hpp:83-149) around two callbacks:
    linearize(T) -> (H, b, e), error(T) -> e.  Returns (T, last outer index, converged)."""
    import oracle as O

    T = np.eye(4)
    converged, it = False, 0
    for it in range(max_iterations):
        if converged:
            it -= 1
            break
        H, b, e = linearize(T)
        success = False
        for _ in range(max_inner):
            d = np.linalg.solve(H + lam * np.eye(6), -b)
            T_new = T @ O.se3_exp(d)
            e_new = error(T_new)
            if e_new <= e:
                converged = bool(np.linalg.norm(d[:3]) <= 0.1 * np.pi / 180 and np.linalg.norm(d[3:]) <= 1e-3)  # termination_criteria.hpp:10-20
                T, e, success = T_new, e_new, True
                lam /= lam_factor
                break
            lam *= lam_factor
        if not success:
            break
    return T, it, converged


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_vgicp_lm_matches_unsharded_and_oracle(world):
    """BASELINE configs[3] in miniature: Gaussian voxel map target (leaf 1.0) replicated on every rank, source sharded,
    LevenbergMarquardt driving linearize + error through the exchange fused into the kernels.  Every rank must walk the
    same trajectory as one context holding the whole source, and end where the CPU oracle's VGICP align ends."""
    import torch

    import oracle as O
    from conftest import pose_error
    from small_gicp_b200.distributed import shard_range

    sg = _sg()
    tgt, tcov, src, scov, Tgt = _pair(100_000)
    n = src.shape[0]

    def vgicp_context(lo, hi):
        c = sg.Context(0)
        c.build_target_voxelmap(tgt, tcov, 1.0)
        c.set_source(src[lo:hi], scov[lo:hi])
        return c

    full = vgicp_context(0, n)
    T_full, it_full, conv_full = _lm(lambda T: full.linearize(T, factor=sg.FACTOR_GICP), full.error)

    ctxs = [vgicp_context(*shard_range(n, r, world)) for r in range(world)]
    boxes = [c.comm_mailbox() for c in ctxs]
    for r, c in enumerate(ctxs):
        c.comm_connect_ptrs(r, world, boxes)
    outs = [torch.zeros(64, dtype=torch.float64, device="cuda") for _ in range(world)]
    errs = [torch.zeros(1, dtype=torch.float64, device="cuda") for _ in range(world)]

    def linearize(T):
        for r in range(world):
            ctxs[r].linearize_device(T, outs[r].data_ptr(), factor=sg.FACTOR_GICP)
        for c in ctxs:
            c.synchronize()
        h = [o.cpu().numpy()[:44] for o in outs]
        for r in range(1, world):
            np.testing.assert_array_equal(h[r], h[0])  # the same sum, in the same order, on every rank
        return h[0][:36].reshape(6, 6).copy(), h[0][36:42].copy(), float(h[0][42])

    def error(T):
        for r in reversed(range(world)):
            ctxs[r].error_device(T, errs[r].data_ptr())
        for c in ctxs:
            c.synchronize()
        e = [float(x.cpu()[0]) for x in errs]
        assert all(x == e[0] for x in e)
        return e[0]

    T_sh, it_sh, conv_sh = _lm(linearize, error)
    assert (it_sh, conv_sh) == (it_full, conv_full)
    rot, trans = pose_error(T_full, T_sh)
    assert rot < 1e-6 and trans < 1e-5, (rot, trans)  # shards re-centre their own boxes: FP32 roundings differ in the last digits
    ninl = int(round(outs[0].cpu().numpy()[43]))
    assert abs(ninl - full.num_inliers()) <= 3

    # the CPU oracle on the same inputs: GaussianVoxelMap target, GICP factor, LM (registration_helper.cpp:130-136)
    tc, sc = O.Cloud(tgt), O.Cloud(src)
    tc.set_features(None, tcov)
    sc.set_features(None, scov)
    ref = O.Registration(factor=O.FACTOR_GICP, num_threads=max(1, O.max_threads())).align(O.GaussianVoxelMap(tc, 1.0), None, sc, np.eye(4))
    rot, trans = pose_error(ref.T_target_source, T_sh)
    assert rot < 1e-4 and trans < 1e-3, (rot, trans)  # BASELINE north_star bar
    assert ref.iterations == it_sh
    rot, trans = pose_error(Tgt, T_sh)
    assert rot < 5e-3 and trans < 5e-2
    for c in ctxs + [full]:
        c.close()


@pytest.mark.parametrize("bind", [True, False])
def test_context_reduction_is_ordered_with_torch(bind):
    """distributed.ContextReduction: the context's kernels and torch's read of the result buffer must be ordered -- either the
    context runs on torch's current stream (bind_stream=True) or the adapter synchronises the context before torch looks.
    Keyword overrides of linearize() reach the kernel."""
    import torch

    from small_gicp_b200.distributed import ContextReduction, ShardedReduction

    sg = _sg()
    tgt, tcov, src, scov, T = _pair(40_000)
    ref = sg.Context(0)
    ref.set_target(tgt, None, tcov)
    ref.build_target_kdtree(0)
    ref.set_source(src, scov)
    ctx = sg.Context(0)
    ctx.set_target(tgt, None, tcov)
    ctx.build_target_kdtree(0)
    ctx.set_source(src, scov)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        red = ShardedReduction(ContextReduction(ctx, sg.FACTOR_GICP, bind_stream=bind), device="cuda")
        for _ in range(20):  # a race would show up as a stale / zero buffer in some repetition
            for pose in (np.eye(4), T):
                H0, b0, e0 = ref.linearize(pose)
                H, b, e, ninl = red.linearize(pose)
                assert np.array_equal(H, H0) and e == e0 and ninl == ref.num_inliers()
                assert red.error(pose) == ref.error(pose)
        H0, b0, e0 = ref.linearize(T, max_dist_sq=0.01)
        H, b, e, _ = red.linearize(T, max_dist_sq=0.01)
        assert np.array_equal(H, H0) and e == e0
    ctx.close()
    ref.close()
