"""The whole device pipeline held to an exact FP64 model of what it stores (np_factors.storage_model), at the source sizes where the
kernels change regime and through every input path of the upload.

Between the caller's buffer and the final sum lie the upload (pageable staging, or the two-stream pipeline for page-locked and device
memory), centring, the Hilbert permutation, the chunked covariance scatter, the leaf-order gathers, the cp.async operand ring of
factor_reduce_kernel, the ticket-tree reduction and the pipelined error().  Against the oracle all of that is checked to 2e-5, which is
more than one point's share of the sums above ~50k points.  Here the GPU sums are compared with numpy evaluated over the GPU's own
correspondences on the modelled arrays, to np_factors.TIGHT = 1e-10, so a single point given another point's operands fails.

The features are random, not estimated: covariances with the (1e-3, 1, 1) spectrum in random orientations and random unit normals, so a
wrong operand changes that point's term by about its own size (estimated features of neighbours are nearly equal).  The covariances'
lower triangles are perturbed: the device reads only the upper one.  The scene sits hundreds of metres from the origin.

Each test prints the worst ratio it reached (run with -s to see it)."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

import np_factors as NF
import oracle as O

pytestmark = pytest.mark.gpu

N_TGT = 200_000
# 32-query chunk; kLinBlock = 128-point tile; kFinishGroup = 16 CTAs per ticket group (16 CTAs, 17, a third group of one CTA);
# covariance upload chunks above 65536 points, all kUploadChunks = 8 of them from 458753; ~9 tiles per factor CTA (the 3-stage ring wraps)
SIZES = [1, 2, 31, 32, 33, 127, 128, 129, 2047, 2048, 2049, 4097, 65536, 65537, 458753, 600_000]
ALL_NINE = (2049, 458753)  # every factor x robust kernel combination at these sizes, the three plain factors at the others
N_PATHS = 600_000  # the input-path tests: all 8 covariance chunks in flight
OFFSET = np.array([310.0, -220.0, 45.0])
TRIALS = ([0.01, -0.02, 0.005, 0.05, -0.03, 0.02], [-0.004, 0.003, 0.01, -0.02, 0.01, 0.03])
SAMPLE = 2000  # queries checked against brute force per call


def _sg():
    import small_gicp_b200 as sg

    return sg


def _unit(rng, n):
    v = rng.normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def _random_covs(rng, n):
    from small_gicp_b200.synthetic import plane_covariances

    c = plane_covariances(_unit(rng, n))  # V diag(1e-3, 1, 1) V^T for a random rotation V (the spectrum only fixes V's first column)
    for a, b in ((1, 0), (2, 0), (2, 1)):
        c[:, a, b] += rng.uniform(-0.1, 0.1, n)  # not read by the device
    return c


def about(centre, delta):
    """se3_exp(delta) applied about `centre` instead of the origin (an exact rotation)"""
    C = np.eye(4)
    C[:3, 3] = centre
    Ci = np.eye(4)
    Ci[:3, 3] = -centre
    return C @ O.se3_exp(np.asarray(delta, dtype=float)) @ Ci


class Data:
    def __init__(self):
        from small_gicp_b200.synthetic import make_pair

        rng = np.random.default_rng(2026)
        tgt, src, T = make_pair(N_TGT, n_source=max(SIZES))
        ones = lambda n: np.ones((n, 1))
        self.tp = np.c_[tgt + OFFSET, ones(len(tgt))]
        self.sp = np.c_[src + T[:3, :3].T @ OFFSET, ones(len(src))]  # T still maps source onto target
        self.tn = np.c_[_unit(rng, len(tgt)), np.zeros(len(tgt))]
        self.tcv = _random_covs(rng, len(tgt))
        self.scv = _random_covs(rng, len(src))
        self.tgt_model = (NF.stored_points(self.tp), NF.stored_normals(self.tn), NF.stored_covs(self.tcv))
        self.scv_model = NF.stored_covs(self.scv)
        self.tree = cKDTree(self.tp[:, :3])
        self.aligned = T
        # misaligned: 1 deg / 0.35 m about the source's centre (about the origin, 300 m away, every pair would be rejected)
        self.misaligned = T @ about(NF.box_centre(self.sp), [0.01, -0.012, 0.008, 0.25, -0.2, 0.15])
        self.rng = rng

    def model(self, n, tgt=None):
        """storage model of source[:n] (its own centre: every set_source re-centres) against the whole target or a given one"""
        tp, tn, tcv = self.tgt_model if tgt is None else tgt
        return NF.stored_points(self.sp[:n]), self.scv_model[:n], tp, tn, tcv


@pytest.fixture(scope="module")
def data():
    return Data()


def _context(tp, tn, tcv):
    ctx = _sg().Context(0)
    ctx.set_target(tp, tn, tcv)
    ctx.build_target_kdtree()
    return ctx


def check_correspondences(corr, d, n, T, tp, max_d):
    """FP64 brute force on a sample of the queries, near ties and rejection-boundary cases allowed (np_factors.compare_correspondences)"""
    sample = np.arange(n) if n <= SAMPLE else np.sort(d.rng.choice(n, SAMPLE, replace=False))
    q = d.sp[sample, :3] @ T[:3, :3].T + T[:3, 3]
    tree = d.tree if tp is d.tp else cKDTree(tp[:, :3])
    dist, k = tree.query(q, distance_upper_bound=np.inf if max_d is None else np.sqrt(max_d) * (1 + 1e-6))
    bf = np.where(np.isinf(dist), NF.NO, k.astype(np.uint64))
    if max_d is not None:
        bf[dist * dist > max_d] = NF.NO
    NF.compare_correspondences(corr[sample], bf, tp, d.sp[sample], T, max_d)


def point_costs(T, corr, factor, model):
    """1/2 r^T M r of every accepted pair (where the robust kernels' knee sits)"""
    sp, scv, tp, tn, tcv = model
    idx = np.nonzero(corr != NF.NO)[0]
    k = corr[idx].astype(np.int64)
    r = tp[k, :3] - (sp[idx, :3] @ T[:3, :3].T + T[:3, 3])
    M = NF.weights(T, factor, sp, scv, tp, tn, tcv, idx, k)
    return 0.5 * np.einsum("ni,nij,nj->n", r, M, r)


def linearize_and_check(ctx, d, n, T, factor, robust, c, model, device_out=None, rejector=1, max_d=1.0, tp=None):
    """one linearize (host call, or linearize_device into `device_out`) and two error() calls, all against the model; returns
    (worst ratio, correspondences)"""
    sg = _sg()
    kw = dict(factor=factor, robust=robust, robust_c=c, rejector=rejector, max_dist_sq=max_d)
    if device_out is None:
        H, b, e = ctx.linearize(T, **kw)
    else:
        ctx.linearize_device(T, device_out.data_ptr(), **kw)
        ctx.synchronize()
        out = device_out.cpu().numpy()
        H, b, e = out[:36].reshape(6, 6), out[36:42], float(out[42])
    corr = ctx.correspondences()
    accepted = int((corr != sg.NO_CORRESPONDENCE).sum())
    assert ctx.num_inliers() == accepted
    if device_out is not None:
        assert out[43] == accepted
    assert np.array_equal(H, H.T)
    check_correspondences(corr, d, n, T, d.tp if tp is None else tp, max_d if rejector else None)
    tag = (n, factor, robust)
    if accepted == 0:
        assert not H.any() and not b.any() and e == 0.0 and ctx.error(T) == 0.0
        return 0.0, corr
    ratios = NF.tight_ratios((H, b, e), NF.linearize(T, corr, factor, robust, c, *model))
    assert max(ratios) <= NF.TIGHT, (tag, "H, b, e:", ratios)
    worst = max(ratios)
    centre = NF.box_centre(d.sp[:n])
    for a in TRIALS:  # LM trial poses: cached correspondences, GICP precision frozen at T
        T2 = T @ about(centre, a)
        e_gpu, e_model = ctx.error(T2), NF.error(T2, T, corr, factor, robust, c, *model)
        r = abs(e_gpu - e_model) / e_model
        assert r <= NF.TIGHT, (tag, "error()", e_gpu, e_model, r)
        worst = max(worst, r)
    return worst, corr


@pytest.fixture(scope="module")
def big_ctx(data):
    ctx = _context(data.tp, data.tn, data.tcv)
    yield ctx
    ctx.close()


@pytest.mark.parametrize("n", SIZES)
def test_sums_match_storage_model_across_sizes(data, big_ctx, n):
    """At each pose the plain factor comes first, and the robust kernels' c is the median per-point cost of its pairs: points on both
    sides of the knee.  The aligned pose is linearized twice (the second search is seeded by the first), the second time through
    linearize_device, whose out[43] must be the inlier count."""
    import torch

    ctx = big_ctx
    ctx.set_source(data.sp[:n], data.scv[:n])
    model = data.model(n)
    out = torch.zeros(64, dtype=torch.float64, device="cuda")
    worst = 0.0
    robusts = (0, 1, 2) if n in ALL_NINE else (0,)
    for factor in (0, 1, 2):
        knee = {}
        for robust in robusts:
            for j, T in enumerate((data.misaligned, data.aligned, data.aligned)):
                c = knee.get(j, 1.0)
                w, corr = linearize_and_check(ctx, data, n, T, factor, robust, c, model, device_out=out if j == 2 else None)
                worst = max(worst, w)
                if robust == 0 and j < 2 and (corr != NF.NO).any():
                    knee[j] = knee[j + 1] = float(np.sqrt(np.median(point_costs(T, corr, factor, model))))
    print(f"worst ratio to the storage model (source {n}): {worst:.2e}")


@pytest.mark.parametrize("m", [1, 5, 33])
def test_tiny_target_large_source(data, m):
    """a target of a few points (one leaf, a degenerate box) under the largest upload; no rejector, so every query matches"""
    n = 65537
    tp, tn, tcv = data.tp[:m], data.tn[:m], data.tcv[:m]
    ctx = _context(tp, tn, tcv)
    ctx.set_source(data.sp[:n], data.scv[:n])
    model = data.model(n, (NF.stored_points(tp), NF.stored_normals(tn), NF.stored_covs(tcv)))
    worst = 0.0
    for factor in (0, 1, 2):
        for T in (data.misaligned, data.aligned, data.aligned):
            w, corr = linearize_and_check(ctx, data, n, T, factor, 0, 1.0, model, rejector=0, tp=tp)
            assert ctx.num_inliers() == n
            worst = max(worst, w)
    ctx.close()
    print(f"worst ratio to the storage model (target {m}): {worst:.2e}")


def _run(ctx, d):
    """what the input-path tests compare bit for bit"""
    res = []
    for T in (d.misaligned, d.aligned):
        H, b, e = ctx.linearize(T, factor=2)
        res.append((H, b, e, ctx.correspondences(), ctx.num_inliers(), ctx.error(T @ about(NF.box_centre(d.sp[:N_PATHS]), TRIALS[0]))))
    return res


def _assert_bitwise(got, ref, tag):
    for (H, b, e, c, ni, err), (H0, b0, e0, c0, ni0, err0) in zip(got, ref):
        assert np.array_equal(H, H0) and np.array_equal(b, b0) and e == e0, tag
        assert np.array_equal(c, c0) and ni == ni0 and err == err0, tag


@pytest.fixture(scope="module")
def pageable(data):
    """the reference run of the input-path tests: numpy (pageable) inputs, checked against the model once"""
    ctx = _context(data.tp, data.tn, data.tcv)
    ctx.set_source(data.sp[:N_PATHS], data.scv[:N_PATHS])
    res = _run(ctx, data)
    model = data.model(N_PATHS)
    for (H, b, e, corr, _, _), T in zip(res, (data.misaligned, data.aligned)):
        assert max(NF.tight_ratios((H, b, e), NF.linearize(T, corr, 2, 0, 1.0, *model))) <= NF.TIGHT
    ctx.close()
    return res


def _torch_inputs(data, how):
    import torch

    arrs = (data.tp, data.tn, data.tcv, data.sp[:N_PATHS], data.scv[:N_PATHS])
    if how == "pinned":
        return [torch.from_numpy(np.ascontiguousarray(a)).pin_memory() for a in arrs]
    out = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrs]
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("how", ["pinned", "cuda"])
def test_input_paths_are_bitwise_equal(data, pageable, how):
    """page-locked host and device inputs take the asynchronous two-stream upload (include/sgicp_b200.h)"""
    tp, tn, tcv, sp, scv = _torch_inputs(data, how)
    ctx = _context(tp, tn, tcv)
    ctx.set_source(sp, scv)
    _assert_bitwise(_run(ctx, data), pageable, how)
    ctx.close()


def test_inputs_produced_on_a_bound_torch_stream(data, pageable):
    """inputs written by torch kernels on the stream the context is bound to, uploaded without any synchronisation: the upload (and
    its copy stream) must be ordered behind the producing kernels"""
    import torch

    base = _torch_inputs(data, "cuda")
    stream = torch.cuda.Stream()
    ctx = _sg().Context(0)
    ctx.set_stream(stream.cuda_stream)
    with torch.cuda.stream(stream):
        tp, tn, tcv, sp, scv = [x.mul(2.0).mul_(0.5) for x in base]  # exact: powers of two
        ctx.set_target(tp, tn, tcv)
        ctx.build_target_kdtree()
        ctx.set_source(sp, scv)
        res = _run(ctx, data)
    _assert_bitwise(res, pageable, "side stream")
    ctx.set_stream(None)
    ctx.close()


def test_back_to_back_uploads(data, pageable):
    """no synchronisation between consecutive uploads: a second set_source replaces the first one's pending copies, and a source upload
    directly behind a target upload shares the staging buffers with it"""
    tp, tn, tcv, sp, scv = _torch_inputs(data, "pinned")
    import torch

    rng = np.random.default_rng(5)
    other_p = torch.from_numpy(np.ascontiguousarray(data.sp[:N_PATHS][::-1] + np.r_[0.2, -0.1, 0.3, 0.0])).pin_memory()
    other_c = torch.from_numpy(_random_covs(rng, N_PATHS)).pin_memory()
    ctx = _context(data.tp, data.tn, data.tcv)
    ctx.set_source(other_p, other_c)
    ctx.set_source(sp, scv)
    _assert_bitwise(_run(ctx, data), pageable, "set_source A then B")
    ctx.close()
    ctx = _sg().Context(0)
    ctx.set_target(tp, tn, tcv)
    ctx.set_source(sp, scv)
    ctx.build_target_kdtree()
    _assert_bitwise(_run(ctx, data), pageable, "set_target then set_source")
    ctx.close()
