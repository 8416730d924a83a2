"""Distinct contexts used at the same time from several host threads (include/sgicp_b200.h: a context is not thread-safe, distinct
contexts are), each bit-identical to its calls alone.

Six workers, each with its own context and its own script, run their script R = 3 times in a row.  Together the scripts launch every
kernel whose dynamic shared memory is opted in above 48 KiB, at different sizes in different threads: joint_step_kernel on windows of 20,
24, 28 and 31 free frames (the most a window holds) on many kd-trees and many voxel maps, batch_knn_kernel and features_kernel on adopted
trees of leaf depth 33, 36 and 40, the single and many-tree builds (kd_refine_smem_kernel, forest_refine_smem_kernel), and the ordinary
hot path around them.  That limit is a property of the kernel on the device, shared by every context of the process, which is why
allow_dynamic_smem only ever raises it (DESIGN.md section 1, "Concurrency").

  1. the serial baseline: every script alone in the main thread, its correspondences, H | b | e, error() and k-NN rows held to the exact
     FP64 models (np_search, np_factors.storage_model), so that a deterministic shared-state bug cannot hide in both runs;
  2. the six scripts on six threads released together, each context on its own stream: every output of every round bit-identical to the
     serial baseline;
  3. the same with every context on a torch stream of its own (set_stream), and two contexts in two threads sharing one stream;
  4. one thread captures align_batch_async into a CUDA graph and replays it while the others run their scripts;
  5. two threads create, use and close short-lived contexts while the others run;
  6. two devices in one process: device 1 after device 0 and then both at once, device 1 bit-identical to device 0 (skipped with fewer
     than two GPUs);
and, for the reference's own pattern in C++, four Registration<GICPFactor, ParallelReductionCUDA>::align() calls of the host mirror on
four std::threads against one shared target (tests/host_threads).

Each case runs its fixed workload once; the file prints its wall time (-s)."""
import contextlib
import os
import subprocess
import tempfile
import threading
import time
import traceback

import numpy as np
import pytest

import np_factors as NF
import np_search as NS
from test_gpu_storage_model import TRIALS, about

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROUNDS = 3
JOINT_FRAMES = 32  # the most frames a window takes, one of them fixed: 31 free frames
T_START = time.perf_counter()


def _sg():
    import small_gicp_b200 as sg

    return sg


def _torch():
    return pytest.importorskip("torch")


# ---------------------------------------------------------------------------------------------------------------------------------
# inputs, made once per module
# ---------------------------------------------------------------------------------------------------------------------------------
class World:
    def __init__(self):
        from test_gpu_align_joint import Frames
        from test_gpu_search_exhaustive import _caterpillar
        from test_gpu_storage_model import Data
        from small_gicp_b200.synthetic import make_world, sample_cloud

        self.d = d = Data()
        self.n_single = 65537
        self.members = [(0, 31), (100, 129), (1000, 4097), (20000, 9000), (40000, 20000)]  # (start, size) in the source
        self.frames = Frames(JOINT_FRAMES, n=1500, seed=11)
        self.trees = {depth: _caterpillar(depth) for depth in (33, 36, 40)}
        rng = np.random.default_rng(31)
        self.tree_queries = {}
        for depth, (pts, _, _) in self.trees.items():
            q = NF._f32(pts[::3] + rng.normal(0.0, 0.05, (len(pts[::3]), 3)))
            self.tree_queries[depth] = np.concatenate([q, [[depth + 30.0, 2.0, 1.0], [-25.0, -4.0, 0.5]]])
        world = make_world(200_000, 5)
        self.clouds = [sample_cloud(world, n, 60 + j) for j, n in enumerate((8000, 21000, 36000))]
        self.cloud_queries = [sample_cloud(world, 3000, 70 + j) + rng.normal(0.0, 0.05, (3000, 3)) for j in range(3)]
        self.small = sample_cloud(world, 5000, 80)  # the short-lived contexts' cloud

    def member(self, m):
        s, n = self.members[m]
        return self.d.sp[s : s + n], self.d.scv[s : s + n]

    def member_poses(self, shift=0):
        d = self.d
        out = []
        for m in range(len(self.members)):
            c = NF.box_centre(self.member(m)[0])
            T = d.aligned if (m + shift) % 2 == 0 else d.misaligned
            out.append(T @ about(c, [0.002 * (m % 5), -0.001 * (m % 3), 0.0015, 0.01 * (m % 4), 0.0, -0.02]))
        return np.array(out)


@pytest.fixture(scope="module")
def world():
    return World()


# ---------------------------------------------------------------------------------------------------------------------------------
# the scripts: each takes (context, world, torch stream or None) and returns a list of (name, array); `checks` collects what the
# serial baseline holds to the FP64 models
# ---------------------------------------------------------------------------------------------------------------------------------
def _host(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def script_hot(ctx, w, stream, checks=None):
    """the single-target hot path on the 200k scene, then a batch of members against it: linearize / error / correspondences,
    linearize_batch / error_batch / correspondences_batch, align_batch"""
    d = w.d
    n = w.n_single
    out = []
    ctx.set_target(d.tp, d.tn, d.tcv)
    ctx.build_target_kdtree()
    ctx.set_source(d.sp[:n], d.scv[:n])
    centre = NF.box_centre(d.sp[:n])
    for j, T in enumerate((d.misaligned, d.aligned)):
        H, b, e = ctx.linearize(T, factor=2)
        corr = ctx.correspondences()
        T2 = T @ about(centre, TRIALS[0])
        err = ctx.error(T2)
        out += [(f"H{j}", H), (f"b{j}", b), (f"e{j}", np.float64(e)), (f"corr{j}", corr), (f"inl{j}", np.int64(ctx.num_inliers())),
                (f"err{j}", np.float64(err))]
        if checks is not None:
            checks.append(("single", T, T2, corr, (H, b, e), err))
    srcs = [w.member(m) for m in range(len(w.members))]
    ctx.set_source_batch([p for p, _ in srcs], [c for _, c in srcs])
    Ts = w.member_poses()
    H, b, e, inl = ctx.linearize_batch(Ts, factor=2)
    corrs = ctx.correspondences_batch()
    T2s = np.array([T @ about(NF.box_centre(p), TRIALS[1]) for T, (p, _) in zip(Ts, srcs)])
    eb = ctx.error_batch(T2s)
    out += [("bH", H), ("bb", b), ("be", e), ("binl", inl), ("berr", eb)] + [(f"bcorr{m}", c) for m, c in enumerate(corrs)]
    if checks is not None:
        checks.append(("batch", Ts, T2s, corrs, (H, b, e), eb))
    r = ctx.align_batch(w.member_poses(1), factor=2)
    out += [("aT", r.T_target_source), ("aconv", r.converged), ("ait", r.iterations), ("ainl", r.num_inliers), ("aerr", r.error), ("aH", r.H)]
    return out


def _async_setup(ctx, w):
    d = w.d
    ctx.set_target(d.tp[:150_000], d.tn[:150_000], d.tcv[:150_000])
    ctx.build_target_kdtree()
    srcs = [w.member(m) for m in range(len(w.members))]
    ctx.set_source_batch([p for p, _ in srcs], [c for _, c in srcs])


def script_async(ctx, w, stream, checks=None):
    """align_batch_async and align_batch_gnc_async on a 150k-point target (the context on a torch stream)"""
    torch = _torch()
    _async_setup(ctx, w)
    T0 = torch.from_numpy(w.member_poses(1)).cuda()
    a = ctx.align_batch_async(T0, factor=2)
    g = ctx.align_batch_gnc_async(T0, 0.25, factor=2, max_dist_sq=0.25)
    ctx.synchronize()
    return [("T16", _host(a.T16)), ("info4", _host(a.info4)), ("Hb42", _host(a.Hb42)), ("gT16", _host(g.T16)), ("ginfo4", _host(g.info4)),
            ("gHb42", _host(g.Hb42)), ("gnc2", _host(g.gnc2))]


def _joint_setup(ctx, w, K, kind):
    from test_gpu_align_joint import _window_edges

    fr = w.frames
    idx = list(range(K))
    pts = [fr.pts[i] for i in idx]
    if kind == "kdtree":
        ctx.build_target_kdtrees(pts, [fr.normals[i] for i in idx], [fr.covs[i] for i in idx])
    else:
        ctx.build_target_voxelmaps(pts, [fr.covs[i] for i in idx], 1.0, 1)
    ctx.set_source_batch(pts, [fr.covs[i] for i in idx])
    edges = _window_edges(K)
    ctx.set_source_pairs(np.array([e[0] for e in edges], dtype=np.uint32), np.array([e[1] for e in edges], dtype=np.uint32))
    return idx


def _joint_script(ctx, w, stream, kind, free):
    """one window of F + 1 frames, its first fixed, per count F of free frames, synchronous and stream-ordered in turn"""
    from test_gpu_align_joint import _perturbed

    torch = _torch()
    out = []
    for j, F in enumerate(free):
        K = F + 1
        idx = _joint_setup(ctx, w, K, kind)
        X = _perturbed(w.frames, idx, 40 + K)
        if j % 2 == 0:
            r = ctx.align_joint(X, factor=2)
            X16, info = r.X, np.c_[r.converged, r.iterations, r.num_inliers, r.error]
        else:
            a = ctx.align_joint_async(torch.from_numpy(np.ascontiguousarray(X)).cuda(), factor=2)
            ctx.synchronize()
            X16, info = _host(a.X16).reshape(K, 4, 4).transpose(0, 2, 1), _host(a.info4)
        out += [(f"X{K}", X16), (f"info{K}", info), (f"corr{K}", np.concatenate(ctx.correspondences_batch()))]
    return out


def script_joint_trees(ctx, w, stream, checks=None):
    return _joint_script(ctx, w, stream, "kdtree", (20, 31, 24, 28))


def script_joint_voxels(ctx, w, stream, checks=None):
    return _joint_script(ctx, w, stream, "voxelmap", (31, 20, 28, 24))


def script_deep_trees(ctx, w, stream, checks=None):
    """adopted trees of leaf depth 33, 36 and 40: batch k-NN at k = 1, 10, 20, 32, features in place at k = 10, 20, 32 (seen through a
    point-to-plane linearize), and estimate_features of the same points on the library's own tree"""
    sg = _sg()
    out = []
    for depth, (pts, nodes, idx) in w.trees.items():
        ctx.set_target(pts)
        ctx.set_target_kdtree(nodes, idx)
        q = w.tree_queries[depth]
        for k in (1, 10, 20, 32):
            kidx, kd2 = ctx.target_batch_knn(q, k)
            out += [(f"knn{depth}_{k}", kidx), (f"d2{depth}_{k}", kd2)]
            if checks is not None:
                checks.append(("knn", depth, k, q, kidx, kd2))
        for k in (10, 20, 32):
            ctx.estimate_target_features(k)
            ctx.set_source(q[:-2])
            H, b, e = ctx.linearize(np.eye(4), factor=sg.FACTOR_PLANE_ICP)
            out += [(f"pH{depth}_{k}", H), (f"pb{depth}_{k}", b), (f"pe{depth}_{k}", np.float64(e))]
        for k in (10, 20, 32):
            nr, cv = ctx.estimate_features(pts, k)
            out += [(f"fn{depth}_{k}", nr), (f"fc{depth}_{k}", cv)]
    return out


def script_preprocess(ctx, w, stream, checks=None):
    """voxelgrid_sampling_batch, estimate_features_batch at k = 10, 20, 32, many voxel maps + linearize_batch + target_knn_maps, many
    kd-trees + target_knn_maps, and single tree builds of different sizes + target_batch_knn"""
    out = []
    clouds = w.clouds
    vp, voff = ctx.voxelgrid_sampling_batch(clouds, 0.25)
    out += [("vox", vp), ("voxoff", voff)]
    covs = None
    for k in (10, 20, 32):
        nr, cv = ctx.estimate_features_batch(clouds, k)
        out += [(f"bn{k}", nr), (f"bc{k}", cv)]
        covs = cv if k == 20 else covs
    off = np.concatenate([[0], np.cumsum([len(c) for c in clouds])])
    cl_covs = [covs[off[j] : off[j + 1]] for j in range(len(clouds))]
    ctx.build_target_voxelmaps(clouds, cl_covs, 1.0, 1)
    qs = w.cloud_queries
    ctx.set_source_batch(qs, [c[: len(q)] for c, q in zip(cl_covs, qs)])
    H, b, e, inl = ctx.linearize_batch(np.array([np.eye(4)] * len(qs)), factor=2)
    vidx, vd2 = ctx.target_knn_maps(qs, 5)
    out += [("vH", H), ("vb", b), ("ve", e), ("vinl", inl), ("vknn", vidx), ("vd2", vd2)]
    ctx.build_target_kdtrees(clouds, None, cl_covs)
    kidx, kd2 = ctx.target_knn_maps(qs, 10)
    out += [("fknn", kidx), ("fd2", kd2)]
    if checks is not None:
        qoff = np.concatenate([[0], np.cumsum([len(q) for q in qs])])
        for s in range(len(qs)):
            checks.append(("knn_map", s, 10, qs[s], kidx[qoff[s] : qoff[s + 1]], kd2[qoff[s] : qoff[s + 1]]))
    for j, c in enumerate(clouds):
        ctx.set_target(c)
        ctx.build_target_kdtree()
        kidx, kd2 = ctx.target_batch_knn(qs[j], 20)
        out += [(f"sknn{j}", kidx), (f"sd2{j}", kd2)]
    return out


def script_short_lived(ctx, w, stream, checks=None):
    """a small job of a short-lived context: tree, features, one linearize"""
    ctx.set_target(w.small)
    ctx.build_target_kdtree()
    nr, cv = ctx.estimate_features(w.small, 10)
    ctx.set_target(w.small, nr, cv)
    ctx.build_target_kdtree()
    ctx.set_source(w.small[::2], cv[::2])
    H, b, e = ctx.linearize(about(NF.box_centre(w.small), [0.01, 0.0, -0.01, 0.05, 0.02, 0.0]), factor=2)
    return [("n", nr), ("c", cv), ("H", H), ("b", b), ("e", np.float64(e)), ("corr", ctx.correspondences())]


# name -> (script, needs a torch stream)
SCRIPTS = {
    "hot": (script_hot, False),
    "async": (script_async, True),
    "joint_trees": (script_joint_trees, True),
    "joint_voxels": (script_joint_voxels, True),
    "deep_trees": (script_deep_trees, False),
    "preprocess": (script_preprocess, False),
}


# ---------------------------------------------------------------------------------------------------------------------------------
# running and comparing
# ---------------------------------------------------------------------------------------------------------------------------------
def _rounds(ctx, w, fn, stream, rounds=ROUNDS, checks=None):
    torch = _torch()
    if stream is not None:
        ctx.set_stream(stream.cuda_stream)
    res = []
    with torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext():
        for r in range(rounds):
            res.append(fn(ctx, w, stream, checks if r == 0 else None))
    if stream is not None:
        stream.synchronize()
    return res


def _same(got, ref, tag):
    assert [n for n, _ in got] == [n for n, _ in ref], tag
    for (name, a), (_, b) in zip(got, ref):
        a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
        assert a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes(), (tag, name, "differs from the serial run")


def _same_rounds(got, ref, tag):
    assert len(got) == len(ref), tag
    for r, (g, s) in enumerate(zip(got, ref)):
        _same(g, s, (tag, "round", r))


class Workers:
    """jobs run on threads released together by a barrier; each job: (tag, fn(barrier) -> result).  Every failure is kept with its
    traceback (an SgbError carries the context's sgb_last_error)."""

    def __init__(self, jobs):
        self.jobs = jobs
        self.barrier = threading.Barrier(len(jobs))
        self.results = {}
        self.errors = {}

    def run(self):
        def work(tag, fn):
            try:
                self.results[tag] = fn(self.barrier)
            except BaseException:
                self.errors[tag] = traceback.format_exc()
                self.barrier.abort()

        threads = [threading.Thread(target=work, args=job) for job in self.jobs]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert not self.errors, "\n".join(f"{k}: {v}" for k, v in self.errors.items())
        return self.results


def _script_job(w, name, device=0, stream=None, rounds=ROUNDS):
    """a worker: its own context (and a torch stream of its own where its script needs one and none is given), released with the
    others, R rounds of its script"""
    fn, needs_stream = SCRIPTS[name] if name in SCRIPTS else (script_short_lived, False)

    def job(barrier):
        torch = _torch()
        sg = _sg()
        with torch.cuda.device(device):
            s = stream if stream is not None else (torch.cuda.Stream() if needs_stream else None)
            ctx = sg.Context(device)
            try:
                barrier.wait(timeout=300)
                return _rounds(ctx, w, fn, s, rounds)
            finally:
                if s is not None:
                    s.synchronize()
                ctx.close()

    return job


@pytest.fixture(scope="module")
def serial(world):
    """every script alone, one fresh context at a time, in the main thread; with the values the FP64 models check"""
    torch = _torch()
    sg = _sg()
    out, checks = {}, {}
    for name, (fn, needs_stream) in SCRIPTS.items():
        ctx = sg.Context(0)
        checks[name] = []
        out[name] = _rounds(ctx, world, fn, torch.cuda.Stream() if needs_stream else None, checks=checks[name])
        ctx.close()
    ctx = sg.Context(0)
    out["short_lived"] = _rounds(ctx, world, script_short_lived, None, rounds=1)
    ctx.close()
    return out, checks


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    yield
    print(f"\ntest_gpu_concurrent_contexts: {time.perf_counter() - T_START:.1f} s wall time")


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. the serial baseline against the FP64 models
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_serial_baseline_matches_fp64_models(world, serial):
    _, checks = serial
    d = world.d
    n = world.n_single
    worst = 0.0
    for kind, T, T2, corr, (H, b, e), err in checks["hot"]:
        if kind == "single":
            NS.check_correspondences(corr, T, d.sp[:n], d.search, 1.0)
            model = d.model(n)
            ratios = NF.tight_ratios((H, b, e), NF.linearize(T, corr, 2, 0, 1.0, *model))
            assert max(ratios) <= NF.TIGHT, ("single", ratios)
            e_model = NF.error(T2, T, corr, 2, 0, 1.0, *model)
            assert abs(err - e_model) <= NF.TIGHT * e_model, ("single error()", err, e_model)
            worst = max(worst, *ratios)
            continue
        for m, (p, cv) in enumerate(world.member(j) for j in range(len(world.members))):
            NS.check_correspondences(corr[m], T[m], p, d.search, 1.0)
            model = (NF.stored_points(p), NF.stored_covs(cv), *d.tgt_model)
            ratios = NF.tight_ratios((H[m], b[m], e[m]), NF.linearize(T[m], corr[m], 2, 0, 1.0, *model))
            assert max(ratios) <= NF.TIGHT, ("member", m, ratios)
            e_model = NF.error(T2[m], T[m], corr[m], 2, 0, 1.0, *model)
            assert abs(err[m] - e_model) <= NF.TIGHT * e_model, ("member error_batch", m, err[m], e_model)
            worst = max(worst, *ratios)
    for _, depth, k, q, kidx, kd2 in checks["deep_trees"]:
        NS.check_knn(kidx, kd2, q, k, NS.Target(world.trees[depth][0]))
    for _, s, k, q, kidx, kd2 in checks["preprocess"]:
        NS.check_knn(kidx, kd2, q, k, NS.Target(world.clouds[s]))
    print(f"serial baseline: worst ratio to the storage model {worst:.2e}; search model: {NS.REPORT}")


# ---------------------------------------------------------------------------------------------------------------------------------
# 2, 3. concurrent: private streams, caller streams, one shared caller stream
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_concurrent_private_streams(world, serial):
    ref, _ = serial
    got = Workers([(name, _script_job(world, name)) for name in SCRIPTS]).run()
    for name in SCRIPTS:
        _same_rounds(got[name], ref[name], ("private streams", name))


@pytest.mark.gpu
def test_concurrent_caller_streams(world, serial):
    torch = _torch()
    ref, _ = serial
    streams = {name: torch.cuda.Stream() for name in SCRIPTS}
    got = Workers([(name, _script_job(world, name, stream=streams[name])) for name in SCRIPTS]).run()
    for name in SCRIPTS:
        _same_rounds(got[name], ref[name], ("caller streams", name))
    shared = torch.cuda.Stream()  # two contexts in two threads, both on one caller stream
    got = Workers([(name, _script_job(world, name, stream=shared)) for name in ("hot", "deep_trees")]).run()
    for name in ("hot", "deep_trees"):
        _same_rounds(got[name], ref[name], ("shared stream", name))


# ---------------------------------------------------------------------------------------------------------------------------------
# 4. a graph capture beside other threads
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_capture_beside_other_threads(world, serial):
    """The capture uses capture_error_mode="thread_local": only the capturing thread is restricted, while the other threads go on
    uploading, growing their contexts' buffers (cudaMalloc) and launching.  Torch's default "global" mode forbids such calls in every
    other thread for the duration of a capture, by torch's own rule, so concurrent work beside a capture is only valid in this mode (or
    "relaxed") and "global" is not tested here."""
    torch = _torch()
    sg = _sg()
    ref, _ = serial
    want = dict(ref["async"][0])

    def capture(barrier):
        s = torch.cuda.Stream()
        ctx = sg.Context(0)
        try:
            ctx.set_stream(s.cuda_stream)
            with torch.cuda.stream(s):
                _async_setup(ctx, world)
                T0 = torch.from_numpy(world.member_poses(1)).cuda()
                out = ctx.align_batch_async(T0, factor=2)  # warm-up outside the capture: buffers sized, the loop graph built
            s.synchronize()
            barrier.wait(timeout=300)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
                ctx.align_batch_async(T0, out=out)
            res = []
            with torch.cuda.stream(s):
                for _ in range(ROUNDS):
                    out.T16.zero_()
                    out.info4.zero_()
                    g.replay()
                    s.synchronize()
                    res.append([("T16", _host(out.T16)), ("info4", _host(out.info4)), ("Hb42", _host(out.Hb42))])
            return res
        finally:
            s.synchronize()
            ctx.close()

    others = [n for n in SCRIPTS if n != "async"]
    got = Workers([("capture", capture)] + [(name, _script_job(world, name)) for name in others]).run()
    for r, res in enumerate(got["capture"]):
        _same(res, [(n, want[n]) for n in ("T16", "info4", "Hb42")], ("replay", r))
    for name in others:
        _same_rounds(got[name], ref[name], ("beside a capture", name))


# ---------------------------------------------------------------------------------------------------------------------------------
# 5. contexts created and closed while others compute
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_create_and_close_while_others_compute(world, serial):
    sg = _sg()
    ref, _ = serial

    def churn(barrier):
        barrier.wait(timeout=300)
        res = []
        for _ in range(ROUNDS):
            ctx = sg.Context(0)
            try:
                res.append(script_short_lived(ctx, world, None))
            finally:
                ctx.close()
        return res

    jobs = [(f"churn{i}", churn) for i in range(2)] + [(name, _script_job(world, name)) for name in SCRIPTS]
    got = Workers(jobs).run()
    for i in range(2):
        for r, res in enumerate(got[f"churn{i}"]):
            _same(res, ref["short_lived"][0], ("short-lived context", i, r))
    for name in SCRIPTS:
        _same_rounds(got[name], ref[name], ("beside short-lived contexts", name))


# ---------------------------------------------------------------------------------------------------------------------------------
# 6. two devices in one process
# ---------------------------------------------------------------------------------------------------------------------------------
def script_two_devices(ctx, w, stream, checks=None):
    """the tree builds and features: one kd-tree (kd_refine_smem_kernel), many kd-trees (forest_refine_smem_kernel), features"""
    d = w.d
    ctx.set_target(d.tp, d.tn, d.tcv)
    ctx.build_target_kdtree()
    ctx.set_source(d.sp[:20000], d.scv[:20000])
    H, b, e = ctx.linearize(d.aligned, factor=2)
    out = [("H", H), ("b", b), ("e", np.float64(e)), ("corr", ctx.correspondences())]
    ctx.build_target_kdtrees(w.clouds)
    idx, d2 = ctx.target_knn_maps(w.cloud_queries, 10)
    nr, cv = ctx.estimate_features(w.clouds[1], 20)
    return out + [("knn", idx), ("d2", d2), ("n", nr), ("c", cv)]


@pytest.mark.gpu
def test_two_devices_in_one_process(world):
    torch = _torch()
    sg = _sg()
    if torch.cuda.device_count() < 2:
        pytest.skip("two devices in one process: needs 2 GPUs, this machine has fewer")
    assert torch.cuda.get_device_name(0) == torch.cuda.get_device_name(1), "device 1's results are compared bit for bit with device 0's"
    alone = {}
    for dev in (0, 1):  # device 0 builds its trees first, then device 1 (whose kernels' attributes were never set)
        with torch.cuda.device(dev):
            ctx = sg.Context(dev)
            alone[dev] = _rounds(ctx, world, script_two_devices, None, rounds=1)
            ctx.close()
    _same_rounds(alone[1], alone[0], "device 1 after device 0")

    def job(dev):
        def run(barrier):
            with torch.cuda.device(dev):
                ctx = sg.Context(dev)
                try:
                    barrier.wait(timeout=300)
                    return _rounds(ctx, world, script_two_devices, None)
                finally:
                    ctx.close()

        return run

    got = Workers([(dev, job(dev)) for dev in (0, 1)]).run()
    for dev in (0, 1):
        _same_rounds(got[dev], alone[0] * ROUNDS, ("two devices at once", dev))


# ---------------------------------------------------------------------------------------------------------------------------------
# the drop-in's own pattern in C++: Registration<>::align() on std::threads
# ---------------------------------------------------------------------------------------------------------------------------------
def _build_host_threads(out_dir):
    binary = os.path.join(out_dir, "sgb_host_threads")
    r = subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "tests", "host_threads"), f"OUT={binary}"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return binary


def test_host_threads_driver_compiles():
    """the C++ driver compiles against the in-repo mirror headers and links against the library (no GPU needed)"""
    with tempfile.TemporaryDirectory() as d:
        assert os.path.exists(_build_host_threads(d))


@pytest.mark.gpu
def test_host_threads_registration_align():
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([_build_host_threads(d)], capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert r.stdout.count("identical") == 4
