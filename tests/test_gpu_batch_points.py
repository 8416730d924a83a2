"""Per-point terms of batched registration (sgb_linearize_batch_points / sgb_error_batch_points, Context.linearize_batch_points /
error_batch_points): every target kind, against the plain calls bit for bit and against an FP64 model of each point's terms.

  1. the member sums, error() and the correspondences are bit-identical to linearize_batch / error_batch, and the calls leave the same state;
  2. every row matches the FP64 storage model of its point (J^T M J, J^T M r, 1/2 r^T M r, robust weight; error() at a trial pose with the
     GICP precision frozen at the linearisation pose) to np_factors.TIGHT;
  3. each member's rows add up to its H | b | e to TIGHT;
  4. rows are zero exactly where there is no correspondence, for inactive members and against an empty target;
  5. a permuted cloud gives permuted rows, and a member's rows are bit-identical at B = 1, 17 and 4096 wherever it sits;
  6. CUDA and page-locked outputs equal host outputs bit for bit;
  7. the launch counts are those of the plain calls;
  8. misuse fails with a message.
Each model test prints the worst ratio it reached (run with -s to see it)."""
import ctypes as C

import numpy as np
import pytest

import np_factors as NF
import np_preprocess as PP
import np_submaps as SM
from test_gpu_storage_model import OFFSET, _random_covs, _unit, about

pytestmark = pytest.mark.gpu

ROBUST = [(0, 1.0), (1, 0.05), (2, 0.01)]
MAX_D = [1.0, 0.05]
LEAF = 1.0


def _sg():
    import small_gicp_b200 as sg

    return sg


def _p4(xyz):
    return np.c_[xyz, np.ones(len(xyz))]


def _n4(rng, n):
    return np.c_[_unit(rng, n), np.zeros(n)]


class Scene:
    """One world 300 m from the origin: a 40k-point target; five maps (one of them empty, one of a single point), each also handed over
    in a frame of its own for the submap lists; five source clouds (one empty, sizes on both sides of the 128-point tile).  Random
    normals and covariances."""

    def __init__(self):
        from small_gicp_b200.synthetic import make_world, sample_cloud

        world = make_world(200_000)
        rng = np.random.default_rng(91)
        self.tp = _p4(sample_cloud(world, 40_000, 1) + OFFSET)
        self.tn = _n4(rng, len(self.tp))
        self.tcv = _random_covs(rng, len(self.tp))
        self.maps = [_p4(sample_cloud(world, n, 10 + j) + OFFSET) if n else np.zeros((0, 4)) for j, n in enumerate([8000, 12000, 0, 6000, 1])]
        self.mnormals = [_n4(rng, len(m)) for m in self.maps]
        self.mcovs = [_random_covs(rng, len(m)) for m in self.maps]
        self.P = [about(OFFSET, np.r_[rng.uniform(-0.3, 0.3, 3), rng.uniform(-2, 2, 3)]) for _ in self.maps]
        self.smaps = [_p4(m[:, :3] @ SM.inverse(P)[:3, :3].T + SM.inverse(P)[:3, 3]) if len(m) else m for m, P in zip(self.maps, self.P)]
        self.srcs = [_p4(sample_cloud(world, n, 50 + j) + OFFSET) if n else np.zeros((0, 4)) for j, n in enumerate([3000, 700, 129, 0, 2000])]
        self.scovs = [_random_covs(rng, len(s)) for s in self.srcs]
        self.centres = [NF.box_centre(s) if len(s) else OFFSET for s in self.srcs]

    def poses(self, clouds, k=0):
        return np.array([about(self.centres[c], [0.003 * ((p + k) % 5) - 0.006, 0.002 * (p % 3), -0.002, 0.04 * ((p + k) % 4) - 0.06, 0.02, -0.03 * k])
                         for p, c in enumerate(clouds)])


@pytest.fixture(scope="module")
def scene():
    return Scene()


# ---- the target kinds: a context, the cloud of each member, and each member's correspondences -> per-point FP64 operands ----
class Kind:
    def __init__(self, name, ctx, clouds, operands, plane=True):
        self.name, self.ctx, self.clouds, self.operands, self.plane = name, ctx, clouds, operands, plane


def _kdtree(s):
    ctx = _sg().Context(0)
    ctx.set_target(s.tp, s.tn, s.tcv)
    ctx.build_target_kdtree()
    ctx.set_source_batch(s.srcs, s.scovs)
    return ctx


def _point_operands(tp, tn, tcv):
    """correspondences = original indices of one stored point cloud"""
    def f(p, c, corr):
        sp, scv, t, n, cv = NF.storage_model(p, c, tp, tn, tcv)
        idx = np.where(corr == NF.NO, -1, corr.astype(np.int64))
        return [(np.eye(4), idx, sp, scv, t, n, cv)]
    return f


def _voxel_operands(tp, tcv):
    coords, means, vcovs, _ = PP.voxelmap_model(tp[:, :3], tcv, LEAF) if len(tp) else (None, np.zeros((0, 4)), np.zeros((0, 4, 4)), None)

    def f(p, c, corr):
        sp, scv, t, _, cv = NF.storage_model(p, c, means, None, vcovs)
        idx = np.where(corr == NF.NO, -1, (corr >> np.uint64(32)).astype(np.int64))
        return [(np.eye(4), idx, sp, scv, t, None, cv)]
    return f


def _submap_operands(s, lists):
    """member p: entry j of its list = stored map lists[p][j] placed by P; the point's terms at P^-1 T against that map as stored"""
    def make(p):
        def f(pts, c, corr):
            out = []
            for j, k in enumerate(lists[p]):
                sp, scv, t, _, cv = NF.storage_model(pts, c, s.smaps[k], None, s.mcovs[k])
                mine = (corr != NF.NO) & ((corr >> np.uint64(32)) == j)
                idx = np.where(mine, (corr & SM.LOW).astype(np.int64), -1)
                out.append((SM.inverse(s.P[k]), idx, sp, scv, t, None, cv))
            return out
        return f
    return make


def kinds(s):
    """every target kind: one kd-tree, one voxel map at 1 / 7 / 27 search offsets, many voxel maps, many kd-trees, pairs with and
    without a maps table, submap lists of 1 and of 5 entries"""
    out = []
    every = list(range(len(s.srcs)))
    out.append(Kind("kdtree", _kdtree(s), every, [_point_operands(s.tp, s.tn, s.tcv)] * len(every)))
    for offs in (1, 7, 27):
        ctx = _sg().Context(0)
        ctx.build_target_voxelmap(s.tp, s.tcv, LEAF, offs)
        ctx.set_source_batch(s.srcs, s.scovs)
        out.append(Kind(f"voxelmap{offs}", ctx, every, [_voxel_operands(s.tp, s.tcv)] * len(every), plane=False))
    ctx = _sg().Context(0)
    ctx.build_target_voxelmaps(s.maps, s.mcovs, LEAF, 7)
    ctx.set_source_batch(s.srcs, s.scovs)
    out.append(Kind("voxelmaps", ctx, every, [_voxel_operands(m, c) for m, c in zip(s.maps, s.mcovs)], plane=False))
    ctx = _sg().Context(0)
    ctx.build_target_kdtrees(s.maps, s.mnormals, s.mcovs)
    ctx.set_source_batch(s.srcs, s.scovs)
    out.append(Kind("kdtrees", ctx, every, [_point_operands(m, n, c) for m, n, c in zip(s.maps, s.mnormals, s.mcovs)]))
    cl, mp = [4, 0, 0, 2, 1, 3, 0], [0, 1, 3, 4, 2, 0, 4]
    ctx = _sg().Context(0)
    ctx.build_target_kdtrees(s.maps, s.mnormals, s.mcovs)
    ctx.set_source_batch(s.srcs, s.scovs)
    ctx.set_source_pairs(cl, mp)
    out.append(Kind("pairs_maps", ctx, cl, [_point_operands(s.maps[k], s.mnormals[k], s.mcovs[k]) for k in mp]))
    cl = [1, 0, 4, 0]
    ctx = _kdtree(s)
    ctx.set_source_pairs(cl)
    out.append(Kind("pairs", ctx, cl, [_point_operands(s.tp, s.tn, s.tcv)] * len(cl)))
    for name, lists in (("submaps1", [[0], [1], [3], [4], [0]]), ("submaps5", [[0, 1, 2, 3, 4], [3, 0, 1, 4, 2], [1, 0, 3, 0, 4], [4, 2, 2, 1, 0], [2, 3, 4, 1, 0]])):
        cl = [0, 4, 1, 2, 3]
        ctx = _sg().Context(0)
        ctx.build_target_kdtrees(s.smaps, None, s.mcovs)
        ctx.set_source_batch(s.srcs, s.scovs)
        ctx.set_source_submaps(lists, [[s.P[k] for k in l] for l in lists], cl)
        make = _submap_operands(s, lists)
        out.append(Kind(name, ctx, cl, [make(p) for p in range(len(cl))], plane=False))
    return out


@pytest.fixture(scope="module")
def all_kinds(scene):
    return kinds(scene)


# ---- the FP64 model of one point's terms (np_factors.linearize / error without the sum) ----
def model_rows(T, idx, factor, robust, c, sp, scv, tp, tn, tcv):
    n = len(idx)
    e, H, b = np.zeros(n), np.zeros((n, 6, 6)), np.zeros((n, 6))
    has = np.nonzero(idx >= 0)[0]
    if len(has) == 0:
        return e, H, b
    k = idx[has]
    R = T[:3, :3]
    p = sp[has, :3]
    r = tp[k, :3] - (p @ R.T + T[:3, 3])
    M = NF.weights(T, factor, sp, scv, tp, tn, tcv, has, k)
    J = np.concatenate([R @ NF._skew_batch(p), np.tile(-R, (len(has), 1, 1))], axis=2)
    Mr = np.einsum("nij,nj->ni", M, r)
    ei = 0.5 * np.einsum("ni,ni->n", r, Mr)
    w = NF.robust_weight(robust, c, np.sqrt(ei))
    e[has] = w * ei
    H[has] = w[:, None, None] * np.einsum("nki,nkj->nij", J, M @ J)
    b[has] = w[:, None] * np.einsum("nki,nk->ni", J, Mr)
    return e, H, b


def model_error_rows(T, T_lin, idx, factor, robust, c, sp, scv, tp, tn, tcv):
    e = np.zeros(len(idx))
    has = np.nonzero(idx >= 0)[0]
    if len(has) == 0:
        return e
    k = idx[has]
    r = tp[k, :3] - (sp[has, :3] @ T[:3, :3].T + T[:3, 3])
    M = NF.weights(T_lin, factor, sp, scv, tp, tn, tcv, has, k)
    ei = 0.5 * np.einsum("ni,nij,nj->n", r, M, r)
    e[has] = NF.robust_weight(robust, c, np.sqrt(ei)) * ei
    return e


def model_member(kind, s, p, T, T1, corr, factor, robust, c):
    """member p's per-point (e, H, b) at T and error() rows at T1, summed over its entries (one unless submaps: a point has one entry)"""
    cloud = kind.clouds[p]
    n = len(s.srcs[cloud])
    e, H, b, ee = np.zeros(n), np.zeros((n, 6, 6)), np.zeros((n, 6)), np.zeros(n)
    for Pinv, idx, sp, scv, tp, tn, tcv in kind.operands[p](s.srcs[cloud], s.scovs[cloud], corr):
        e1, H1, b1 = model_rows(Pinv @ T, idx, factor, robust, c, sp, scv, tp, tn, tcv)
        e, H, b = e + e1, H + H1, b + b1
        ee += model_error_rows(Pinv @ T1, Pinv @ T, idx, factor, robust, c, sp, scv, tp, tn, tcv)
    return e, H, b, ee


def row_ratios(e, H, b, e0, H0, b0):
    """each row against the model, relative to its own size plus the member's mean row: the residual of a point matched at 0.1 mm is
    carried by FP64 coordinates 300 m from the origin to about 1e-10 of itself only"""
    me, mH = e0.mean(), np.linalg.norm(H0, axis=(1, 2)).mean()
    dH = np.diagonal(H0, axis1=1, axis2=2) + np.diagonal(H0, axis1=1, axis2=2).mean(0)
    re = np.abs(e - e0) / (e0 + me)
    rh = np.linalg.norm(H - H0, axis=(1, 2)) / (np.linalg.norm(H0, axis=(1, 2)) + mH)
    rb = np.abs(b - b0) / np.sqrt(2.0 * (e0 + me)[:, None] * dH)
    return float(rh.max()), float(rb.max()), float(re.max())


def _factors(kind):
    return (0, 1, 2) if kind.plane else (0, 2)


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


# ---- 1, 2, 3, 4: every kind, factor, robust kernel and rejection distance ----
def test_sums_state_and_rows_against_the_model(scene, all_kinds):
    s = scene
    worst = {}
    for kind in all_kinds:
        ctx = kind.ctx
        B = len(kind.clouds)
        T, T1 = s.poses(kind.clouds), s.poses(kind.clouds, 1)
        for factor in _factors(kind):
            for robust, c in ROBUST:
                for max_d in MAX_D:
                    tag = (kind.name, factor, robust, max_d)
                    args = dict(factor=factor, robust=robust, robust_c=c, max_dist_sq=max_d)
                    plain = ctx.linearize_batch(T, **args)
                    corr = ctx.correspondences_batch()
                    err = ctx.error_batch(T1)
                    r = ctx.linearize_batch_points(T, **args)
                    assert _same(plain, (r.H, r.b, r.e, r.num_inliers)), tag
                    assert _same(corr, ctx.correspondences_batch()), tag
                    e1, pe = ctx.error_batch_points(T1)
                    assert np.array_equal(e1, err), tag
                    # the state afterwards: the plain calls give what they gave
                    assert _same(plain, ctx.linearize_batch(T, **args)) and _same(corr, ctx.correspondences_batch()), tag
                    assert np.array_equal(ctx.error_batch(T1), err), tag
                    off = r.offsets
                    assert len(r.point_e) == off[-1] == len(pe)
                    for p in range(B):
                        rows = slice(off[p], off[p + 1])
                        e, H, b = r.point_e[rows], r.point_H[rows], r.point_b[rows]
                        none = corr[p] == NF.NO
                        # 4. zero rows exactly where there is no correspondence; H symmetric
                        assert not e[none].any() and not H[none].any() and not b[none].any() and not pe[rows][none].any(), (tag, p)
                        assert np.array_equal(H, H.transpose(0, 2, 1)), (tag, p)
                        if none.all():
                            continue
                        # 2. every row against the FP64 model
                        e0, H0, b0, ee0 = model_member(kind, s, p, T[p], T1[p], corr[p], factor, robust, c)
                        rat = row_ratios(e, H, b, e0, H0, b0)
                        rerr = float((np.abs(pe[rows] - ee0) / (ee0 + ee0.mean())).max())
                        assert max(rat) <= NF.TIGHT and rerr <= NF.TIGHT, (tag, p, rat, rerr)
                        # 3. the rows add up to the member
                        sums = NF.tight_ratios((H.sum(0), b.sum(0), e.sum()), (r.H[p], r.b[p], r.e[p]))
                        assert max(sums) <= NF.TIGHT and abs(pe[rows].sum() - err[p]) <= NF.TIGHT * err[p], (tag, p, sums)
                        assert (~none).sum() == r.num_inliers[p], (tag, p)
                        w = worst.setdefault(kind.name, [0.0, 0.0])
                        w[0], w[1] = max(w[0], *rat, rerr), max(w[1], *sums)
    print("worst (row vs model, rows summed vs member):", worst)


def test_inactive_members_and_hessians_off(scene, all_kinds):
    s = scene
    for kind in all_kinds:
        ctx = kind.ctx
        B = len(kind.clouds)
        T, T1 = s.poses(kind.clouds), s.poses(kind.clouds, 1)
        full = ctx.linearize_batch_points(T)
        _, full_pe = ctx.error_batch_points(T1)
        active = np.arange(B) % 2 == 1
        r = ctx.linearize_batch_points(T, active=active)
        _, pe = ctx.error_batch_points(T1, active=active)
        e_only = ctx.linearize_batch_points(T, active=active, hessians=False)
        assert e_only.point_H is None and np.array_equal(e_only.point_e, r.point_e), kind.name
        for p in range(B):
            rows = slice(r.offsets[p], r.offsets[p + 1])
            if active[p]:
                assert _same((r.point_e[rows], r.point_Hb42[rows], pe[rows]), (full.point_e[rows], full.point_Hb42[rows], full_pe[rows])), (kind.name, p)
            else:
                assert not r.point_e[rows].any() and not r.point_Hb42[rows].any() and not pe[rows].any(), (kind.name, p)
                assert not r.H[p].any() and r.e[p] == 0


def test_empty_target(scene):
    s = scene
    ctx = _sg().Context(0)
    ctx.set_target(np.zeros((0, 4)), None, np.zeros((0, 4, 4)))
    ctx.build_target_kdtree()
    ctx.set_source_batch(s.srcs, s.scovs)
    T = s.poses(range(len(s.srcs)))
    for factor in (0, 2):
        # rows that held something are cleared: the outputs are given pre-filled
        n = sum(len(x) for x in s.srcs)
        oe, ohb = np.full(n, 7.0), np.full((n, 42), 7.0)
        r = ctx.linearize_batch_points(T, factor=factor, out_e=oe, out_Hb42=ohb)
        assert r.point_e is oe and not oe.any() and not ohb.any() and not r.H.any() and not r.e.any()
        pe = np.full(n, 7.0)
        e, got = ctx.error_batch_points(T, out_e=pe)
        assert got is pe and not pe.any() and not e.any()


# ---- 5. order and independence ----
def test_permuted_cloud_gives_permuted_rows(scene):
    s = scene
    rng = np.random.default_rng(5)
    perm = rng.permutation(len(s.srcs[0]))
    ctx = _kdtree(s)
    ctx2 = _sg().Context(0)
    ctx2.set_target(s.tp, s.tn, s.tcv)
    ctx2.build_target_kdtree()
    ctx2.set_source_batch([s.srcs[0][perm]], [s.scovs[0][perm]])
    T, T1 = s.poses([0]), s.poses([0], 1)
    for factor in (0, 1, 2):
        a = ctx.linearize_batch_points(np.repeat(T, len(s.srcs), 0), factor=factor, robust=1, robust_c=0.05)
        _, ae = ctx.error_batch_points(np.repeat(T1, len(s.srcs), 0))
        b = ctx2.linearize_batch_points(T, factor=factor, robust=1, robust_c=0.05)
        _, be = ctx2.error_batch_points(T1)
        n = len(perm)
        assert np.array_equal(b.point_e, a.point_e[:n][perm]) and np.array_equal(b.point_Hb42, a.point_Hb42[:n][perm]), factor
        assert np.array_equal(be, ae[:n][perm]), factor


def test_member_rows_independent_of_the_batch(scene):
    s = scene
    from small_gicp_b200.synthetic import make_world, sample_cloud

    filler = _p4(sample_cloud(make_world(50_000), 9000, 7) + OFFSET)
    fcov = _random_covs(np.random.default_rng(3), len(filler))
    X, Xc = s.srcs[0], s.scovs[0]
    TX, TX1 = s.poses([0])[0], s.poses([0], 1)[0]
    ref = None
    for B, at in ((1, 0), (17, 9), (4096, 4000)):
        sizes = [(37 * j) % 200 + 1 for j in range(B)]
        starts = np.concatenate([[0], np.cumsum(sizes)]) % (len(filler) - 200)
        srcs = [filler[starts[j] : starts[j] + sizes[j]] for j in range(B)]
        covs = [fcov[starts[j] : starts[j] + sizes[j]] for j in range(B)]
        srcs[at], covs[at] = X, Xc
        ctx = _sg().Context(0)
        ctx.set_target(s.tp, s.tn, s.tcv)
        ctx.build_target_kdtree()
        ctx.set_source_batch(srcs, covs)
        T = np.array([about(NF.box_centre(p), [0.001 * (j % 7), 0.0, -0.002, 0.03, -0.01 * (j % 3), 0.02]) for j, p in enumerate(srcs)])
        T1 = T.copy()
        T[at], T1[at] = TX, TX1
        got = []
        for factor in (0, 1, 2):
            r = ctx.linearize_batch_points(T, factor=factor, robust=2, robust_c=0.01)
            _, pe = ctx.error_batch_points(T1)
            rows = slice(r.offsets[at], r.offsets[at + 1])
            got += [r.H[at], r.b[at], r.e[at], r.point_e[rows].copy(), r.point_Hb42[rows].copy(), pe[rows].copy()]
        if ref is None:
            ref = got
        assert _same(ref, got), B


# ---- 6. device and page-locked outputs ----
def test_device_outputs_equal_host_outputs(scene, all_kinds):
    import torch

    s = scene
    for kind in all_kinds:
        ctx = kind.ctx
        T, T1 = s.poses(kind.clouds), s.poses(kind.clouds, 1)
        n = int(ctx._batch_offsets[-1])
        host = ctx.linearize_batch_points(T, factor=2)
        _, host_pe = ctx.error_batch_points(T1)
        for pin in (False, True):
            if pin:
                de, dhb, dpe = (torch.full(shape, 7.0, dtype=torch.float64).pin_memory() for shape in ((n,), (n, 42), (n,)))
            else:
                de, dhb, dpe = (torch.full(shape, 7.0, dtype=torch.float64, device="cuda") for shape in ((n,), (n, 42), (n,)))
            r = ctx.linearize_batch_points(T, factor=2, out_e=de, out_Hb42=dhb)
            _, got_pe = ctx.error_batch_points(T1, out_e=dpe)
            assert r.point_e is de and got_pe is dpe and r.point_H.shape == (n, 6, 6)
            assert _same((host.H, host.b, host.e), (r.H, r.b, r.e)), (kind.name, pin)
            assert np.array_equal(de.cpu().numpy(), host.point_e) and np.array_equal(dhb.cpu().numpy(), host.point_Hb42), (kind.name, pin)
            assert np.array_equal(dpe.cpu().numpy(), host_pe), (kind.name, pin)


# ---- 7. launch counts ----
def test_launch_counts_equal_the_plain_calls(scene, all_kinds):
    s = scene
    for kind in all_kinds:
        ctx = kind.ctx
        T = s.poses(kind.clouds)
        active = np.arange(len(kind.clouds)) != 1
        counts = []
        for call in (lambda: ctx.linearize_batch(T, active=active), lambda: ctx.linearize_batch_points(T, active=active),
                     lambda: ctx.linearize_batch_points(T, active=active, hessians=False), lambda: ctx.error_batch(T, active=active),
                     lambda: ctx.error_batch_points(T, active=active)):
            before = ctx.kernel_launches
            call()
            counts.append(ctx.kernel_launches - before)
        assert counts[0] == counts[1] == counts[2] and counts[3] == counts[4], (kind.name, counts)


# ---- 8. misuse ----
def test_misuse_fails_with_a_message(scene, all_kinds):
    sg = _sg()
    s = scene
    L = sg.capi._lib()
    dp = C.POINTER(C.c_double)

    def raw_lin(ctx, out44, pe, phb, factor=2, T=None):
        T = np.zeros((max(len(ctx._batch_offsets) - 1, 1), 16)) if T is None else T
        return L.sgb_linearize_batch_points(ctx._h, factor, 0, 1.0, 1, 1.0, T.ctypes.data_as(dp), None, out44, pe, phb)

    def msg(ctx):
        return L.sgb_last_error(ctx._h).decode()

    ctx = _kdtree(s)
    B, n = len(s.srcs), int(ctx._batch_offsets[-1])
    T = np.ascontiguousarray(s.poses(range(B)).transpose(0, 2, 1))
    out44, pe, phb = np.zeros((B, 44)), np.zeros(n), np.zeros((n, 42))
    assert raw_lin(ctx, out44.ctypes.data_as(dp), None, None, T=T) == 1 and "null per-point outputs" in msg(ctx)
    assert raw_lin(ctx, None, pe.ctypes.data_as(dp), None, T=T) == 1 and "null output" in msg(ctx)
    assert L.sgb_linearize_batch_points(ctx._h, 3, 0, 1.0, 1, 1.0, T.ctypes.data_as(dp), None, out44.ctypes.data_as(dp), pe.ctypes.data_as(dp), None) == 1
    assert "invalid factor/robust/rejector kind" in msg(ctx)
    # error() before any linearize, and with a null per-point output
    assert L.sgb_error_batch_points(ctx._h, T.ctypes.data_as(dp), None, out44.ctypes.data_as(dp), pe.ctypes.data_as(dp)) == 1
    assert "no preceding sgb_linearize_batch" in msg(ctx)
    ctx.linearize_batch_points(s.poses(range(B)))
    assert L.sgb_error_batch_points(ctx._h, T.ctypes.data_as(dp), None, out44.ctypes.data_as(dp), None) == 1 and "null per-point output" in msg(ctx)
    assert L.sgb_error_batch_points(ctx._h, T.ctypes.data_as(dp), None, None, pe.ctypes.data_as(dp)) == 1 and "null output" in msg(ctx)
    # no batch: a single source
    single = sg.Context(0)
    single.set_target(s.tp, s.tn, s.tcv)
    single.build_target_kdtree()
    single.set_source(s.srcs[0], s.scovs[0])
    assert L.sgb_linearize_batch_points(single._h, 2, 0, 1.0, 1, 1.0, T.ctypes.data_as(dp), None, out44.ctypes.data_as(dp), pe.ctypes.data_as(dp), None) == 1
    assert "holds no batch" in msg(single)
    assert L.sgb_error_batch_points(single._h, T.ctypes.data_as(dp), None, out44.ctypes.data_as(dp), pe.ctypes.data_as(dp)) == 1 and "holds no batch" in msg(single)
    # point-to-plane against submaps
    sub = next(k for k in all_kinds if k.name == "submaps5")
    with pytest.raises(sg.SgbError, match="sgb_linearize_batch_points: SGB_FACTOR_PLANE_ICP is not available against submaps"):
        sub.ctx.linearize_batch_points(s.poses(sub.clouds), factor=1)
    # Python-side shape checks of given outputs
    with pytest.raises(sg.SgbError, match="shape"):
        ctx.linearize_batch_points(s.poses(range(B)), out_e=np.zeros(n + 1))
