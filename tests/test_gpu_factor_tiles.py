"""linearize's per-tile warp sums (factor_reduce_kernel: every tile of 128 points summed across each warp, one running sum per lane)
held to the exact FP64 storage model (np_factors.TIGHT) where the tiling changes: partial tiles and warps, one point either side of a
full one-wave grid of tiles, CTAs with unequal tile counts, a million points, tiles and warps without a single accepted point, and a
cloud 5.8 km from the origin.  Every combination of factor and robust kernel; the sums must also repeat bit for bit and H must be
bitwise symmetric, rejected correspondences must be cleared, and error() after such a linearize must match the model."""
import numpy as np
import pytest

import np_factors as NF
from test_gpu_storage_model import _context, _random_covs, _unit, about, linearize_and_check, point_costs

pytestmark = pytest.mark.gpu

N_TGT = 200_000
N_MAX = 1_000_000
CTAS_PER_SM = 6  # resident CTAs of the linearize factor kernel (80 registers, 80 B of landing zone per point and stage)
FAR = np.array([5800.0, -2300.0, 310.0])  # the far cloud: ~6.2 km from the origin


class Data:
    def __init__(self, offset):
        from small_gicp_b200.synthetic import make_pair

        rng = np.random.default_rng(7)
        tgt, src, T = make_pair(N_TGT, n_source=N_MAX)
        ones = lambda n: np.ones((n, 1))
        self.tp = np.c_[tgt + offset, ones(len(tgt))]
        self.sp = np.c_[src + T[:3, :3].T @ offset, ones(len(src))]
        self.tn = np.c_[_unit(rng, len(tgt)), np.zeros(len(tgt))]
        self.tcv = _random_covs(rng, len(tgt))
        self.scv = _random_covs(rng, len(src))
        self.tgt_model = (NF.stored_points(self.tp), NF.stored_normals(self.tn), NF.stored_covs(self.tcv))
        self.scv_model = NF.stored_covs(self.scv)
        import np_search as NS

        self.search = NS.Target(self.tp)
        self.aligned = T
        self.misaligned = T @ about(NF.box_centre(self.sp), [0.01, -0.012, 0.008, 0.25, -0.2, 0.15])

    def model(self, n, sp=None):
        tp, tn, tcv = self.tgt_model
        return NF.stored_points(self.sp[:n] if sp is None else sp), self.scv_model[:n], tp, tn, tcv


@pytest.fixture(scope="module")
def data():
    return Data(np.array([310.0, -220.0, 45.0]))


@pytest.fixture(scope="module")
def ctx(data):
    c = _context(data.tp, data.tn, data.tcv)
    yield c
    c.close()


def _grid_points():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count * CTAS_PER_SM * 128


def _sizes():
    return [1, 31, 127, 128, 129, "grid-1", "grid+1", "unequal"]


def _n(size):
    g = _grid_points()
    return {"grid-1": g - 1, "grid+1": g + 1, "unequal": 2 * g + 37 * 128 + 5}.get(size, size)


def _all_nine(ctx, d, n, model, poses=None):
    """every factor x robust kernel; the robust kernels' c is the median per-point cost (points on both sides of the knee)"""
    worst = 0.0
    for factor in (0, 1, 2):
        knee = {}
        for robust in (0, 1, 2):
            for j, T in enumerate(poses or (d.misaligned, d.aligned)):
                w, corr = linearize_and_check(ctx, d, n, T, factor, robust, knee.get(j, 1.0), model)
                worst = max(worst, w)
                if robust == 0 and (corr != NF.NO).any():
                    knee[j] = float(np.sqrt(np.median(point_costs(T, corr, factor, model))))
    return worst


@pytest.mark.parametrize("size", _sizes())
def test_tile_sums_match_storage_model(data, ctx, size):
    n = _n(size)
    ctx.set_source(data.sp[:n], data.scv[:n])
    worst = _all_nine(ctx, data, n, data.model(n))
    print(f"worst ratio to the storage model (source {n}): {worst:.2e}")


def test_tile_sums_million_points(data, ctx):
    ctx.set_source(data.sp[:N_MAX], data.scv[:N_MAX])
    worst = _all_nine(ctx, data, N_MAX, data.model(N_MAX), poses=(data.aligned,))
    print(f"worst ratio to the storage model (source {N_MAX}): {worst:.2e}")


def test_sums_repeat_bitwise(data, ctx):
    import small_gicp_b200 as sg

    n = _n("unequal")
    ctx.set_source(data.sp[:n], data.scv[:n])
    for factor in (0, 1, 2):
        for robust in (0, 1, 2):
            kw = dict(factor=factor, robust=robust, robust_c=0.5)
            H0, b0, e0 = ctx.linearize(data.aligned, **kw)
            c0 = ctx.correspondences()
            for _ in range(3):
                H, b, e = ctx.linearize(data.aligned, **kw)
                assert np.array_equal(H, H0) and np.array_equal(b, b0) and e == e0, kw
                assert np.array_equal(H, H.T)
                assert np.array_equal(ctx.correspondences(), c0)
            assert ctx.num_inliers() == int((c0 != sg.NO_CORRESPONDENCE).sum())


def test_all_points_rejected(data, ctx):
    """a pose 50 m off: nothing within the rejector's reach, zero sums and no correspondence left"""
    import small_gicp_b200 as sg

    n = _n("grid+1")
    ctx.set_source(data.sp[:n], data.scv[:n])
    far = data.aligned @ about(NF.box_centre(data.sp[:n]), [0.0, 0.0, 0.0, 50.0, 0.0, 0.0])
    for factor in (0, 1, 2):
        H, b, e = ctx.linearize(far, factor=factor, robust=1, robust_c=0.5)
        assert not H.any() and not b.any() and e == 0.0
        assert ctx.num_inliers() == 0 and (ctx.correspondences() == sg.NO_CORRESPONDENCE).all()
        assert ctx.error(far) == 0.0


def test_tiles_and_warps_without_inliers(data, ctx):
    """source tiles 0 and 2 (all 128 lanes) and warp 1 of tile 5 (32 lanes) moved 50 m away: every lane of them is rejected, the others
    are not, and the sums over the rest match the model"""
    n = 40 * 128 + 77
    sp = data.sp[:n].copy()
    moved = np.r_[0:128, 256:384, 5 * 128 + 32 : 5 * 128 + 64]
    sp[moved, 0] += 50.0
    ctx.set_source(sp, data.scv[:n])

    class View:  # what linearize_and_check reads of the data: the moved source, the same target
        pass

    d = View()
    d.sp, d.tp, d.search = sp, data.tp, data.search
    model = data.model(n, sp=sp)
    worst = _all_nine(ctx, d, n, model, poses=(data.aligned,))
    corr = ctx.correspondences()
    assert (corr[moved] == NF.NO).all() and (corr != NF.NO).sum() > n // 2
    print(f"worst ratio to the storage model (moved tiles): {worst:.2e}")


def test_far_from_origin():
    """a cloud 5.8 km from the origin: the absolute source point enters H_rr and H_rt (skew(p)), so the sums are large and cancel"""
    d = Data(FAR)
    c = _context(d.tp, d.tn, d.tcv)
    try:
        for size in (129, "unequal"):
            n = _n(size)
            c.set_source(d.sp[:n], d.scv[:n])
            worst = _all_nine(c, d, n, d.model(n))
            print(f"worst ratio to the storage model (source {n}, {np.linalg.norm(FAR):.0f} m out): {worst:.2e}")
    finally:
        c.close()
