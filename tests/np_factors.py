"""Independent numpy evaluation of the reduced system for a GIVEN correspondence set (third leg of the parity
triangle: oracle <-> numpy <-> GPU).  Follows the reference formulas literally:
  icp_factor.hpp:43-51, plane_icp_factor.hpp:43-55, gicp_factor.hpp:59-70, robust_kernel.hpp:24-27,47,84-89.
Used to make the GPU parity checks immune to legitimate FP32 near-ties / rejection-boundary flips: the GPU sums are
compared against numpy sums over the GPU's own correspondences, and the correspondences themselves are compared
against the oracle's with an explicit near-tie rule."""
import numpy as np

NO = np.uint64(0xFFFFFFFFFFFFFFFF)

# GPU sums against this module evaluated on storage_model() inputs: FP64 algebra on identical operands, only the summation order and
# fma contraction differ.  One point's share of the sums at 1M points is ~1e-6, so a point given wrong operands misses this by far.
TIGHT = 1e-10


def _f32(a):
    return np.asarray(a, dtype=np.float64).astype(np.float32).astype(np.float64)


def finite_rows(pts):
    """rows whose x, y and z are all finite; a row with a NaN or an infinity is inert (include/sgicp_b200.h)"""
    return np.isfinite(np.asarray(pts, dtype=np.float64)[:, :3]).all(1)


def box_centre(pts):
    """the centre every upload (source, target, voxel means) is stored relative to: 0.5 (min + max) per axis in FP64 over the finite
    rows, 0 if there are none"""
    p = np.asarray(pts, dtype=np.float64)[:, :3]
    p = p[finite_rows(p)] if len(p) else p
    if len(p) == 0:
        return np.zeros(3)
    return 0.5 * (p.min(0) + p.max(0))


def stored_points(pts, centre=None):
    """convert_kernel: float32(p - c) with round-to-nearest, read back as that + c in FP64; c = box_centre of the whole upload.  A
    non-finite row is stored as NaN in all three coordinates."""
    c = box_centre(pts) if centre is None else centre
    out = np.array(pts, dtype=np.float64)
    fin = finite_rows(out)
    out[:, :3] = np.where(fin[:, None], _f32(np.where(fin[:, None], out[:, :3], 0.0) - c) + c, np.nan)
    return out


def stored_normals(normals):
    out = np.zeros((len(normals), 4))
    out[:, :3] = _f32(np.asarray(normals)[:, :3])
    return out


def stored_covs(covs):
    """pack_covA / pack_covB: the upper triangle (0,0) (0,1) (0,2) (1,1) (1,2) (2,2) rounded to FP32 and mirrored; the lower triangle
    and the fourth row / column are never read"""
    covs = np.asarray(covs)
    out = np.zeros((len(covs), 4, 4))
    for a, b in ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)):
        out[:, a, b] = out[:, b, a] = _f32(covs[:, a, b])
    return out


def storage_model(src_pts, src_covs, tgt_pts, tgt_normals, tgt_covs, src_centre=None, tgt_centre=None):
    """what the device holds for one (source, target) upload, as FP64 arrays for linearize() / error(); absent features stay None.
    The centres default to the boxes of the arrays given (pass them when the arrays are a subset of what was uploaded)."""
    return (stored_points(src_pts, src_centre), None if src_covs is None else stored_covs(src_covs), stored_points(tgt_pts, tgt_centre),
            None if tgt_normals is None else stored_normals(tgt_normals), None if tgt_covs is None else stored_covs(tgt_covs))


def orthonormal(T):
    """T_target_source.txt carries 6 digits: R^T R differs from I by 1e-6.  The source-frame formulation uses R^T R = I (an
    Isometry3d is a rotation; every pose the optimizers produce is one to 1e-16), so the exact-algebra check needs a true rotation."""
    U, _, Vt = np.linalg.svd(T[:3, :3])
    out = T.copy()
    out[:3, :3] = U @ Vt
    return out


def tight_ratios(got, ref):
    """(H, b, e) against a reference: relative Frobenius norm of H, relative e, and b per component relative to sqrt(2 e H_kk)
    (Cauchy-Schwarz scale of b_k); each is held to TIGHT"""
    (H, b, e), (H0, b0, e0) = got, ref
    rh = np.linalg.norm(H - H0) / np.linalg.norm(H0)
    re = abs(e - e0) / e0
    rb = float((np.abs(b - b0) / np.sqrt(2.0 * e0 * np.diag(H0))).max())
    return float(rh), float(rb), float(re)


def _skew_batch(p):
    S = np.zeros((len(p), 3, 3))
    S[:, 0, 1], S[:, 0, 2] = -p[:, 2], p[:, 1]
    S[:, 1, 0], S[:, 1, 2] = p[:, 2], -p[:, 0]
    S[:, 2, 0], S[:, 2, 1] = -p[:, 1], p[:, 0]
    return S


def robust_weight(kind, c, x):
    if kind == 1:
        ax = np.abs(x)
        return np.where(ax < c, 1.0, c / np.maximum(ax, 1e-300))
    if kind == 2:
        return c / (c + x * x)
    return np.ones_like(x)


def weights(T, factor, src_pts, src_covs, tgt_pts, tgt_normals, tgt_covs, idx, k):
    """per-point 3x3 weight matrix M (identity / diag(n^2) / fused GICP precision at pose T)"""
    n = len(idx)
    if factor == 0:
        return np.tile(np.eye(3), (n, 1, 1))
    if factor == 1:
        nn = tgt_normals[k, :3]
        M = np.zeros((n, 3, 3))
        for a in range(3):
            M[:, a, a] = nn[:, a] ** 2
        return M
    R = T[:3, :3]
    RCR = tgt_covs[k, :3, :3] + R @ src_covs[idx, :3, :3] @ R.T
    return np.linalg.inv(RCR)


def _check_inert(corr, src_pts, tgt_pts):
    """a non-finite source row has no correspondence, and no correspondence names a non-finite target row"""
    corr = np.asarray(corr, dtype=np.uint64)
    hit = corr != NO
    assert not (hit & ~finite_rows(src_pts)).any(), ("non-finite source rows with a correspondence", np.nonzero(hit & ~finite_rows(src_pts))[0][:10])
    k = corr[hit].astype(np.int64)
    assert finite_rows(np.asarray(tgt_pts)[k]).all() if len(k) else True, "a correspondence names a non-finite target row"


def linearize(T, corr, factor, robust, robust_c, src_pts, src_covs, tgt_pts, tgt_normals, tgt_covs):
    """sum over accepted correspondences of J^T M J, J^T M r, 1/2 r^T M r (robust-weighted)"""
    _check_inert(corr, src_pts, tgt_pts)
    idx = np.nonzero(corr != NO)[0]
    if len(idx) == 0:
        return np.zeros((6, 6)), np.zeros(6), 0.0
    k = corr[idx].astype(np.int64)
    R = T[:3, :3]
    p = src_pts[idx, :3]
    q = p @ R.T + T[:3, 3]
    r = tgt_pts[k, :3] - q
    M = weights(T, factor, src_pts, src_covs, tgt_pts, tgt_normals, tgt_covs, idx, k)
    J = np.concatenate([R @ _skew_batch(p), np.tile(-R, (len(idx), 1, 1))], axis=2)  # (n,3,6)
    MJ = M @ J
    Mr = np.einsum("nij,nj->ni", M, r)
    e = 0.5 * np.einsum("ni,ni->n", r, Mr)
    w = robust_weight(robust, robust_c, np.sqrt(e))
    H = np.einsum("n,nki,nkj->ij", w, J, MJ)
    b = np.einsum("n,nki,nk->i", w, J, Mr)
    return H, b, float((w * e).sum())


def error(T_trial, T_lin, corr, factor, robust, robust_c, src_pts, src_covs, tgt_pts, tgt_normals, tgt_covs):
    """Reduction::error: residuals at T_trial, GICP precision frozen at T_lin (gicp_factor.hpp:81-89)"""
    _check_inert(corr, src_pts, tgt_pts)
    idx = np.nonzero(corr != NO)[0]
    if len(idx) == 0:
        return 0.0
    k = corr[idx].astype(np.int64)
    q = src_pts[idx, :3] @ T_trial[:3, :3].T + T_trial[:3, 3]
    r = tgt_pts[k, :3] - q
    M = weights(T_lin, factor, src_pts, src_covs, tgt_pts, tgt_normals, tgt_covs, idx, k)
    e = 0.5 * np.einsum("ni,nij,nj->n", r, M, r)
    return float((robust_weight(robust, robust_c, np.sqrt(e)) * e).sum())


def compare_correspondences(gpu, cpu, tgt_pts, src_pts, T, max_dist_sq=1.0, max_mismatch_frac=2e-3):
    """GPU (FP32 search on centred FP32 coordinates) vs oracle (FP64): identical except
       * near-ties: both candidates' squared distances agree to 1e-5 relative + 1e-7
       * rejection boundary: one side rejected, the other's squared distance within 1e-4 of max_dist_sq.
    Returns the number of differing entries."""
    mism = np.nonzero(gpu != cpu)[0]
    assert len(mism) <= max(3, max_mismatch_frac * len(cpu)), (len(mism), len(cpu))
    q = src_pts[:, :3] @ T[:3, :3].T + T[:3, 3]
    for i in mism:
        dg = np.inf if gpu[i] == NO else ((tgt_pts[int(gpu[i]), :3] - q[i]) ** 2).sum()
        dc = np.inf if cpu[i] == NO else ((tgt_pts[int(cpu[i]), :3] - q[i]) ** 2).sum()
        if np.isinf(dg) or np.isinf(dc):
            fin = dc if np.isinf(dg) else dg
            assert max_dist_sq is not None and abs(fin - max_dist_sq) < 1e-4 * max(1.0, max_dist_sq), (i, dg, dc)
        else:
            assert abs(dg - dc) <= 1e-5 * dc + 1e-7, (i, dg, dc)
    return len(mism)
