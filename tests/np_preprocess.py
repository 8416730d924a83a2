"""Exact FP64 models of the device's per-cloud preparation and of the VGICP correspondence search, in numpy.

  voxelgrid_model       voxel_keys_kernel + stable radix sort + voxel_means_kernel (sgb_voxelgrid_sampling): bit-identical
  voxelmap_model        the same grouping + voxel_stats_kernel (sgb_target_build_voxelmap): bit-identical means and covariances
  features_model        features_kernel (sgb_estimate_features): exact neighbours, FP64 covariance, LAPACK eigenvectors
  vgicp_correspondences linearize_vox_kernel's probe of 1 / 7 / 27 voxels, on the stored (centred FP32) voxel means

The device sums each voxel in ascending original index, one point after the other.  numpy's add.reduce / reduceat sum pairwise, so
the models add the points of all voxels in lockstep (one numpy addition per position within a voxel; voxels of more than 256 points
one at a time with cumsum), which is the same sequence of FP64 additions, and the result is bit for bit the device's."""
import numpy as np
from scipy.spatial import cKDTree

NO = np.uint64(0xFFFFFFFFFFFFFFFF)
COORD_BITS = 21
COORD_OFFSET = 1 << (COORD_BITS - 1)
COORD_MASK = (1 << COORD_BITS) - 1


def voxel_coords(points, leaf):
    """integer voxel coordinates floor(p * (1 / leaf)): a multiply by the FP64 reciprocal, as the kernels and the reference compute it.
    A row with a non-finite coordinate (or one whose scaled coordinate overflows) gets coordinates outside the 21-bit range, so that
    coord_keys drops it, as the reference's fast_floor (INT_MIN) does; numpy's cast of NaN to int64 is not relied on."""
    c = np.floor(np.asarray(points, dtype=np.float64)[:, :3] * (1.0 / leaf))
    fin = np.isfinite(c).all(1)
    out = np.where(fin[:, None], np.clip(np.where(fin[:, None], c, 0.0), -(1 << 40), 1 << 40), 0.0).astype(np.int64)
    out[~fin] = COORD_MASK + 1
    return out


def coord_keys(c):
    """63-bit key of integer voxel coordinates (x in bits 0-20, y 21-41, z 42-62); NO where a coordinate leaves the 21-bit range"""
    s = c + COORD_OFFSET
    ok = np.all((s >= 0) & (s <= COORD_MASK), axis=1)
    s = np.where(ok[:, None], s, 0).astype(np.uint64)
    keys = s[:, 0] | (s[:, 1] << np.uint64(COORD_BITS)) | (s[:, 2] << np.uint64(2 * COORD_BITS))
    return np.where(ok, keys, NO)


def _segments(points, leaf):
    """(order, starts, counts, keys of the voxels): points of each voxel in ascending original index, voxels in ascending key"""
    keys = coord_keys(voxel_coords(points, leaf))
    order = np.argsort(keys, kind="stable")
    order = order[keys[order] != NO]
    sk = keys[order]
    heads = np.ones(len(sk), dtype=bool)
    heads[1:] = sk[1:] != sk[:-1]
    starts = np.nonzero(heads)[0]
    counts = np.diff(np.r_[starts, len(sk)])
    return order, starts, counts, sk[starts]


def _sequential_means(values, order, starts, counts):
    """per segment: ((v[0] + v[1]) + v[2]) + ... in segment order, divided by the count (FP64, as the kernels do it)"""
    sums = np.zeros((len(starts), values.shape[1]))
    small = counts <= 256
    for j in range(int(counts[small].max()) if small.any() else 0):
        live = np.nonzero(small & (counts > j))[0]
        sums[live] += values[order[starts[live] + j]]
    for s in np.nonzero(~small)[0]:  # large voxels one at a time: cumsum (add.accumulate) adds strictly left to right
        sums[s] = np.cumsum(values[order[starts[s]:starts[s] + counts[s]]], axis=0)[-1]
    return sums / counts[:, None].astype(np.float64)


def voxelgrid_model(points, leaf):
    """sgb_voxelgrid_sampling: (M, 4) voxel means (w = 1), voxels in ascending key order"""
    p = np.asarray(points, dtype=np.float64)[:, :3]
    order, starts, counts, _ = _segments(p, leaf)
    out = np.ones((len(starts), 4))
    if len(starts):
        out[:, :3] = _sequential_means(p, order, starts, counts)
    return out


def voxelmap_model(points, covs, leaf):
    """sgb_target_build_voxelmap: (coords (M,3) int, means (M,4), covs (M,4,4) or None, counts (M,)), voxel id = row, ascending key"""
    p = np.asarray(points, dtype=np.float64)[:, :3]
    order, starts, counts, keys = _segments(p, leaf)
    m = len(starts)
    coords = np.stack([(keys >> np.uint64(s)) & np.uint64(COORD_MASK) for s in (0, COORD_BITS, 2 * COORD_BITS)], axis=1).astype(np.int64) - COORD_OFFSET
    means = np.ones((m, 4))
    cv = None
    if m:
        means[:, :3] = _sequential_means(p, order, starts, counts)
    if covs is not None:
        cv = np.zeros((m, 4, 4))
        if m:
            cv = _sequential_means(np.asarray(covs, dtype=np.float64).reshape(-1, 16), order, starts, counts).reshape(m, 4, 4)
    return coords, means, cv, counts


class Features:
    """features_model's result: normals (N,4), covs (N,4,4), eigenvalues (N,3) ascending, eigenvectors (N,3,3) in columns, the squared
    distances of the k + 1 nearest neighbours (N, k+1; inf where the cloud has fewer points) and the neighbour count used"""


def features_model(points, k):
    """estimate_normals_covariances (normal_estimation.hpp) as features_kernel computes it, in FP64 on the caller's coordinates: the k
    nearest points (the query included) by an exact search, their covariance about its mean, the eigenvector of the smallest
    eigenvalue (LAPACK) flipped so that p . n <= 0, covariance I - 0.999 v v^T.  Fewer than 5 neighbours: zero normal, identity."""
    p = np.asarray(points, dtype=np.float64)[:, :3]
    n = len(p)
    kk = min(k + 1, n)
    d, idx = cKDTree(p).query(p, k=kk, workers=-1)
    d, idx = d.reshape(n, kk), idx.reshape(n, kk)
    m = min(k, n)
    X = p[idx[:, :m]]
    X = X - X.mean(axis=1, keepdims=True)
    C = np.einsum("nki,nkj->nij", X, X) / m
    lam, E = np.linalg.eigh(C)
    v = E[:, :, 0]
    sgn = np.where(np.einsum("ni,ni->n", p, v) > 0.0, -1.0, 1.0)
    f = Features()
    f.count = m
    f.eigenvalues, f.eigenvectors = lam, E
    f.d2 = np.full((n, k + 1), np.inf)
    f.d2[:, :kk] = d * d
    f.normals = np.zeros((n, 4))
    f.covs = np.zeros((n, 4, 4))
    f.covs[:, :3, :3] = np.eye(3)
    if m >= 5:
        f.normals[:, :3] = sgn[:, None] * v
        f.covs[:, :3, :3] = np.eye(3) - (1.0 - 1e-3) * v[:, :, None] * v[:, None, :]
    return f


def vox_offsets(num):
    """vox_offset of sgb_kernels.cu: 27 lexicographic (x slowest), else centre, +x, +y, +z, -x, -y, -z (first `num` of them)"""
    if num == 27:
        return [(i, j, k) for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1)]
    return [(0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (-1, 0, 0), (0, -1, 0), (0, 0, -1)][:num]


def vgicp_correspondences(queries, leaf, num_offsets, vox_coords, stored_means, max_dist_sq):
    """The voxel each query (FP64, target frame) is matched to: the voxels at the probe offsets around floor(q / leaf) in the kernel's
    order, the nearest STORED mean wins (strict <: on a tie the first found), then the distance rejector (d2 > max rejects).
    vox_coords must be in ascending key order (voxelmap_model's, the device's voxel ids).  Returns (ids as uint64 / NO, clear):
    clear is False where the device may legitimately differ -- the query within 1e-6 m of a voxel face, two candidate distances within
    compare_correspondences' tie rule, or the best distance that close to max_dist_sq."""
    q = np.asarray(queries, dtype=np.float64)[:, :3]
    keys = coord_keys(np.asarray(vox_coords, dtype=np.int64))
    assert np.all(keys[1:] > keys[:-1])
    base = voxel_coords(q, leaf)
    n = len(q)
    best = np.full(n, np.inf)
    second = np.full(n, np.inf)
    ids = np.full(n, -1, dtype=np.int64)
    for off in vox_offsets(num_offsets):
        ck = coord_keys(base + np.array(off))
        pos = np.minimum(np.searchsorted(keys, ck), len(keys) - 1)
        hit = (ck != NO) & (keys[pos] == ck)
        d = np.full(n, np.inf)
        d[hit] = ((stored_means[pos[hit], :3] - q[hit]) ** 2).sum(1)
        closer = d < best
        second = np.where(closer, best, np.minimum(second, d))
        ids = np.where(closer, pos, ids)
        best = np.where(closer, d, best)
    rejected = best > max_dist_sq
    out = np.where((ids < 0) | rejected, NO, ids.astype(np.uint64))
    frac = q * (1.0 / leaf)
    face = np.abs(frac - np.round(frac)).min(axis=1) * leaf < 1e-6
    with np.errstate(invalid="ignore"):  # inf - inf where fewer than two voxels were found
        tie = np.isfinite(second) & (np.abs(second - best) <= 1e-5 * best + 1e-7)
        edge = np.isfinite(best) & (np.abs(best - max_dist_sq) < 1e-4 * max(1.0, max_dist_sq))
    return out, ~(face | tie | edge)
