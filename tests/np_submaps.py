"""FP64 models of submap members (sgb_source_set_submaps): a source at pose T (source -> common frame) against the union of several maps,
map k placed by the rigid pose P_k (map -> common frame).

The device never places a map.  It carries the member's pose into each map's stored frame, T_k = P_k^-1 T, and works there:
  * sums: a point's share of H | b | e is np_factors.linearize / error at T_k against the UN-placed map of its correspondence
    (union_linearize / union_error) -- equal to the factor at T against the placed union (placed_union) because r^T M r and its
    derivatives by the right perturbation of T do not change under P_k (test_np_submaps.py), except for point-to-plane;
  * search: each entry is searched with its own FP32 query, float32 of the FP64 query at T_k centred on map k, against map k's stored FP32
    points (np_search), and the entry with the smallest FP32 squared distance wins, the earlier one at an exact tie.  check_union holds
    every returned (entry, index) to that: its distance within np_search.BAND of the smallest over all entries, the rejector applied to
    the FP64 residual in the entry's frame.
Correspondences are (entry << 32) | index within that entry's map, as sgb_correspondences_batch reports them."""
import numpy as np

import np_factors as NF
import np_search as NS

NO = NF.NO
LOW = np.uint64(0xFFFFFFFF)


def inverse(P):
    out = np.eye(4)
    out[:3, :3] = P[:3, :3].T
    out[:3, 3] = -P[:3, :3].T @ P[:3, 3]
    return out


def relative(P, T):
    """the member's pose in the stored frame of a map placed by P"""
    return inverse(P) @ T


def split(corr, n_entries):
    """per entry: the correspondences that lie in it (index within its map), NO elsewhere"""
    corr = np.asarray(corr, dtype=np.uint64)
    hit = corr != NO
    entry = np.where(hit, corr >> np.uint64(32), np.uint64(n_entries))
    return [np.where(entry == np.uint64(e), corr & LOW, NO) for e in range(n_entries)]


def union_linearize(T, corr, factor, robust, robust_c, src_pts, src_covs, maps, poses):
    """maps: per entry (points, normals | None, covs | None) as stored; the sum over the entries of the factor at P_k^-1 T on map k"""
    H, b, e = np.zeros((6, 6)), np.zeros(6), 0.0
    for (pts, normals, covs), P, ck in zip(maps, poses, split(corr, len(maps))):
        h, g, f = NF.linearize(relative(P, T), ck, factor, robust, robust_c, src_pts, src_covs, pts, normals, covs)
        H, b, e = H + h, b + g, e + f
    return H, b, e


def union_error(T_trial, T_lin, corr, factor, robust, robust_c, src_pts, src_covs, maps, poses):
    return sum(NF.error(relative(P, T_trial), relative(P, T_lin), ck, factor, robust, robust_c, src_pts, src_covs, pts, normals, covs)
               for (pts, normals, covs), P, ck in zip(maps, poses, split(corr, len(maps))))


def placed_union(maps, poses):
    """ONE cloud: every map's points, normals and covariances carried into the common frame (P q, R n, R C R^T), and the first
    position of each entry in it"""
    pts, normals, covs, first = [], [], [], [0]
    for (p, n, c), P in zip(maps, poses):
        R4 = np.eye(4)
        R4[:3, :3] = P[:3, :3]
        q = np.ones((len(p), 4))
        q[:, :3] = p[:, :3] @ P[:3, :3].T + P[:3, 3]
        pts.append(q)
        normals.append(None if n is None else n @ R4.T)
        covs.append(None if c is None else R4 @ c @ R4.T)
        first.append(first[-1] + len(p))
    cat = lambda xs, shape: None if any(x is None for x in xs) else (np.concatenate(xs) if xs else np.zeros(shape))
    return cat(pts, (0, 4)), cat(normals, (0, 4)), cat(covs, (0, 4, 4)), np.array(first)


def to_union(corr, first):
    """(entry, index) correspondences as positions in placed_union's cloud"""
    corr = np.asarray(corr, dtype=np.uint64)
    hit = corr != NO
    e = np.where(hit, corr >> np.uint64(32), np.uint64(0)).astype(np.int64)
    return np.where(hit, (first[e] + (corr & LOW).astype(np.int64)).astype(np.uint64), NO)


def _d2(a, b):
    return ((a - b) ** 2).sum(-1)


def _judge(c, q, q32, targets, max_d):
    """one query against the model, given its FP64 and FP32 query per entry: 0 fine, 1 fine at the rejection boundary, -1 wrong"""
    dmin = np.full(len(targets), np.inf)
    near = [None] * len(targets)
    for e, t in enumerate(targets):
        if t.n:
            _, j = t.tree.query(q32[e])
            dmin[e], near[e] = _d2(q32[e], t.f[j]), j
    best = dmin.min()
    if c != NO:
        e, r = int(c >> np.uint64(32)), int(c & LOW)
        if e >= len(targets) or r >= targets[e].n:
            return -1
        ok = _d2(q32[e], targets[e].f[r]) <= best * (1.0 + NS.BAND)
        if max_d is not None:
            ok = ok and _d2(targets[e].f[r], q[e]) <= max_d * (1.0 + 1e-12)
        return 0 if ok else -1
    if not np.isfinite(best):
        return 0  # nothing to match
    if max_d is None:
        return -1  # NullRejector: a non-empty union matches every query
    if best * (1.0 + NS.BAND) >= NS.search_bound(max_d):
        return 0
    # some point of the tie band, in whichever entry, that the rejector refuses
    for e, t in enumerate(targets):
        if dmin[e] <= best * (1.0 + NS.BAND):
            r2 = _d2(t.f[NS._band_points(t, q32[e], dmin[e])], q[e][None])
            if (r2 > max_d * (1.0 - 1e-12)).any():
                return 1
    return -1


def check_union(corr, T, src_pts, targets, poses, max_dist_sq=1.0, src_centre=None, report=NS.REPORT):
    """every correspondence of one member; targets: one np_search.Target per entry (the same object may repeat).  Raises
    AssertionError naming the first wrong queries; returns the number of queries checked."""
    corr = np.asarray(corr, dtype=np.uint64)
    n = len(corr)
    assert len(src_pts) == n
    report.queries += n
    if n == 0:
        return 0
    E = len(targets)
    if E == 0:
        assert (corr == NO).all(), "an empty list gives no correspondences"
        return n
    Q = [NS.queries(relative(P, T), src_pts, t.centre, src_centre) for t, P in zip(targets, poses)]
    q = np.stack([x[0] for x in Q], 1)      # (n, E, 3)
    q32 = np.stack([x[1] for x in Q], 1)
    amb = np.stack([x[2] for x in Q], 1)
    other = np.stack([x[3] for x in Q], 1)
    # vectorised pass for the overwhelming majority: the returned point within the band of the smallest distance over all entries
    dmin = np.full((n, E), np.inf)
    for e, t in enumerate(targets):
        if t.n:
            _, j = t.tree.query(q32[:, e], workers=-1)
            dmin[:, e] = _d2(q32[:, e], t.f[j])
    best = dmin.min(1)
    done = np.zeros(n, dtype=bool)
    hit = np.nonzero(corr != NO)[0]
    he, hr = (corr[hit] >> np.uint64(32)).astype(np.int64), (corr[hit] & LOW).astype(np.int64)
    for e, t in enumerate(targets):
        s = (he == e) & (hr < t.n)
        i, r = hit[s], hr[s]
        ok = _d2(q32[i, e], t.f[r]) <= best[i] * (1.0 + NS.BAND)
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.where(best[i] > 0, (_d2(q32[i, e], t.f[r]) / best[i] - 1.0) / NS.BAND, 0.0)
        if max_dist_sq is not None:
            ok &= _d2(t.f[r], q[i, e]) <= max_dist_sq * (1.0 + 1e-12)
        done[i[ok]] = True
        if ok.any():
            report.worst_band = max(report.worst_band, float(ratio[ok].max()))
    # the rest one by one: misses, and hits that only pass with the other rounding of an ambiguous FP32 query coordinate
    still = []
    report.ambiguous += int(amb.any((1, 2)).sum())
    for i in np.nonzero(~done)[0]:
        s = _judge(corr[i], q[i], q32[i], targets, max_dist_sq)
        if s < 0 and amb[i].any():
            where = np.argwhere(amb[i])
            for mask in range(1, 1 << min(len(where), 8)):
                alt = q32[i].copy()
                for b, (e, a) in enumerate(where[:8]):
                    if mask >> b & 1:
                        alt[e, a] = other[i, e, a]
                s = _judge(corr[i], q[i], alt, targets, max_dist_sq)
                if s >= 0:
                    report.other_rounding += 1
                    break
        if s < 0:
            still.append(int(i))
        report.boundary += int(s == 1)
    if still:
        i = still[0]
        got = "NO" if corr[i] == NO else f"entry {int(corr[i] >> np.uint64(32))} index {int(corr[i] & LOW)}"
        raise AssertionError(f"{len(still)} of {n} queries wrong; first: query {i} got {got}, nearest d2 per entry {dmin[i]}, max_dist_sq {max_dist_sq}, "
                             f"queries {still[:10]}")
    return n
