"""Exact model of the nearest-neighbour search, checked on EVERY query (not a sample).

The device searches with the FP32 query q32 = float32(R s_f + t') in the target-centred frame (t' = R c_s + t - c_t, evaluated in FP64,
centred_translation / centred_query_f32) against the stored FP32 centred target points, then applies the DistanceRejector (d2 > max) to
the FP64 residual of the stored operands.  This module rebuilds q32 and the stored points exactly and holds every returned index to:

  * nearest: D_r <= D_min (1 + BAND), D = exact squared distance between the FP32 query and the FP32 point.  BAND = 32 * 2^-24 covers
    the FP32 rounding of the device's distances (probe fma form, seed and leaf-scan form) and its FP32 box pruning; nothing else is
    allowed, so a query given any other point than a nearest one to a few ulps fails;
  * rejector: an inlier has r2 <= max (1 + 1e-12) (r2 = FP64 residual); NO_CORRESPONDENCE only where the device could not have
    returned an acceptable point: some point of the tie band has r2 > max (1 - 1e-12), or the band lies beyond the FP32 search bound
    (search_bound in sgb_capi.cu); with NullRejector a non-empty target matches every query.

The device contracts the query's FP64 multiply-adds into fmas, so a coordinate whose FP64 value lies within the rounding uncertainty of an
FP32 midpoint may round either way: those queries are accepted if either rounding passes (ambiguous, counted).

batch_knn (sgb_target_batch_knn): the reported d2 is the FP64 squared distance between the stored point and the FP64 centred query (to
1e-12 relative), rows are non-decreasing, the index set is the model's k-set except where its k-th and (k+1)-th distances are within the
band, and rows are padded with UINT64_MAX / DBL_MAX when the target has fewer than k points."""
import numpy as np
from scipy.spatial import cKDTree

from np_factors import NO, _f32, box_centre, finite_rows

BAND = 32 * 2.0**-24
DBL_MAX = np.finfo(np.float64).max


def search_bound(max_dist_sq):
    """sgb::search_bound: the FP32 bound a hair above the rejector's threshold (strict <)"""
    b = np.nextafter(np.float32(max_dist_sq * (1.0 + 4e-6) + 1e-12), np.float32(np.inf))
    return float(min(b, np.finfo(np.float32).max))


class Target:
    """the stored target: FP32 coordinates centred on the box centre (held as FP64) and a cKDTree over them.  Non-finite rows are
    inert (include/sgicp_b200.h): f holds NaN there, the tree holds only the finite rows, and every index the tree returns is mapped
    back to the row it came from (tree.query's answers go through .rows)."""

    def __init__(self, pts):
        pts = np.asarray(pts, dtype=np.float64)[:, :3]
        self.n = len(pts)
        self.centre = box_centre(pts)
        fin = finite_rows(pts)
        self.f = np.where(fin[:, None], _f32(np.where(fin[:, None], pts, 0.0) - self.centre), np.nan)
        self.rows = np.nonzero(fin)[0]
        self.n_finite = len(self.rows)
        self.tree = _RowTree(self.f[self.rows], self.rows, self.n) if self.n_finite else None


class _RowTree:
    """cKDTree over the finite rows whose query returns row indices of the whole target (n where cKDTree reports a missing neighbour)"""

    def __init__(self, f, rows, n):
        self._t, self._rows = cKDTree(f), np.append(rows, n)

    def query(self, x, k=1, **kw):
        d, j = self._t.query(x, k=k, **kw)
        return d, self._rows[j]


def _rows(T, x):
    """R x + t row by row, summed left to right like the device (x: (n, 3))"""
    return np.stack([T[a, 0] * x[:, 0] + T[a, 1] * x[:, 1] + T[a, 2] * x[:, 2] for a in range(3)], axis=1)


def queries(T, src_pts, tgt_centre, src_centre=None):
    """(FP64 centred query, its FP32 rounding, per-coordinate ambiguity mask, the other FP32 rounding) of every stored source point"""
    src = np.asarray(src_pts, dtype=np.float64)[:, :3]
    cs = box_centre(src) if src_centre is None else np.asarray(src_centre, dtype=np.float64)
    sf = _f32(src - cs)
    tp = np.array([T[a, 0] * cs[0] + T[a, 1] * cs[1] + T[a, 2] * cs[2] + T[a, 3] - tgt_centre[a] for a in range(3)])
    q = _rows(T, sf) + tp
    # rounding uncertainty of the FP64 query: 2^-40 relative, or 2^-50 of the sum of the magnitudes that went into it (t' cancels
    # large centres far from the origin; each of its ~6 roundings is at most 2^-53 of that sum)
    scale = np.abs(_rows(np.abs(T), np.abs(sf))) + (np.abs(T[:3, :3]) @ np.abs(cs) + np.abs(T[:3, 3]) + np.abs(tgt_centre))[None]
    eps = np.maximum(2.0**-40 * np.abs(q), 2.0**-50 * scale)
    q32 = _f32(q)
    # the FP32 midpoint next to q on the side away from q32
    other = np.where(q >= q32, np.nextafter(q32.astype(np.float32), np.float32(np.inf)), np.nextafter(q32.astype(np.float32), np.float32(-np.inf))).astype(np.float64)
    # (where the FP32 spacing itself is below the uncertainty -- coordinates within ~1e-13 m of 0 -- either rounding moves the query by
    # less than that, which the band absorbs)
    amb = (np.abs(q - 0.5 * (q32 + other)) <= eps) & (np.abs(other - q32) > 2.0 * eps)
    return q, q32, amb, other


def _d2(a, b):
    return ((a - b) ** 2).sum(-1)


def _band_points(tgt, q32, dmin):
    """indices of every target point within the tie band of one query"""
    lim = dmin * (1.0 + BAND)
    k = min(8, tgt.n_finite)
    while True:
        d, j = tgt.tree.query(q32, k=k)
        d, j = np.atleast_1d(d) ** 2, np.atleast_1d(j)
        if d[-1] > lim or k == tgt.n_finite:
            return j[d <= lim * (1 + 1e-15)]
        k = min(4 * k, tgt.n_finite)


def _check_nn(tgt, corr, q, q32, max_d):
    """per query: 0 = fine, 1 = fine at the rejection boundary, -1 = wrong; and the band ratio of each returned point"""
    n = len(q)
    _, j = tgt.tree.query(q32, k=1, workers=-1)
    dmin = _d2(q32, tgt.f[j])  # exact squared distance of the nearest point (cKDTree's own is the square of a square root)
    status = np.full(n, -1, dtype=np.int64)
    ratio = np.zeros(n)
    hit = corr != NO
    h = np.nonzero(hit)[0]
    r = corr[h].astype(np.int64)
    valid = r < tgt.n
    h, r = h[valid], r[valid]
    dr = _d2(q32[h], tgt.f[r])
    ok = dr <= dmin[h] * (1.0 + BAND)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio[h] = np.where(dmin[h] > 0, (dr / dmin[h] - 1.0) / BAND, np.where(dr > 0, np.inf, 0.0))
    if max_d is not None:
        ok &= _d2(tgt.f[r], q[h]) <= max_d * (1.0 + 1e-12)
    status[h[ok]] = 0
    miss = np.nonzero(~hit)[0]
    if max_d is None:
        return status, ratio  # NullRejector: every query of a non-empty target matches
    # NO_CORRESPONDENCE: the band beyond the FP32 search bound, or a point of the band that the rejector refuses (the nearest point
    # itself decides almost every case; the band is enumerated only where it does not)
    r2n = _d2(tgt.f[j[miss]], q[miss])
    beyond = dmin[miss] * (1.0 + BAND) >= search_bound(max_d)
    refused = r2n > max_d * (1.0 - 1e-12)
    status[miss[beyond | refused]] = np.where(r2n[beyond | refused] <= max_d, 1, 0)
    for i in miss[~(beyond | refused)]:
        r2 = _d2(tgt.f[_band_points(tgt, q32[i], dmin[i])], q[i][None])
        if (r2 > max_d * (1.0 - 1e-12)).any():
            status[i] = 1
    return status, ratio


class Report:
    def __init__(self):
        self.queries = self.ambiguous = self.other_rounding = self.boundary = 0
        self.worst_band = 0.0

    def __str__(self):
        return (f"{self.queries} queries, worst band ratio {self.worst_band:.3g}, {self.ambiguous} ambiguous FP32 queries "
                f"({self.other_rounding} right only with the other rounding), {self.boundary} rejection-boundary cases")


REPORT = Report()  # totals over the whole process (the tests print them)


def check_correspondences(corr, T, src_pts, tgt, max_dist_sq=1.0, src_centre=None, report=REPORT):
    """every query of one linearize against the model; tgt: a Target, max_dist_sq None = NullRejector.  Raises AssertionError naming
    the first wrong queries.  Returns the number of queries checked."""
    corr = np.asarray(corr, dtype=np.uint64)
    n = len(corr)
    assert len(src_pts) == n
    report.queries += n
    if n == 0:
        return 0
    fin = finite_rows(src_pts)
    assert (corr[~fin] == NO).all(), ("non-finite queries with a correspondence", np.nonzero(~fin & (corr != NO))[0][:10])
    if tgt.n_finite == 0:
        assert (corr == NO).all()
        return n
    cs = box_centre(src_pts) if src_centre is None else src_centre
    src = np.where(fin[:, None], np.asarray(src_pts, dtype=np.float64)[:, :3], cs)  # (checked above; the finite rows are the queries)
    q, q32, amb, other = queries(T, src, tgt.centre, cs)
    status, ratio = _check_nn(tgt, corr, q, q32, max_dist_sq)
    status[~fin] = 0
    ratio[~fin] = 0.0
    amb[~fin] = False
    bad = np.nonzero(status < 0)[0]
    amb_any = amb.any(1)
    report.ambiguous += int(amb_any.sum())
    still = []
    for i in bad:
        if not amb_any[i]:
            still.append(i)
            continue
        # every combination of the ambiguous coordinates' two roundings
        axes = np.nonzero(amb[i])[0]
        passed = False
        for mask in range(1, 1 << len(axes)):
            alt = q32[i].copy()
            for b, a in enumerate(axes):
                if mask >> b & 1:
                    alt[a] = other[i, a]
            s, rr = _check_nn(tgt, corr[i : i + 1], q[i : i + 1], alt[None], max_dist_sq)
            if s[0] >= 0:
                passed, status[i], ratio[i] = True, s[0], rr[0]
                report.other_rounding += 1
                break
        if not passed:
            still.append(i)
    if still:
        i = still[0]
        dmin = tgt.tree.query(q32[i])[0] ** 2
        got = "NO" if corr[i] == NO else f"{int(corr[i])} at d2 {_d2(q32[i], tgt.f[int(corr[i])]) if corr[i] < tgt.n else 'out of range'}"
        raise AssertionError(f"{len(still)} of {n} queries wrong; first: query {i} got {got}, nearest d2 {dmin}, max_dist_sq {max_dist_sq}, "
                             f"queries {still[:10]}")
    report.boundary += int((status == 1).sum())
    fin = ratio[np.isfinite(ratio)]
    if len(fin):
        report.worst_band = max(report.worst_band, float(fin.max()))
    return n


def check_knn(idx, d2, queries_xyz, k, tgt, report=REPORT):
    """every row of one sgb_target_batch_knn call against the model"""
    idx, d2 = np.asarray(idx, dtype=np.uint64), np.asarray(d2, dtype=np.float64)
    qw = np.asarray(queries_xyz, dtype=np.float64)[:, :3]
    n = len(qw)
    assert idx.shape == (n, k) and d2.shape == (n, k)
    report.queries += n
    # a non-finite query has no neighbours: its row is all padding
    fin = finite_rows(qw)
    assert (idx[~fin] == NO).all() and (d2[~fin] == DBL_MAX).all(), ("non-finite queries with neighbours", np.nonzero(~fin & (idx[:, 0] != NO))[0][:10])
    idx, d2, qw = idx[fin], d2[fin], qw[fin]
    n = len(qw)
    m = min(k, tgt.n_finite)
    # padding
    assert (idx[:, m:] == NO).all() and (d2[:, m:] == DBL_MAX).all(), "padding"
    if m == 0 or n == 0:
        return n
    assert (idx[:, :m] < tgt.n).all(), "index out of range or missing"
    qc = qw - tgt.centre  # the device's FP64 centred query
    j = idx[:, :m].astype(np.int64)
    want = _d2(tgt.f[j], qc[:, None, :])
    assert np.all(np.abs(d2[:, :m] - want) <= 1e-12 * want), ("reported d2", np.nonzero(np.abs(d2[:, :m] - want) > 1e-12 * want)[0][:10])
    assert np.all(np.diff(d2, axis=1) >= 0), ("rows not ascending", np.nonzero((np.diff(d2, axis=1) < 0).any(1))[0][:10])
    assert all(len(set(row)) == m for row in j.tolist()), "duplicate index in a row"
    # the model's FP64 k-set: k + 8 candidates re-ranked by the exact FP64 distance
    kk = min(tgt.n_finite, m + 8)
    _, cand = tgt.tree.query(qc, k=kk, workers=-1)
    cand = cand.reshape(n, kk)
    cd = _d2(tgt.f[cand], qc[:, None, :])
    order = np.argsort(cd, axis=1, kind="stable")
    cd = np.take_along_axis(cd, order, 1)
    cand = np.take_along_axis(cand, order, 1)
    dk = cd[:, m - 1]
    # every reported point within the band of the k-th distance, and every point clearly nearer than the k-th reported
    assert np.all(want <= dk[:, None] * (1.0 + BAND) + 1e-300), ("k-set", np.nonzero((want > dk[:, None] * (1.0 + BAND)).any(1))[0][:10])
    strict = cd[:, :m] < dk[:, None] / (1.0 + BAND)
    for i in np.nonzero(strict.any(1))[0]:
        need = set(cand[i, :m][strict[i]].tolist())
        assert need <= set(j[i].tolist()), ("k-set misses a nearer point", i)
    pos = dk > 0
    if pos.any():
        report.worst_band = max(report.worst_band, float(((want[pos] / dk[pos, None] - 1.0) / BAND).max()))
    return n
