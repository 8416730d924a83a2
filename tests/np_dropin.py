"""Call-by-call check of the drop-in reduction: every linearize() and error() the reference's Registration<> makes on
include/small_gicp/registration/reduction_cuda.hpp (or on its own ParallelReductionOMP), as logged by href_align_log
(tests/host_ref/host_ref_capi.cpp), against the FP64 models.

For each logged call:
  * correspondences: a kd-tree target against the exact search model of np_search (the target as sgb_target_set_points stores it);
    a voxel map against the probe of its flat_voxels (coordinates in any order and range, stored means), with vgicp_correspondences'
    tie rule;
  * target_index: the original point index (kd-tree) or the flat_voxels position << 32 (voxel map, calc_index(voxel, 0) of
    incremental_voxelmap.hpp), SIZE_MAX for outliers; the factor vector shows them after every linearize (sync_every_linearize), or is
    left as Registration::align constructed it except factor 0's source_index (the drop-in's "linearized" mark);
  * H | b | e against np_factors.linearize over that call's own correspondences, within `tol` (np_factors.TIGHT on the storage model);
  * error() against np_factors.error at its trial pose, the precision frozen at the preceding linearize pose;
  * num_inliers of the align() result: the inliers of its last linearize (0 when nothing was synced).
compare_arms() holds every CUDA call to the FP64 reference on FP64 inputs at its own pose and correspondences within 2e-5 (DESIGN §2;
the OMP arm is that reference), and the CUDA log to the OMP log: the same call sequence until their correspondences first differ, and
that first difference only inside the tie band.

A failed check raises AssertionError naming the call ("align a, call c (linearize)") and the quantity."""
import os
from dataclasses import dataclass, field

import numpy as np
from scipy.spatial import cKDTree

import np_factors as NF
import np_search as NS
from np_preprocess import vox_offsets

NO = NF.NO
STRUCTURES = {0: "KdTree", 1: "UnsafeKdTree", 2: "KdTreeBuilderOMP", 3: "GaussianVoxelMap"}
ORACLE_TOL = 2e-5  # DESIGN §2: GPU against the FP64 reference on FP64 inputs
CALL = 61  # doubles per call record
ALIGN = 21  # doubles per align record


@dataclass
class Call:
    kind: int  # 0 linearize, 1 error
    align: int
    T: np.ndarray
    H: np.ndarray
    b: np.ndarray
    e: float
    source_index: np.ndarray = None  # linearize only: the factor vector after the call
    target_index: np.ndarray = None
    corr: np.ndarray = None  # the correspondences the reduction used (the context's, read into a copy)

    @property
    def name(self):
        return "linearize" if self.kind == 0 else "error"


@dataclass
class Log:
    calls: list
    aligns: list  # (structure, T, iterations, converged, num_inliers, error)
    vox_coords: np.ndarray
    vox_means: np.ndarray
    vox_covs: np.ndarray
    n_src: int = 0
    extra: dict = field(default_factory=dict)


def parse(calls, idx, aligns, vox_coords, vox_means, vox_covs, n_src):
    calls = np.asarray(calls, dtype=np.float64).reshape(-1, CALL)
    out, pos = [], 0
    for r in calls:
        c = Call(int(r[0]), int(r[1]), r[2:18].reshape(4, 4).copy(), r[18:54].reshape(6, 6).copy(), r[54:60].copy(), float(r[60]))
        if c.kind == 0:
            c.source_index, c.target_index, c.corr = (idx[pos + k * n_src : pos + (k + 1) * n_src].copy() for k in range(3))
            pos += 3 * n_src
        out.append(c)
    assert pos == len(idx)
    al = [(int(a[0]), a[1:17].reshape(4, 4).copy(), int(a[17]), bool(a[18]), int(a[19]), float(a[20])) for a in np.asarray(aligns).reshape(-1, ALIGN)]
    return Log(out, al, np.asarray(vox_coords).reshape(-1, 3), np.asarray(vox_means).reshape(-1, 4), np.asarray(vox_covs).reshape(-1, 4, 4), n_src)


@dataclass
class Problem:
    """what the reduction was given: source and target exactly as the cloud type holds them (FP64 arrays), the factor setting, and the
    voxel map's search parameters"""
    src_pts: np.ndarray
    src_covs: np.ndarray
    tgt_pts: np.ndarray
    tgt_normals: np.ndarray
    tgt_covs: np.ndarray
    factor: int
    robust: int
    robust_c: float
    max_dist_sq: float  # None: NullRejector
    leaf: float = 1.0
    offsets: int = 1
    sync: bool = True


# ---------------------------------------------------------------- voxel probe on flat_voxels
def voxel_correspondences(q, leaf, num_offsets, coords, means, max_dist_sq):
    """the flat_voxels position each query q (FP64, target frame) is matched to: the voxels at the probe offsets around floor(q / leaf),
    nearest mean wins (strict <, first found on a tie), then the rejector.  Coordinates may be in any order and any int32 range (a
    host-filled table).  Returns (ids, clear) with vgicp_correspondences' rule for `clear`."""
    q = np.asarray(q, dtype=np.float64)[:, :3]
    n = len(q)
    base = np.floor(q * (1.0 / leaf)).astype(np.int64)
    table = {tuple(c): i for i, c in enumerate(np.asarray(coords, dtype=np.int64).tolist())}
    ub, inv = np.unique(base, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    best, second = np.full(n, np.inf), np.full(n, np.inf)
    ids = np.full(n, -1, dtype=np.int64)
    for off in vox_offsets(num_offsets):
        found = np.array([table.get((int(x) + off[0], int(y) + off[1], int(z) + off[2]), -1) for x, y, z in ub], dtype=np.int64)[inv]
        hit = found >= 0
        d = np.full(n, np.inf)
        d[hit] = ((means[found[hit], :3] - q[hit]) ** 2).sum(1)
        closer = d < best
        second = np.where(closer, best, np.minimum(second, d))
        ids = np.where(closer, found, ids)
        best = np.where(closer, d, best)
    rejected = best > (np.inf if max_dist_sq is None else max_dist_sq)
    out = np.where((ids < 0) | rejected, NO, ids.astype(np.uint64))
    frac = q * (1.0 / leaf)
    face = np.abs(frac - np.round(frac)).min(axis=1) * leaf < 1e-6
    with np.errstate(invalid="ignore"):
        tie = np.isfinite(second) & (np.abs(second - best) <= 1e-5 * best + 1e-7)
        edge = np.isfinite(best) & (max_dist_sq is not None) & (np.abs(best - (max_dist_sq or 0.0)) < 1e-4 * max(1.0, max_dist_sq or 0.0))
    return out, ~(face | tie | edge)


# ---------------------------------------------------------------- the checker
class Checker:
    """holds one log to the models.  exact=False: the device's storage model, np_search, np_factors.TIGHT; exact=True: the FP64 inputs
    themselves, an FP64 nearest search, `tol` 1e-9 (the OMP arm)."""

    def __init__(self, prob, log, exact=False, tol=None):
        self.p, self.log, self.exact = prob, log, exact
        self.tol = tol if tol is not None else (1e-9 if exact else NF.TIGHT)
        self.worst = 0.0
        self.checked = 0
        self._kd = None

    def where(self, j):
        c = self.log.calls[j]
        return f"align {c.align} ({STRUCTURES[self.log.aligns[c.align][0]]}), call {j} ({c.name})"

    def on_map(self, c):
        return self.log.aligns[c.align][0] == 3

    def inputs(self, on_map):
        p = self.p
        if on_map:
            tgt = (self.log.vox_means, None, self.log.vox_covs)
        else:
            tgt = (p.tgt_pts, p.tgt_normals, p.tgt_covs)
        if self.exact:
            return (np.asarray(p.src_pts, dtype=np.float64), p.src_covs) + tgt
        return NF.storage_model(p.src_pts, p.src_covs, *tgt)

    def ids(self, j):
        """the correspondences of linearize call j as indices into the model's target (voxel: position in flat_voxels)"""
        c = self.log.calls[j]
        corr = c.corr
        if not self.on_map(c):
            return corr
        hit = corr != NO
        assert not (corr[hit] & np.uint64(0xFFFFFFFF)).any(), f"{self.where(j)}: target_index of a voxel is not calc_index(voxel, 0)"
        return np.where(hit, corr >> np.uint64(32), NO)

    def check_correspondences(self, j):
        c, p = self.log.calls[j], self.p
        ids = self.ids(j)
        hit = ids != NO
        if self.on_map(c):
            m = len(self.log.vox_coords)
            assert (ids[hit] < m).all(), f"{self.where(j)}: correspondences: voxel index out of range"
            model_in = self.inputs(True)
            q = model_in[0][:, :3] @ c.T[:3, :3].T + c.T[:3, 3]
            means = model_in[2]
            ref, clear = voxel_correspondences(q, p.leaf, p.offsets, self.log.vox_coords, means, p.max_dist_sq)
            bad = np.nonzero((ids != ref) & clear)[0]
            assert len(bad) == 0, (f"{self.where(j)}: correspondences: {len(bad)} voxel matches differ from the probe model; first: point {bad[0]} "
                                   f"got {ids[bad[0]]}, model {ref[bad[0]]}")
            return
        assert (ids[hit] < len(p.tgt_pts)).all(), f"{self.where(j)}: correspondences: target_index out of range"
        if self.exact:
            if self._kd is None:
                self._kd = cKDTree(np.asarray(p.tgt_pts)[:, :3])
            q = np.asarray(p.src_pts)[:, :3] @ c.T[:3, :3].T + c.T[:3, 3]
            d, _ = self._kd.query(q, k=1)
            dmin = d * d
            dr = np.full(len(q), np.inf)
            dr[hit] = ((np.asarray(p.tgt_pts)[ids[hit].astype(np.int64), :3] - q[hit]) ** 2).sum(1)
            lim = dmin * (1 + 1e-9) + 1e-18
            wrong = hit & (dr > lim)
            if p.max_dist_sq is not None:
                wrong |= hit & (dr > p.max_dist_sq)
                wrong |= ~hit & (dmin <= p.max_dist_sq * (1 - 1e-12))
            else:
                wrong |= ~hit
            bad = np.nonzero(wrong)[0]
            assert len(bad) == 0, f"{self.where(j)}: correspondences: {len(bad)} not a nearest point; first: point {bad[0]} d2 {dr[bad[0]]}, nearest {dmin[bad[0]]}"
            return
        if not hasattr(self, "_tgt"):
            self._tgt = NS.Target(p.tgt_pts)
        try:
            NS.check_correspondences(ids, c.T, p.src_pts, self._tgt, p.max_dist_sq)
        except AssertionError as e:
            raise AssertionError(f"{self.where(j)}: correspondences: {e}") from None

    def check_factors(self, j):
        c, n = self.log.calls[j], self.log.n_src
        if self.p.sync:
            assert np.array_equal(c.source_index, np.arange(n, dtype=np.uint64)), f"{self.where(j)}: source_index of the factor vector"
            assert np.array_equal(c.target_index, c.corr), f"{self.where(j)}: target_index of the factor vector differs from the correspondences used"
        else:
            want = np.full(n, NO)
            if n:
                want[0] = 0
            assert np.array_equal(c.source_index, want) and (c.target_index == NO).all(), f"{self.where(j)}: factor vector synced although sync_every_linearize is false"

    def check_sums(self, j):
        c, p = self.log.calls[j], self.p
        ids = self.ids(j)
        model = NF.linearize(c.T, ids, p.factor, p.robust, p.robust_c, *self.inputs(self.on_map(c)))
        if not (ids != NO).any():
            assert not c.H.any() and not c.b.any() and c.e == 0.0, f"{self.where(j)}: H | b | e not zero without correspondences"
            return
        rh, rb, re = NF.tight_ratios((c.H, c.b, c.e), model)
        for name, r in (("H", rh), ("b", rb), ("e", re)):
            assert r <= self.tol, f"{self.where(j)}: {name} off the model by {r:.3g} (limit {self.tol:.3g})"
        self.worst = max(self.worst, rh, rb, re)

    def check_error(self, j, lin):
        c, p, L = self.log.calls[j], self.p, self.log.calls[lin]
        ids = self.ids(lin)
        want = NF.error(c.T, L.T, ids, p.factor, p.robust, p.robust_c, *self.inputs(self.on_map(L)))
        r = abs(c.e - want) / want if want > 0 else abs(c.e)
        assert r <= self.tol, f"{self.where(j)}: e off the model by {r:.3g} (limit {self.tol:.3g}; got {c.e}, model {want})"
        self.worst = max(self.worst, r)

    def run(self):
        lin = None
        last = {}
        for j, c in enumerate(self.log.calls):
            if c.kind == 0:
                self.check_correspondences(j)
                self.check_factors(j)
                self.check_sums(j)
                lin = j
                last[c.align] = j
            else:
                assert lin is not None and self.log.calls[lin].align == c.align, f"{self.where(j)}: error() before any linearize of its align()"
                self.check_error(j, lin)
            self.checked += 1
        for a, (_, _, _, _, inl, _) in enumerate(self.log.aligns):
            want = int((self.log.calls[last[a]].corr != NO).sum()) if (self.p.sync and a in last) else 0
            assert inl == want, f"align {a}: num_inliers {inl}, the last linearize has {want}"
        return self


def check(prob, log, exact=False, tol=None):
    return Checker(prob, log, exact, tol).run()


def _outside_tie_band(gi, oi, tgt_pts, src_pts, Tg, To, max_dist_sq):
    """the first query whose two correspondences (CUDA's gi chosen at pose Tg, OMP's oi at To) are not both acceptable, or None.  The
    distances are taken at Tg.  Each arm's choice is nearest at its own pose (check() shows it), and moving a query by |dq| moves a squared
    distance d by at most 2 sqrt(d) |dq| + |dq|^2, so the two distances may differ by the tie band (np_factors.compare_correspondences)
    plus that much for each; a rejected query, by the rejection band plus that much.  At the first call both poses are the initial
    guess and this is the tie band alone."""
    mism = np.nonzero(gi != oi)[0]
    p = src_pts[mism, :3]
    qg, qo = p @ Tg[:3, :3].T + Tg[:3, 3], p @ To[:3, :3].T + To[:3, 3]
    dq = np.sqrt(((qg - qo) ** 2).sum(1))
    for k, i in enumerate(mism):
        d = [np.inf if x == NO else float(((tgt_pts[int(x), :3] - qg[k]) ** 2).sum()) for x in (gi[i], oi[i])]
        slack = sum(2.0 * np.sqrt(x) * dq[k] + dq[k] ** 2 for x in d if np.isfinite(x))
        if np.isinf(d[0]) or np.isinf(d[1]):
            fin = d[1] if np.isinf(d[0]) else d[0]
            ok = max_dist_sq is not None and abs(fin - max_dist_sq) < 1e-4 * max(1.0, max_dist_sq) + slack
        else:
            ok = abs(d[0] - d[1]) <= 1e-5 * d[1] + 1e-7 + slack
        if not ok:
            return (int(i), d[0], d[1], float(dq[k]))
    return None


def compare_arms(prob, cuda, omp):
    """CUDA log against the OMP arm.  The OMP arm is the FP64 model (check(..., exact=True) holds it there to 1e-9), so every CUDA call is
    held to that model on the FP64 inputs at the CUDA arm's own pose and correspondences, within ORACLE_TOL.  The two arms' logged sums
    are not compared with each other: their poses part after the first step (each solves its own system; at UTM-like coordinates the
    world origin's lever arm turns a rounding-level difference in a step into a visible one in the pose), and sums at different poses
    differ by more than the sums' own error.  The logs must make the same calls until their correspondences first differ, and that first
    difference must lie inside the tie band.  Returns the number of calls before the arms part (the log's length if they never do)."""
    fp = Checker(prob, cuda, exact=True)
    om = Checker(prob, omp, exact=True)
    parted, lin = None, None
    for j, g in enumerate(cuda.calls):
        where = f"align {g.align}, call {j} ({g.name})"
        on_map = cuda.aligns[g.align][0] == 3
        inp = fp.inputs(on_map)
        if g.kind == 0:
            ids = fp.ids(j)
            lin = j
            if (ids != NO).any():
                ratios = NF.tight_ratios((g.H, g.b, g.e), NF.linearize(g.T, ids, prob.factor, prob.robust, prob.robust_c, *inp))
                for name, r in zip(("H", "b", "e"), ratios):
                    assert r <= ORACLE_TOL, f"{where}: {name} off the FP64 reference on FP64 inputs by {r:.3g} (limit {ORACLE_TOL:g})"
        else:
            want = NF.error(g.T, cuda.calls[lin].T, fp.ids(lin), prob.factor, prob.robust, prob.robust_c, *inp)
            assert abs(g.e - want) <= ORACLE_TOL * want, f"{where}: e off the FP64 reference on FP64 inputs ({g.e} against {want})"
        if parted is not None:
            continue
        assert j < len(omp.calls), f"{where}: the OMP arm made only {len(omp.calls)} calls"
        o = omp.calls[j]
        assert g.kind == o.kind and g.align == o.align, f"{where}: call sequence differs from the OMP arm ({o.name} of align {o.align})"
        if g.kind == 0:
            gi, oi = fp.ids(j), om.ids(j)
            if not np.array_equal(gi, oi):
                if on_map:  # a query on a voxel face may be probed from either side
                    q = inp[0][:, :3] @ g.T[:3, :3].T + g.T[:3, 3]
                    clear = voxel_correspondences(q, prob.leaf, prob.offsets, cuda.vox_coords, inp[2], prob.max_dist_sq)[1]
                    gi = np.where(clear, gi, oi)
                bad = _outside_tie_band(gi, oi, inp[2], inp[0], g.T, o.T, prob.max_dist_sq)
                assert bad is None, f"{where}: correspondences differ from the OMP arm outside the tie band: {bad}"
                parted = j
    if parted is None:
        assert len(cuda.calls) == len(omp.calls), f"call count {len(cuda.calls)} differs from the OMP arm's {len(omp.calls)}"
    return len(cuda.calls) if parted is None else parted


# ---------------------------------------------------------------- running the harness
def _f32(a):
    return None if a is None else np.asarray(a, dtype=np.float64).astype(np.float32).astype(np.float64)


def as_cloud_type(cloud_type, pts, normals, covs):
    """the FP64 arrays the reduction reads from a cloud of this type: PointCloud holds the input; the harness' FP32 struct holds every
    field rounded to FP32 (covariances: the upper triangle, mirrored)"""
    if cloud_type == 0:
        return pts, normals, covs
    p = np.array(pts, dtype=np.float64)
    p[:, :3] = _f32(p[:, :3])
    p[:, 3] = 1.0
    n = None
    if normals is not None:
        n = np.zeros((len(normals), 4))
        n[:, :3] = _f32(np.asarray(normals)[:, :3])
    c = None
    if covs is not None:
        c = NF.stored_covs(covs)
    return p, n, c


def run(lib, backend, tgt_pts, tgt_normals, tgt_covs, src_pts, src_covs, init_T=None, factor=2, robust=0, robust_c=1.0, max_dist_sq=1.0,
        optimizer=1, max_iterations=20, num_threads=4, structure=0, max_leaf_size=20, voxel_resolution=1.0, offsets=1, lru_horizon=100,
        lru_clear_cycle=10, cloud_type=0, sync=True, generation=0, scenario=0, insert_poses=None):
    """href_align_log through ctypes: (Problem, Log).  max_dist_sq None = NullRejector."""
    import ctypes as C

    dp = C.POINTER(C.c_double)
    f64 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)  # noqa: E731
    d = lambda a: None if a is None else a.ctypes.data_as(dp)  # noqa: E731
    tp, tn, tc, sp, sc = f64(tgt_pts), f64(tgt_normals), f64(tgt_covs), f64(src_pts), f64(src_covs)
    poses = f64(np.eye(4)[None] if insert_poses is None else insert_poses)
    rejector = 0 if max_dist_sq is None else 1
    args = np.array([backend, factor, robust, robust_c, rejector, max_dist_sq or 0.0, optimizer, max_iterations, num_threads, structure, max_leaf_size,
                     voxel_resolution, offsets, lru_horizon, lru_clear_cycle, cloud_type, int(sync), generation, scenario, len(poses), 0], dtype=np.float64)
    T0 = f64(np.eye(4) if init_T is None else init_T)
    rc = lib.href_align_log(d(args), C.c_size_t(len(tp)), d(tp), d(tn), d(tc), C.c_size_t(len(sp)), d(sp), d(sc), d(T0), d(poses))
    if rc != 0:
        raise RuntimeError(lib.href_last_error().decode())
    sizes = np.zeros(4, dtype=np.uint64)
    lib.href_log_sizes(sizes.ctypes.data_as(C.c_void_p))
    nc, ni, na, nv = (int(s) for s in sizes)
    calls, idx, al = np.zeros(nc), np.zeros(ni, dtype=np.uint64), np.zeros(na)
    vc, vm, vv = np.zeros(nv * 3, dtype=np.int32), np.zeros(nv * 4), np.zeros(nv * 16)
    lib.href_log_copy(*(a.ctypes.data_as(C.c_void_p) for a in (calls, idx, al, vc, vm, vv)))
    log = parse(calls, idx, al, vc, vm, vv, len(sp))
    p, n, c = as_cloud_type(cloud_type, tp, tn, tc)
    s, _, scv = as_cloud_type(cloud_type, sp, None, sc)
    # ParallelReductionOMP fills the factor vector on every linearize whatever sync_every_linearize says (a CUDA-only switch)
    prob = Problem(s, scv, p, n, c, factor, robust, robust_c, max_dist_sq, voxel_resolution, offsets, sync or backend == 0)
    return prob, log


# ---------------------------------------------------------------- loading the harness
def load_harness(path):
    """oracle/_ref/libsgb_host_ref.so for the tests, or a skip where it cannot be had.  It is built only where the reference's sources
    are at hand (tests/host_ref/Makefile, which rebuilds it whenever its sources' content changes); a library without href_align_log was
    built from older sources and, like a missing one, can only be rebuilt there."""
    import ctypes as C

    import pytest

    if not os.path.exists(path):
        pytest.skip("oracle/_ref/libsgb_host_ref.so not built (needs the reference's sources: `make -C tests/host_ref REF=<reference checkout>`)")
    L = C.CDLL(path)
    if not hasattr(L, "href_align_log"):
        pytest.skip("oracle/_ref/libsgb_host_ref.so was built from older sources (no href_align_log); rebuild it: `make -C tests/host_ref REF=<reference checkout>`")
    L.href_last_error.restype = C.c_char_p
    return L
