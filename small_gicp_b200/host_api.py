"""ctypes front-end of libsgicp_b200_host.so: the C++ host mirror of the reference's template surface
(Registration<Factor, ParallelReductionCUDA, ...>::align, KdTree<PointCloud>) instantiated behind one C entry point.
Used by the tests; C++ users include small_gicp_b200/host/include/small_gicp_b200/*.hpp directly."""
import ctypes as C
import os

import numpy as np

from . import capi

_dp = C.POINTER(C.c_double)
_u64p = C.POINTER(C.c_uint64)
_LIB = None

TREE_HOST_KDTREE, TREE_DEVICE_KDTREE, TREE_VOXELMAP = 0, 1, 2
OPT_GN, OPT_LM = 0, 1


def library_path():
    return os.path.join(os.path.dirname(capi.library_path()), "libsgicp_b200_host.so")


def _lib():
    global _LIB
    if _LIB is None:
        capi._lib()  # libsgicp_b200.so first (the host library links against it)
        path = library_path()
        if not os.path.exists(path):
            raise capi.SgbError(f"{path} is missing: build it with __graft_entry__.build()")
        L = C.CDLL(path)
        L.sgbh_last_error.restype = C.c_char_p
        L.sgbh_align.restype = C.c_int
        L.sgbh_align.argtypes = [C.c_size_t, _dp, _dp, _dp, C.c_size_t, _dp, _dp, _dp, _dp, _dp, _dp, _dp, _dp]
        L.sgbh_kdtree_knn.restype = C.c_int
        L.sgbh_kdtree_knn.argtypes = [C.c_size_t, _dp, C.c_size_t, _dp, C.c_int, _u64p, _dp]
        _LIB = L
    return _LIB


def _d(a):
    return None if a is None else a.ctypes.data_as(_dp)


def _f64(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64)


class Result:
    pass


def align(
    target_points,
    source_points,
    target_normals=None,
    target_covs=None,
    source_covs=None,
    init_T=None,
    factor=capi.FACTOR_GICP,
    robust=capi.ROBUST_NONE,
    robust_c=1.0,
    rejector=capi.REJECT_DISTANCE,
    max_dist_sq=1.0,
    optimizer=OPT_LM,
    max_iterations=20,
    rotation_eps=0.1 * np.pi / 180.0,
    translation_eps=1e-3,
    tree=TREE_HOST_KDTREE,
    voxel_resolution=1.0,
    voxel_search_offsets=1,
    dof_mask=None,
    device=0,
):
    """Registration<Factor, ParallelReductionCUDA, GeneralFactor, Rejector, Optimizer>::align (C++ host mirror)."""
    L = _lib()
    tp, sp = capi._points4(target_points), capi._points4(source_points)
    tn, tc, sc = _f64(target_normals), _f64(target_covs), _f64(source_covs)
    opts = np.zeros(21)
    opts[:13] = [factor, robust, robust_c, rejector, max_dist_sq, optimizer, max_iterations, rotation_eps, translation_eps, tree, voxel_resolution, voxel_search_offsets, 0 if dof_mask is None else 1]
    opts[13:19] = 1.0 if dof_mask is None else np.asarray(dof_mask, dtype=float)
    opts[19] = device
    T0 = np.ascontiguousarray((np.eye(4) if init_T is None else np.asarray(init_T, dtype=float)).T)
    T = np.empty(16)
    sc4 = np.empty(4)
    H = np.empty(36)
    b = np.empty(6)
    rc = L.sgbh_align(tp.shape[0], _d(tp), _d(tn), _d(tc), sp.shape[0], _d(sp), _d(sc), _d(opts), _d(T0), _d(T), _d(sc4), _d(H), _d(b))
    if rc != 0:
        raise capi.SgbError(L.sgbh_last_error().decode())
    r = Result()
    r.T_target_source = T.reshape(4, 4).T.copy()
    r.converged = bool(sc4[0])
    r.iterations = int(sc4[1])
    r.num_inliers = int(sc4[2])
    r.error = float(sc4[3])
    r.H = H.reshape(6, 6).copy()
    r.b = b.copy()
    return r


def align_batch(
    target_points,
    sources,
    target_normals=None,
    target_covs=None,
    source_covs=None,
    init_Ts=None,
    factor=capi.FACTOR_GICP,
    robust=capi.ROBUST_NONE,
    robust_c=1.0,
    rejector=capi.REJECT_DISTANCE,
    max_dist_sq=1.0,
    optimizer=OPT_LM,
    max_iterations=20,
    rotation_eps=0.1 * np.pi / 180.0,
    translation_eps=1e-3,
    tree=TREE_HOST_KDTREE,
    voxel_resolution=1.0,
    voxel_search_offsets=1,
    dof_mask=None,
    device=0,
    cloud_of_member=None,
):
    """BatchRegistration<Factor, GeneralFactor, Rejector, Optimizer>::align (C++ host mirror): every source (a list of (N_m, 3|4) arrays)
    from its initial pose (init_Ts: (B, 4, 4), default identity); source_covs: None or a list of (N_m, 4, 4).  Keyword arguments as align().
    cloud_of_member (or None: one member per source): member p is source cloud_of_member[p], each source uploaded once (multi-start;
    one initial pose per member).  Returns capi.BatchAlignResult (per-member arrays)."""
    L = _lib()
    if not hasattr(L.sgbh_align_batch, "_typed"):
        L.sgbh_align_batch.restype = C.c_int
        L.sgbh_align_batch.argtypes = [C.c_size_t, _dp, _dp, _dp, C.c_size_t, C.POINTER(C.c_size_t), _dp, _dp, _dp, _dp, _dp, _dp, _dp, _dp, C.c_size_t,
                                       C.POINTER(C.c_size_t)]
        L.sgbh_align_batch._typed = True
    tp = capi._points4(target_points)
    tn, tc = _f64(target_normals), _f64(target_covs)
    members = [capi._points4(s) for s in sources]
    B = len(members)
    offsets = np.zeros(B + 1, dtype=np.uintp)
    offsets[1:] = np.cumsum([m.shape[0] for m in members])
    sp = np.ascontiguousarray(np.concatenate(members) if B else np.zeros((0, 4)))
    sc = None if source_covs is None else np.ascontiguousarray(np.concatenate([_f64(c) for c in source_covs]) if B else np.zeros((0, 4, 4)))
    opts = np.zeros(21)
    opts[:13] = [factor, robust, robust_c, rejector, max_dist_sq, optimizer, max_iterations, rotation_eps, translation_eps, tree, voxel_resolution, voxel_search_offsets, 0 if dof_mask is None else 1]
    opts[13:19] = 1.0 if dof_mask is None else np.asarray(dof_mask, dtype=float)
    opts[19] = device
    n_sources = B
    com = None if cloud_of_member is None else np.ascontiguousarray(cloud_of_member, dtype=np.uintp).reshape(-1)
    if com is not None:
        B = com.size
    Ts = np.tile(np.eye(4), (B, 1, 1)) if init_Ts is None else np.asarray(init_Ts, dtype=float).reshape(B, 4, 4)
    T0 = np.ascontiguousarray(Ts.transpose(0, 2, 1))
    T, sc4, H, b = np.zeros((max(B, 1), 16)), np.zeros((max(B, 1), 4)), np.zeros((max(B, 1), 36)), np.zeros((max(B, 1), 6))
    rc = L.sgbh_align_batch(tp.shape[0], _d(tp), _d(tn), _d(tc), n_sources, offsets.ctypes.data_as(C.POINTER(C.c_size_t)), _d(sp), _d(sc), _d(opts), _d(T0), _d(T),
                            _d(sc4), _d(H), _d(b), B, None if com is None else com.ctypes.data_as(C.POINTER(C.c_size_t)))
    if rc != 0:
        raise capi.SgbError(L.sgbh_last_error().decode())
    return capi.BatchAlignResult(T[:B], sc4[:B], np.concatenate([H, b], axis=1)[:B])


def align_batch_pairs(
    targets,
    sources,
    target_covs=None,
    source_covs=None,
    init_Ts=None,
    factor=capi.FACTOR_GICP,
    robust=capi.ROBUST_NONE,
    robust_c=1.0,
    rejector=capi.REJECT_DISTANCE,
    max_dist_sq=1.0,
    optimizer=OPT_LM,
    max_iterations=20,
    rotation_eps=0.1 * np.pi / 180.0,
    translation_eps=1e-3,
    voxel_resolution=1.0,
    voxel_search_offsets=1,
    dof_mask=None,
    device=0,
    tree=TREE_VOXELMAP,
    target_normals=None,
    pairs=None,
):
    """BatchRegistration<...>::align(targets, sources, init_Ts, voxel_resolution, search_offsets) (C++ host mirror): source m against a
    Gaussian voxel map of targets[m], every pair in one batched call; with tree=TREE_DEVICE_KDTREE BatchRegistration<...>::align(targets,
    sources, init_Ts): source m against a kd-tree of targets[m].  targets / sources: lists of (N_m, 3|4) arrays; target_covs / source_covs:
    None or lists of (N_m, 4, 4); target_normals: None or a list of (N_m, 4) (point-to-plane, kd-trees only).  pairs (or None: source m
    against target m): a (P, 2) list of (source index, target index), the pair-list overloads -- each target built once, each source
    uploaded once, one initial pose per pair.  Keyword arguments as align_batch().  Returns capi.BatchAlignResult."""
    L = _lib()
    if tree not in (TREE_VOXELMAP, TREE_DEVICE_KDTREE):
        raise capi.SgbError("align_batch_pairs: tree must be TREE_VOXELMAP or TREE_DEVICE_KDTREE")
    if not hasattr(L.sgbh_align_batch_pairs, "_typed"):
        L.sgbh_align_batch_pairs.restype = C.c_int
        L.sgbh_align_batch_pairs.argtypes = [C.c_size_t, C.POINTER(C.c_size_t), _dp, _dp, _dp, C.POINTER(C.c_size_t), _dp, _dp, _dp, _dp, _dp, _dp, _dp, _dp,
                                             C.c_size_t, C.c_size_t, C.POINTER(C.c_size_t)]
        L.sgbh_align_batch_pairs._typed = True
    pl = None if pairs is None else np.ascontiguousarray(pairs, dtype=np.uintp).reshape(-1, 2)
    if pl is None:
        assert len(targets) == len(sources), "one target per source"
    B = len(sources) if pl is None else pl.shape[0]

    def concat(clouds, covs):
        members = [capi._points4(c) for c in clouds]
        offsets = np.zeros(len(members) + 1, dtype=np.uintp)
        offsets[1:] = np.cumsum([m.shape[0] for m in members])
        p = np.ascontiguousarray(np.concatenate(members) if members else np.zeros((0, 4)))
        c = None if covs is None else np.ascontiguousarray(np.concatenate([_f64(x) for x in covs]) if members else np.zeros((0, 4, 4)))
        return offsets, p, c

    to, tp, tc = concat(targets, target_covs)
    so, sp, sc = concat(sources, source_covs)
    tn = None if target_normals is None else np.ascontiguousarray(np.concatenate([_f64(x) for x in target_normals]) if len(targets) else np.zeros((0, 4)))
    if tn is not None:
        assert tn.shape == (tp.shape[0], 4)
    opts = np.zeros(21)
    opts[:13] = [factor, robust, robust_c, rejector, max_dist_sq, optimizer, max_iterations, rotation_eps, translation_eps, tree, voxel_resolution,
                 voxel_search_offsets, 0 if dof_mask is None else 1]
    opts[13:19] = 1.0 if dof_mask is None else np.asarray(dof_mask, dtype=float)
    opts[19] = device
    Ts = np.tile(np.eye(4), (B, 1, 1)) if init_Ts is None else np.asarray(init_Ts, dtype=float).reshape(B, 4, 4)
    T0 = np.ascontiguousarray(Ts.transpose(0, 2, 1))
    T, sc4, H, b = np.zeros((max(B, 1), 16)), np.zeros((max(B, 1), 4)), np.zeros((max(B, 1), 36)), np.zeros((max(B, 1), 6))
    rc = L.sgbh_align_batch_pairs(B, to.ctypes.data_as(C.POINTER(C.c_size_t)), _d(tp), _d(tn), _d(tc), so.ctypes.data_as(C.POINTER(C.c_size_t)), _d(sp), _d(sc),
                                  _d(opts), _d(T0), _d(T), _d(sc4), _d(H), _d(b), len(targets), len(sources),
                                  None if pl is None else pl.ctypes.data_as(C.POINTER(C.c_size_t)))
    if rc != 0:
        raise capi.SgbError(L.sgbh_last_error().decode())
    return capi.BatchAlignResult(T[:B], sc4[:B], np.concatenate([H, b], axis=1)[:B])


def align_batch_submaps(maps, sources, lists, poses, map_covs=None, source_covs=None, init_Ts=None, cloud_of_member=None, factor=capi.FACTOR_GICP,
                        robust=capi.ROBUST_NONE, robust_c=1.0, rejector=capi.REJECT_DISTANCE, max_dist_sq=1.0, optimizer=OPT_LM, max_iterations=20,
                        rotation_eps=0.1 * np.pi / 180.0, translation_eps=1e-3, dof_mask=None, device=0):
    """BatchRegistration<...>::align(maps, sources, cloud_of_member, submaps, init_Ts) (C++ host mirror): member p = sources[cloud_of_member[p]]
    (None: source p) from init_Ts[p] against the union of the maps lists[p], map lists[p][j] placed by the 4x4 pose poses[p][j] (map ->
    common frame); each map's kd-tree is built once and none is transformed.  maps / sources: lists of (N_m, 3|4) arrays; map_covs /
    source_covs: None or lists of (N_m, 4, 4).  ICP and GICP; point-to-plane raises.  Returns capi.BatchAlignResult."""
    L = _lib()
    szp = C.POINTER(C.c_size_t)
    if not hasattr(L.sgbh_align_batch_submaps, "_typed"):
        L.sgbh_align_batch_submaps.restype = C.c_int
        L.sgbh_align_batch_submaps.argtypes = [C.c_size_t, C.c_size_t, szp, _dp, _dp, C.c_size_t, szp, _dp, _dp, szp, szp, szp, _dp, _dp, _dp, _dp, _dp, _dp, _dp]
        L.sgbh_align_batch_submaps._typed = True
    B = len(lists)

    def concat(clouds, covs):
        members = [capi._points4(c) for c in clouds]
        offsets = np.zeros(len(members) + 1, dtype=np.uintp)
        offsets[1:] = np.cumsum([m.shape[0] for m in members])
        p = np.ascontiguousarray(np.concatenate(members) if members else np.zeros((0, 4)))
        c = None if covs is None else np.ascontiguousarray(np.concatenate([_f64(x) for x in covs]) if members else np.zeros((0, 4, 4)))
        return offsets, p, c

    mo, mp, mc = concat(maps, map_covs)
    so, sp, sc = concat(sources, source_covs)
    cl = np.ascontiguousarray(np.arange(B) if cloud_of_member is None else cloud_of_member, dtype=np.uintp).reshape(B)
    off = np.zeros(B + 1, dtype=np.uintp)
    off[1:] = np.cumsum([len(l) for l in lists])
    em = np.ascontiguousarray([k for l in lists for k in l], dtype=np.uintp)
    assert all(len(poses[p]) == len(lists[p]) for p in range(B)), "one pose per list entry"
    ep = np.ascontiguousarray(np.array([np.asarray(P, dtype=float).reshape(4, 4).T for ps in poses for P in ps]).reshape(-1, 16)) if em.size else np.zeros((1, 16))
    opts = np.zeros(21)
    opts[:13] = [factor, robust, robust_c, rejector, max_dist_sq, optimizer, max_iterations, rotation_eps, translation_eps, TREE_DEVICE_KDTREE, 1.0, 1,
                 0 if dof_mask is None else 1]
    opts[13:19] = 1.0 if dof_mask is None else np.asarray(dof_mask, dtype=float)
    opts[19] = device
    Ts = np.tile(np.eye(4), (B, 1, 1)) if init_Ts is None else np.asarray(init_Ts, dtype=float).reshape(B, 4, 4)
    T0 = np.ascontiguousarray(Ts.transpose(0, 2, 1))
    T, sc4, H, b = np.zeros((max(B, 1), 16)), np.zeros((max(B, 1), 4)), np.zeros((max(B, 1), 36)), np.zeros((max(B, 1), 6))
    rc = L.sgbh_align_batch_submaps(B, len(maps), mo.ctypes.data_as(szp), _d(mp), _d(mc), len(sources), so.ctypes.data_as(szp), _d(sp), _d(sc),
                                    cl.ctypes.data_as(szp), off.ctypes.data_as(szp), em.ctypes.data_as(szp), _d(ep), _d(opts), _d(T0), _d(T), _d(sc4), _d(H), _d(b))
    if rc != 0:
        raise capi.SgbError(L.sgbh_last_error().decode())
    return capi.BatchAlignResult(T[:B], sc4[:B], np.concatenate([H, b], axis=1)[:B])


ICP, PLANE_ICP, GICP, VGICP = 0, 1, 2, 3  # RegistrationSetting::RegistrationType


def helper_align(target_points, source_points, init_T=None, type=GICP, voxel_resolution=1.0, downsampling_resolution=0.25, max_correspondence_distance=1.0,
                 rotation_eps=0.1 * np.pi / 180.0, translation_eps=1e-3, max_iterations=20, device=0):
    """small_gicp::align(target, source, init_T, RegistrationSetting) on raw points (registration_helper.cpp:58-69):
    device voxel-grid sampling (0.25 m), k = 10 normals + covariances, kd-tree, LM registration with the CUDA reduction."""
    L = _lib()
    if not hasattr(L.sgbh_helper_align, "_typed"):
        L.sgbh_helper_align.restype = C.c_int
        L.sgbh_helper_align.argtypes = [C.c_size_t, _dp, C.c_size_t, _dp, _dp, _dp, _dp, _dp, _dp]
        L.sgbh_helper_align._typed = True
    tp, sp = capi._points4(target_points), capi._points4(source_points)
    s = np.array([type, voxel_resolution, downsampling_resolution, max_correspondence_distance, rotation_eps, translation_eps, max_iterations, device], dtype=np.float64)
    T0 = np.ascontiguousarray((np.eye(4) if init_T is None else np.asarray(init_T, dtype=float)).T)
    T, sc4, sizes = np.empty(16), np.empty(4), np.empty(2)
    rc = L.sgbh_helper_align(tp.shape[0], _d(tp), sp.shape[0], _d(sp), _d(s), _d(T0), _d(T), _d(sc4), _d(sizes))
    if rc != 0:
        raise capi.SgbError(L.sgbh_last_error().decode())
    r = Result()
    r.T_target_source = T.reshape(4, 4).T.copy()
    r.converged, r.iterations, r.num_inliers, r.error = bool(sc4[0]), int(sc4[1]), int(sc4[2]), float(sc4[3])
    r.target_size, r.source_size = int(sizes[0]), int(sizes[1])
    return r


def preprocess_points(clouds, downsampling_resolution=0.25, num_neighbors=10, batch=False, device=0):
    """preprocess_points(cloud, ...).first of every cloud (C++ host mirror), or with batch=True preprocess_points_batch(clouds, ...):
    clouds is a list of (N_m, 3|4) arrays.  Returns a list of (points (M_m, 4), normals (M_m, 4), covs (M_m, 4, 4))."""
    L = _lib()
    if not hasattr(L.sgbh_preprocess_points, "_typed"):
        L.sgbh_preprocess_points.restype = C.c_int
        L.sgbh_preprocess_points.argtypes = [C.c_size_t, C.POINTER(C.c_size_t), _dp, C.c_double, C.c_int, C.c_int, C.c_int, _dp, _dp, _dp,
                                             C.POINTER(C.c_size_t)]
        L.sgbh_preprocess_points._typed = True
    members = [capi._points4(c) for c in clouds]
    B = len(members)
    offsets = np.zeros(B + 1, dtype=np.uintp)
    offsets[1:] = np.cumsum([m.shape[0] for m in members])
    p = np.ascontiguousarray(np.concatenate(members) if B else np.zeros((0, 4)))
    n = max(p.shape[0], 1)
    pts, nrm, cov = np.zeros((n, 4)), np.zeros((n, 4)), np.zeros((n, 4, 4))
    out_off = np.zeros(B + 1, dtype=np.uintp)
    rc = L.sgbh_preprocess_points(B, offsets.ctypes.data_as(C.POINTER(C.c_size_t)), _d(p), float(downsampling_resolution), int(num_neighbors), int(device),
                                  int(bool(batch)), _d(pts), _d(nrm), _d(cov), out_off.ctypes.data_as(C.POINTER(C.c_size_t)))
    if rc != 0:
        raise capi.SgbError(L.sgbh_last_error().decode())
    return [(pts[a:b].copy(), nrm[a:b].copy(), cov[a:b].copy()) for a, b in zip(out_off[:-1].astype(np.int64), out_off[1:].astype(np.int64))]


def kdtree_knn(points, queries, k):
    """KdTree<PointCloud>(points).knn_search for each query (host mirror, CPU)."""
    L = _lib()
    p, q = capi._points4(points), capi._points4(queries)
    idx = np.empty((q.shape[0], k), dtype=np.uint64)
    d2 = np.empty((q.shape[0], k))
    rc = L.sgbh_kdtree_knn(p.shape[0], _d(p), q.shape[0], _d(q), k, idx.ctypes.data_as(_u64p), _d(d2))
    if rc != 0:
        raise capi.SgbError(L.sgbh_last_error().decode())
    return idx, d2


def read_points_cpp(filename, kind="ply"):
    """read_ply / read_points of the C++ host mirror (small_gicp_b200/host/include/small_gicp_b200/read_points.hpp) -> (N, 4) float32."""
    L = _lib()
    n = C.c_size_t(0)
    k = 0 if kind == "ply" else 1
    fn = str(filename).encode()
    L.sgbh_read_points.restype = C.c_int
    L.sgbh_read_points.argtypes = [C.c_char_p, C.c_int, C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t)]
    if L.sgbh_read_points(fn, k, 0, None, C.byref(n)) != 0:
        raise capi.SgbError(L.sgbh_last_error().decode())
    out = np.empty((n.value, 4), dtype=np.float32)
    if n.value and L.sgbh_read_points(fn, k, n.value, out.ctypes.data_as(C.c_void_p), C.byref(n)) != 0:
        raise capi.SgbError(L.sgbh_last_error().decode())
    return out


def write_points_cpp(filename, points):
    """write_points of the C++ host mirror: (N, 4) float32 -> KITTI-style .bin"""
    L = _lib()
    p = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 4)
    L.sgbh_write_points.restype = C.c_int
    L.sgbh_write_points.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p]
    if L.sgbh_write_points(str(filename).encode(), p.shape[0], p.ctypes.data_as(C.c_void_p)) != 0:
        raise capi.SgbError(L.sgbh_last_error().decode())
