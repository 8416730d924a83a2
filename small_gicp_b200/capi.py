"""ctypes binding of include/sgicp_b200.h.  numpy in, numpy out; poses are 4x4 row-major numpy arrays
(transposed to Eigen's column-major at the boundary)."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)

FACTOR_ICP, FACTOR_PLANE_ICP, FACTOR_GICP = 0, 1, 2
ROBUST_NONE, ROBUST_HUBER, ROBUST_CAUCHY = 0, 1, 2
REJECT_NONE, REJECT_DISTANCE = 0, 1
OPT_GAUSS_NEWTON, OPT_LEVENBERG_MARQUARDT = 0, 1
GNC_GEMAN_MCCLURE, GNC_TLS = 0, 1
NO_CORRESPONDENCE = np.uint64(0xFFFFFFFFFFFFFFFF)

_dp = C.POINTER(C.c_double)
_u64p = C.POINTER(C.c_uint64)
_i32p = C.POINTER(C.c_int32)
_vp = C.c_void_p


class AlignOptions(C.Structure):
    """sgb_align_options"""

    _fields_ = [
        ("factor_kind", C.c_int),
        ("robust_kind", C.c_int),
        ("robust_c", C.c_double),
        ("rejector_kind", C.c_int),
        ("max_dist_sq", C.c_double),
        ("optimizer_kind", C.c_int),
        ("max_iterations", C.c_int),
        ("gn_lambda", C.c_double),
        ("max_inner_iterations", C.c_int),
        ("init_lambda", C.c_double),
        ("lambda_factor", C.c_double),
        ("rotation_eps", C.c_double),
        ("translation_eps", C.c_double),
        ("dof_mask", C.c_double * 6),
    ]


def _align_options(factor=FACTOR_GICP, robust=ROBUST_NONE, robust_c=1.0, rejector=REJECT_DISTANCE, max_dist_sq=1.0, optimizer=OPT_LEVENBERG_MARQUARDT,
                   max_iterations=20, gn_lambda=1e-6, max_inner_iterations=10, init_lambda=1e-3, lambda_factor=10.0, rotation_eps=0.1 * np.pi / 180.0,
                   translation_eps=1e-3, dof_mask=None):
    """the sgb_align_options of the align_batch keywords"""
    o = AlignOptions(int(factor), int(robust), float(robust_c), int(rejector), float(max_dist_sq), int(optimizer), int(max_iterations), float(gn_lambda),
                     int(max_inner_iterations), float(init_lambda), float(lambda_factor), float(rotation_eps), float(translation_eps))
    o.dof_mask[:] = [1.0] * 6 if dof_mask is None else [float(x) for x in dof_mask]
    return o


def _windows(windows, fixed, K, who):
    """the window offsets and fixed flags of a joint call over K frames"""
    off = np.ascontiguousarray(np.array([0, K] if windows is None else windows, dtype=np.uintp).reshape(-1))
    if off.size < 1:
        raise SgbError(f"{who}: windows needs at least one entry")
    fx = None if fixed is None else np.ascontiguousarray(np.asarray(fixed).astype(np.uint8).reshape(-1))
    if fx is not None and fx.size != K:
        raise SgbError(f"{who}: fixed needs {K} entries")
    return off, fx


class GncOptions(C.Structure):
    """sgb_gnc_options"""

    _fields_ = [("kind", C.c_int), ("noise_bound_sq", C.c_double), ("max_stages", C.c_int), ("stage_iterations", C.c_int)]

# name -> (restype, argtypes): every symbol include/sgicp_b200.h declares
_SIGNATURES = {
    "sgb_create": (C.c_int, [C.c_int, C.POINTER(_vp)]),
    "sgb_destroy": (None, [_vp]),
    "sgb_last_error": (C.c_char_p, [_vp]),
    "sgb_set_stream": (C.c_int, [_vp, _vp]),
    "sgb_synchronize": (C.c_int, [_vp]),
    "sgb_kernel_launches": (C.c_uint64, [_vp]),
    "sgb_comm_handle": (C.c_int, [_vp, _vp]),
    "sgb_comm_connect": (C.c_int, [_vp, C.c_int, C.c_int, _vp]),
    "sgb_comm_mailbox": (C.c_int, [_vp, C.POINTER(_vp)]),
    "sgb_comm_connect_ptrs": (C.c_int, [_vp, C.c_int, C.c_int, C.POINTER(_vp)]),
    "sgb_comm_disconnect": (C.c_int, [_vp]),
    "sgb_comm_set_timeout_ms": (C.c_int, [_vp, C.c_int]),
    "sgb_comm_status": (C.c_int, [_vp, C.POINTER(C.c_int)]),
    "sgb_comm_wait_ns": (C.c_int, [_vp, _u64p, _u64p]),
    "sgb_drop_seeds": (C.c_int, [_vp]),
    "sgb_target_set_points": (C.c_int, [_vp, C.c_size_t, _dp, _dp, _dp]),
    "sgb_target_set_kdtree": (C.c_int, [_vp, _vp, C.c_size_t, C.c_uint32, _u64p]),
    "sgb_target_build_kdtree": (C.c_int, [_vp, C.c_int]),
    "sgb_target_set_voxelmap": (C.c_int, [_vp, C.c_double, C.c_size_t, _i32p, _dp, _dp, C.c_int]),
    "sgb_target_build_voxelmap": (C.c_int, [_vp, C.c_size_t, _dp, _dp, C.c_double, C.c_int]),
    "sgb_target_build_voxelmaps": (C.c_int, [_vp, C.c_size_t, C.POINTER(C.c_size_t), _dp, _dp, C.c_double, C.c_int]),
    "sgb_target_build_kdtrees": (C.c_int, [_vp, C.c_size_t, C.POINTER(C.c_size_t), _dp, _dp, _dp]),
    "sgb_target_batch_knn": (C.c_int, [_vp, C.c_size_t, _dp, C.c_int, _u64p, _dp]),
    "sgb_target_batch_knn_maps": (C.c_int, [_vp, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_uint32), _dp, C.c_int, _u64p, _dp]),
    "sgb_target_batch_knn_submaps": (C.c_int, [_vp, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_uint32), _dp, _dp, C.c_int, _u64p,
                                               _dp]),
    "sgb_target_size": (C.c_size_t, [_vp]),
    "sgb_source_set_points": (C.c_int, [_vp, C.c_size_t, _dp, _dp]),
    "sgb_source_size": (C.c_size_t, [_vp]),
    "sgb_linearize": (C.c_int, [_vp, C.c_int, C.c_int, C.c_double, C.c_int, C.c_double, _dp, _dp]),
    "sgb_error": (C.c_int, [_vp, _dp, _dp]),
    "sgb_linearize_device": (C.c_int, [_vp, C.c_int, C.c_int, C.c_double, C.c_int, C.c_double, _dp, _vp]),
    "sgb_error_device": (C.c_int, [_vp, _dp, _vp]),
    "sgb_correspondences": (C.c_int, [_vp, _u64p]),
    "sgb_num_inliers": (C.c_int, [_vp, C.POINTER(C.c_size_t)]),
    "sgb_source_set_batch": (C.c_int, [_vp, C.c_size_t, C.POINTER(C.c_size_t), _dp, _dp]),
    "sgb_source_set_pairs": (C.c_int, [_vp, C.c_size_t, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    "sgb_source_set_submaps": (C.c_int, [_vp, C.c_size_t, C.POINTER(C.c_uint32), C.POINTER(C.c_size_t), C.POINTER(C.c_uint32), _dp]),
    "sgb_source_set_weights": (C.c_int, [_vp, _dp]),
    "sgb_linearize_batch": (C.c_int, [_vp, C.c_int, C.c_int, C.c_double, C.c_int, C.c_double, _dp, C.POINTER(C.c_uint8), _dp]),
    "sgb_error_batch": (C.c_int, [_vp, _dp, C.POINTER(C.c_uint8), _dp]),
    "sgb_correspondences_batch": (C.c_int, [_vp, _u64p]),
    "sgb_linearize_batch_points": (C.c_int, [_vp, C.c_int, C.c_int, C.c_double, C.c_int, C.c_double, _dp, C.POINTER(C.c_uint8), _dp, _dp, _dp]),
    "sgb_error_batch_points": (C.c_int, [_vp, _dp, C.POINTER(C.c_uint8), _dp, _dp]),
    "sgb_align_batch": (C.c_int, [_vp, C.POINTER(AlignOptions), _dp, _dp, _dp, _dp]),
    "sgb_align_batch_async": (C.c_int, [_vp, C.POINTER(AlignOptions), _dp, _dp, _dp, _dp]),
    "sgb_align_batch_gnc": (C.c_int, [_vp, C.POINTER(AlignOptions), C.POINTER(GncOptions), _dp, _dp, _dp, _dp, _dp, _dp]),
    "sgb_align_batch_gnc_async": (C.c_int, [_vp, C.POINTER(AlignOptions), C.POINTER(GncOptions), _dp, _dp, _dp, _dp, _dp, _dp]),
    "sgb_align_joint": (C.c_int, [_vp, C.POINTER(AlignOptions), C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_uint8), _dp, _dp, _dp]),
    "sgb_align_joint_async": (C.c_int, [_vp, C.POINTER(AlignOptions), C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_uint8), _dp, _dp, _dp]),
    "sgb_align_joint_gnc_async": (C.c_int, [_vp, C.POINTER(AlignOptions), C.POINTER(GncOptions), C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_uint8),
                                            _dp, _dp, _dp, _dp, _dp]),
    "sgb_joint_edge_poses": (C.c_int, [_vp, C.c_size_t, C.POINTER(C.c_size_t), _dp, _dp]),
    "sgb_align_joint_gnc": (C.c_int, [_vp, C.POINTER(AlignOptions), C.POINTER(GncOptions), C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_uint8), _dp,
                                      _dp, _dp, _dp, _dp]),
    "sgb_estimate_features": (C.c_int, [_vp, C.c_size_t, _dp, C.c_int, _dp, _dp]),
    "sgb_target_estimate_features": (C.c_int, [_vp, C.c_int]),
    "sgb_source_estimate_features": (C.c_int, [_vp, C.c_int]),
    "sgb_target_adopt_source": (C.c_int, [_vp]),
    "sgb_voxelgrid_sampling": (C.c_int, [_vp, C.c_size_t, _dp, C.c_double, _dp, C.POINTER(C.c_size_t)]),
    "sgb_voxelgrid_sampling_batch": (C.c_int, [_vp, C.c_size_t, C.POINTER(C.c_size_t), _dp, C.c_double, _dp, C.POINTER(C.c_size_t)]),
    "sgb_estimate_features_batch": (C.c_int, [_vp, C.c_size_t, C.POINTER(C.c_size_t), _dp, C.c_int, _dp, _dp]),
}


class SgbError(RuntimeError):
    pass


class BatchAlignResult:
    """per-member RegistrationResult fields of a batched align, from T16 (column-major), info4 and H|b 42 rows"""

    def __init__(self, T16, info4, Hb42):
        B = T16.shape[0]
        self.T_target_source = np.ascontiguousarray(T16.reshape(B, 4, 4).transpose(0, 2, 1))
        self.converged = info4[:, 0] != 0
        self.iterations = info4[:, 1].astype(np.int64)
        self.num_inliers = info4[:, 2].astype(np.int64)
        self.error = info4[:, 3].copy()
        self.H = np.ascontiguousarray(Hb42[:, :36].reshape(B, 6, 6).transpose(0, 2, 1))
        self.b = Hb42[:, 36:42].copy()


class GncAlignResult(BatchAlignResult):
    """what Context.align_batch_gnc returns: the BatchAlignResult fields of each member's last stage (iterations summed over its stages),
    stages (B,) the stages it ran, mu (B,) the surrogate's shape at its last stage (TLS without outliers: 0), and point_w (N,) each point's
    final GNC weight g in the layout of correspondences_batch (None unless requested)"""

    def __init__(self, T16, info4, Hb42, gnc2, point_w):
        super().__init__(T16, info4, Hb42)
        self.stages = gnc2[:, 0].astype(np.int64)
        self.mu = gnc2[:, 1].copy()
        self.point_w = point_w


class BatchPointTerms:
    """what Context.linearize_batch_points returns: the member arrays of linearize_batch, H (B,6,6), b (B,6), e (B,) and num_inliers (B,),
    and one row per source point in the layout of correspondences_batch (member m's rows are offsets[m] .. offsets[m + 1], in its
    cloud's original order): point_e (N,), point_H (N,6,6) and point_b (N,6) (None with hessians=False).  The point arrays are views of
    the raw rows point_e and point_Hb42 (N,42) = H (36, row-major) | b, numpy arrays or the CUDA tensors passed as out_e / out_Hb42."""

    def __init__(self, H, b, e, num_inliers, offsets, point_e, point_Hb42):
        self.H, self.b, self.e, self.num_inliers, self.offsets = H, b, e, num_inliers, offsets
        self.point_e, self.point_Hb42 = point_e, point_Hb42
        n = point_e.shape[0]
        self.point_H = None if point_Hb42 is None else point_Hb42[:, :36].reshape(n, 6, 6)
        self.point_b = None if point_Hb42 is None else point_Hb42[:, 36:42]


class JointAlignResult:
    """what Context.align_joint returns: per frame X (K,4,4); per window converged (W,) bool, iterations (W,), num_inliers (W,) and error
    (W,), the last two summed over the window's edges"""

    def __init__(self, X16, info4):
        K = X16.shape[0]
        self.X = np.ascontiguousarray(X16.reshape(K, 4, 4).transpose(0, 2, 1))
        self.converged = info4[:, 0] != 0
        self.iterations = info4[:, 1].astype(np.int64)
        self.num_inliers = info4[:, 2].astype(np.int64)
        self.error = info4[:, 3].copy()


class JointGncAlignResult(JointAlignResult):
    """what Context.align_joint_gnc returns: the JointAlignResult fields of each window's last stage (iterations summed over its stages),
    stages (W,) the stages it ran, mu (W,) the surrogate's shape at its last stage (TLS without outliers: 0), and point_w (N,) each edge
    point's final GNC weight g in the layout of correspondences_batch (None unless requested)"""

    def __init__(self, X16, info4, gnc2, point_w):
        super().__init__(X16, info4)
        self.stages = gnc2[:, 0].astype(np.int64)
        self.mu = gnc2[:, 1].copy()
        self.point_w = point_w


class AsyncAlignResult:
    """what Context.align_batch_async enqueued: CUDA float64 tensors filled in stream order.  T_target_source (B,4,4), H (B,6,6) and b
    (B,6) as in BatchAlignResult; converged (1.0 / 0.0), iterations, num_inliers and error are (B,) float64 views of the info rows.  All
    are views of the raw outputs T16 (B,16), info4 (B,4) and Hb42 (B,42), which pass as out= to reuse them (graph capture needs fixed
    buffers)."""

    def __init__(self, T16, info4, Hb42):
        B = T16.shape[0]
        self.T16, self.info4, self.Hb42 = T16, info4, Hb42
        self.T_target_source = T16.view(B, 4, 4).transpose(1, 2)
        self.converged = info4[:, 0]
        self.iterations = info4[:, 1]
        self.num_inliers = info4[:, 2]
        self.error = info4[:, 3]
        self.H = Hb42[:, :36].view(B, 6, 6).transpose(1, 2)
        self.b = Hb42[:, 36:42]


class AsyncGncAlignResult(AsyncAlignResult):
    """what Context.align_batch_gnc_async enqueued: the AsyncAlignResult views (iterations summed over the stages), stages (B,) and mu (B,)
    as float64 views of the raw gnc2 (B,2), and point_w (N,) each point's final g (None unless requested).  The raw outputs T16, info4,
    Hb42, gnc2 and point_w pass as out= to reuse them (graph capture needs fixed buffers)."""

    def __init__(self, T16, info4, Hb42, gnc2, point_w):
        super().__init__(T16, info4, Hb42)
        self.gnc2, self.point_w = gnc2, point_w
        self.stages = gnc2[:, 0]
        self.mu = gnc2[:, 1]


class AsyncJointAlignResult:
    """what Context.align_joint_async enqueued: CUDA float64 tensors filled in stream order.  X (K,4,4) per frame; converged (1.0 / 0.0),
    iterations, num_inliers and error (W,) per window, as in JointAlignResult.  All are views of the raw outputs X16 (K,16) and info4 (W,4),
    which pass as out= to reuse them (graph capture needs fixed buffers)."""

    def __init__(self, X16, info4):
        K = X16.shape[0]
        self.X16, self.info4 = X16, info4
        self.X = X16.view(K, 4, 4).transpose(1, 2)
        self.converged = info4[:, 0]
        self.iterations = info4[:, 1]
        self.num_inliers = info4[:, 2]
        self.error = info4[:, 3]


class AsyncJointGncAlignResult(AsyncJointAlignResult):
    """what Context.align_joint_gnc_async enqueued: the AsyncJointAlignResult views (iterations summed over each window's stages), stages
    (W,) and mu (W,) as float64 views of the raw gnc2 (W,2), and point_w (N,) each edge point's final g (None unless requested).  The raw
    outputs X16, info4, gnc2 and point_w pass as out= to reuse them (graph capture needs fixed buffers)."""

    def __init__(self, X16, info4, gnc2, point_w):
        super().__init__(X16, info4)
        self.gnc2, self.point_w = gnc2, point_w
        self.stages = gnc2[:, 0]
        self.mu = gnc2[:, 1]


def library_path(profiling=False):
    """the product library; profiling=True: the same sources built with -DSGB_PROFILING (experiment switches read from SGB_*
    environment variables in sgb_create + the superseded A/B kernels) -- A/B scripts and the structure-agreement test only"""
    if os.environ.get("SGB_LIBRARY", "") == "prev" and not profiling:  # A/B against a saved build of the product library (scripts/gpu_ab.sh)
        return os.path.join(_HERE, "lib", "libsgicp_b200_prev.so")
    return os.path.join(_HERE, "lib", "libsgicp_b200_prof.so" if profiling else "libsgicp_b200.so")


def exported_symbols():
    return sorted(_SIGNATURES)


_LIBS = {}


def _lib(profiling=False):
    if profiling not in _LIBS:
        path = library_path(profiling)
        if not os.path.exists(path):
            raise SgbError(
                f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `make -C small_gicp_b200/csrc`). There is no CPU fallback."
            )
        L = C.CDLL(path)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the library does not export it
            fn.restype = res
            fn.argtypes = args
        _LIBS[profiling] = L
    return _LIBS[profiling]


def _is_dev(a):
    """a torch tensor (host or CUDA): passed by address -- the library copies with cudaMemcpyDefault, so device-resident producers
    hand their buffers over without a host round trip"""
    return hasattr(a, "data_ptr") and hasattr(a, "is_contiguous")


def _f64(a):
    if _is_dev(a):
        import torch

        assert a.dtype == torch.float64 and a.is_contiguous(), "torch inputs must be contiguous float64"
        return a
    return np.ascontiguousarray(a, dtype=np.float64)


def _d(a):
    if a is None:
        return None
    if _is_dev(a):
        return C.cast(C.c_void_p(a.data_ptr()), _dp)
    return a.ctypes.data_as(_dp)


def _pose(T):
    T = _f64(T)
    assert T.shape == (4, 4)
    return np.ascontiguousarray(T.T)  # row-major transpose == column-major original


def _points4(p):
    if _is_dev(p):
        assert p.dim() == 2 and p.shape[1] == 4, "torch point inputs must be (N, 4) = (x, y, z, 1)"
        return _f64(p)
    p = _f64(p)
    assert p.ndim == 2 and p.shape[1] in (3, 4)
    if p.shape[1] == 3:
        p = np.concatenate([p, np.ones((p.shape[0], 1))], axis=1)
    return np.ascontiguousarray(p)


class Context:
    """One GPU, one stream (sgb_ctx)."""

    def __init__(self, device=0, profiling=None):
        if profiling is None:  # A/B scripts select the profiling build for a whole process
            profiling = os.environ.get("SGB_LIBRARY", "") == "prof"
        self._L = _lib(bool(profiling))
        h = _vp()
        rc = self._L.sgb_create(int(device), C.byref(h))
        if rc != 0:
            raise SgbError(self._L.sgb_last_error(None).decode())
        self._h = h
        self.device = int(device)
        self._stream = None  # set_stream's stream (None: the context's own)
        self._async_in = None  # align_batch_async's column-major poses
        self._joint_in = None  # align_joint_async's column-major frame poses

    def close(self):
        if getattr(self, "_h", None):
            self._L.sgb_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            raise SgbError(self._L.sgb_last_error(self._h).decode())

    # ---- plumbing ----
    def set_stream(self, cuda_stream_ptr):
        self._check(self._L.sgb_set_stream(self._h, _vp(cuda_stream_ptr) if cuda_stream_ptr else None))
        self._stream = int(cuda_stream_ptr) if cuda_stream_ptr else None

    def synchronize(self):
        self._check(self._L.sgb_synchronize(self._h))

    @property
    def kernel_launches(self):
        return int(self._L.sgb_kernel_launches(self._h))

    # ---- target ----
    def set_target(self, points, normals=None, covs=None):
        p = _points4(points)
        n = _f64(normals) if normals is not None else None
        c = _f64(covs) if covs is not None else None
        if n is not None:
            assert tuple(n.shape) == (p.shape[0], 4)
        if c is not None:
            assert tuple(c.shape) == (p.shape[0], 4, 4)
        self._check(self._L.sgb_target_set_points(self._h, p.shape[0], _d(p), _d(n), _d(c)))

    def set_target_kdtree(self, nodes24, indices, root=0):
        nodes24 = np.ascontiguousarray(nodes24, dtype=np.uint8)
        indices = np.ascontiguousarray(indices, dtype=np.uint64)
        self._check(self._L.sgb_target_set_kdtree(self._h, nodes24.ctypes.data_as(_vp), nodes24.shape[0], int(root), indices.ctypes.data_as(_u64p)))

    def build_target_kdtree(self, max_leaf_size=0):
        self._check(self._L.sgb_target_build_kdtree(self._h, int(max_leaf_size)))

    def set_target_voxelmap(self, leaf_size, coords, means, covs, search_offsets=1):
        coords = np.ascontiguousarray(coords, dtype=np.int32)
        m = _points4(means)
        c = _f64(covs) if covs is not None else None
        self._check(self._L.sgb_target_set_voxelmap(self._h, float(leaf_size), m.shape[0], coords.ctypes.data_as(_i32p), _d(m), _d(c), int(search_offsets)))

    def build_target_voxelmap(self, points, covs, leaf_size, search_offsets=1):
        """GaussianVoxelMap(leaf_size).insert(points) built on the device (incremental_voxelmap.hpp:55-92)"""
        p = _points4(points)
        c = _f64(covs) if covs is not None else None
        if c is not None:
            assert tuple(c.shape) == (p.shape[0], 4, 4)
        self._check(self._L.sgb_target_build_voxelmap(self._h, p.shape[0], _d(p), _d(c), float(leaf_size), int(search_offsets)))

    def build_target_voxelmaps(self, points_list, covs_list=None, leaf_size=1.0, search_offsets=1):
        """one Gaussian voxel map per cloud, as ONE target of the batched calls: member m of the batch is aligned against map m.
        points_list: a list of (N_m, 3|4) arrays, or (points (N, 3|4), offsets (B + 1,)) with the clouds concatenated (numpy or torch).
        covs_list: None, a list of (N_m, 4, 4) arrays, or one (N, 4, 4) array."""
        if isinstance(points_list, tuple):
            points, offsets = points_list
            p = _points4(points)
            offsets = np.ascontiguousarray(offsets, dtype=np.uintp)
            if offsets.ndim != 1 or offsets.size < 1 or int(offsets[-1]) != p.shape[0]:
                raise SgbError(f"build_target_voxelmaps: offsets must have B + 1 entries ending at the point count {p.shape[0]}")
        else:
            members = [_points4(x) for x in points_list]
            offsets = np.zeros(len(members) + 1, dtype=np.uintp)
            offsets[1:] = np.cumsum([m.shape[0] for m in members])
            p = np.concatenate(members) if members else np.zeros((0, 4))
        c = None
        if covs_list is not None:
            c = _f64(covs_list) if not isinstance(covs_list, (list, tuple)) else (np.concatenate([_f64(x) for x in covs_list]) if len(covs_list) else np.zeros((0, 4, 4)))
            assert tuple(c.shape) == (p.shape[0], 4, 4)
        self._check(self._L.sgb_target_build_voxelmaps(self._h, offsets.size - 1, offsets.ctypes.data_as(C.POINTER(C.c_size_t)), _d(p), _d(c),
                                                       float(leaf_size), int(search_offsets)))

    def build_target_kdtrees(self, points_list, normals_list=None, covs_list=None):
        """one kd-tree per cloud, as ONE target of the batched calls: member m of the batch is aligned against map m (ICP, point-to-plane
        with normals, GICP with covariances).  points_list: a list of (N_m, 3|4) arrays, or (points (N, 3|4), offsets (B + 1,)) with the
        clouds concatenated (numpy or torch).  normals_list / covs_list: None, a list of (N_m, 4) / (N_m, 4, 4) arrays, or one
        (N, 4) / (N, 4, 4) array."""
        if isinstance(points_list, tuple):
            points, offsets = points_list
            p = _points4(points)
            offsets = np.ascontiguousarray(offsets, dtype=np.uintp)
            if offsets.ndim != 1 or offsets.size < 1 or int(offsets[-1]) != p.shape[0]:
                raise SgbError(f"build_target_kdtrees: offsets must have B + 1 entries ending at the point count {p.shape[0]}")
        else:
            members = [_points4(x) for x in points_list]
            offsets = np.zeros(len(members) + 1, dtype=np.uintp)
            offsets[1:] = np.cumsum([m.shape[0] for m in members])
            p = np.concatenate(members) if members else np.zeros((0, 4))

        def _joined(xs, shape):
            if xs is None:
                return None
            a = _f64(xs) if not isinstance(xs, (list, tuple)) else (np.concatenate([_f64(x) for x in xs]) if len(xs) else np.zeros((0,) + shape))
            assert tuple(a.shape) == (p.shape[0],) + shape
            return a

        n = _joined(normals_list, (4,))
        c = _joined(covs_list, (4, 4))
        self._check(self._L.sgb_target_build_kdtrees(self._h, offsets.size - 1, offsets.ctypes.data_as(C.POINTER(C.c_size_t)), _d(p), _d(n), _d(c)))

    def target_batch_knn(self, queries, k=1):
        """KdTree.batch_knn_search(queries, k) on the device -> (indices (N,k) uint64, squared distances (N,k))"""
        q = _points4(queries)
        idx = np.empty((q.shape[0], int(k)), dtype=np.uint64)
        d = np.empty((q.shape[0], int(k)))
        self._check(self._L.sgb_target_batch_knn(self._h, q.shape[0], _d(q), int(k), idx.ctypes.data_as(_u64p), _d(d)))
        return idx, d

    @staticmethod
    def _query_sets(queries, who):
        """a list of (N_s, 3|4) arrays, or (points (N, 4), offsets (S + 1,)) -> (points (N, 4), offsets as size_t)"""
        if isinstance(queries, tuple):
            points, offsets = queries
            q = _points4(points)
            offsets = np.ascontiguousarray(offsets, dtype=np.uintp)
            if offsets.ndim != 1 or offsets.size < 1 or int(offsets[-1]) != q.shape[0]:
                raise SgbError(f"{who}: offsets must have S + 1 entries ending at the query count {q.shape[0]}")
            return q, offsets
        sets = [_points4(x) for x in queries]
        offsets = np.zeros(len(sets) + 1, dtype=np.uintp)
        offsets[1:] = np.cumsum([s.shape[0] for s in sets])
        if sets and all(_is_dev(s) for s in sets):
            import torch

            return torch.cat(sets).contiguous(), offsets
        return (np.concatenate([np.asarray(s.cpu()) if _is_dev(s) else s for s in sets]) if sets else np.zeros((0, 4))), offsets

    @staticmethod
    def _knn_rows(q, k):
        """the (N, k) outputs of a k-NN call: torch tensors on the queries' device for torch queries, numpy arrays otherwise"""
        if _is_dev(q):
            import torch

            return torch.empty((q.shape[0], k), dtype=torch.uint64, device=q.device), torch.empty((q.shape[0], k), dtype=torch.float64, device=q.device)
        return np.empty((q.shape[0], k), dtype=np.uint64), np.empty((q.shape[0], k))

    @staticmethod
    def _u64(a):
        return C.cast(C.c_void_p(a.data_ptr()), _u64p) if _is_dev(a) else a.ctypes.data_as(_u64p)

    def target_knn_maps(self, queries, k=1, maps=None):
        """k nearest neighbours of query sets, set s in map maps[s] of the target (None: map s): many kd-trees, many voxel maps, or the
        one kd-tree / voxel map (map 0).  queries: a list of (N_s, 3|4) arrays, or (points (N, 4), offsets (S + 1,)), numpy or torch
        (CUDA tensors stay on the device).  -> (indices (N, k) uint64, squared distances (N, k)); kd-trees: index within the map, voxel
        maps: voxel id within the map << 32."""
        q, off = self._query_sets(queries, "target_knn_maps")
        mp = None if maps is None else np.ascontiguousarray(maps, dtype=np.uint32).reshape(-1)
        if mp is not None and mp.size != off.size - 1:
            raise SgbError(f"target_knn_maps: {off.size - 1} query sets but {mp.size} maps")
        idx, d = self._knn_rows(q, int(k))
        self._check(self._L.sgb_target_batch_knn_maps(self._h, off.size - 1, off.ctypes.data_as(C.POINTER(C.c_size_t)),
                                                      None if mp is None else mp.ctypes.data_as(C.POINTER(C.c_uint32)), _d(q), int(k), self._u64(idx), _d(d)))
        return idx, d

    def target_knn_submaps(self, queries, lists, poses=None, k=1):
        """k nearest neighbours of query sets, set s in the union of the maps lists[s] of a many-kd-trees target, map lists[s][j] placed by
        the rigid 4x4 pose poses[s][j] (map -> common frame; None: identity), as set_source_submaps takes them; queries in the common
        frame, as for target_knn_maps.  -> (indices (N, k) uint64 = (entry within the list) << 32 | index within that map, squared
        distances (N, k))."""
        q, off = self._query_sets(queries, "target_knn_submaps")
        lists = [np.asarray(l, dtype=np.uint32).reshape(-1) for l in lists]
        S = len(lists)
        if S != off.size - 1:
            raise SgbError(f"target_knn_submaps: {off.size - 1} query sets but {S} lists")
        loff = np.zeros(S + 1, dtype=np.uintp)
        loff[1:] = np.cumsum([l.size for l in lists])
        maps = np.ascontiguousarray(np.concatenate(lists) if S else np.zeros(0), dtype=np.uint32)
        pc = None
        if poses is not None:
            if len(poses) != S or any(len(poses[s]) != lists[s].size for s in range(S)):
                raise SgbError("target_knn_submaps: one pose per list entry")
            flat = [np.asarray(T, dtype=np.float64).reshape(4, 4).T for s in range(S) for T in poses[s]]  # column-major
            pc = np.ascontiguousarray(np.array(flat).reshape(-1, 16)) if flat else np.zeros((1, 16))
        idx, d = self._knn_rows(q, int(k))
        self._check(self._L.sgb_target_batch_knn_submaps(self._h, S, off.ctypes.data_as(C.POINTER(C.c_size_t)), loff.ctypes.data_as(C.POINTER(C.c_size_t)),
                                                         maps.ctypes.data_as(C.POINTER(C.c_uint32)), _d(pc), _d(q), int(k), self._u64(idx), _d(d)))
        return idx, d

    @property
    def target_size(self):
        return int(self._L.sgb_target_size(self._h))

    # ---- source ----
    def set_source(self, points, covs=None):
        p = _points4(points)
        c = _f64(covs) if covs is not None else None
        if c is not None:
            assert tuple(c.shape) == (p.shape[0], 4, 4)
        self._check(self._L.sgb_source_set_points(self._h, p.shape[0], _d(p), _d(c)))

    @property
    def source_size(self):
        return int(self._L.sgb_source_size(self._h))

    # ---- hot path ----
    def linearize(self, T, factor=FACTOR_GICP, robust=ROBUST_NONE, robust_c=1.0, rejector=REJECT_DISTANCE, max_dist_sq=1.0):
        """Reduction::linearize -> (H 6x6, b 6, e)"""
        Tc = _pose(T)
        out = np.empty(43)
        self._check(self._L.sgb_linearize(self._h, factor, robust, float(robust_c), rejector, float(max_dist_sq), _d(Tc), _d(out)))
        return out[:36].reshape(6, 6).copy(), out[36:42].copy(), float(out[42])

    def error(self, T):
        Tc = _pose(T)
        e = C.c_double(0.0)
        self._check(self._L.sgb_error(self._h, _d(Tc), C.byref(e)))
        return e.value

    def linearize_device(self, T, d_out_ptr, factor=FACTOR_GICP, robust=ROBUST_NONE, robust_c=1.0, rejector=REJECT_DISTANCE, max_dist_sq=1.0):
        """asynchronous; d_out_ptr = device address of >= 44 doubles (H | b | e | num_inliers)"""
        Tc = _pose(T)
        self._check(self._L.sgb_linearize_device(self._h, factor, robust, float(robust_c), rejector, float(max_dist_sq), _d(Tc), _vp(d_out_ptr)))

    def error_device(self, T, d_out_ptr):
        Tc = _pose(T)
        self._check(self._L.sgb_error_device(self._h, _d(Tc), _vp(d_out_ptr)))

    def correspondences(self):
        out = np.empty(self.source_size, dtype=np.uint64)
        self._check(self._L.sgb_correspondences(self._h, out.ctypes.data_as(_u64p)))
        return out

    # ---- batched registration: many sources ("members") against the one target, each at its own pose ----
    def set_source_batch(self, sources, covs=None):
        """sources: a list of (N_m, 3|4) arrays, or (points (N, 3|4), offsets (B + 1,)) with the members concatenated.
        covs: None, a list of (N_m, 4, 4) arrays, or one (N, 4, 4) array."""
        if isinstance(sources, tuple):
            points, offsets = sources
            p = _points4(points)
            offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
            if offsets.ndim != 1 or offsets.size < 1 or int(offsets[-1]) != p.shape[0]:
                raise SgbError(f"set_source_batch: offsets must have B + 1 entries ending at the point count {p.shape[0]}")
        else:
            members = [_points4(s) for s in sources]
            offsets = np.zeros(len(members) + 1, dtype=np.uint64)
            offsets[1:] = np.cumsum([m.shape[0] for m in members])
            p = np.concatenate(members) if members else np.zeros((0, 4))
        c = None
        if covs is not None:
            c = _f64(covs) if not isinstance(covs, (list, tuple)) else (np.concatenate([_f64(x) for x in covs]) if len(covs) else np.zeros((0, 4, 4)))
            assert tuple(c.shape) == (p.shape[0], 4, 4)
        offsets = offsets.astype(np.uintp)
        self._check(self._L.sgb_source_set_batch(self._h, offsets.size - 1, offsets.ctypes.data_as(C.POINTER(C.c_size_t)), _d(p), _d(c)))
        self._batch_offsets = offsets.astype(np.int64)
        self._cloud_offsets = self._batch_offsets

    def set_source_pairs(self, clouds=None, maps=None):
        """the batch's members become (cloud, map) pairs of the clouds of the last set_source_batch, without a new upload: member p is
        cloud clouds[p] (None: cloud p, one member per cloud) aligned against map maps[p] of a many-maps / many-kd-trees target (None:
        map p, or the one target).  The batched calls then take and return one pose / result per member."""
        cl = None if clouds is None else np.ascontiguousarray(clouds, dtype=np.uint32).reshape(-1)
        mp = None if maps is None else np.ascontiguousarray(maps, dtype=np.uint32).reshape(-1)
        n_clouds = self._cloud_offsets.size - 1 if hasattr(self, "_cloud_offsets") else 0
        P = cl.size if cl is not None else (mp.size if mp is not None else n_clouds)
        if cl is not None and mp is not None and mp.size != P:
            raise SgbError(f"set_source_pairs: {cl.size} clouds but {mp.size} maps")
        u32p = C.POINTER(C.c_uint32)
        self._check(self._L.sgb_source_set_pairs(self._h, P, None if cl is None else cl.ctypes.data_as(u32p), None if mp is None else mp.ctypes.data_as(u32p)))
        sizes = np.diff(self._cloud_offsets)
        self._batch_offsets = np.concatenate([[0], np.cumsum(sizes[cl] if cl is not None else sizes)]).astype(np.int64)

    def set_source_submaps(self, lists, poses=None, clouds=None):
        """the batch's members become (cloud, submap) pairs: member p is cloud clouds[p] (None: cloud p) aligned against the union of the
        maps lists[p] (map indices of a many-kd-trees target), map lists[p][j] placed by the rigid 4x4 pose poses[p][j] (map -> common
        frame; poses None: all identity).  Each map stays as built; ICP and GICP.  The batched calls then take and return one pose per
        member, source -> common frame, and correspondences_batch reports (entry within the list) << 32 | index within that map."""
        lists = [np.asarray(l, dtype=np.uint32).reshape(-1) for l in lists]
        P = len(lists)
        off = np.zeros(P + 1, dtype=np.uintp)
        off[1:] = np.cumsum([l.size for l in lists])
        maps = np.ascontiguousarray(np.concatenate(lists) if P else np.zeros(0), dtype=np.uint32)
        pc = None
        if poses is not None:
            if len(poses) != P or any(len(poses[p]) != lists[p].size for p in range(P)):
                raise SgbError("set_source_submaps: one pose per list entry")
            flat = [np.asarray(T, dtype=np.float64).reshape(4, 4).T for p in range(P) for T in poses[p]]  # column-major
            pc = np.ascontiguousarray(np.array(flat).reshape(-1, 16)) if flat else np.zeros((1, 16))
        cl = None if clouds is None else np.ascontiguousarray(clouds, dtype=np.uint32).reshape(-1)
        if cl is not None and cl.size != P:
            raise SgbError(f"set_source_submaps: {cl.size} clouds but {P} lists")
        u32p = C.POINTER(C.c_uint32)
        self._check(self._L.sgb_source_set_submaps(self._h, P, None if cl is None else cl.ctypes.data_as(u32p), off.ctypes.data_as(C.POINTER(C.c_size_t)),
                                                   maps.ctypes.data_as(u32p), _d(pc)))
        sizes = np.diff(self._cloud_offsets)
        self._batch_offsets = np.concatenate([[0], np.cumsum(sizes[cl] if cl is not None else sizes)]).astype(np.int64)

    def set_source_weights(self, w):
        """per-point weights of every batched call (sgb_source_set_weights): w (N,) float64 in the row layout of correspondences_batch
        (member m's rows are offsets m .. m + 1, in its cloud's original order), a numpy array or a contiguous float64 torch tensor (CUDA on
        the context's device, or host / page-locked); None clears them.  Each point's H | b | e (and its error() share) is multiplied by its
        weight after the robust kernel; correspondences and num_inliers do not change.  Every weight must be finite and >= 0, else the call
        fails naming the row and the weights in force stay.  set_source_batch / _pairs / _submaps / set_source clear the weights."""
        if w is None:
            self._check(self._L.sgb_source_set_weights(self._h, None))
            return
        offsets = getattr(self, "_batch_offsets", None)
        n = int(offsets[-1]) if offsets is not None else None
        if _is_dev(w):
            import torch

            if w.dtype != torch.float64 or not w.is_contiguous():
                raise SgbError("set_source_weights: a torch tensor of weights must be contiguous float64")
            if w.is_cuda and w.device.index != self.device:
                raise SgbError(f"set_source_weights: the weights are on {w.device}, the context on cuda:{self.device}")
        else:
            w = np.ascontiguousarray(w, dtype=np.float64)
        if n is not None and tuple(w.shape) != (n,):
            raise SgbError(f"set_source_weights: need ({n},) weights, one per member point in the layout of correspondences_batch; got {tuple(w.shape)}")
        self._check(self._L.sgb_source_set_weights(self._h, _d(w)))

    def _batch_args(self, Ts, active):
        Ts = np.asarray(Ts, dtype=np.float64)
        B = self._batch_offsets.size - 1
        assert Ts.shape == (B, 4, 4), f"need ({B}, 4, 4) poses"
        Tc = np.ascontiguousarray(Ts.transpose(0, 2, 1))  # each pose column-major
        a = None if active is None else np.ascontiguousarray(np.asarray(active).astype(np.uint8).reshape(B))
        return B, Tc, a, (None if a is None else a.ctypes.data_as(C.POINTER(C.c_uint8)))

    def linearize_batch(self, Ts, active=None, factor=FACTOR_GICP, robust=ROBUST_NONE, robust_c=1.0, rejector=REJECT_DISTANCE, max_dist_sq=1.0):
        """Reduction::linearize of every member at its pose -> (H (B,6,6), b (B,6), e (B,), inliers (B,)); inactive members: zeros.  The
        weights in force (set_source_weights) apply."""
        B, Tc, a, ap = self._batch_args(Ts, active)
        out = np.zeros((max(B, 1), 44))
        self._check(self._L.sgb_linearize_batch(self._h, factor, robust, float(robust_c), rejector, float(max_dist_sq), _d(Tc), ap, _d(out)))
        out = out[:B]
        return out[:, :36].reshape(B, 6, 6).copy(), out[:, 36:42].copy(), out[:, 42].copy(), out[:, 43].astype(np.int64)

    def error_batch(self, Ts, active=None):
        """Reduction::error of every active member at its trial pose (cached correspondences) -> (B,); the weights in force apply"""
        B, Tc, a, ap = self._batch_args(Ts, active)
        out = np.zeros(max(B, 1))
        self._check(self._L.sgb_error_batch(self._h, _d(Tc), ap, _d(out)))
        return out[:B].copy()

    def _rows(self, out, cols, who):
        """a per-point output: a new numpy array, or `out` (numpy or torch, CUDA tensors included) checked for shape and layout"""
        n = int(self._batch_offsets[-1])
        shape = (n,) if cols == 1 else (n, cols)
        if out is None:
            return np.zeros((max(n, 1),) + shape[1:])[:n]
        if tuple(out.shape) != shape:
            raise SgbError(f"{who}: the per-point output must have shape {shape}")
        if _is_dev(out):
            _f64(out)
        elif not (out.dtype == np.float64 and out.flags.c_contiguous):
            raise SgbError(f"{who}: the per-point output must be contiguous float64")
        return out

    def linearize_batch_points(self, Ts, active=None, factor=FACTOR_GICP, robust=ROBUST_NONE, robust_c=1.0, rejector=REJECT_DISTANCE, max_dist_sq=1.0,
                               hessians=True, out_e=None, out_Hb42=None):
        """linearize_batch plus every source point's terms (sgb_linearize_batch_points) -> BatchPointTerms.  The member sums are
        bit-identical to linearize_batch's.  point_e = the point's w e, point_H / point_b its J^T M J / J^T M r (robust-weighted); zero rows
        for rejected or unmatched points and inactive members.  hessians=False: point_e only (H | b rows not computed).  out_e (N,) and
        out_Hb42 (N, 42): float64 outputs to write in place (numpy, or CUDA tensors on the context's device, written by the kernel).  With
        weights in force (set_source_weights) the rows are the weighted terms."""
        B, Tc, a, ap = self._batch_args(Ts, active)
        e_rows = self._rows(out_e, 1, "linearize_batch_points")
        hb_rows = self._rows(out_Hb42, 42, "linearize_batch_points") if hessians else None
        out = np.zeros((max(B, 1), 44))
        self._check(self._L.sgb_linearize_batch_points(self._h, factor, robust, float(robust_c), rejector, float(max_dist_sq), _d(Tc), ap, _d(out),
                                                       _d(e_rows), _d(hb_rows)))
        out = out[:B]
        return BatchPointTerms(out[:, :36].reshape(B, 6, 6).copy(), out[:, 36:42].copy(), out[:, 42].copy(), out[:, 43].astype(np.int64),
                               self._batch_offsets.copy(), e_rows, hb_rows)

    def error_batch_points(self, Ts, active=None, out_e=None):
        """error_batch plus every source point's share of its member's e (sgb_error_batch_points) -> (e (B,), point_e (N,)), point_e in the
        layout of correspondences_batch; out_e as in linearize_batch_points; the weights in force apply to both"""
        B, Tc, a, ap = self._batch_args(Ts, active)
        e_rows = self._rows(out_e, 1, "error_batch_points")
        out = np.zeros(max(B, 1))
        self._check(self._L.sgb_error_batch_points(self._h, _d(Tc), ap, _d(out), _d(e_rows)))
        return out[:B].copy(), e_rows

    def correspondences_batch(self):
        """list of per-member correspondence arrays (original target indices, NO_CORRESPONDENCE = rejected)"""
        off = self._batch_offsets
        out = np.empty(max(int(off[-1]), 1), dtype=np.uint64)
        self._check(self._L.sgb_correspondences_batch(self._h, out.ctypes.data_as(_u64p)))
        return [out[off[m] : off[m + 1]].copy() for m in range(off.size - 1)]

    def align_batch(self, init_Ts, factor=FACTOR_GICP, robust=ROBUST_NONE, robust_c=1.0, rejector=REJECT_DISTANCE, max_dist_sq=1.0,
                    optimizer=OPT_LEVENBERG_MARQUARDT, max_iterations=20, gn_lambda=1e-6, max_inner_iterations=10, init_lambda=1e-3,
                    lambda_factor=10.0, rotation_eps=0.1 * np.pi / 180.0, translation_eps=1e-3, dof_mask=None):
        """Registration<...>::align of every member from its initial pose (sgb_align_batch) -> a Result with per-member arrays
        T_target_source (B,4,4), converged (B,) bool, iterations (B,), num_inliers (B,), error (B,), H (B,6,6), b (B,6).  The weights in
        force (set_source_weights) apply to every round."""
        B, Tc, _, _ = self._batch_args(init_Ts, None)
        o = _align_options(factor, robust, robust_c, rejector, max_dist_sq, optimizer, max_iterations, gn_lambda, max_inner_iterations, init_lambda,
                           lambda_factor, rotation_eps, translation_eps, dof_mask)
        T = np.zeros((max(B, 1), 16))
        info = np.zeros((max(B, 1), 4))
        Hb = np.zeros((max(B, 1), 42))
        self._check(self._L.sgb_align_batch(self._h, C.byref(o), _d(Tc), _d(T), _d(info), _d(Hb)))
        return BatchAlignResult(T[:B], info[:B], Hb[:B])

    def align_batch_gnc(self, init_Ts, noise_bound_sq, gnc=GNC_TLS, max_stages=64, stage_iterations=3, point_weights=False, **align):
        """Graduated non-convexity over every member (sgb_align_batch_gnc) -> a GncAlignResult.  Each stage re-estimates every point's weight
        g on the device from its residual r^2 = 2 e at the member's pose (gnc: GNC_GEMAN_MCCLURE or GNC_TLS, noise_bound_sq = c^2 on that
        scale), then runs align_batch from there with the weights w * g (w: the weights in force, which the call leaves unchanged) and
        max_iterations = stage_iterations, or align's max_iterations at the member's last stage.  At most max_stages stages.
        point_weights=True: each point's final g too.  align: the keywords of align_batch (robust must stay ROBUST_NONE)."""
        B, Tc, _, _ = self._batch_args(init_Ts, None)
        o = _align_options(**align)
        g = GncOptions(int(gnc), float(noise_bound_sq), int(max_stages), int(stage_iterations))
        T = np.zeros((max(B, 1), 16))
        info = np.zeros((max(B, 1), 4))
        Hb = np.zeros((max(B, 1), 42))
        gnc2 = np.zeros((max(B, 1), 2))
        pw = np.zeros(max(int(self._batch_offsets[-1]), 1)) if point_weights else None
        self._check(self._L.sgb_align_batch_gnc(self._h, C.byref(o), C.byref(g), _d(Tc), _d(T), _d(info), _d(Hb), _d(gnc2), _d(pw)))
        return GncAlignResult(T[:B], info[:B], Hb[:B], gnc2[:B], None if pw is None else pw[: int(self._batch_offsets[-1])])

    def align_joint(self, init_X, windows=None, fixed=None, factor=FACTOR_GICP, robust=ROBUST_NONE, robust_c=1.0, rejector=REJECT_DISTANCE, max_dist_sq=1.0,
                    optimizer=OPT_LEVENBERG_MARQUARDT, max_iterations=20, gn_lambda=1e-6, max_inner_iterations=10, init_lambda=1e-3,
                    lambda_factor=10.0, rotation_eps=0.1 * np.pi / 180.0, translation_eps=1e-3, dof_mask=None):
        """Joint registration of windows of frames (sgb_align_joint) -> a JointAlignResult.  Frame k is cloud k of set_source_batch with map k
        of the many-maps target; the edges are the members of set_source_pairs(clouds, maps), edge p = cloud clouds[p] against map maps[p] at
        X_j^-1 X_i.  init_X (K,4,4) row-major frame poses; windows: the window offsets (W + 1,) from 0 to K (None: one window of all
        frames); fixed (K,) flags of frames held at their initial pose (None: the first frame of each window); the other keywords as in
        align_batch.  The weights in force (set_source_weights, one per edge point) apply."""
        K, Xc, off, fx = self._joint_args(init_X, windows, fixed, "align_joint")
        W = off.size - 1
        o = _align_options(factor, robust, robust_c, rejector, max_dist_sq, optimizer, max_iterations, gn_lambda, max_inner_iterations, init_lambda,
                           lambda_factor, rotation_eps, translation_eps, dof_mask)
        out = np.zeros((max(K, 1), 16))
        info = np.zeros((max(W, 1), 4))
        self._check(self._L.sgb_align_joint(self._h, C.byref(o), W, off.ctypes.data_as(C.POINTER(C.c_size_t)),
                                            None if fx is None else fx.ctypes.data_as(C.POINTER(C.c_uint8)), _d(Xc), _d(out), _d(info)))
        return JointAlignResult(out[:K], info[:W])

    def _joint_args(self, X, windows, fixed, who):
        """the column-major frame poses, window offsets and fixed flags of a joint call"""
        X = np.asarray(X, dtype=np.float64)
        K = self._cloud_offsets.size - 1 if hasattr(self, "_cloud_offsets") else 0
        if X.shape != (K, 4, 4):
            raise SgbError(f"{who}: need ({K}, 4, 4) frame poses")
        off, fx = _windows(windows, fixed, K, who)
        return K, np.ascontiguousarray(X.transpose(0, 2, 1)), off, fx

    def joint_edge_poses(self, X, windows=None):
        """The edge poses the joint aligns linearise at (sgb_joint_edge_poses) -> (E, 4, 4) row-major, T_p = X_j^-1 X_i for pairing member p
        (cloud i against map j), computed on the device with the joint align's own kernel: bit for bit the poses align_joint and
        align_joint_gnc use, ready for linearize_batch_points.  X (K,4,4) row-major frame poses; windows as in align_joint."""
        K, Xc, off, _ = self._joint_args(X, windows, None, "joint_edge_poses")
        E = self._batch_offsets.size - 1
        out = np.zeros((max(E, 1), 16))
        self._check(self._L.sgb_joint_edge_poses(self._h, off.size - 1, off.ctypes.data_as(C.POINTER(C.c_size_t)), _d(Xc), _d(out)))
        return np.ascontiguousarray(out[:E].reshape(E, 4, 4).transpose(0, 2, 1))

    def align_joint_gnc(self, init_X, noise_bound_sq, windows=None, fixed=None, gnc=GNC_TLS, max_stages=64, stage_iterations=3, point_weights=False,
                        **align):
        """Graduated non-convexity over joint windows (sgb_align_joint_gnc) -> a JointGncAlignResult.  Per window, each stage re-estimates every
        edge point's weight g on the device from its residual r^2 = 2 e at the window's edge poses (one mu per window; gnc: GNC_GEMAN_MCCLURE
        or GNC_TLS, noise_bound_sq = c^2 on that scale), then runs align_joint from there with the weights w * g (w: the weights in force,
        which the call leaves unchanged) and max_iterations = stage_iterations, or align's max_iterations at the window's last stage.  At
        most max_stages stages.  point_weights=True: each point's final g too.  init_X, windows and fixed as in align_joint; align: the
        keywords of align_joint (robust must stay ROBUST_NONE)."""
        K, Xc, off, fx = self._joint_args(init_X, windows, fixed, "align_joint_gnc")
        W = off.size - 1
        o = _align_options(**align)
        g = GncOptions(int(gnc), float(noise_bound_sq), int(max_stages), int(stage_iterations))
        out = np.zeros((max(K, 1), 16))
        info = np.zeros((max(W, 1), 4))
        gnc2 = np.zeros((max(W, 1), 2))
        n = int(self._batch_offsets[-1]) if hasattr(self, "_batch_offsets") else 0
        pw = np.zeros(max(n, 1)) if point_weights else None
        self._check(self._L.sgb_align_joint_gnc(self._h, C.byref(o), C.byref(g), W, off.ctypes.data_as(C.POINTER(C.c_size_t)),
                                                None if fx is None else fx.ctypes.data_as(C.POINTER(C.c_uint8)), _d(Xc), _d(out), _d(info), _d(gnc2),
                                                _d(pw)))
        return JointGncAlignResult(out[:K], info[:W], gnc2[:W], None if pw is None else pw[:n])

    def align_batch_async(self, init_Ts, factor=FACTOR_GICP, robust=ROBUST_NONE, robust_c=1.0, rejector=REJECT_DISTANCE, max_dist_sq=1.0,
                          optimizer=OPT_LEVENBERG_MARQUARDT, max_iterations=20, gn_lambda=1e-6, max_inner_iterations=10, init_lambda=1e-3,
                          lambda_factor=10.0, rotation_eps=0.1 * np.pi / 180.0, translation_eps=1e-3, dof_mask=None, out=None):
        """align_batch enqueued on the context's stream without a host synchronisation (sgb_align_batch_async).  init_Ts: CUDA float64
        (B, 4, 4) row-major, on the context's device; the context's stream must have been set (set_stream) to a torch stream, on which the
        poses are transposed into the library's column-major layout.  Returns an AsyncAlignResult of CUDA tensors (out: a previous result
        whose buffers are reused).  Inside torch.cuda.graph (with the capture stream set) the align is captured: each replay re-runs it
        from what init_Ts holds then, with the weights in force then (set_source_weights)."""

        def outputs(B, N, zeros):
            if out is None:
                return AsyncAlignResult(zeros(B, 16), zeros(B, 4), zeros(B, 42))
            if tuple(out.T16.shape) != (B, 16):
                raise SgbError(f"align_batch_async: out holds {out.T16.shape[0]} members, the batch {B}")
            return out

        res = self._batch_async_in(init_Ts, "align_batch_async", outputs)
        o = _align_options(factor, robust, robust_c, rejector, max_dist_sq, optimizer, max_iterations, gn_lambda, max_inner_iterations, init_lambda,
                           lambda_factor, rotation_eps, translation_eps, dof_mask)
        self._check(self._L.sgb_align_batch_async(self._h, C.byref(o), _d(self._async_in), _d(res.T16), _d(res.info4), _d(res.Hb42)))
        return res

    def _batch_async_in(self, init_Ts, who, outputs):
        """the outputs of a stream-ordered batch call, with init_Ts transposed into _async_in (column-major) on the context's stream;
        outputs(B, N, zeros) returns the call's result buffers for B members of N points in all, zeros(rows, cols) a new float64 tensor there"""
        import torch

        if self._stream is None:
            raise SgbError(f"{who}: set the context's stream to a torch stream first (set_stream): the poses are prepared on it")
        offsets = getattr(self, "_batch_offsets", None)  # (no batch yet: the library says so)
        B = int(offsets.size) - 1 if offsets is not None else int(init_Ts.shape[0])
        N = int(offsets[-1]) if offsets is not None else 0
        if not (isinstance(init_Ts, torch.Tensor) and init_Ts.is_cuda and init_Ts.dtype == torch.float64 and tuple(init_Ts.shape) == (B, 4, 4)):
            raise SgbError(f"{who}: init_Ts must be a CUDA float64 tensor of shape ({B}, 4, 4)")
        dev = init_Ts.device
        with torch.cuda.stream(torch.cuda.ExternalStream(self._stream, device=dev)):
            res = outputs(B, N, lambda rows, cols: torch.zeros((max(rows, 1), cols), dtype=torch.float64, device=dev)[:rows])
            if self._async_in is None or self._async_in.shape[0] != B or self._async_in.device != dev:
                self._async_in = torch.empty((max(B, 1), 16), dtype=torch.float64, device=dev)[:B]
            self._async_in.view(B, 4, 4).copy_(init_Ts.transpose(1, 2))  # column-major
        return res

    def align_batch_gnc_async(self, init_Ts, noise_bound_sq, gnc=GNC_TLS, max_stages=64, stage_iterations=3, point_weights=False, out=None, **align):
        """align_batch_gnc enqueued on the context's stream without a host synchronisation (sgb_align_batch_gnc_async): every stage and round
        runs on the device.  init_Ts and the stream as in align_batch_async; the other arguments as in align_batch_gnc.  Returns an
        AsyncGncAlignResult of CUDA tensors (out: a previous result whose buffers are reused; it must hold point_w if point_weights).  Inside
        torch.cuda.graph (with the capture stream set) the whole GNC is captured: each replay re-runs it from what init_Ts holds then, with
        the weights in force then (set_source_weights)."""

        def outputs(B, N, zeros):
            if out is None:
                return AsyncGncAlignResult(zeros(B, 16), zeros(B, 4), zeros(B, 42), zeros(B, 2), zeros(N, 1)[:, 0] if point_weights else None)
            if tuple(out.T16.shape) != (B, 16):
                raise SgbError(f"align_batch_gnc_async: out holds {out.T16.shape[0]} members, the batch {B}")
            if point_weights and (out.point_w is None or tuple(out.point_w.shape) != (N,)):
                raise SgbError(f"align_batch_gnc_async: point_weights needs out.point_w of {N} rows")
            return out

        res = self._batch_async_in(init_Ts, "align_batch_gnc_async", outputs)
        o = _align_options(**align)
        g = GncOptions(int(gnc), float(noise_bound_sq), int(max_stages), int(stage_iterations))
        pw = res.point_w if point_weights else None
        self._check(self._L.sgb_align_batch_gnc_async(self._h, C.byref(o), C.byref(g), _d(self._async_in), _d(res.T16), _d(res.info4), _d(res.Hb42),
                                                      _d(res.gnc2), _d(pw)))
        return res

    def align_joint_async(self, init_X, windows=None, fixed=None, factor=FACTOR_GICP, robust=ROBUST_NONE, robust_c=1.0, rejector=REJECT_DISTANCE,
                          max_dist_sq=1.0, optimizer=OPT_LEVENBERG_MARQUARDT, max_iterations=20, gn_lambda=1e-6, max_inner_iterations=10, init_lambda=1e-3,
                          lambda_factor=10.0, rotation_eps=0.1 * np.pi / 180.0, translation_eps=1e-3, dof_mask=None, out=None):
        """align_joint enqueued on the context's stream without a host synchronisation (sgb_align_joint_async).  init_X: CUDA float64 (K, 4, 4)
        row-major frame poses on the context's device, transposed on the context's stream (set_stream: a torch stream); windows, fixed and the
        other keywords as in align_joint.  Returns an AsyncJointAlignResult of CUDA tensors (out: a previous result whose buffers are reused).
        Inside torch.cuda.graph (with the capture stream set) the align is captured: each replay re-runs it from what init_X holds then.
        The weights in force (set_source_weights) apply, at a replay those in force then."""
        o = _align_options(factor, robust, robust_c, rejector, max_dist_sq, optimizer, max_iterations, gn_lambda, max_inner_iterations, init_lambda,
                           lambda_factor, rotation_eps, translation_eps, dof_mask)

        def outputs(K, W, zeros):
            if out is None:
                return AsyncJointAlignResult(zeros(K, 16), zeros(W, 4))
            if tuple(out.X16.shape) != (K, 16) or tuple(out.info4.shape) != (W, 4):
                raise SgbError(f"align_joint_async: out holds {out.X16.shape[0]} frames and {out.info4.shape[0]} windows, the call {K} and {W}")
            return out

        W, off, fx, res = self._joint_async_in(init_X, windows, fixed, "align_joint_async", outputs)
        self._check(self._L.sgb_align_joint_async(self._h, C.byref(o), W, off.ctypes.data_as(C.POINTER(C.c_size_t)),
                                                  None if fx is None else fx.ctypes.data_as(C.POINTER(C.c_uint8)), _d(self._joint_in), _d(res.X16),
                                                  _d(res.info4)))
        return res

    def _joint_async_in(self, init_X, windows, fixed, who, outputs):
        """the window offsets, fixed flags and outputs of a stream-ordered joint call, with init_X transposed into _joint_in (column-major) on
        the context's stream; outputs(K, W, zeros) returns the call's result buffers, zeros(rows, cols) a new float64 tensor there"""
        import torch

        if self._stream is None:
            raise SgbError(f"{who}: set the context's stream to a torch stream first (set_stream): the poses are prepared on it")
        K = self._cloud_offsets.size - 1 if hasattr(self, "_cloud_offsets") else 0
        if not (isinstance(init_X, torch.Tensor) and init_X.is_cuda and init_X.dtype == torch.float64 and tuple(init_X.shape) == (K, 4, 4)):
            raise SgbError(f"{who}: init_X must be a CUDA float64 tensor of shape ({K}, 4, 4)")
        off, fx = _windows(windows, fixed, K, who)
        W = off.size - 1
        dev = init_X.device
        with torch.cuda.stream(torch.cuda.ExternalStream(self._stream, device=dev)):
            res = outputs(K, W, lambda rows, cols: torch.zeros((max(rows, 1), cols), dtype=torch.float64, device=dev)[:rows])
            if self._joint_in is None or self._joint_in.shape[0] != K or self._joint_in.device != dev:
                self._joint_in = torch.empty((max(K, 1), 16), dtype=torch.float64, device=dev)[:K]
            self._joint_in.view(K, 4, 4).copy_(init_X.transpose(1, 2))  # column-major
        return W, off, fx, res

    def align_joint_gnc_async(self, init_X, noise_bound_sq, windows=None, fixed=None, gnc=GNC_TLS, max_stages=64, stage_iterations=3, point_weights=False,
                              out=None, **align):
        """align_joint_gnc enqueued on the context's stream without a host synchronisation (sgb_align_joint_gnc_async): every stage and joint
        round runs on the device.  init_X and the stream as in align_joint_async; the other arguments as in align_joint_gnc.  Returns an
        AsyncJointGncAlignResult of CUDA tensors (out: a previous result whose buffers are reused; it must hold point_w if point_weights).
        Inside torch.cuda.graph (with the capture stream set) the whole GNC is captured: each replay re-runs it from what init_X holds then,
        with the weights in force then (set_source_weights)."""
        o = _align_options(**align)
        g = GncOptions(int(gnc), float(noise_bound_sq), int(max_stages), int(stage_iterations))
        N = int(self._batch_offsets[-1]) if hasattr(self, "_batch_offsets") else 0

        def outputs(K, W, zeros):
            if out is None:
                return AsyncJointGncAlignResult(zeros(K, 16), zeros(W, 4), zeros(W, 2), zeros(N, 1)[:, 0] if point_weights else None)
            if tuple(out.X16.shape) != (K, 16) or tuple(out.info4.shape) != (W, 4):
                raise SgbError(f"align_joint_gnc_async: out holds {out.X16.shape[0]} frames and {out.info4.shape[0]} windows, the call {K} and {W}")
            if point_weights and (out.point_w is None or tuple(out.point_w.shape) != (N,)):
                raise SgbError(f"align_joint_gnc_async: point_weights needs out.point_w of {N} rows")
            return out

        W, off, fx, res = self._joint_async_in(init_X, windows, fixed, "align_joint_gnc_async", outputs)
        pw = res.point_w if point_weights else None
        self._check(self._L.sgb_align_joint_gnc_async(self._h, C.byref(o), C.byref(g), W, off.ctypes.data_as(C.POINTER(C.c_size_t)),
                                                      None if fx is None else fx.ctypes.data_as(C.POINTER(C.c_uint8)), _d(self._joint_in), _d(res.X16),
                                                      _d(res.info4), _d(res.gnc2), _d(pw)))
        return res

    # ---- multi-GPU: all-reduce of H|b|e fused into the reduction kernel (peer memory over NVLink) ----
    COMM_HANDLE_BYTES = 64

    def comm_handle(self):
        """64-byte CUDA IPC handle of this context's mailbox (to be all-gathered across the ranks)"""
        buf = (C.c_ubyte * self.COMM_HANDLE_BYTES)()
        self._check(self._L.sgb_comm_handle(self._h, C.cast(buf, _vp)))
        return bytes(buf)

    def comm_connect(self, rank, world, handles):
        """handles: world x 64 bytes in rank order; afterwards linearize()/error() return the sum over all ranks"""
        blob = b"".join(handles) if not isinstance(handles, (bytes, bytearray)) else bytes(handles)
        assert len(blob) == world * self.COMM_HANDLE_BYTES
        buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
        self._check(self._L.sgb_comm_connect(self._h, int(rank), int(world), C.cast(buf, _vp)))

    def comm_mailbox(self):
        """device address of this context's mailbox (wiring contexts of one process: tests)"""
        p = _vp()
        self._check(self._L.sgb_comm_mailbox(self._h, C.byref(p)))
        return int(p.value)

    def comm_connect_ptrs(self, rank, world, mailboxes):
        arr = (_vp * world)(*[_vp(int(m)) for m in mailboxes])
        self._check(self._L.sgb_comm_connect_ptrs(self._h, int(rank), int(world), arr))

    def comm_disconnect(self):
        self._check(self._L.sgb_comm_disconnect(self._h))

    def comm_set_timeout_ms(self, ms):
        self._check(self._L.sgb_comm_set_timeout_ms(self._h, int(ms)))

    def comm_status(self):
        """0 = fine, bit 0 = an exchange gave up on a peer, bit 1 = a peer reported a failed call (sticky until the next connect)"""
        st = C.c_int(0)
        self._check(self._L.sgb_comm_status(self._h, C.byref(st)))
        return int(st.value)

    def comm_wait_ns(self):
        """(ring of the last 64 exchanges' waiting times in ns indexed by call number % 64, number of exchanges so far)"""
        ring = np.zeros(64, dtype=np.uint64)
        calls = C.c_uint64(0)
        self._check(self._L.sgb_comm_wait_ns(self._h, ring.ctypes.data_as(_u64p), C.byref(calls)))
        return ring, int(calls.value)

    def drop_seeds(self):
        self._check(self._L.sgb_drop_seeds(self._h))

    def num_inliers(self):
        n = C.c_size_t(0)
        self._check(self._L.sgb_num_inliers(self._h, C.byref(n)))
        return int(n.value)

    # ---- per-cloud preparation on the device ----
    def estimate_features(self, points, num_neighbors=20, normals=True, covs=True):
        """estimate_normals_covariances (util/normal_estimation.hpp): returns (normals (N,4) | None, covs (N,4,4) | None)"""
        p = _points4(points)
        if _is_dev(p) and p.is_cuda:  # device in, device out
            import torch

            n_out = torch.empty((p.shape[0], 4), dtype=torch.float64, device=p.device) if normals else None
            c_out = torch.empty((p.shape[0], 4, 4), dtype=torch.float64, device=p.device) if covs else None
        else:
            n_out = np.empty((p.shape[0], 4)) if normals else None
            c_out = np.empty((p.shape[0], 4, 4)) if covs else None
        self._check(self._L.sgb_estimate_features(self._h, p.shape[0], _d(p), int(num_neighbors), _d(n_out), _d(c_out)))
        return n_out, c_out

    def estimate_target_features(self, num_neighbors=20):
        self._check(self._L.sgb_target_estimate_features(self._h, int(num_neighbors)))

    def estimate_source_features(self, num_neighbors=20):
        self._check(self._L.sgb_source_estimate_features(self._h, int(num_neighbors)))

    def adopt_source_as_target(self):
        """frame streams: the current source (points, its device-built tree, covariances) becomes the target; no source afterwards"""
        self._check(self._L.sgb_target_adopt_source(self._h))

    def voxelgrid_sampling(self, points, leaf_size):
        """voxelgrid_sampling (util/downsampling.hpp:22-78): returns the (M,4) down-sampled points"""
        p = _points4(points)
        out = np.empty_like(p)
        m = C.c_size_t(0)
        self._check(self._L.sgb_voxelgrid_sampling(self._h, p.shape[0], _d(p), float(leaf_size), _d(out), C.byref(m)))
        return out[: int(m.value)].copy()

    # ---- many clouds at once (frames of a sequence): plain concatenated arrays in the caller's order ----
    @staticmethod
    def _clouds(points_list, who):
        """a list of (N_m, 3|4) clouds, or (points (N, 3|4), offsets (B + 1,)) -> (points (N, 4), offsets as size_t); CUDA tensors stay
        on the device"""
        if isinstance(points_list, tuple):
            points, offsets = points_list
            p = _points4(points)
            offsets = np.ascontiguousarray(offsets.cpu().numpy() if _is_dev(offsets) else offsets, dtype=np.uintp)
            if offsets.ndim != 1 or offsets.size < 1 or int(offsets[-1]) != p.shape[0]:
                raise SgbError(f"{who}: offsets must have B + 1 entries ending at the point count {p.shape[0]}")
            return p, offsets
        members = [_points4(x) for x in points_list]
        offsets = np.zeros(len(members) + 1, dtype=np.uintp)
        offsets[1:] = np.cumsum([m.shape[0] for m in members])
        if members and all(_is_dev(m) for m in members):
            import torch

            return torch.cat(members).contiguous(), offsets
        p = np.concatenate([m.cpu().numpy() if _is_dev(m) else m for m in members]) if members else np.zeros((0, 4))
        return np.ascontiguousarray(p), offsets

    def voxelgrid_sampling_batch(self, points_list, leaf_size):
        """voxelgrid_sampling of every cloud in one call: points_list as for build_target_voxelmaps.  Returns (points (M, 4), offsets
        (B + 1,) int64): cloud c's voxels are points[offsets[c]:offsets[c+1]], bit-identical to voxelgrid_sampling of that cloud alone.
        CUDA tensors in give a CUDA tensor out."""
        p, offsets = self._clouds(points_list, "voxelgrid_sampling_batch")
        out = p.new_empty(p.shape) if _is_dev(p) else np.empty_like(p)
        out_off = np.zeros(offsets.size, dtype=np.uintp)
        self._check(self._L.sgb_voxelgrid_sampling_batch(self._h, offsets.size - 1, offsets.ctypes.data_as(C.POINTER(C.c_size_t)), _d(p), float(leaf_size),
                                                         _d(out), out_off.ctypes.data_as(C.POINTER(C.c_size_t))))
        m = int(out_off[-1])
        return (out[:m].clone() if _is_dev(out) else out[:m].copy()), out_off.astype(np.int64)

    def estimate_features_batch(self, points_list, num_neighbors=20, normals=True, covs=True):
        """estimate_features of every cloud in one call: points_list as for build_target_voxelmaps.  Returns (normals (N, 4) | None,
        covs (N, 4, 4) | None) in the concatenated order; CUDA tensors in give CUDA tensors out."""
        p, offsets = self._clouds(points_list, "estimate_features_batch")
        if _is_dev(p) and p.is_cuda:
            import torch

            n_out = torch.empty((p.shape[0], 4), dtype=torch.float64, device=p.device) if normals else None
            c_out = torch.empty((p.shape[0], 4, 4), dtype=torch.float64, device=p.device) if covs else None
        else:
            n_out = np.empty((p.shape[0], 4)) if normals else None
            c_out = np.empty((p.shape[0], 4, 4)) if covs else None
        self._check(self._L.sgb_estimate_features_batch(self._h, offsets.size - 1, offsets.ctypes.data_as(C.POINTER(C.c_size_t)), _d(p), int(num_neighbors),
                                                        _d(n_out), _d(c_out)))
        return n_out, c_out
