"""H100-native small_gicp hot path: ctypes front-end of libsgicp_b200.so (C-ABI in include/sgicp_b200.h).

There is no CPU fallback: importing works anywhere (the library only needs libcudart), but creating a
Context without an H100 raises, and a missing library raises at import of `capi`.
"""
from .capi import (  # noqa: F401
    Context,
    SgbError,
    FACTOR_ICP,
    FACTOR_PLANE_ICP,
    FACTOR_GICP,
    ROBUST_NONE,
    ROBUST_HUBER,
    ROBUST_CAUCHY,
    REJECT_NONE,
    REJECT_DISTANCE,
    NO_CORRESPONDENCE,
    GNC_GEMAN_MCCLURE,
    GNC_TLS,
    library_path,
    exported_symbols,
)
