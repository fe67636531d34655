"""spicedb-kubeapi-proxy_b200 -- host side of libzgpu (H100-native batched Zanzibar
permission checks behind the reference proxy's v1.PermissionsServiceClient boundary).

The directory name contains '-', so import it through the root-level shim:

    import zgpu                      # loads this package as spicedb_kubeapi_proxy_b200
    eng = zgpu.Engine(schema_text)

Only what the hot path needs lives here: csrc/ (CUDA kernels + C ABI), the ctypes
binding, a client that mirrors v1.PermissionsServiceClient, and the synthetic
workload generators of SURVEY.md section 8(d).
"""
from ._lib import (  # noqa: F401
    CHECK_DTYPE, TUPLE_DTYPE, UPDATE_DTYPE, HAS_PERMISSION, ITEM_ERROR, NO_PERMISSION, SREL_NONE, SREL_WILDCARD,
    Engine, ZgpuError, build_library, library_path,
)
from .client import PermissionsClient  # noqa: F401
