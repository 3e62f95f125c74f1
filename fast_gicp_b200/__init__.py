"""fast_gicp_b200 -- H100-native VGICP registration engine behind the fast_gicp FastVGICPCuda / pygicp API.

The numerical work lives in lib/libvgicp_b200.so (hand-written sm_90a CUDA, C ABI in include/vgicp_b200.h).
Importing the package requires the built library; there is no CPU fallback.
"""
from .core import Core, VgicpError, load_library, default_params, LIB_PATH  # noqa: F401
from .registration import (  # noqa: F401
    FastVGICPCuda,
    LsqRegistration,
    LSQ_OPTIMIZER_TYPE,
    NDTCuda,
    NDTDistanceMode,
    NearestNeighborMethod,
    NeighborSearchMethod,
    RegularizationMethod,
)

load_library()  # fail loudly at import time when the extension is missing
