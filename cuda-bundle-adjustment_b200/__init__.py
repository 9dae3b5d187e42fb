"""cuda-bundle-adjustment_b200: H100-native LM bundle adjustment behind the reference's graph API.

This Python package is only a thin ctypes mirror of the C ABI in include/cuba_b200.h (the product is
libcuba_b200.so: hand-written sm_90a kernels + a C++ host).  There is NO CPU fallback: if the library
is missing or no CUDA device is present, everything that computes raises.
"""
from . import graphio  # noqa: F401
from . import binding  # noqa: F401
from .binding import (Engine, CubaError, load_library, library_path, build_structure_host, pcg_partition_host, pcg5_plan_host, pcg5_plan_apc_host, transfer_bytes,  # noqa: F401
                      ROBUST_NONE, ROBUST_HUBER, ROBUST_TUKEY, EDGE_MONOCULAR, EDGE_STEREO, PROFILE_ITEMS, PoseRound, orbslam2_pose_schedule, Sim3Params,
                      BATCH_STATUS, batch_status_message, stats_view)
from . import synth  # noqa: F401
from . import sharding  # noqa: F401
