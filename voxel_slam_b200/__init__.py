"""voxel_slam_b200 — H100-native (sm_90a CUDA) bundle-adjustment hot path of hku-mars/Voxel-SLAM.

The product is the C-ABI shared library ``lib/libvxs.so`` (``include/vxs.h``); this package is the thin Python
mirror used by the tests and ``bench.py``.  There is no CPU fallback: importing works anywhere (so that the
CPU-only checks can verify the ABI), but every compute entry point needs a CUDA device and raises otherwise.
"""
from .api import (  # noqa: F401
    VxsError, lib, Context, Factor, LocalMap, MapParams, LmTrace, VoxelId, ImuHooks, declared_symbols, LIB_PATH,
)

__all__ = ["VxsError", "lib", "Context", "Factor", "LocalMap", "MapParams", "LmTrace", "VoxelId", "ImuHooks", "declared_symbols", "LIB_PATH"]
