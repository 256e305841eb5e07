"""gs_icp_slam_b200 — H100-native (sm_90a) hot paths of GS-ICP-SLAM behind the reference's APIs.

  rasterizer  : Gaussian-splat rasterizer forward/backward  (diff_gaussian_rasterization drop-in)
  gicp        : Generalized-ICP tracker                      (pygicp drop-in)
  knn         : distCUDA2                                    (simple_knn._C drop-in)
  loss        : fused mapper loss (N2)          frontend : tracker front-end (N1)
  map_table   : fused Adam, table maintenance, device hand-over, scene.ply (N3, N4)
  wire        : SIBR viewer wire format (N4)    sharding : multi-GPU exchange group (ShardGroup)

All compute is in gs_icp_slam_b200/libgsicp_b200.so (C ABI: include/gsicp_b200.h); importing the
package fails loudly when that library is missing — there is no CPU fallback.
"""
from . import _lib  # noqa: F401  (raises ImportError if the CUDA library is not built)

__all__ = ["_lib"]
