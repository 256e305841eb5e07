"""Drop-in `pygicp` module backed by libgsicp_b200.so (sm_90a CUDA), for the reference's
mp_Tracker.py / mp_Tracker_unlimit.py (`self.reg = pygicp.FastGICP()`, mp_Tracker.py:53).

Exports the two registration classes the reference's pygicp binds: FastGICP, the class the trackers use, and
FastVGICP, its voxelized variant (submodules/fast_gicp/src/python/main.cpp:264-279).  The reference's free functions
align_points and downsample (main.cpp:47-147) are outside the SLAM hot path (SURVEY.md §2 rows 20-21) and raise
NotImplementedError.  FastVGICPCuda and NDTCuda are not exported: the reference builds them only with its CUDA option.
"""
from gs_icp_slam_b200.gicp import FastGICP, FastVGICP

__version__ = "b200"


def _out_of_scope(name):
    def f(*a, **k):
        raise NotImplementedError(f"pygicp.{name} is outside the GS-ICP-SLAM hot path and is not provided by gs_icp_slam_b200")

    f.__name__ = name
    return f


align_points = _out_of_scope("align_points")
downsample = _out_of_scope("downsample")

__all__ = ["FastGICP", "FastVGICP", "align_points", "downsample"]
