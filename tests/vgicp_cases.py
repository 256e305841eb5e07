"""Call sequences of the FastVGICP parity tests.  Every case takes a `make()` factory returning an object with the
pygicp.FastVGICP interface (this repo's CUDA drop-in, or the reference's own pybind11 module built by `make -C oracle ref`)
and returns a dict of numpy results: poses ("pose*"), final Hessians ("H*") and the voxel map as ("vmean", "vcov"),
sorted by mean so that the order in which a map lists its voxels does not matter.  get_source_correspondence is never
called (the reference returns uninitialised memory for a FastVGICP)."""
import os

import numpy as np

from gs_icp_slam_b200 import synthetic as S
from tests import vgicp_model as VM

HERE = os.path.dirname(os.path.abspath(__file__))


def _filter_all(n):
    return np.arange(1, n + 1, dtype=np.int32)


def _make(make, res, method):
    r = make()
    r.set_max_knn_distance(99999)
    r.set_resolution(res)
    r.set_neighbor_search_method(method)
    return r


def voxels(r):
    mu, C = r.get_voxel_mean_cov()
    mean, cov = VM.sort_by_mean(np.array(mu).reshape(-1, 4), np.array(C).reshape(-1, 4, 4))
    return dict(vmean=mean, vcov=cov.reshape(-1, 16))


def kitti(make, res, method):
    """The reference's KITTI fixture (FG/src/test/gicp_test.cpp)."""
    k = np.load(os.path.join(HERE, "golden", "gicp_kitti_pair.npz"))
    r = _make(make, res, method)
    r.set_input_target(k["target"])
    r.set_input_source(k["source"])
    r.set_source_filter(len(k["source"]), _filter_all(len(k["source"])))
    out = dict(pose=np.array(r.align(np.eye(4, dtype=np.float32))), H=np.array(r.get_final_hessian()))
    out.update(voxels(r))
    return out


def tracker_c3(make, res, P=100000, frames=(1, 2, 3), keyframe_at=2):
    """The C3 tracker shape of tests/gicp_cases.tracker_c3 with a FastVGICP: 12 416-point frames with the trackable-subset
    filter against a P-Gaussian target from (q, s), seeded with the previous estimated pose, target refreshed at
    `keyframe_at`."""
    cam = S.TUM
    g = S.gaussian_map(P, 3)
    r = _make(make, res, "DIRECT1")
    r.set_max_correspondence_distance(0.03)
    r.set_input_target(g["means3D"].astype(np.float64))
    r.set_target_covariances_fromqs(g["rotations"].reshape(-1), g["scales"].reshape(-1))
    pose = S.trajectory_pose(frames[0] - 1, 200).astype(np.float32)
    out = {}
    for f in frames:
        pts, tr = S.tracker_cloud(S.raycast_depth(S.trajectory_pose(f, 200), cam)[0], cam)
        r.set_input_source(pts)
        r.set_source_filter(len(tr), S.trackable_filter(len(pts), tr))
        pose = np.array(r.align(pose))
        out[f"pose{f}"], out[f"H{f}"] = pose, np.array(r.get_final_hessian())
        if f == keyframe_at:
            r.set_input_target(g["means3D"].astype(np.float64))
            r.set_target_covariances_fromqs(g["rotations"].reshape(-1), g["scales"].reshape(-1))
    out.update(voxels(r))
    return out


def c1_and_swap(make, res=0.25, method="DIRECT7", n=4000):
    """C1 pair through calculate_target_covariance_with_filter, then swap_source_and_target and a second align."""
    tgt, src, _ = S.gicp_pair(n, n)
    r = _make(make, res, method)
    r.set_input_target(tgt)
    r.set_target_filter(len(tgt), _filter_all(len(tgt)))
    r.calculate_target_covariance_with_filter()
    r.set_input_source(src)
    r.set_source_filter(len(src), _filter_all(len(src)))
    out = dict(pose=np.array(r.align(np.eye(4, dtype=np.float32))), H=np.array(r.get_final_hessian()))
    out.update(voxels(r))
    r.swap_source_and_target()
    r.set_source_filter(len(tgt), _filter_all(len(tgt)))
    out["pose_swapped"] = np.array(r.align(np.eye(4, dtype=np.float32)))
    out["H_swapped"] = np.array(r.get_final_hessian())
    v = voxels(r)
    out["vmean_swapped"], out["vcov_swapped"] = v["vmean"], v["vcov"]
    return out


def no_overlap(make, res=0.25):
    """Source 100 m away from the target: no voxel correspondences; the reference returns the guess and a zero Hessian."""
    tgt, src, _ = S.gicp_pair(3000, 2000)
    r = _make(make, res, "DIRECT27")
    r.set_input_target(tgt)
    r.set_input_source(src + 100.0)
    r.set_source_filter(len(src), _filter_all(len(src)))
    guess = np.eye(4, dtype=np.float32)
    guess[:3, 3] = (0.01, -0.02, 0.03)
    return dict(pose=np.array(r.align(guess)), H=np.array(r.get_final_hessian()))


def lattice_target(res=0.25):
    """Target points exactly on voxel faces ((k + 0.5) * res), the same lattice jittered, offset by 1000 m."""
    g = np.arange(-8, 8) * res + 0.5 * res
    X, Y, Z = np.meshgrid(g, g, g[:6], indexing="ij")
    tgt = np.c_[X.ravel(), Y.ravel(), Z.ravel()] + 1000.0
    rng = np.random.default_rng(3)
    return np.r_[tgt, tgt + rng.normal(0, 0.02, tgt.shape)]


def lattice(make, res=0.25):
    """Voxel statistics of lattice_target (the pose is not compared: the lattice is degenerate by design)."""
    tgt = lattice_target(res)
    src = tgt[::2] + [0.01, 0.0, -0.01]
    r = _make(make, res, "DIRECT7")
    r.set_input_target(tgt)
    r.set_input_source(src)
    r.set_source_filter(len(src), _filter_all(len(src)))
    r.align(np.eye(4, dtype=np.float32))
    return voxels(r)


# name -> (function, keyword arguments, whether the case's pose and Hessian are compared)
CASES = {f"kitti_r{res}_d{d}": (kitti, dict(res=res, method=f"DIRECT{d}"), True) for res in (1.0, 0.5) for d in (1, 7, 27)}
CASES.update({
    "c3_r0.05": (tracker_c3, dict(res=0.05), True),
    "c3_r0.1": (tracker_c3, dict(res=0.1), True),
    "c1_swap": (c1_and_swap, {}, True),
    "no_overlap": (no_overlap, {}, True),
    "lattice": (lattice, {}, False),
})
