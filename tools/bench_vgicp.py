"""FastVGICP vs FastGICP align() time on the C3 tracker frames (12 416-point frames with the trackable filter against a
P-Gaussian target from (q, s), seeded with the previous estimated pose; tests/gicp_cases.tracker_c3).
Host clock around a synchronised align(), after warm-up aligns; median and spread over the timed aligns.  Writes one JSON
document (stdout, and --out if given) with the device name and its enforced power limit beside the numbers:
    python tools/bench_vgicp.py [--P 300000] [--frames 20] [--warmup 3] [--out result.json]"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import pygicp  # noqa: E402
from gs_icp_slam_b200 import synthetic as S  # noqa: E402


def device_info():
    info = {"device": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        import pynvml as nv

        nv.nvmlInit()
        info["power_limit_w"] = nv.nvmlDeviceGetEnforcedPowerLimit(nv.nvmlDeviceGetHandleByIndex(0)) / 1000.0
    except Exception as ex:  # no NVML here: the limit stays unknown
        info["power_limit_error"] = type(ex).__name__
    return info


def run(make, g, frames, warmup):
    r = make()
    r.set_max_knn_distance(99999)
    r.set_max_correspondence_distance(0.03)
    r.set_input_target(g["means3D"])
    r.set_target_covariances_fromqs(g["rotations"].reshape(-1), g["scales"].reshape(-1))
    pose = S.trajectory_pose(0, 200).astype(np.float32)
    ts = []
    for i, (pts, n_tr, f) in enumerate(frames):
        r.set_input_source(pts)
        r.set_source_filter(n_tr, f)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pose = r.align(pose)
        torch.cuda.synchronize()
        if i >= warmup:
            ts.append((time.perf_counter() - t0) * 1e3)
    return {"align_ms_median": float(np.median(ts)), "align_ms_min": float(np.min(ts)), "align_ms_max": float(np.max(ts)),
            "aligns": len(ts), "last_pose_err": float(np.abs(pose - S.trajectory_pose(len(frames), 200)).max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=300000)
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    g = S.gaussian_map(args.P, 3)
    frames = []
    for f in range(1, args.warmup + args.frames + 1):
        pts, tr = S.tracker_cloud(S.raycast_depth(S.trajectory_pose(f, 200), S.TUM)[0], S.TUM)
        frames.append((np.asarray(pts, np.float32), len(tr), S.trackable_filter(len(pts), tr)))
    res = dict(device_info(), target_gaussians=args.P, source_points=int(len(frames[0][0])),
               trackable=frames[0][1], runs={})
    res["runs"]["FastGICP"] = run(pygicp.FastGICP, g, frames, args.warmup)
    for method in ("DIRECT1", "DIRECT7"):
        for rv in (0.05, 0.1):
            def make(method=method, rv=rv):
                r = pygicp.FastVGICP()
                r.set_resolution(rv)
                r.set_neighbor_search_method(method)
                return r

            res["runs"][f"FastVGICP_{method}_r{rv}"] = run(make, g, frames, args.warmup)
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
