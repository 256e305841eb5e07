"""Cost of the deterministic render backward: device time of one gsicp_raster_backward call (render backward + per-Gaussian
backward) on one saved forward state, default mode against deterministic mode, alternated call by call, CUDA events,
median over --iters calls after --warmup calls of each.

    python tools/bench_raster_det.py [--shapes c3,c4] [--iters 60] [--warmup 10]

C3 = 300k Gaussians at 640x480, C4 = 1M Gaussians at 1280x960 (the shapes of tools/bench_raster.py).  Prints the card and
its power limit with the numbers, and one JSON line per shape."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gs_icp_slam_b200 import rasterizer as R  # noqa: E402
from gs_icp_slam_b200 import synthetic as S  # noqa: E402

SHAPES = {"c3": (640, 480, 300000, 1.0, 3, 200), "c4": (1280, 960, 1000000, 2.0, 4, 20)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0)


def bench(which, iters, warmup, dev):
    W, H, P, sc, seed, n_traj = SHAPES[which]
    cam = dict(S.TUM)
    cam.update(W=W, H=H, fx=cam["fx"] * sc, fy=cam["fy"] * sc, cx=cam["cx"] * sc, cy=cam["cy"] * sc)
    g = S.gaussian_map(P, seed, scale=sc)
    cm = S.camera_matrices(S.trajectory_pose(3, n_traj, scale=sc), cam)
    t = {k: torch.from_numpy(v).to(dev) for k, v in g.items()}
    c = {k: (torch.from_numpy(v).to(dev) if isinstance(v, np.ndarray) else v) for k, v in cm.items()}
    bg, e = torch.zeros(3, device=dev), torch.Tensor([])
    n, depth, color, radii, _, geom, binning, img = R.rasterize_gaussians(
        bg, t["means3D"], e, t["opacities"], t["scales"], t["rotations"], 1.0, e, c["viewmatrix"], c["projmatrix"],
        c["tanfovx"], c["tanfovy"], H, W, t["shs"], 0, c["campos"], False, False)
    gen = torch.Generator(device="cpu").manual_seed(5)
    gcol, gdep = torch.randn((3, H, W), generator=gen).to(dev), torch.randn((1, H, W), generator=gen).to(dev)

    def backward():
        return R.rasterize_gaussians_backward(bg, t["means3D"], radii, e, t["scales"], t["rotations"], 1.0, e, c["viewmatrix"],
                                              c["projmatrix"], c["tanfovx"], c["tanfovy"], gdep, gcol, t["shs"], 0, c["campos"],
                                              geom, n, binning, img, False)

    times = {False: [], True: []}
    grads = {}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        for i in range(warmup + iters):
            for det in (False, True):
                torch.use_deterministic_algorithms(det)
                ev0.record()
                out = backward()
                ev1.record()
                ev1.synchronize()
                if i >= warmup:
                    times[det].append(ev0.elapsed_time(ev1) * 1e3)
                grads[det] = out
    finally:
        torch.use_deterministic_algorithms(prev)
    err = max(float((a - b).abs().max() / (b.abs().max() + 1e-30)) for a, b in zip(grads[True], grads[False]) if b.numel())
    d, x = float(np.median(times[False])), float(np.median(times[True]))
    return dict(shape=which, P=P, W=W, H=H, visible=int((radii > 0).sum()), rendered=int(n), iters=iters,
                default_us=round(d, 1), deterministic_us=round(x, 1), ratio=round(x / d, 3), max_rel_grad_diff=err)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c3,c4")
    ap.add_argument("--iters", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_raster_det.py needs a CUDA device")
    dev = torch.device("cuda:0")
    name = card()
    print(f"card: {name}", flush=True)
    for which in a.shapes.split(","):
        r = bench(which, a.iters, a.warmup, dev)
        r["card"] = name
        print(f"{which}: default {r['default_us']} us, deterministic {r['deterministic_us']} us ({r['ratio']}x), "
              f"gradients within {r['max_rel_grad_diff']:.2e} of max", flush=True)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
