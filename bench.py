#!/usr/bin/env python
"""bench.py — SLAM frames/s on the synthetic TUM-shape workload (BASELINE.json metric).

One "step" = one SLAM frame of the two hot paths, in the order the reference's processes run them:
  tracker  (mp_Tracker.py:191-231,256-288): set_input_source(12 416-pt cloud) -> set_source_filter ->
            align(previous ESTIMATED pose, mp_Tracker.py:199) -> get_source_correspondence; every 5th frame is a tracking
            keyframe: get_source_rotationsq/scales, set_input_target(map points) + set_target_covariances_fromqs(map q, s)
  mapper   (mp_Mapper.py:219-242, one training iteration): GaussianRasterizer forward on the 300k-Gaussian map at the
            frame's camera -> the mapper's loss against the frame's RGB-D (masked L1 + 0.2 DSSIM + 0.1 depth L1) -> backward
            through the rasterizer.  Adam is outside the hot path (SURVEY.md §8f N3).
Workload = BASELINE config C3: 640x480, fx 517.3 ..., downsample 5, max_corr 0.03, 300 000 Gaussians (seed 3).
The two halves of a frame are independent and run CONCURRENTLY, as in the reference (tracker and mapper are two
processes, gs_icp_slam.py:121-131): ours = two host threads + two CUDA streams in one process, reference arm = tracker
(CPU) in its own process next to the mapper (GPU).  One fixed schedule; `schedules` also lists the back-to-back time.

HEADLINE (`value`, `e2e`) = the configuration an unmodified mp_Mapper.py runs: this repo's drop-in rasterizer / tracker
with the mapper's loss evaluated by the reference's own PyTorch ops (utils/loss_utils.py) — identical to the reference
arm's config.  `fused_loss` reports the same frame with the loss through gs_icp_slam_b200.loss.mapping_loss (SURVEY §8f N2).

Printed JSON (one line, rank 0): `value` = frames/s with every input already resident in HBM; `e2e.value` = frames/s
through the public drop-in APIs with HOST inputs (numpy clouds / pinned images copied H2D inside the step; pose,
correspondences and loss read back D2H); `roofline` = the kernel with the largest device time in the step, measured with
CUDA events around its launches (gsicp_prof_*); `cpu_baseline` = the reference's CPU tracker (fast_gicp built from
/root/reference into oracle/_ref) + the CPU raster oracle on a bounded sample.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--config c3|c2|c4|c5] [--multi replicas|shard]
                  [--dump-outputs DIR]
`--dump-outputs DIR` writes what the headline run's last timed step returned to its caller (pose, correspondences, loss,
rendered images, radii, parameter gradients) as DIR/<name>.npy in float32 / float64, at most 60 MB (per-Gaussian arrays
are cut to a fixed, seeded sample of Gaussians beyond that), for comparing two builds output for output: the inputs
depend on the arguments only.
`--impl reference` = the reference's own implementation of the same frame on this box: fast_gicp (its unmodified
sources + pybind module, oracle/_ref/fast_gicp) on all host cores in a tracker process + the reference's CUDA
rasterizer through its own torch extension (oracle/_ref/site, stock build path) and PyTorch loss in the mapper process.
`--config c4|c5` = the large strong-scaling configs (rasterizer only, 1280x960, 1M Gaussians, tile-sharded; GICP on a
2M x 2M point pair, source-sharded) under the same JSON contract with "scaling": "strong".
"""
import argparse
import json
import math
import os
import sys
import threading
import time

# The CPU legs (reference arm, cpu_baseline) run OpenMP teams of one thread per logical CPU next to a thread that drives the
# GPU.  libgomp's default is to spin after every parallel region; on a shared host that starves the GPU-driving thread and the
# teams themselves (measured on one box: 1.5 frames/s spinning vs 12.7 passive, same run).  Must be set before libgomp loads.
os.environ.setdefault("OMP_WAIT_POLICY", "passive")

import numpy as np  # noqa: E402

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

KEYFRAME_EVERY = 5
N_TRAJ = 200       # frames of the full synthetic trajectory (SURVEY §8d)
UNIQUE_FRAMES = 48  # distinct frames kept resident; longer runs walk them back and forth (consecutive poses stay adjacent)
MAP_SEED = {"c3": 3, "c2": 2}
METRIC = "SLAM frames/sec (synthetic 640x480 RGB-D, 300k Gaussians)"


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--config", default="c3", choices=["c3", "c2", "c1", "c4", "c5"],
                    help="c3 (default, the metric's config): TUM-shape 640x480, 300k Gaussians; c2: Replica-shape, 100k Gaussians; "
                         "c1: GICP align of two 10k-point clouds (the reference's CPU-runnable case); "
                         "c4 / c5: the large rasterizer-only / GICP-only strong-scaling configs")
    ap.add_argument("--gaussians", type=int, default=None)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the outputs of the last timed step of the headline run as DIR/<name>.npy (c3 / c2, --impl ours)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-roofline", action="store_true")
    ap.add_argument("--no-variants", action="store_true", help="skip the fused-loss and back-to-back passes")
    ap.add_argument("--multi", default="replicas", choices=["replicas", "shard"],
                    help="N>1 with c3/c2: replicas = one independent SLAM sequence per GPU, no collective (the SLAM loop is "
                         "sequential in time: SURVEY §8e 'replicas only'); shard = ONE sequence, raster tiles + GICP source "
                         "points sharded over the ranks (pays only at C4/C5 sizes)")
    ap.add_argument("--loss", default="torch", choices=["torch", "fused", "l1"],
                    help="mapper loss of the HEADLINE leg.  torch (default) = the reference's PyTorch ops (what an unmodified "
                         "mp_Mapper.py runs, and what the reference arm runs); fused = gs_icp_slam_b200.loss.mapping_loss; "
                         "l1 = simplified L1 colour + depth in PyTorch ops")
    a = ap.parse_args()
    if a.warmup < 3:
        a.warmup = 3
    if a.gaussians is None:
        a.gaussians = {"c3": 300000, "c2": 100000, "c1": 10000, "c4": 1000000, "c5": 2000000}[a.config]
    return a


# ----------------------------------------------------------------------------------------------
# the mapper's loss as the reference's PyTorch code evaluates it (caller code, not part of the library)
# ----------------------------------------------------------------------------------------------
_WINDOWS = {}


def torch_mapper_loss(image, depth, gt_image, gt_depth, lambda_dssim=0.2):
    """mp_Mapper.py:225-242 with utils/loss_utils.py:17-69: masked L1 + DSSIM (11x11 Gaussian window, sigma 1.5, depthwise
    conv2d) + 0.1 * L1 of depth / 10, every step a separate PyTorch op like in the reference (pinned to the reference's own
    loss_utils.py by tests/test_loss_oracle.py)."""
    import torch
    import torch.nn.functional as F

    def l1(x, gt):
        return torch.where(gt != 0, torch.abs(x - gt), 0.).mean()

    key = (image.device, image.dtype)
    if key not in _WINDOWS:
        g = torch.Tensor([math.exp(-(x - 5) ** 2 / float(2 * 1.5 ** 2)) for x in range(11)])
        g = (g / g.sum()).unsqueeze(1)
        _WINDOWS[key] = g.mm(g.t()).float().unsqueeze(0).unsqueeze(0).expand(3, 1, 11, 11).contiguous().to(image.device)
    w = _WINDOWS[key]
    gt_image = gt_image * (gt_depth > 0.)
    ll1 = l1(image, gt_image)
    x = torch.where(gt_image != 0, image, 0.)
    mu1, mu2 = F.conv2d(x, w, padding=5, groups=3), F.conv2d(gt_image, w, padding=5, groups=3)
    mu1_sq, mu2_sq, mu12 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    s1 = F.conv2d(x * x, w, padding=5, groups=3) - mu1_sq
    s2 = F.conv2d(gt_image * gt_image, w, padding=5, groups=3) - mu2_sq
    s12 = F.conv2d(x * gt_image, w, padding=5, groups=3) - mu12
    ssim = (((2 * mu12 + 0.01 ** 2) * (2 * s12 + 0.03 ** 2)) / ((mu1_sq + mu2_sq + 0.01 ** 2) * (s1 + s2 + 0.03 ** 2))).mean()
    return (1.0 - lambda_dssim) * ll1 + lambda_dssim * (1.0 - ssim) + 0.1 * l1(depth / 10., gt_depth / 10.)


# ----------------------------------------------------------------------------------------------
# synthetic sequence
# ----------------------------------------------------------------------------------------------
def slam_config(name):
    from gs_icp_slam_b200 import synthetic as S

    if name == "c2":
        return dict(S.REPLICA), 0.02, "C2 Replica-shape"
    return dict(S.TUM), 0.03, "C3 TUM-shape"


def frame_index(i, n_unique):
    """Walk the unique frames back and forth: 0 1 ... n-1 n-2 ... 1 0 1 ..."""
    if n_unique <= 1:
        return 0
    period = 2 * (n_unique - 1)
    r = i % period
    return r if r < n_unique else period - r


def make_sequence(n_steps, cfg_name, P, need_images=True):
    from gs_icp_slam_b200 import synthetic as S

    cam, max_corr, label = slam_config(cfg_name)
    gmap = S.gaussian_map(P, MAP_SEED.get(cfg_name, 3))
    n_unique = min(n_steps + 1, UNIQUE_FRAMES)
    frames = []
    for i in range(n_unique):
        c2w = S.trajectory_pose(i, N_TRAJ)
        depth, hit = S.raycast_depth(c2w, cam)
        pts, tr = S.tracker_cloud(depth, cam)
        f = dict(c2w=c2w, pts=pts, filt=S.trackable_filter(len(pts), tr), n_trk=len(tr))
        if need_images:
            f["depth"] = depth[None].copy()
            f["rgb"] = S.texture(hit).astype(np.float32).reshape(cam["H"], cam["W"], 3).transpose(2, 0, 1).copy()
            f["cam"] = S.camera_matrices(c2w, cam)
        frames.append(f)
    return cam, max_corr, label, gmap, frames


class ClockSampler:
    """SM clock / throttle reasons sampled every 20 ms during the timed region (NVML through pynvml)."""

    def __init__(self, index):
        self.samples, self.reasons, self.max_mhz = [], set(), None
        self._stop = threading.Event()
        self.index = index
        self.th = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        try:
            import pynvml as nv

            nv.nvmlInit()
            h = nv.nvmlDeviceGetHandleByIndex(self.index)
            self.max_mhz = nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM)
            names = {"hw_slowdown": nv.nvmlClocksThrottleReasonHwSlowdown,
                     "hw_thermal_slowdown": nv.nvmlClocksThrottleReasonHwThermalSlowdown,
                     "sw_thermal_slowdown": nv.nvmlClocksThrottleReasonSwThermalSlowdown,
                     "sw_power_cap": nv.nvmlClocksThrottleReasonSwPowerCap}
            while not self._stop.is_set():
                self.samples.append(nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM))
                r = nv.nvmlDeviceGetCurrentClocksThrottleReasons(h)
                for k, bit in names.items():
                    if r & bit:
                        self.reasons.add(k)
                time.sleep(0.02)
        except Exception as ex:  # no NVML in this environment
            self.reasons.add(f"unavailable:{type(ex).__name__}")

    def __enter__(self):
        self.th.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        self.th.join(timeout=2)

    def summary(self):
        return {"sm_mhz": float(np.median(self.samples)) if self.samples else None, "sm_max_mhz": self.max_mhz,
                "reasons": sorted(self.reasons)}


# ----------------------------------------------------------------------------------------------
# our implementation
# ----------------------------------------------------------------------------------------------
class Ours:
    def __init__(self, cam, max_corr, gmap, frames, dev, world, rank, shard=False, loss="torch"):
        import torch

        import pygicp
        from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
        from gs_icp_slam_b200 import _lib, rasterizer
        from gs_icp_slam_b200 import loss as fused

        self.torch, self.dev, self.cam, self.frames = torch, dev, cam, frames
        self.world, self.rank = world, rank
        self.fused = fused
        self.loss_kind = loss
        if loss != "l1" and shard:
            raise SystemExit("--multi shard needs --loss l1 (the SSIM window crosses tile shards)")
        self.Settings, self.Rasterizer, self._lib = GaussianRasterizationSettings, GaussianRasterizer, _lib
        self.map_np = gmap
        self.map = {k: torch.from_numpy(v).to(dev).requires_grad_(True) for k, v in gmap.items()}
        self.means2D = torch.zeros_like(self.map["means3D"], requires_grad=True)
        self.bg = torch.zeros(3, device=dev)
        self.reg = pygicp.FastGICP()
        self.reg.set_max_correspondence_distance(max_corr)
        self.reg.set_max_knn_distance(99999)
        H, W = cam["H"], cam["W"]
        # per-frame resident copies (value mode) and pinned host copies (e2e mode)
        for f in frames:
            f["pts32"] = np.ascontiguousarray(f["pts"], dtype=np.float32)
            f["d_pts"] = torch.from_numpy(f["pts32"]).to(dev)
            f["d_rgb"] = torch.from_numpy(f["rgb"]).to(dev)
            f["d_depth"] = torch.from_numpy(f["depth"]).to(dev)
            f["h_rgb"] = torch.from_numpy(f["rgb"]).pin_memory()
            f["h_depth"] = torch.from_numpy(f["depth"]).pin_memory()
            f["d_cam"] = {k: (torch.from_numpy(v).to(dev) if isinstance(v, np.ndarray) else v) for k, v in f["cam"].items()}
        self.stage_rgb = torch.empty((3, H, W), device=dev)
        self.stage_depth = torch.empty((1, H, W), device=dev)
        self.flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
        self.pix_mask = None
        self.count_stats = False
        if world > 1:
            import torch.distributed as dist

            self.dist = dist
        if world > 1 and shard:
            from gs_icp_slam_b200 import sharding

            self.sharding = sharding
            self.group = sharding.ShardGroup(dev, world, rank)  # in-kernel exchange over peer memory (NCCL callbacks as fallback)
            self.group.attach_rasterizer()
            self.group.attach_gicp(self.reg)
            self.pix_mask = sharding.tile_owner_mask(H, W, world, rank, dev)
        self.pose = frames[0]["c2w"].astype(np.float32)
        self.pool = None
        self.gicp_stream = None
        self.stats = dict(R=0, V=0, n_src=0, n_corr=0, n_tgt=0, frames=0, h2d=0, d2h=0, n_lin=0, pose_err=0.0)
        self.keep_outputs = False  # hold on to each step's results for --dump-outputs (references only, no copies)
        self.last_outputs = {}
        self.refresh_target(resident=True)

    def set_loss(self, kind):
        self.loss_kind = kind

    def refresh_target(self, resident):
        m = self.map
        if resident:
            self.reg.set_input_target(m["means3D"].detach())
            self.reg.set_target_covariances_fromqs(m["rotations"].detach(), m["scales"].detach())
        else:
            # host float32 numpy, as mp_Tracker receives it from SharedTargetPoints.get_values_np() (scene/shared_objs.py:118-126)
            g = self.map_np
            self.reg.set_input_target(g["means3D"])
            self.reg.set_target_covariances_fromqs(g["rotations"].reshape(-1), g["scales"].reshape(-1))
            self.stats["h2d"] += g["means3D"].nbytes + g["rotations"].nbytes + g["scales"].nbytes

    def tracker_part(self, step, resident):
        """mp_Tracker.py:191-231 (+ :256-288 on keyframes) for step `step` (frame index walks the resident frames)."""
        f = self.frames[frame_index(step + 1, len(self.frames))]
        st = self.stats
        if resident:
            self.reg.set_input_source(f["d_pts"])
        else:
            self.reg.set_input_source(f["pts32"])  # host float32 numpy, as downsample_and_make_pointcloud2 returns it
            st["h2d"] += f["pts32"].nbytes
        self.reg.set_source_filter(f["n_trk"], f["filt"])
        st["h2d"] += f["filt"].nbytes
        pose = self.reg.align(self.pose)  # seeded with the previous ESTIMATED pose (mp_Tracker.py:199)
        corr, sqd = self.reg.get_source_correspondence()
        st["d2h"] += 64 + corr.nbytes + sqd.nbytes
        st["n_src"] += len(corr)
        st["n_corr"] += int((corr >= 0).sum())
        st["n_tgt"] += self.map["means3D"].shape[0]
        st["n_lin"] += self.reg.last_iterations
        st["pose_err"] = max(st["pose_err"], float(np.abs(pose.astype(np.float64) - f["c2w"]).max()))
        self.pose = pose
        if self.keep_outputs:
            self.last_outputs.update(pose=pose, correspondences=corr, squared_distances=sqd)
        if (step + 1) % KEYFRAME_EVERY == 0:
            rots, scales = self.reg.get_source_rotationsq(), self.reg.get_source_scales()
            st["d2h"] += rots.nbytes + scales.nbytes
            self.refresh_target(resident)

    def mapper_part(self, step, resident):
        """One training iteration of mp_Mapper.py:219-242 at the camera of the step's frame."""
        torch = self.torch
        f = self.frames[frame_index(step + 1, len(self.frames))]
        st = self.stats
        if resident:
            gt_rgb, gt_depth = f["d_rgb"], f["d_depth"]
        else:
            self.stage_rgb.copy_(f["h_rgb"], non_blocking=True)
            self.stage_depth.copy_(f["h_depth"], non_blocking=True)
            gt_rgb, gt_depth = self.stage_rgb, self.stage_depth
            st["h2d"] += f["h_rgb"].numel() * 4 + f["h_depth"].numel() * 4
        c, cam, m = f["d_cam"], self.cam, self.map
        rs = self.Settings(cam["H"], cam["W"], c["tanfovx"], c["tanfovy"], self.bg, 1.0, c["viewmatrix"], c["projmatrix"], 0,
                           c["campos"], False, False)
        depth, color, radii, is_used = self.Rasterizer(rs)(means3D=m["means3D"], means2D=self.means2D,
                                                           opacities=m["opacities"], shs=m["shs"], scales=m["scales"],
                                                           rotations=m["rotations"])
        if self.loss_kind == "fused":
            loss = self.fused.mapping_loss(color, depth, gt_rgb, gt_depth)
        elif self.loss_kind == "torch":
            loss = torch_mapper_loss(color, depth, gt_rgb, gt_depth)
        elif self.pix_mask is None:
            loss = (color - gt_rgb).abs().mean() + 0.1 * (depth - gt_depth).abs().mean()
        else:
            sh = self.sharding
            loss = sh.sharded_l1(color, gt_rgb, self.pix_mask, gt_rgb.numel()) + 0.1 * sh.sharded_l1(depth, gt_depth, self.pix_mask, gt_depth.numel())
        n_rendered = getattr(color.grad_fn, "num_rendered", 0) if color.grad_fn is not None else 0
        loss.backward()
        lv = float(loss.item())  # D2H read of the step's result
        st["d2h"] += 8
        if self.keep_outputs:
            self.last_outputs.update(loss=lv, color=color, depth=depth, radii=radii, grad_means2D=self.means2D.grad,
                                     **{"grad_" + k: v.grad for k, v in m.items()})
        for k in m:
            m[k].grad = None
        self.means2D.grad = None
        st["R"] += n_rendered
        if self.count_stats:  # bench bookkeeping (a reduction + D2H sync): only in the profiled pass
            st["V"] += int((radii > 0).sum())
        st["frames"] += 1
        return lv

    def step(self, i, resident):
        """One SLAM frame.  Tracker and mapper are independent within a frame (two concurrent processes in the reference,
        gs_icp_slam.py:121-131): with the concurrent schedule they run on two host threads / two CUDA streams."""
        if self.pool is None:
            self.tracker_part(i, resident)
            return self.mapper_part(i, resident)
        fut = self.pool.submit(self._tracker_thread, i, resident)
        lv = self.mapper_part(i, resident)
        fut.result()
        # the step ends when both halves have: the main stream waits for the tracker's stream (asynchronous target uploads)
        self.torch.cuda.current_stream(self.dev).wait_stream(self.gicp_stream)
        return lv

    def _tracker_thread(self, i, resident):
        self.torch.cuda.set_device(self.dev)
        self.tracker_part(i, resident)

    def enable_concurrent(self, on=True):
        from concurrent.futures import ThreadPoolExecutor

        if not on:
            if self.pool is not None:
                self.pool.shutdown(wait=True)
                self.pool = None
                self.torch.cuda.synchronize()
                self.reg.set_stream(self.torch.cuda.current_stream(self.dev).cuda_stream)
                sys.setswitchinterval(self._switch0)
            return
        if self.pool is not None:
            return
        # two Python threads hand the GIL over every switch interval (default 5 ms) when both want it: make it short
        self._switch0 = sys.getswitchinterval()
        sys.setswitchinterval(2e-5)
        self.pool = ThreadPoolExecutor(max_workers=1)
        if self.gicp_stream is None:
            self.gicp_stream = self.torch.cuda.Stream(device=self.dev)
        self.reg.set_stream(self.gicp_stream.cuda_stream)

    def close(self):
        """Orderly teardown (worker thread, library handle) before the interpreter exits normally."""
        self.enable_concurrent(False)
        self.torch.cuda.synchronize()
        if getattr(self, "group", None) is not None:
            self.group.close()
            self.group = None
        self.reg = None

    def run(self, steps, warmup, resident, profile=False):
        """W untimed + K timed steps; returns (sum of the K per-step CUDA-event times in ms, launches, stats)."""
        torch = self.torch
        self._lib.prof_enable(False)
        for k in self.stats:
            self.stats[k] = 0
        self.pose = self.frames[0]["c2w"].astype(np.float32)
        self.refresh_target(resident=True)
        times = []
        for i in range(warmup + steps):
            if i == warmup:
                for k in self.stats:
                    self.stats[k] = 0
                if self.world > 1:
                    self.dist.barrier()
                torch.cuda.synchronize()
                self._lib.prof_reset()
                self._lib.prof_enable(profile)
                self.count_stats = profile
                self.launch0 = self._lib.launch_count()
            self.flush.fill_(i & 0xff)  # L2 flush between steps (outside the timed events)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            self.step(i, resident)
            e1.record()
            torch.cuda.synchronize()
            if i >= warmup:
                times.append(e0.elapsed_time(e1))
        if self.world > 1:
            self.dist.barrier()
        torch.cuda.synchronize()
        self._lib.prof_enable(False)
        self.count_stats = False
        launches = self._lib.launch_count() - self.launch0
        self.last_times = times
        return float(np.sum(times)), launches, dict(self.stats)


# ----------------------------------------------------------------------------------------------
# reference arm / CPU baseline
# ----------------------------------------------------------------------------------------------
def host_threads():
    try:
        return len(os.sched_getaffinity(0))
    except Exception:
        return os.cpu_count() or 1


def make_cpu_tracker(max_corr, gmap):
    """The reference's CPU tracker: fast_gicp itself (oracle/_ref/fast_gicp, built from /root/reference) when present
    ("reference"), the oracle restatement otherwise ("port").  All host threads."""
    from oracle import ref_gicp

    n = host_threads()
    if ref_gicp.available():
        reg, kind = ref_gicp.FastGICP(), "reference"
        reg.set_num_threads(n)  # fgi:36-44 (torchrun exports OMP_NUM_THREADS=1)
    else:
        from oracle import gicp_oracle as G

        G.set_num_threads(n)
        reg, kind = G.FastGICP(), "port"
    reg.set_max_correspondence_distance(max_corr)
    reg.set_max_knn_distance(99999)
    reg.set_input_target(gmap["means3D"].astype(np.float64))
    reg.set_target_covariances_fromqs(gmap["rotations"].reshape(-1), gmap["scales"].reshape(-1))
    return reg, kind, n


def cpu_tracker_step(reg, gmap, frames, step, pose):
    f = frames[frame_index(step + 1, len(frames))]
    reg.set_input_source(f["pts"])
    reg.set_source_filter(f["n_trk"], f["filt"])
    pose = reg.align(np.asarray(pose, dtype=np.float32))
    reg.get_source_correspondence()
    if (step + 1) % KEYFRAME_EVERY == 0:
        reg.get_source_rotationsq()
        reg.get_source_scales()
        reg.set_input_target(gmap["means3D"].astype(np.float64))
        reg.set_target_covariances_fromqs(gmap["rotations"].reshape(-1), gmap["scales"].reshape(-1))
    return pose


def cpu_baseline(cfg_name, max_corr, gmap, frames, budget_s=20.0):
    from oracle import raster_oracle

    reg, kind, n = make_cpu_tracker(max_corr, gmap)
    pose = frames[0]["c2w"].astype(np.float32)
    t0, k, t_trk = time.time(), 0, 0.0
    while k < min(3, len(frames) - 1) and (time.time() - t0 < budget_s or k == 0):
        ta = time.time()
        pose = cpu_tracker_step(reg, gmap, frames, k, pose)
        t_trk += time.time() - ta
        f = frames[frame_index(k + 1, len(frames))]
        H, W = f["rgb"].shape[1:]
        o = raster_oracle.forward_backward(gmap, f["cam"], H, W, np.zeros(3, np.float32))
        gc = np.sign(o.color - f["rgb"]).astype(np.float32) / o.color.size
        gd = 0.1 * np.sign(o.depth - f["depth"]).astype(np.float32) / o.depth.size
        raster_oracle.forward_backward(gmap, f["cam"], H, W, np.zeros(3, np.float32), dL_dcolor=gc, dL_ddepth=gd)
        k += 1
    dt = time.time() - t0
    return {"value": k / dt, "unit": "frames/s", "cores": n, "kind": kind,
            "tracker_ms_per_frame": t_trk / k * 1e3,
            "sample": f"{k} frame(s) of {cfg_name}: " + ("fast_gicp (reference sources, oracle/_ref/fast_gicp; PCL k-NN through oracle/pcl_shim)"
                                                         if kind == "reference" else "oracle restatement of fast_gicp") +
                      f" align on {n} threads + CPU raster oracle fwd+bwd on 1 thread (the reference has no CPU rasterizer: port), "
                      f"{gmap['means3D'].shape[0]} Gaussians"}


def _ref_tracker_worker(conn, cfg_name, P, steps, warmup):
    """Tracker process of the reference arm (mp_Tracker.py runs as its own process): fast_gicp on all host threads."""
    try:
        cam, max_corr, label, gmap, frames = make_sequence(steps + warmup, cfg_name, P, need_images=False)
        reg, kind, n = make_cpu_tracker(max_corr, gmap)
        pose = frames[0]["c2w"].astype(np.float32)
        for i in range(warmup):
            pose = cpu_tracker_step(reg, gmap, frames, i, pose)
        conn.send(("ready", kind, n))
        conn.recv()  # go
        t0 = time.perf_counter()
        err = 0.0
        for i in range(warmup, warmup + steps):
            pose = cpu_tracker_step(reg, gmap, frames, i, pose)
            err = max(err, float(np.abs(pose.astype(np.float64) - frames[frame_index(i + 1, len(frames))]["c2w"]).max()))
        conn.send(("done", time.perf_counter() - t0, err))
    except Exception as ex:  # report instead of hanging the parent
        conn.send(("error", repr(ex)))


def reference_arm(args):
    """Reference implementation of the frame on this box: tracker process = fast_gicp (CPU, all host threads), mapper =
    the reference's CUDA rasterizer through its own torch extension + its PyTorch loss, running concurrently."""
    import multiprocessing as mp

    from oracle import ref_ext

    use_gpu = False
    try:
        import torch

        use_gpu = torch.cuda.is_available() and ref_ext.available()
    except Exception:
        pass
    ctx = mp.get_context("spawn")
    parent, child = ctx.Pipe()
    proc = ctx.Process(target=_ref_tracker_worker, args=(child, args.config, args.gaussians, args.steps, args.warmup), daemon=True)
    proc.start()
    cam, max_corr, label, gmap, frames = make_sequence(args.steps + args.warmup, args.config, args.gaussians)
    if use_gpu:
        dgr = ref_ext.diff_gaussian_rasterization()
        dev = torch.device("cuda:0")
        m = {k: torch.from_numpy(v).to(dev).requires_grad_(True) for k, v in gmap.items()}
        means2D = torch.zeros_like(m["means3D"], requires_grad=True)
        bg = torch.zeros(3, device=dev)
        for f in frames:
            f["d_rgb"], f["d_depth"] = torch.from_numpy(f["rgb"]).to(dev), torch.from_numpy(f["depth"]).to(dev)
            f["d_cam"] = {k: (torch.from_numpy(v).to(dev) if isinstance(v, np.ndarray) else v) for k, v in f["cam"].items()}

    def mapper_step(i):
        f = frames[frame_index(i + 1, len(frames))]
        if use_gpu:
            c = f["d_cam"]
            rs = dgr.GaussianRasterizationSettings(cam["H"], cam["W"], c["tanfovx"], c["tanfovy"], bg, 1.0, c["viewmatrix"],
                                                   c["projmatrix"], 0, c["campos"], False, False)
            depth, color, radii, is_used = dgr.GaussianRasterizer(rs)(means3D=m["means3D"], means2D=means2D,
                                                                      opacities=m["opacities"], shs=m["shs"],
                                                                      scales=m["scales"], rotations=m["rotations"])
            if args.loss == "l1":
                loss = (color - f["d_rgb"]).abs().mean() + 0.1 * (depth - f["d_depth"]).abs().mean()
            else:
                loss = torch_mapper_loss(color, depth, f["d_rgb"], f["d_depth"])
            loss.backward()
            lv = float(loss.item())
            for k in m:
                m[k].grad = None
            means2D.grad = None
            return lv
        from oracle import raster_oracle

        H, W = f["rgb"].shape[1:]
        o = raster_oracle.forward_backward(gmap, f["cam"], H, W, np.zeros(3, np.float32))
        gc = np.sign(o.color - f["rgb"]).astype(np.float32) / o.color.size
        gd = 0.1 * np.sign(o.depth - f["depth"]).astype(np.float32) / o.depth.size
        raster_oracle.forward_backward(gmap, f["cam"], H, W, np.zeros(3, np.float32), dL_dcolor=gc, dL_ddepth=gd)

    for i in range(args.warmup):
        mapper_step(i)
    msg = parent.recv()
    if msg[0] != "ready":
        raise SystemExit(f"reference tracker process failed: {msg}")
    _, kind, cores = msg
    if use_gpu:
        torch.cuda.synchronize()
    parent.send("go")
    t0 = time.perf_counter()
    for i in range(args.warmup, args.warmup + args.steps):
        mapper_step(i)
    if use_gpu:
        torch.cuda.synchronize()
    t_map = time.perf_counter() - t0
    msg = parent.recv()
    dt = time.perf_counter() - t0
    if msg[0] != "done":
        raise SystemExit(f"reference tracker process failed: {msg}")
    t_trk, pose_err = msg[1], msg[2]
    proc.join(timeout=10)
    fps = args.steps / dt
    mapper = ("reference CUDA rasterizer through its own torch extension (oracle/_ref/site, sm_90a) + PyTorch loss on cuda:0"
              if use_gpu else "CPU raster oracle (1 thread)")
    tracker = ("fast_gicp (reference sources + pybind module, oracle/_ref/fast_gicp; PCL k-NN through oracle/pcl_shim)"
               if kind == "reference" else "oracle restatement of fast_gicp")
    args.loss_impl = "torch"
    return {"metric": METRIC, "value": fps, "unit": "frames/s", "impl": "reference", "n_gpus": args.gpus, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": dt / args.steps * 1e3, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "f64 (GICP) / f32 (rasterizer)", "data": "synthetic",
            "config": workload_config(args, label),
            "reference_impl": {"tracker": tracker, "mapper": mapper,
                               "schedule": "tracker process (CPU) and mapper process (GPU) run concurrently, like gs_icp_slam.py:121-131"},
            "phase_ms_per_step": {"tracker_cpu_ms": t_trk / args.steps * 1e3, "mapper_ms": t_map / args.steps * 1e3},
            "tracker_max_pose_error": pose_err,
            "cpu_baseline": {"value": fps, "unit": "frames/s", "cores": cores, "kind": kind,
                             "sample": f"{args.steps} frames: {tracker} on {cores} threads || {mapper}"},
            "e2e": {"value": fps, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}


def workload_config(args, label, **extra):
    """Identical for both arms (the driver compares it): names the workload only."""
    loss = {"torch": "the reference mapper's loss (masked L1 + 0.2 DSSIM + 0.1 depth L1, mp_Mapper.py:225-242) in the reference's "
                     "PyTorch ops",
            "fused": "the reference mapper's loss through gs_icp_slam_b200.loss.mapping_loss (2 CUDA kernels)",
            "l1": "L1 colour + 0.1 L1 depth in PyTorch ops"}[getattr(args, "loss", "torch")]
    cam, max_corr, _ = slam_config(args.config)
    n_src = (int(cam["H"] / cam["downsample"]) + 1) * len(range(0, cam["W"], cam["downsample"]))
    c = {"workload": f"{label}: {cam['W']}x{cam['H']} RGB-D, {args.gaussians} Gaussians (seed {MAP_SEED.get(args.config, 3)}), "
                     f"{n_src} source points/frame, max_corr {max_corr}, align seeded with the previous estimated pose, keyframe every "
                     f"{KEYFRAME_EVERY} (target refresh), 1 mapper iteration (raster fwd + loss + raster bwd) per frame; loss = {loss}; "
                     f"tracker and mapper run concurrently",
         "l2": "256 MiB write between steps, excluded from the per-step CUDA-event time"}
    c.update(extra)
    return c


def ncu_traffic():
    """DRAM bytes and warp instructions per launch from an ncu capture of this build, summarised into
    profiles/ncu_traffic.json by tools/ncu_summary.py; {} (roofline.traffic null, no roofline.issue) until one is taken."""
    try:
        return json.load(open(os.path.join(ROOT, "profiles", "ncu_traffic.json")))
    except Exception:
        return {}


DUMP_LIMIT = 60_000_000  # bytes of array data written by --dump-outputs (the .npy headers add 128 bytes a file)


def dump_outputs(out_dir, outputs, n_gaussians):
    """DIR/<name>.npy for every output of a step: float32 arrays and integers below 2**24 as float32, other integers and the
    loss as float64.  When the whole set would pass DUMP_LIMIT, the per-Gaussian arrays (radii, grad_*) keep a fixed, seeded
    sample of Gaussians, whose indices are written as gaussian_rows.npy."""
    import torch

    arrays = {}
    for name, v in outputs.items():
        a = v.detach().cpu().numpy() if torch.is_tensor(v) else np.asarray(v)
        small_int = a.dtype.kind in "iu" and (a.size == 0 or int(np.abs(a).max()) < (1 << 24))
        arrays[name] = a.astype(np.float32) if (a.dtype.kind == "f" and a.dtype.itemsize <= 4) or small_int else a.astype(np.float64)
    per_gaussian = [k for k in arrays if k == "radii" or k.startswith("grad_")]
    if sum(a.nbytes for a in arrays.values()) > DUMP_LIMIT:
        other = sum(a.nbytes for k, a in arrays.items() if k not in per_gaussian)
        per_row = 8 + sum(arrays[k].nbytes // n_gaussians for k in per_gaussian)
        keep = max(0, min(n_gaussians, (DUMP_LIMIT - other) // per_row))
        rows = np.sort(np.random.default_rng(0).choice(n_gaussians, size=keep, replace=False))
        for k in per_gaussian:
            arrays[k] = arrays[k][rows]
        arrays["gaussian_rows"] = rows.astype(np.float64)
    os.makedirs(out_dir, exist_ok=True)
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"), a)


def bind_to_gpu_numa(local_rank, world):
    """N > 1 on one host: pin this rank (its Python threads, the library's spin-waits, pinned-staging copies) to the CPUs
    of its GPU's NUMA node, split evenly among the ranks that share the node (r1: e2e replica efficiency 0.71 at N = 8 with
    16 unpinned host threads hopping between the two sockets).  Returns a description for the JSON line, or None."""
    try:
        import pynvml as nv

        nv.nvmlInit()
        ncpu = os.cpu_count() or 1
        words = (ncpu + 63) // 64

        def cpus_of(i):
            mask = nv.nvmlDeviceGetCpuAffinity(nv.nvmlDeviceGetHandleByIndex(i), words)
            return tuple(c for c in range(ncpu) if (mask[c // 64] >> (c % 64)) & 1)

        mine = cpus_of(local_rank)
        allowed = set(os.sched_getaffinity(0))
        mine = tuple(c for c in mine if c in allowed)
        if not mine:
            return None
        sharing = [r for r in range(world) if cpus_of(r) == cpus_of(local_rank)]
        k, n = sharing.index(local_rank), len(sharing)
        per = max(2, len(mine) // n)
        part = mine[k * per:(k + 1) * per] or mine
        os.sched_setaffinity(0, part)
        return {"cpus": len(part), "of_node": len(mine), "ranks_on_node": n}
    except Exception:
        return None


def main():
    args = parse()
    rank = int(os.environ.get("RANK", 0))
    local_rank = int(os.environ.get("LOCAL_RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    if args.dump_outputs is not None and (args.config in ("c1", "c4", "c5") or args.impl != "ours"
                                          or (world > 1 and args.multi == "shard")):
        raise SystemExit("bench.py: --dump-outputs covers the SLAM frame of --impl ours (--config c3 or c2, not --multi shard, "
                         "whose ranks each hold a part of the frame)")
    if args.config in ("c1", "c4", "c5"):
        from tools import bench_large

        return bench_large.main(args, rank, local_rank, world)
    if args.impl == "reference":
        if rank != 0:
            return
        print(json.dumps(reference_arm(args)))
        return

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device — gs_icp_slam_b200 has no CPU path (use --impl reference for the CPU arm)")
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    affinity = None
    if world > 1:
        import torch.distributed as dist

        affinity = bind_to_gpu_numa(local_rank, world)
        dist.init_process_group("nccl", device_id=dev)
    cam, max_corr, label, gmap, frames = make_sequence(args.steps + args.warmup, args.config, args.gaussians)
    shard = world > 1 and args.multi == "shard"
    if shard and args.loss != "l1":
        args.loss = "l1"
    eng = Ours(cam, max_corr, gmap, frames, dev, world, rank, shard=shard, loss=args.loss)
    from gs_icp_slam_b200 import _lib

    K, Wm = args.steps, args.warmup
    pre = min(K, 5)
    # untimed pre-pass: CUDA module loading, caching-allocator growth and library scratch growth happen here
    eng.run(pre, 1, resident=False)
    eng.run(pre, 1, resident=True)

    def max_over_ranks(x):
        if world == 1:
            return x
        t = torch.tensor([x], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    seqs = 1 if shard else world  # replicas: every rank walks its own K frames

    def fps(t_ms):
        return seqs * K / (t_ms * 1e-3)

    concurrent = not shard  # the sharded run drives one stream (the collectives are ordered on it)
    with ClockSampler(local_rank) as clk:
        eng.enable_concurrent(concurrent)
        if concurrent:
            eng.run(pre, 1, resident=True)  # stream / thread start-up, untimed
        eng.keep_outputs = args.dump_outputs is not None
        r = eng.run(K, Wm, resident=True)
        eng.keep_outputs = False
        res_times = list(eng.last_times)
        if args.dump_outputs is not None and rank == 0:
            dump_outputs(args.dump_outputs, eng.last_outputs, args.gaussians)
        e = eng.run(K, Wm, resident=False)
        e2e_times = list(eng.last_times)
    clocks = clk.summary()
    t_res, t_e2e = max_over_ranks(r[0]), max_over_ranks(e[0])
    _, launches, st_res = r
    _, _, st_e2e = e

    extra = {}
    if not args.no_variants and not shard:
        # the same frame with the mapper's loss through the fused op (SURVEY §8f N2) / through PyTorch ops
        other = "fused" if args.loss != "fused" else "torch"
        eng.set_loss(other)
        eng.run(pre, 1, resident=True)
        tv = max_over_ranks(eng.run(K, Wm, resident=True)[0])
        te = max_over_ranks(eng.run(K, Wm, resident=False)[0])
        extra[other + "_loss"] = {"value": fps(tv), "e2e": fps(te), "ms_per_step": tv / K,
                                  "note": "same frame, mapper loss through " +
                                          ("gs_icp_slam_b200.loss.mapping_loss (fused CUDA op)" if other == "fused" else "the reference's PyTorch ops")}
        eng.set_loss(args.loss)
        # the back-to-back schedule (one host thread, one stream) for comparison
        eng.enable_concurrent(False)
        eng.run(pre, 1, resident=True)
        tb = max_over_ranks(eng.run(K, Wm, resident=True)[0])
        tbe = max_over_ranks(eng.run(K, Wm, resident=False)[0])
        extra["schedules"] = {"concurrent": {"value": fps(t_res), "e2e": fps(t_e2e),
                                             "value_ms_p50_max": [float(np.median(res_times)), float(np.max(res_times))],
                                             "e2e_ms_p50_max": [float(np.median(e2e_times)), float(np.max(e2e_times))]},
                              "back_to_back": {"value": fps(tb), "e2e": fps(tbe)},
                              "headline": "concurrent"}
    eng.enable_concurrent(False)
    prof, st_p = {}, st_res
    if not args.no_roofline:
        _, _, st_p = eng.run(K, Wm, resident=True, profile=True)
        prof = _lib.prof_read()
    eng.close()
    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return

    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm_peak, peak_src = (peaks["hbm_gbs"], "measured (MEASURED_PEAKS.json)") if "hbm_gbs" in peaks else (3350.0, "H100 SXM data sheet (3.35 TB/s HBM3)")

    roofline, kernels = None, {}
    if prof:
        tiles = ((cam["W"] + 15) // 16) * ((cam["H"] + 15) // 16)
        npix = cam["W"] * cam["H"]
        R, V = st_p["R"] / K, st_p["V"] / K
        n_src, n_corr, n_tgt = st_p["n_src"] / K, st_p["n_corr"] / K, st_p["n_tgt"] / K
        P = args.gaussians
        alg = {  # algorithmic bytes per launch (SURVEY.md §8d / DESIGN.md §5)
            "render_forward": 8 * tiles + 52 * R + 36 * npix,
            "render_backward": 8 * tiles + 52 * R + 36 * npix + 56 * V,
            # one launch of the device-resident LM loop = n_lin x (linearize + >= 1 compute_error) (SURVEY §8d per-call figures)
            "gicp_linearize": (st_p["n_lin"] / K) * ((60 * n_src + 60 * n_corr + 12 * n_tgt + 224) + (12 * n_src + 60 * n_corr + 8)),
            "gicp_error": 12 * n_src + 60 * n_corr + 8,
            "preprocess": 56 * P + 5 * P + 79 * V,
            "gaussian_backward": V * 139 + P * 64,
            "tile_sort": 12 * R,
            "tile_scan": 24 * tiles,
            "emit_instances": 52 * V + 4 * P + 8 * R,
            "gicp_covariance": 160 * n_src + 60 * n_src,
        }
        traffic = ncu_traffic()
        for name, (ms, n) in prof.items():
            if n > 0:
                per = ms / n
                kernels[name] = {"launches_per_step": n / K, "ms_per_launch": per, "ms_per_step": ms / K}
                if alg.get(name):
                    kernels[name]["achieved_GBps"] = alg[name] / (per * 1e-3) / 1e9
        cand = [k for k in kernels if alg.get(k)]
        top = max(cand, key=lambda k: kernels[k]["ms_per_step"])
        ach = kernels[top]["achieved_GBps"]
        tr = traffic.get(top, {})
        roofline = {"kernel": top, "bound": "hbm", "achieved": ach, "peak": hbm_peak, "unit": "GB/s", "frac": ach / hbm_peak,
                    "traffic": tr.get("dram_bytes"), "traffic_source": tr.get("source"),
                    "peak_source": peak_src, "algorithmic_bytes_per_launch": alg[top],
                    "ms_per_launch": kernels[top]["ms_per_launch"]}
        if tr.get("warp_instructions"):
            a = tr["warp_instructions"] / (kernels[top]["ms_per_launch"] * 1e-3) / 1e9
            pk = 132 * 4 * ((clocks or {}).get("sm_mhz") or 1980.0) * 1e6 / 1e9
            roofline["issue"] = {"warp_instructions_per_launch": tr["warp_instructions"], "achieved": a, "peak": pk,
                                 "unit": "G warp-inst/s", "frac": a / pk,
                                 "note": "instruction count from an ncu capture summarised into profiles/ncu_traffic.json by tools/ncu_summary.py; "
                                         "peak = 132 SMs x 4 schedulers x SM clock (H100 SXM)"}
        if "render_forward" in kernels and "render_backward" in kernels:
            roofline["render_fwd_bwd_GBps"] = ((alg["render_forward"] + alg["render_backward"]) / 1e9 /
                                              ((kernels["render_forward"]["ms_per_launch"] + kernels["render_backward"]["ms_per_launch"]) * 1e-3))

    parallelism = ("single GPU" if world == 1 else
                   f"{world} GPUs, one sequence, raster tiles + GICP source points sharded, in-library exchange over peer memory" if shard else
                   f"{world} independent SLAM sequences (replicas), one per GPU, no collective")
    out = {"metric": METRIC, "value": fps(t_res), "unit": "frames/s", "n_gpus": world, "steps": K, "warmup": Wm,
           "ms_per_step": t_res / K, "higher_is_better": True, "scaling": "strong" if shard else "weak", "vs_baseline": None,
           "dtype": "f64 (GICP algebra on f32 points) / f32 (rasterizer)", "data": "synthetic",
           "config": workload_config(args, label),
           "parallelism": parallelism, "host_affinity": affinity,
           "loss_impl": {"torch": "PyTorch ops (unmodified mp_Mapper.py)", "fused": "gs_icp_slam_b200.loss.mapping_loss",
                         "l1": "PyTorch ops (L1 only)"}[args.loss],
           "frame_stats": {"lm_iterations_per_frame": st_res["n_lin"] / K, "tile_instances_per_frame": st_res["R"] / K,
                           "visible_gaussians_per_frame": st_p["V"] / K, "max_pose_error_vs_ground_truth": st_res["pose_err"]},
           "clocks": clocks, "gpu_launches": launches,
           "e2e": {"value": fps(t_e2e), "unit": "frames/s", "ms_per_step": t_e2e / K,
                   "h2d_bytes_per_step": st_e2e["h2d"] / K, "d2h_bytes_per_step": st_e2e["d2h"] / K},
           "roofline": roofline, "kernels": kernels}
    out.update(extra)
    if world == 1 and not args.no_cpu_baseline:
        out["cpu_baseline"] = cpu_baseline(label, max_corr, gmap, frames)
    print(json.dumps(out))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
