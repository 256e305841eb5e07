"""Deterministic render backward (gsicp_raster_set_deterministic, selected by torch.use_deterministic_algorithms).

The default render backward adds each Gaussian's 12 moments over its (sub-tile, survivor group) contributions with float
atomics, in whatever order the CTAs get there.  The deterministic mode runs the kernel twice with integer atomics only
(raster_backward.cu, DetRow): pass A takes, per Gaussian and moment, the largest biased fp32 exponent field E of the
contributions and, per Gaussian, their count n; pass B adds llrint(c 2^(S + 126 - E)) into an int64 with
S = 62 - ceil(log2 n); the result is float(double(acc) 2^(E - 126 - S)).

CPU: a numpy model of that rule against exact sums (every fp32 value is an integer multiple of 2^-149, so Python integers
sum them exactly): no int64 overflow in any order, and |fixed-point sum - exact| <= n/2 2^(E - 126 - S).
GPU: bit-identical gradients and moments over repeated backwards, permuted tile launch orders, every backward path and
tile shards; the per-Gaussian float64 bound of test_raster_bwd_bound.py; the 2e-4 bar against the default mode and the
reference's golden records; the torch switch; and whole mapper iterations.
"""
import contextlib
from fractions import Fraction

import numpy as np
import pytest

from tests.test_raster_bwd_bound import GPU_CASES, U, GpuRun, _gpu_case, _reference, check_gradients, check_tap
from tests.util import rel_err


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the exponent / count / scale rule
# ---------------------------------------------------------------------------------------------------------------------
def det_sum(c):
    """(float32 result, int64 accumulator, E, S) of the deterministic sum of the float32 terms c (finite)."""
    c = np.asarray(c, np.float32)
    n = len(c)
    nz = c[c != 0]
    if len(nz) == 0:
        return np.float32(0.0), 0, 0, 62
    E = int(((nz.view(np.uint32) >> 23) & 0xFF).max())
    S = 62 - (n - 1).bit_length()
    q = np.rint(np.ldexp(nz.astype(np.float64), S + 126 - E)).astype(np.int64)  # exact scaling, round half to even
    assert np.abs(q).max() <= 2 ** S and n * 2 ** S <= 2 ** 62  # so no partial sum, in any order, overflows int64
    acc = int(q.sum())
    assert acc == sum(int(x) for x in q)
    with np.errstate(over="ignore"):  # a sum beyond the float32 range becomes +-inf, as on the GPU
        out = np.float32(np.float64(acc) * 2.0 ** (E - 126 - S))
    return out, acc, E, S


def exact_sum(c):
    """The exact sum of float32 terms, as a Fraction."""
    k = np.ldexp(np.asarray(c, np.float32).astype(np.float64), 149)  # integers, exactly
    return Fraction(sum(int(x) for x in k), 2 ** 149)


def check_rule(c):
    c = np.asarray(c, np.float32)
    out, acc, E, S = det_sum(c)
    ex = exact_sum(c)
    n = len(c)
    fixed = Fraction(acc) * Fraction(2) ** (E - 126 - S)
    bound = Fraction(n, 2) * Fraction(2) ** (E - 126 - S)
    assert abs(fixed - ex) <= bound, (float(abs(fixed - ex)), float(bound))
    if np.isfinite(out):  # double(acc) and the float conversion round once each
        assert abs(Fraction(float(out)) - ex) <= bound + Fraction(2) ** -23 * (abs(ex) + bound) + Fraction(2) ** -149
    else:  # overflow to inf only where the exact sum is beyond the float32 range
        assert abs(ex) >= Fraction(float(np.finfo(np.float32).max))


@pytest.mark.parametrize("sign", [1.0, -1.0])
@pytest.mark.parametrize("n", [1, 2, 3, 1000, 2 ** 16 + 1, 2 ** 20])
def test_rule_equal_sign_max_magnitude(n, sign):
    big = np.float32(sign * np.finfo(np.float32).max)
    c = np.full(n, big, np.float32)
    out, acc, E, S = det_sum(c)
    assert E == 254 and abs(acc) <= 2 ** 62
    check_rule(c)
    half = np.full(n, np.float32(sign * 2.0 ** 100), np.float32)  # representable sum: exact
    out, acc, E, S = det_sum(half)
    assert out == np.float32(sign * n * 2.0 ** 100)


@pytest.mark.parametrize("seed", range(4))
def test_rule_whole_fp32_range_with_subnormals(seed):
    rng = np.random.default_rng(seed)
    n = [5000, 2 ** 17, 77, 2 ** 20][seed]
    e = rng.integers(-149, 128, size=n)
    m = rng.uniform(1.0, 2.0, size=n)
    c = (np.ldexp(m, e) * rng.choice([-1.0, 1.0], size=n)).astype(np.float32)
    c[: n // 10] = (rng.integers(1, 2 ** 23, size=n // 10) * 2.0 ** -149 * rng.choice([-1.0, 1.0], size=n // 10)).astype(np.float32)
    assert np.any((c != 0) & (np.abs(c) < np.finfo(np.float32).tiny))  # subnormals present
    c = c[np.isfinite(c)]
    check_rule(c)
    sub = c[(c != 0) & (np.abs(c) < np.finfo(np.float32).tiny)]  # subnormals only: E = 0, still within the bound
    out, acc, E, S = det_sum(sub)
    assert E == 0
    check_rule(sub)


@pytest.mark.parametrize("n", [2, 1001, 2 ** 20])
def test_rule_heavy_cancellation(n):
    rng = np.random.default_rng(n)
    x = (rng.normal(size=n // 2) * 1e30).astype(np.float32)
    c = np.concatenate([x, -x, (rng.normal(size=n - 2 * (n // 2)) * 1e-3).astype(np.float32)])
    c[0] = np.float32(3e30)
    c = c[rng.permutation(len(c))]
    check_rule(c)


@pytest.mark.parametrize("n", [1, 7, 2 ** 20])
def test_rule_all_zeros(n):
    c = np.zeros(n, np.float32)
    c[::2] = -0.0
    out, acc, E, S = det_sum(c)
    assert out == 0 and acc == 0


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def torch_deterministic(on):
    """torch.use_deterministic_algorithms(on) for the block; the previous setting is restored."""
    import torch

    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


@pytest.fixture
def restore_switch():
    import torch

    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


@contextlib.contextmanager
def tile_order(mode, seed=0):
    from gs_icp_slam_b200 import _lib

    _lib.lib.gsicp_test_set_bwd_tile_order(mode, seed)
    try:
        yield
    finally:
        _lib.lib.gsicp_test_set_bwd_tile_order(0, 0)


def last_mode():
    from gs_icp_slam_b200 import _lib

    return _lib.lib.gsicp_test_last_bwd_mode()


def bits(x):
    x = np.ascontiguousarray(x)
    return x.view({4: np.int32, 8: np.int64}[x.dtype.itemsize])


def same_bits(a, b):
    """(tap, grads) of two backwards are bit-identical."""
    return np.array_equal(bits(a[0]), bits(b[0])) and all(np.array_equal(bits(x), bits(y)) for x, y in zip(a[1], b[1]))


def det_backward(run, gc, gd):
    with torch_deterministic(True):
        out = run.backward(gc, gd)
    assert last_mode() == 1, "the deterministic path did not run"
    return out


def repeat_identical(run, gc, gd, name, k=5):
    first = det_backward(run, gc, gd)
    for i in range(k - 1):
        assert same_bits(first, det_backward(run, gc, gd)), f"{name}: deterministic backward {i + 2} differs from the first"
    return first


@pytest.mark.gpu
@pytest.mark.parametrize("name", GPU_CASES)
def test_deterministic_repeat_order_and_bound(cuda, name, restore_switch):
    g, cm, W, H, bg, deg, gc, gd = _gpu_case(name)
    run = GpuRun(cuda, g, cm, W, H, bg, deg)
    det = repeat_identical(run, gc, gd, name)
    for mode, seed in ((1, 0), (2, 12345)):
        with tile_order(mode, seed):
            assert same_bits(det, det_backward(run, gc, gd)), f"{name}: tile order {mode} changes the deterministic result"
    # default mode: the same permutation, for information only
    with torch_deterministic(False):
        dflt = run.backward(gc, gd)
        assert last_mode() == 0
        with tile_order(2, 12345):
            dflt_perm = run.backward(gc, gd)
    print(f"\n[det] {name}: default mode {'differs' if not same_bits(dflt, dflt_perm) else 'does not differ'} under a shuffled "
          f"tile order")
    # accuracy: the per-Gaussian float64 bound, and the 2e-4 bar against the default mode
    tap, grads = det
    ref, vis, _ = _reference(run, gc, gd, bg)
    finite = name == "far_and_needles"
    worst, med = check_tap(name, tap, ref, vis, finite_only=finite)
    check_gradients(name, tap, grads, ref, vis)
    for a, b in zip(grads, dflt[1]):
        if finite:
            keep = np.isfinite(a) & np.isfinite(b)
            assert np.array_equal(np.isfinite(a), np.isfinite(b))
            a, b = a[keep], b[keep]
        if b.size:
            assert rel_err(a, b) <= 2e-4
    print(f"[det] {name}: |err|/B worst {worst:.3g} median {med:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("switch", ["variant1", "nocull"])
@pytest.mark.parametrize("name", ["fb_20000", "deep", "edge_17x33"])
def test_deterministic_every_backward_path(cuda, name, switch, restore_switch):
    from gs_icp_slam_b200 import _lib

    g, cm, W, H, bg, deg, gc, gd = _gpu_case(name)
    set_fn, on, off = {"variant1": (_lib.lib.gsicp_test_set_bwd_variant, 1, 0),
                       "nocull": (_lib.lib.gsicp_test_set_render_cull, 0, 1)}[switch]
    set_fn(on)
    try:
        run = GpuRun(cuda, g, cm, W, H, bg, deg)
        tap, grads = repeat_identical(run, gc, gd, f"{name}/{switch}")
        with tile_order(1):
            assert same_bits((tap, grads), det_backward(run, gc, gd))
    finally:
        set_fn(off)
    ref, vis, _ = _reference(run, gc, gd, bg)
    worst, med = check_tap(f"{name}/{switch}", tap, ref, vis)
    check_gradients(f"{name}/{switch}", tap, grads, ref, vis)
    print(f"\n[det] {name}/{switch}: |err|/B worst {worst:.3g} median {med:.3g}")


@pytest.mark.gpu
def test_deterministic_tile_shards(cuda, restore_switch):
    g, cm, W, H, bg, deg, gc, gd = _gpu_case("fb_20000")
    full = GpuRun(cuda, g, cm, W, H, bg, deg)
    ref, vis, _ = _reference(full, gc, gd, bg)
    taps = []
    for k in range(3):
        run = GpuRun(cuda, g, cm, W, H, bg, deg, shard=(3, k))
        tap, _ = repeat_identical(run, gc, gd, f"shard {k}")
        with tile_order(2, 7):
            assert same_bits((tap, _), det_backward(run, gc, gd)), f"shard {k}: tile order"
        tap[~vis] = 0.0
        taps.append(tap.astype(np.float32))
    total = (taps[0] + taps[1] + taps[2]).astype(np.float64)
    extra = 2 * U * 3 * (np.abs(taps[0]) + np.abs(taps[1]) + np.abs(taps[2]))
    worst, med = check_tap("det shards", total, ref, vis, extra=extra)
    print(f"\n[det] shards 3: |err|/B worst {worst:.3g} median {med:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("P,size,degree,seed", [(20000, (320, 240), 0, 2), (100000, (640, 480), 0, 3), (30000, (333, 211), 3, 5)])
def test_deterministic_vs_reference_golden(cuda, P, size, degree, seed, restore_switch):
    import torch

    from gs_icp_slam_b200 import rasterizer as R
    from tests.test_raster_gpu import GRADS, _gold, _ours, case_fb

    t, c, bg, gcol, gdep = case_fb(cuda, P, size, degree, seed)
    W, H = size
    n, depth, color, radii, is_used, geom, binning, img = _ours(t, c, H, W, bg, degree)
    ref = _gold(f"fb_{P}_{degree}_{seed}")
    e = torch.Tensor([])
    with torch_deterministic(True):
        ours = R.rasterize_gaussians_backward(bg, t["means3D"], radii, e, t["scales"], t["rotations"], 1.0, e, c["viewmatrix"],
                                              c["projmatrix"], c["tanfovx"], c["tanfovy"], gdep, gcol, t["shs"], degree,
                                              c["campos"], geom, n, binning, img, False)
    assert last_mode() == 1
    for name, o in zip(GRADS, ours):
        err = ref.rel_err("grad_" + name, o.cpu().numpy())
        assert err <= 2e-4, f"grad {name}: rel err {err}"


def _autograd_grads(cuda, t, c, H, W):
    import torch
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer

    p = {k: v.detach().clone().requires_grad_(True) for k, v in t.items()}
    m2 = torch.zeros_like(p["means3D"], requires_grad=True)
    rs = GaussianRasterizationSettings(H, W, c["tanfovx"], c["tanfovy"], torch.tensor([0.1, 0.2, 0.3], device=cuda), 1.0,
                                       c["viewmatrix"], c["projmatrix"], 0, c["campos"], False, False)
    depth, color, radii, _ = GaussianRasterizer(rs)(means3D=p["means3D"], means2D=m2, opacities=p["opacities"], shs=p["shs"],
                                                    scales=p["scales"], rotations=p["rotations"])
    gen = torch.Generator(device="cpu").manual_seed(5)
    loss = (color * torch.randn(color.shape, generator=gen).to(cuda)).sum() + (depth * torch.randn(depth.shape, generator=gen).to(cuda)).sum()
    loss.backward()
    out = {k: v.grad.cpu().numpy() for k, v in p.items()}
    out["means2D"] = m2.grad.cpu().numpy()
    return out


@pytest.mark.gpu
def test_torch_switch_selects_the_mode(cuda, restore_switch):
    import torch

    from tests.util import scene_tensors

    _, _, t, c, _ = scene_tensors(30000, 8, cuda, size=(320, 240))
    torch.use_deterministic_algorithms(True)
    a = _autograd_grads(cuda, t, c, 240, 320)
    assert last_mode() == 1
    b = _autograd_grads(cuda, t, c, 240, 320)
    assert all(np.array_equal(bits(a[k]), bits(b[k])) for k in a), "autograd gradients differ under the torch switch"
    torch.use_deterministic_algorithms(False)
    d = _autograd_grads(cuda, t, c, 240, 320)
    assert last_mode() == 0
    for k in a:
        assert rel_err(a[k], d[k]) <= 2e-4, k


def _mapper_run(cuda, iters=20, P=100000, seed=4):
    """`iters` mapper iterations (forward, fused loss, backward, FusedAdam) with a tracker align() between them."""
    import torch

    import pygicp
    from diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    from gs_icp_slam_b200 import loss as L
    from gs_icp_slam_b200 import synthetic as S
    from gs_icp_slam_b200.map_table import FusedAdam

    g = S.gaussian_map(P, seed)
    params = {k: torch.from_numpy(v).to(cuda).requires_grad_(True) for k, v in g.items()}
    lrs = {"means3D": 1e-4, "shs": 2.5e-3, "opacities": 5e-2, "scales": 5e-3, "rotations": 1e-3}
    opt = FusedAdam([{"params": [params[k]], "lr": lrs.get(k, 1e-3), "name": k} for k in params], lr=0.0, eps=1e-15)
    means2D = torch.zeros_like(params["means3D"], requires_grad=True)
    gen = torch.Generator(device="cpu").manual_seed(seed)
    gt_rgb = torch.rand((3, 480, 640), generator=gen).to(cuda)
    gt_depth = (torch.rand((1, 480, 640), generator=gen) * 3.0).to(cuda)
    tgt, src, _ = S.gicp_pair(4000, 3000, 50, 51)
    reg = pygicp.FastGICP()
    reg.set_max_correspondence_distance(0.05)
    reg.set_max_knn_distance(99999)
    reg.set_input_target(tgt)
    reg.calculate_target_covariance_with_filter()
    reg.set_input_source(src)
    pose, poses, losses = np.eye(4), [], []
    for it in range(iters):
        cm = S.camera_matrices(S.trajectory_pose(it % 10, 20), S.TUM)
        c = {k: (torch.from_numpy(v).to(cuda) if isinstance(v, np.ndarray) else v) for k, v in cm.items()}
        rs = GaussianRasterizationSettings(480, 640, c["tanfovx"], c["tanfovy"], torch.zeros(3, device=cuda), 1.0,
                                           c["viewmatrix"], c["projmatrix"], 0, c["campos"], False, False)
        depth, color, radii, _ = GaussianRasterizer(rs)(means3D=params["means3D"], means2D=means2D, opacities=params["opacities"],
                                                        shs=params["shs"], scales=params["scales"], rotations=params["rotations"])
        loss = L.mapping_loss(color, depth, gt_rgb, gt_depth)
        loss.backward()
        opt.step()
        for p in params.values():
            p.grad = None
        means2D.grad = None
        losses.append(float(loss.detach()))
        pose = reg.align(pose)
        poses.append(np.array(pose))
    torch.cuda.synchronize()
    state = {k: v.detach().cpu().numpy() for k, v in params.items()}
    for k, p in params.items():
        st = opt.state[p]
        state[k + "/exp_avg"] = st["exp_avg"].cpu().numpy()
        state[k + "/exp_avg_sq"] = st["exp_avg_sq"].cpu().numpy()
    return state, np.stack(poses), losses


@pytest.mark.gpu
def test_mapper_iterations_bit_identical(cuda, restore_switch):
    import torch

    torch.use_deterministic_algorithms(True)
    a, pa, la = _mapper_run(cuda)
    assert last_mode() == 1
    b, pb, lb = _mapper_run(cuda)
    assert la == lb, "losses differ"
    assert np.array_equal(bits(pa), bits(pb)), "tracker poses differ"
    for k in a:
        assert np.array_equal(bits(a[k]), bits(b[k])), f"{k} differs after 20 deterministic mapper iterations"
    assert la[-1] < la[0]
    print(f"\n[det] 20 mapper iterations, 100000 Gaussians, 640x480: bit-identical; loss {la[0]:.5f} -> {la[-1]:.5f}")
