"""Per-Gaussian check of the rasterizer's render backward against an error-bounded float64 replay of the forward's own state.

render_backward_kernel reduces, per (8x4 sub-tile, instance), twelve moments of t = G dL/dalpha and w = alpha T over the
warp's pixels on the tensor cores, shifts them from the warp's integer frame to the Gaussian's centre and adds them into
[P][12] with float atomics; gaussian_backward_kernel turns them into the render gradients.  The array-wide checks of
test_raster_gpu.py (max |a - b| <= 2e-4 max |b|) are dominated by a few large Gaussians, so a Gaussian that loses a
sub-tile, or a pixel column attributed to its neighbour, can pass them.  Here every Gaussian and every moment is checked
against oracle/raster_oracle.c:ro_moment_reference, which replays the GPU's SAVED state (splat records, instance list,
tile ranges, n_contrib) in float64 and returns, per Gaussian, the moments, the render gradients and an error bound.

Derivation of the bound (u = 2^-23, the float32 unit roundoff).  For an active pair k of pixel p, let s_k be the absolute
shadow of its expression: for t
    s_t = G ((sum_c (|c| + |acc_c|) |dp_c| + (|depth| + |acc_d|) |dpd|) T + T_final (sum_c |bg_c dp_c| + 15 |dpd|) / (1 - alpha))
(acc = the colour / depth blended behind, accumulated with absolute values; |depth| = the absolute shadow of the conditioned
depth), and for w, s_w = alpha T.  Every float32 step of the GPU changes the pair's term by at most 2u s_k times its basis
shadow b_k: 1, X, Y, X^2, XY, Y^2 for the t-moments, |dpd| {1, X, Y} and |dp_c| for the w-moments, with X = |dx| + 16 and
Y = |dy| + 8.  The offsets are the warp frame: the GPU sums i^a j^b t over pixel offsets i in 0..7, j in 0..3 and forms
e.g. cx^2 S0 - 2 cx S1 + S_ii with |cx| <= |dx| + 7, so its cancelling terms are bounded by (|dx| + 14)^2 |t|.  The number
of steps counted per pair is
    3 n_p                      T: final_T carries n_p products, the backward recovers T through n_p reciprocals
                               (rcp.approx, 1 ulp) and n_p products; also covers the n_p-step blend-behind recurrences
    e_p = sum_j (4 + q_j) / (1 - alpha_j)   the pixel's alphas: expf (2 ulp), the rounding of power (shadow
                               q = |A dx^2| + |C dy^2| + 2 |B dx dy|) and the product with the opacity, amplified through
                               T by 1 / (1 - alpha); a clearly clamped alpha is the float 0.99 on both sides and adds nothing
    q_k + 64                   the pair's own G, the split tf32 MMA (22-bit products, 8 accumulating MMAs of 8-term sums
                               per k-step pair), the centre shift and the epilogue
    S_g                        the float atomics over the Gaussian's S_g sub-tiles (added per Gaussian)
so  B_moment = 2u sum_k (3 n_p + e_p + q_k + 64 + S_g) s_k b_k.
A pair is ambiguous when power, or ln(255 alpha), lies within 64u (1 + q) of its threshold: the GPU's float32 decision
there cannot be known.  Such a pair adds its own |term| s_k b_k to its Gaussian's bound, and 2 alpha / (1 - alpha) times
the shadows of every other pair of its pixel (their T and blend-behind change by that factor).  A Gaussian with no active
or ambiguous pair has reference 0 and bound 0: the GPU must return exactly 0.  The render gradients are linear in the
moments (gaussian_backward_kernel); their bound is sum_i |coef_i| (B_i + 8u |m_i|), with |coef| the absolute shadow of the
coefficient expression.

The constants are validated on the CPU, without a GPU: the float32 restatement ro_backward (DGR's per-pair expression
trees, a different association from the moments, exact divisions, glibc expf) must lie within the bound for every
Gaussian and component in four scenes, and planted errors must be caught.  The worst |err| / B on the float32 restatement
is 2e-3 .. 3e-2 per scene (4e-1 on a denser low-opacity crowd, where near-equal alphas round the transmittance in one
direction and its error grows linearly with n_p), so the bound is within two orders of magnitude of errors that occur.
It is loosest for mean2D (worst ~1e-3), whose bound carries the warp-frame offsets that the restatement does not have.
"""
import ctypes as C

import numpy as np
import pytest

from gs_icp_slam_b200 import synthetic as S
from oracle import raster_oracle as RO

U = 2.0 ** -23
MOM = RO.MOMENTS
GRD = RO.RENDER_GRADS


# ---------------------------------------------------------------------------------------------------------------------
# scenes (numpy), shared by the CPU and GPU parts
# ---------------------------------------------------------------------------------------------------------------------
def scene(P, seed, size, degree=0, frame=3):
    cam = dict(S.TUM)
    W, H = size
    sx, sy = W / cam["W"], H / cam["H"]
    cam.update(W=W, H=H, fx=cam["fx"] * sx, fy=cam["fy"] * sy, cx=cam["cx"] * sx, cy=cam["cy"] * sy)
    g = S.gaussian_map(P, seed, sh_degree=degree)
    cm = S.camera_matrices(S.trajectory_pose(frame, 20), cam)
    return g, cm


def crowd(g, cm, spread, opacity=None):
    """Pull every Gaussian towards a point 2 m in front of the camera (a few tiles hold thousands of instances)."""
    centre = cm["campos"] + 2.0 * cm["viewmatrix"][:3, 2]
    g["means3D"] = (centre + spread * (g["means3D"] - g["means3D"].mean(0))).astype(np.float32)
    g["means3D"][100:200] = g["means3D"][300:400]  # exact duplicates: equal depth keys
    if opacity is not None:
        g["opacities"][:] = opacity
    return g


def far_and_needles(g, cm):
    """Wide Gaussians centred hundreds of pixels outside the frame, and 1 km x 2 cm needles."""
    view = cm["viewmatrix"]  # (world -> view)^T
    right, down, fwd = view[:3, 0], view[:3, 1], view[:3, 2]
    cp = cm["campos"]
    k = 0
    for z, ox, oy in [(3.0, 2.5, 0.0), (3.0, -2.2, 0.4), (4.0, 0.3, 2.6), (2.5, -1.8, -1.9), (5.0, 4.0, 1.0), (3.0, 0.0, -3.0)]:
        g["means3D"][k] = cp + z * fwd + ox * z * right + oy * z * down
        g["scales"][k] = [1.5 * z, 1.2 * z, 0.3]
        g["opacities"][k] = 0.9
        k += 1
    g["scales"][10:14, 0] = 1000.0  # needles
    return g


def _dpix(seed, H, W):
    rng = np.random.default_rng(seed)
    return rng.normal(size=(3, H, W)).astype(np.float32), rng.normal(size=(1, H, W)).astype(np.float32)


def _dpix_structured(kind, H, W):
    gc, gd = np.zeros((3, H, W), np.float32), np.zeros((1, H, W), np.float32)
    if kind == "impulses":  # sub-tile and tile corners (x = 0, 7, 8, 15 mod 16; y = 0, 3, 4, 7, 8, 11, 12, 15 mod 16)
        xs = [x for x in range(W) if x % 16 in (0, 7, 8, 15)]
        ys = [y for y in range(H) if y % 4 in (0, 3)]
        rng = np.random.default_rng(1)
        gc[:, np.ix_(ys, xs)[0], np.ix_(ys, xs)[1]] = rng.normal(size=(3, len(ys), len(xs)))
        gd[:, np.ix_(ys, xs)[0], np.ix_(ys, xs)[1]] = rng.normal(size=(1, len(ys), len(xs)))
    elif kind == "colour_only":
        gc = _dpix(2, H, W)[0]
    elif kind == "depth_only":
        gd = _dpix(3, H, W)[1]
    elif kind == "dynamic_range":  # 1e-6 .. 1e3 within every warp, random signs
        rng = np.random.default_rng(4)
        mag = 10.0 ** rng.uniform(-6, 3, size=(4, H, W))
        sgn = rng.choice([-1.0, 1.0], size=(4, H, W))
        gc, gd = (mag[:3] * sgn[:3]).astype(np.float32), (mag[3:] * sgn[3:]).astype(np.float32)
    return gc, gd


# CPU scenes of the soundness check: (name, builder -> (g, cm, W, H, bg, degree))
def _cpu_scenes():
    def fb0():
        g, cm = scene(20000, 2, (320, 240))
        return g, cm, 320, 240, np.array([0.1, 0.2, 0.3], np.float32), 0

    def sh3():
        g, cm = scene(30000, 5, (333, 211), degree=3)
        return g, cm, 333, 211, np.array([0.1, 0.2, 0.3], np.float32), 3

    def crowded():
        g, cm = scene(9000, 31, (160, 120))
        return crowd(g, cm, 0.02), cm, 160, 120, np.array([0.3, 0.6, 0.9], np.float32), 0

    def deep():
        g, cm = scene(40000, 31, (160, 120))
        return crowd(g, cm, 0.02, opacity=0.02), cm, 160, 120, np.zeros(3, np.float32), 0

    return {"fb_320x240": fb0, "sh3_333x211": sh3, "crowded_160x120": crowded, "deep_160x120": deep}


CPU_SCENES = _cpu_scenes()


def flagged(value, ref_value, bound):
    """Rows (Gaussians) where |value - ref| > bound in some component (NaN counts as a violation)."""
    ok = np.abs(value - ref_value) <= bound
    return np.flatnonzero(~ok.all(1))


def describe(name, labels, value, ref, ref_value, bound, rows, k=6):
    out = []
    for g in rows[:k]:
        ratio = np.abs(value[g] - ref_value[g]) / np.maximum(bound[g], 1e-300)
        i = int(np.nan_to_num(ratio, nan=np.inf).argmax())
        out.append(f"Gaussian {g} {labels[i]}: value {value[g, i]:.9g} ref {ref_value[g, i]:.9g} err {abs(value[g, i] - ref_value[g, i]):.3g} "
                   f"bound {bound[g, i]:.3g} S_g {ref.S_g[g]} pairs {ref.n_pairs[g]} deepest {ref.deepest[g]} ambiguous {ref.n_amb[g]}")
    return f"{name}: {len(rows)} Gaussians outside the bound:\n  " + "\n  ".join(out)


def ratio_stats(value, ref_value, bound, rows):
    r = np.abs(value[rows] - ref_value[rows]) / np.maximum(bound[rows], 1e-300)
    r = r[bound[rows] > 0]
    return (float(r.max()), float(np.median(r))) if r.size else (0.0, 0.0)


def footprint(splats, point_list, ranges, n_contrib, g, W):
    """Pixels (x, y) at which Gaussian g is an active contributor (float64 decisions), per the saved state."""
    H = n_contrib.shape[0]
    pos = np.flatnonzero(point_list == g)
    tiles = np.searchsorted(ranges[:, 1], pos, side="right")
    tiles_x = (W + 15) // 16
    s = splats[g].astype(np.float64)
    out = []
    for p, t in zip(pos, tiles):
        k1 = int(p - ranges[t, 0]) + 1
        x0, y0 = (t % tiles_x) * 16, (t // tiles_x) * 16
        ys, xs = np.mgrid[y0:min(y0 + 16, H), x0:min(x0 + 16, W)]
        dx, dy = s[0] - xs, s[1] - ys
        power = -0.5 * (s[2] * dx * dx + s[4] * dy * dy) - s[3] * dx * dy
        alpha = np.minimum(np.float64(np.float32(0.99)), s[5] * np.exp(power))
        act = (power <= 0) & (alpha >= np.float64(np.float32(1 / 255))) & (k1 <= n_contrib[ys, xs])
        out += list(zip(xs[act].tolist(), ys[act].tolist()))
    return out


def pixel_weight(splats, point_list, ranges, n_contrib, g, x, y, W):
    """w = alpha T of Gaussian g at pixel (x, y), replayed front to back in float64."""
    t = (y // 16) * ((W + 15) // 16) + x // 16
    T = 1.0
    for k in range(int(ranges[t, 0]), int(ranges[t, 0]) + int(n_contrib[y, x])):
        s = splats[point_list[k]].astype(np.float64)
        dx, dy = s[0] - x, s[1] - y
        power = -0.5 * (s[2] * dx * dx + s[4] * dy * dy) - s[3] * dx * dy
        alpha = min(float(np.float32(0.99)), s[5] * np.exp(power))
        if power > 0 or alpha < float(np.float32(1 / 255)):
            continue
        if point_list[k] == g:
            return alpha * T
        T *= 1.0 - alpha
    return 0.0


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the bound holds on an independent float32 implementation, and planted errors are caught
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cpu_states():
    out = {}
    for name, build in CPU_SCENES.items():
        g, cm, W, H, bg, deg = build()
        st = RO.State(g, cm, H, W, bg, sh_degree=deg)
        gc, gd = _dpix(7, H, W)
        ref = RO.moment_reference(st.splats, st.point_list, st.ranges, st.n_contrib, W, H, bg, gc, gd)
        out[name] = (st, gc, gd, ref)
    yield out
    for st, *_ in out.values():
        st.free()


@pytest.mark.parametrize("name", list(CPU_SCENES))
def test_bound_holds_on_float32_restatement(cpu_states, name):
    st, gc, gd, ref = cpu_states[name]
    acc = st.backward_acc(gc, gd)
    rows = flagged(acc, ref.grad, ref.grad_bound)
    assert len(rows) == 0, describe(name, GRD, acc, ref, ref.grad, ref.grad_bound, rows)
    vis = np.flatnonzero(ref.n_pairs > 0)
    worst, med = ratio_stats(acc, ref.grad, ref.grad_bound, vis)
    print(f"\n{name}: {len(vis)} Gaussians, {ref.pairs} pairs, {ref.ambiguous} ambiguous, deepest list {ref.max_contrib}: "
          f"|err|/B worst {worst:.3g} median {med:.3g}")
    assert worst >= 1e-3, "the bound is too loose to catch anything"
    # Gaussians without a pair have exactly zero gradient on both sides
    assert np.all(acc[ref.n_pairs + ref.n_amb == 0] == 0)
    if name.startswith("deep"):
        assert ref.max_contrib > 512 and int((st.ranges[:, 1] - st.ranges[:, 0]).max()) > 16384


def _pick_small(ref, lo, hi):
    cand = np.flatnonzero((ref.n_pairs >= lo) & (ref.n_pairs <= hi) & (ref.n_amb == 0))
    return int(cand[np.lexsort((cand, ref.deepest[cand], ref.n_pairs[cand]))][0])


def test_planted_errors_are_caught(cpu_states):
    st, gc, gd, ref = cpu_states["fb_320x240"]
    W, H = st.W, st.H
    pl, rg, nc = st.point_list.astype(np.int64), st.ranges.astype(np.int64), st.n_contrib.astype(np.int64)

    # 1. one pixel's dL/dpix zeroed on the restatement's side only
    g = _pick_small(ref, 1, 4)
    fp = footprint(st.splats, pl, rg, nc, g, W)
    assert fp, g
    x, y = fp[0]
    gc2, gd2 = gc.copy(), gd.copy()
    gc2[:, y, x] = 0.0
    gd2[:, y, x] = 0.0
    rows = flagged(st.backward_acc(gc2, gd2), ref.grad, ref.grad_bound)
    assert g in rows, ("zeroed dL/dpix not caught", g, x, y)
    tile = (y // 16) * ((W + 15) // 16) + x // 16
    assert set(rows.tolist()) <= set(pl[rg[tile, 0]:rg[tile, 1]].tolist())

    # 2. one pixel's T scaled by 1 + 1e-4, at the (Gaussian, pixel) where that change of w dL/dpix is largest against the
    # Gaussian's colour bound
    best = (0.0, None)
    for g in np.flatnonzero((ref.n_pairs >= 1) & (ref.n_pairs <= 8) & (ref.n_amb == 0)):
        for x, y in footprint(st.splats, pl, rg, nc, g, W):
            w = pixel_weight(st.splats, pl, rg, nc, g, x, y, W)
            r = (1e-4 * w * np.abs(gc[:, y, x]) / np.maximum(ref.grad_bound[g, :3], 1e-300)).max()
            best = max(best, (r, (int(g), x, y)))
    assert best[0] > 2.0, ("no pixel can show a 1e-4 change of T", best)
    g, x, y = best[1]
    keep = float(st.final_T[y, x])
    st.final_T[y, x] = np.float32(keep * (1.0 + 1e-4))
    try:
        rows = flagged(st.backward_acc(gc, gd), ref.grad, ref.grad_bound)
    finally:
        st.final_T[y, x] = keep
    assert g in rows, ("T scaled by 1 + 1e-4 not caught", g, x, y)

    # 3. one sub-tile's pixels shifted by one column for a Gaussian covering 50..500 pixels
    g = _pick_small(ref, 50, 500)
    fp = footprint(st.splats, pl, rg, nc, g, W)
    subs = {}
    for x, y in fp:
        subs[(x // 8 * 8, y // 4 * 4)] = subs.get((x // 8 * 8, y // 4 * 4), 0) + 1
    x0, y0 = max(subs, key=lambda k: (subs[k], k))
    rows = flagged(st.backward_acc(gc, gd, shift=(g, x0, y0)), ref.grad, ref.grad_bound)
    assert list(rows) == [g], ("column shift not caught", g, x0, y0, rows[:8])

    # and the unperturbed restatement is still inside
    assert len(flagged(st.backward_acc(gc, gd), ref.grad, ref.grad_bound)) == 0


# ---------------------------------------------------------------------------------------------------------------------
# GPU: every Gaussian's moments against the float64 replay of the GPU's own saved state
# ---------------------------------------------------------------------------------------------------------------------
def _gpu_case(name):
    """(g, cm, W, H, bg, degree, dL/dpix colour, dL/dpix depth) of a GPU case."""
    if name.startswith("fb_"):
        P, W, H, deg, seed = {"fb_20000": (20000, 320, 240, 0, 2), "fb_100000": (100000, 640, 480, 0, 3),
                              "fb_30000_sh3": (30000, 333, 211, 3, 5)}[name]
        g, cm = scene(P, seed, (W, H), degree=deg)
        return (g, cm, W, H, np.array([0.1, 0.2, 0.3], np.float32), deg) + _dpix(seed + 5, H, W)
    if name.startswith("edge_"):
        W, H = {"edge_333x211": (333, 211), "edge_17x33": (17, 33)}[name]
        g, cm = scene(15000, 40, (W, H), degree=3)
        return (g, cm, W, H, np.array([0.7, 0.1, 0.4], np.float32), 2) + _dpix(77, H, W)
    if name == "deep":
        g, cm = scene(40000, 31, (160, 120))
        return (crowd(g, cm, 0.02, opacity=0.02), cm, 160, 120, np.array([0.2, 0.1, 0.4], np.float32), 0) + _dpix(9, 120, 160)
    if name == "far_and_needles":
        g, cm = scene(3000, 17, (200, 152))
        return (far_and_needles(g, cm), cm, 200, 152, np.array([0.3, 0.6, 0.9], np.float32), 0) + _dpix(3, 152, 200)
    if name.startswith("dpix_"):
        g, cm = scene(20000, 2, (320, 240))
        return (g, cm, 320, 240, np.array([0.1, 0.2, 0.3], np.float32), 0) + _dpix_structured(name[5:], 240, 320)
    raise KeyError(name)


class GpuRun:
    """One forward on the GPU, and backwards with the moment tap set."""

    def __init__(self, cuda, g, cm, W, H, bg, degree, shard=None):
        import torch

        from gs_icp_slam_b200 import rasterizer as R

        self.torch, self.R, self.cuda, self.W, self.H, self.degree = torch, R, cuda, W, H, degree
        self.t = {k: torch.from_numpy(v).to(cuda) for k, v in g.items()}
        self.c = {k: (torch.from_numpy(v).to(cuda) if isinstance(v, np.ndarray) else v) for k, v in cm.items()}
        self.bg = torch.from_numpy(bg).to(cuda)
        e = torch.Tensor([])
        if shard is not None:
            R.set_tile_shard(*shard)
        try:
            t, c = self.t, self.c
            (self.n, self.depth, self.color, self.radii, self.is_used, self.geom, self.binning, self.img) = R.rasterize_gaussians(
                self.bg, t["means3D"], e, t["opacities"], t["scales"], t["rotations"], 1.0, e, c["viewmatrix"],
                c["projmatrix"], c["tanfovx"], c["tanfovy"], H, W, t["shs"], degree, c["campos"], False, False)
        finally:
            R.set_tile_shard(1, 0)
        self.shard = shard

    def backward(self, gc, gd):
        """(moment tap [P][12], the eight gradients) of one backward on the saved state."""
        torch, R, t, c = self.torch, self.R, self.t, self.c
        from gs_icp_slam_b200 import _lib

        P = t["means3D"].shape[0]
        tap = torch.full((P, 12), float("nan"), device=self.cuda)
        e = torch.Tensor([])
        if self.shard is not None:
            R.set_tile_shard(*self.shard)
        _lib.lib.gsicp_test_set_moment_tap(tap.data_ptr())
        try:
            grads = R.rasterize_gaussians_backward(self.bg, t["means3D"], self.radii, e, t["scales"], t["rotations"], 1.0, e,
                                                   c["viewmatrix"], c["projmatrix"], c["tanfovx"], c["tanfovy"],
                                                   torch.from_numpy(gd).to(self.cuda), torch.from_numpy(gc).to(self.cuda),
                                                   t["shs"], self.degree, c["campos"], self.geom, self.n, self.binning,
                                                   self.img, False)
            torch.cuda.synchronize()
        finally:
            _lib.lib.gsicp_test_set_moment_tap(None)
            R.set_tile_shard(1, 0)
        return tap.cpu().numpy().astype(np.float64), [x.cpu().numpy() for x in grads]

    def state(self):
        """(splats [P][12], point_list, ranges, n_contrib [H, W], final_T [H, W]) of the saved forward state."""
        torch, R = self.torch, self.R
        from gs_icp_slam_b200 import _lib

        P, W, H = self.t["means3D"].shape[0], self.W, self.H
        sp = torch.zeros((P, 12), dtype=torch.float32, device=self.cuda)
        ft = torch.zeros((H, W), dtype=torch.float32, device=self.cuda)
        nc = torch.zeros((H, W), dtype=torch.int32, device=self.cuda)
        a = _lib.RasterArgs()
        a.width, a.height = W, H
        _lib.check(_lib.lib.gsicp_test_raster_state(C.byref(a), P, int(self.n), self.geom.data_ptr(), self.img.data_ptr(),
                                                    sp.data_ptr(), ft.data_ptr(), nc.data_ptr(),
                                                    torch.cuda.current_stream(self.cuda).cuda_stream), "gsicp_test_raster_state")
        pl, rg = R.export_binning(self.n, H, W, self.binning, self.img)
        torch.cuda.synchronize()
        return (sp.cpu().numpy(), pl.cpu().numpy(), rg.cpu().numpy(), nc.cpu().numpy().view(np.uint32), ft.cpu().numpy())


def check_tap(name, tap, ref, vis, extra=None, finite_only=False):
    """|tap - ref| <= B for every visible Gaussian and moment; returns (worst, median) of |err| / B."""
    bound = ref.mom_bound if extra is None else ref.mom_bound + extra
    ref_m = ref.mom
    if finite_only:
        keep = np.isfinite(ref_m).all(1) & np.isfinite(bound).all(1)
        vis = vis & keep
    rows = np.flatnonzero(vis)
    bad = rows[flagged(tap[rows], ref_m[rows], bound[rows])]
    assert len(bad) == 0, describe(name, MOM, tap, ref, ref_m, bound, bad)
    return ratio_stats(tap, ref_m, bound, rows)


def check_gradients(name, tap, grads, ref, vis):
    """dL_dcolors / dL_dopacity are tap columns 9..11 / 0 bit for bit; dL_dmeans2D is within the propagated bound."""
    m2, col, opa = grads[0], grads[1], grads[2]
    rows = np.flatnonzero(vis)
    tap32 = tap.astype(np.float32)
    assert np.array_equal(col[rows], tap32[rows, 9:12]), f"{name}: dL_dcolors differ from the moments"
    assert np.array_equal(opa[rows, 0], tap32[rows, 0]), f"{name}: dL_dopacity differs from the moments"
    m2v = np.zeros((len(m2), 12))
    m2v[:, 4:6] = m2[:, :2]
    bnd = ref.grad_bound.copy()
    keep = np.isfinite(ref.grad[:, 4:6]).all(1) & np.isfinite(bnd[:, 4:6]).all(1)
    rows = np.flatnonzero(vis & keep)
    sub = np.zeros_like(bnd)
    sub[:, 4:6] = bnd[:, 4:6]
    refg = np.zeros_like(ref.grad)
    refg[:, 4:6] = ref.grad[:, 4:6]
    bad = rows[flagged(m2v[rows], refg[rows], sub[rows])]
    assert len(bad) == 0, describe(name + " dL_dmeans2D", GRD, m2v, ref, refg, sub, bad)
    # invisible Gaussians: every gradient row is exactly zero
    inv = ~vis
    for x in grads:
        assert not np.any(x.reshape(len(vis), -1)[inv]), f"{name}: gradient of an invisible Gaussian"


def _reference(run, gc, gd, bg):
    sp, pl, rg, nc, ft = run.state()
    ref = RO.moment_reference(sp, pl, rg, nc, run.W, run.H, bg, gc, gd)
    vis = run.radii.cpu().numpy() > 0
    assert np.all(ref.n_pairs[~vis] == 0)  # only visible Gaussians are in the instance list
    return ref, vis, (sp, pl, rg, nc, ft)


GPU_CASES = ["fb_20000", "fb_100000", "fb_30000_sh3", "edge_333x211", "edge_17x33", "deep", "far_and_needles",
             "dpix_impulses", "dpix_colour_only", "dpix_depth_only", "dpix_dynamic_range"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", GPU_CASES)
def test_moments_per_gaussian(cuda, name):
    g, cm, W, H, bg, deg, gc, gd = _gpu_case(name)
    run = GpuRun(cuda, g, cm, W, H, bg, deg)
    tap, grads = run.backward(gc, gd)
    ref, vis, (sp, pl, rg, nc, ft) = _reference(run, gc, gd, bg)
    finite = name == "far_and_needles"
    worst, med = check_tap(name, tap, ref, vis, finite_only=finite)
    check_gradients(name, tap, grads, ref, vis)
    print(f"\n[bwd-bound] {name}: visible {int(vis.sum())}, pairs {ref.pairs}, ambiguous {ref.ambiguous}, deepest "
          f"{ref.max_contrib}: |err|/B worst {worst:.3g} median {med:.3g}")
    if name == "deep":
        assert int(nc.max()) > 512 and int((rg[:, 1] - rg[:, 0]).max()) > 16384, "scene does not reach the intended depth"
        assert int((nc > 256).sum()) > 0
    if name == "far_and_needles":
        far = np.flatnonzero(ref.n_pairs[:6] > 0)
        assert len(far) >= 3, "no far-centred Gaussian reaches the frame"
        assert np.abs(sp[far, :2] - [W / 2, H / 2]).max() > 300


@pytest.mark.gpu
@pytest.mark.parametrize("switch", ["variant1", "nocull"])
@pytest.mark.parametrize("name", ["fb_20000", "deep", "edge_17x33"])
def test_moments_every_backward_path(cuda, name, switch):
    from gs_icp_slam_b200 import _lib

    g, cm, W, H, bg, deg, gc, gd = _gpu_case(name)
    set_fn, on, off = {"variant1": (_lib.lib.gsicp_test_set_bwd_variant, 1, 0),
                       "nocull": (_lib.lib.gsicp_test_set_render_cull, 0, 1)}[switch]
    set_fn(on)
    try:
        run = GpuRun(cuda, g, cm, W, H, bg, deg)
        tap, grads = run.backward(gc, gd)
    finally:
        set_fn(off)
    ref, vis, _ = _reference(run, gc, gd, bg)
    worst, med = check_tap(f"{name}/{switch}", tap, ref, vis)
    check_gradients(f"{name}/{switch}", tap, grads, ref, vis)
    print(f"\n[bwd-bound] {name}/{switch}: ambiguous {ref.ambiguous}: |err|/B worst {worst:.3g} median {med:.3g}")


@pytest.mark.gpu
def test_moments_tile_shards_sum(cuda):
    """Three one-GPU tile shards: the sum of their taps against the reference of the unsharded state."""
    g, cm, W, H, bg, deg, gc, gd = _gpu_case("fb_20000")
    full = GpuRun(cuda, g, cm, W, H, bg, deg)
    ref, vis, _ = _reference(full, gc, gd, bg)
    taps = []
    for k in range(3):
        run = GpuRun(cuda, g, cm, W, H, bg, deg, shard=(3, k))
        tap, _ = run.backward(gc, gd)
        tap[~vis] = 0.0
        taps.append(tap.astype(np.float32))
    total = (taps[0] + taps[1] + taps[2]).astype(np.float64)
    extra = 2 * U * 3 * (np.abs(taps[0]) + np.abs(taps[1]) + np.abs(taps[2]))  # three more roundings
    worst, med = check_tap("shards", total, ref, vis, extra=extra)
    print(f"\n[bwd-bound] shards 3: |err|/B worst {worst:.3g} median {med:.3g}")


@pytest.mark.gpu
def test_second_backward_same_state(cuda):
    """The moments are consumed and re-zeroed: a second backward on the same saved state meets the same bound."""
    g, cm, W, H, bg, deg, gc, gd = _gpu_case("fb_20000")
    run = GpuRun(cuda, g, cm, W, H, bg, deg)
    tap1, _ = run.backward(gc, gd)
    tap2, grads2 = run.backward(gc, gd)
    ref, vis, _ = _reference(run, gc, gd, bg)
    check_tap("first backward", tap1, ref, vis)
    worst, med = check_tap("second backward", tap2, ref, vis)
    check_gradients("second backward", tap2, grads2, ref, vis)
    print(f"\n[bwd-bound] second backward: |err|/B worst {worst:.3g} median {med:.3g}")


@pytest.mark.gpu
def test_gpu_negative_control(cuda):
    """A reference fed a dL/dpix that differs from the GPU's at one pixel must flag a Gaussian active there."""
    g, cm, W, H, bg, deg, gc, gd = _gpu_case("fb_20000")
    run = GpuRun(cuda, g, cm, W, H, bg, deg)
    tap, _ = run.backward(gc, gd)
    ref, vis, (sp, pl, rg, nc, ft) = _reference(run, gc, gd, bg)
    gsel = _pick_small(ref, 1, 4)
    x, y = footprint(sp, pl.astype(np.int64), rg.astype(np.int64), nc.astype(np.int64), gsel, W)[0]
    gc2 = gc.copy()
    gc2[:, y, x] += 1.0
    ref2 = RO.moment_reference(sp, pl, rg, nc, W, H, bg, gc2, gd)
    rows = np.flatnonzero(vis)
    bad = rows[flagged(tap[rows], ref2.mom[rows], ref2.mom_bound[rows])]
    assert gsel in bad, (gsel, x, y, bad[:8])
