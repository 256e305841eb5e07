"""Per-Gaussian check of the rasterizer's parameter gradients: dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations.

gaussian_backward_kernel (raster_backward.cu) turns each visible Gaussian's render gradients into the five arrays the
optimiser steps on.  The array-wide checks of test_raster_gpu.py (max |a - b| <= 2e-4 max |b|) are set by the largest
Gaussian, so a small Gaussian's gradient can be wrong and pass.  Here every Gaussian and component is checked against
tests/param_grad_model.py: a float64 restatement of the kernel's chain, quirks included, with a running error bound
K u S (u = 2^-24, K = 64; derivation and the count of roundings in that module's docstring) plus a charge for Gaussians
whose float32 decisions (t / t_z clamp, SH colour clamp, denom^2 overflow) lie within rounding of their threshold.

On the CPU, without a GPU:
  - structure: with every quirk off the restatement is torch.func.vjp of camera_grad_model.project, per Gaussian;
  - soundness of K: oracle/raster_oracle.c's ro_backward_ex, an independent float32 restatement, lies within the bound
    for every Gaussian and component when the chain is fed the oracle's own float32 render gradients;
  - sensitivity: planted errors in the oracle's outputs are caught, and so is each quirk switched off in the reference
    (the 1e-7 of denom2inv, at most 1.2e-5 relative, only raises the worst |err|/B tenfold: see the control's docstring).
On the GPU, the chain is fed the kernel's own moment tap and splat records.
"""
import contextlib

import numpy as np
import pytest
import torch

from tests import camera_grad_model as CM
from tests import param_grad_model as PM
from tests.test_raster_bwd_bound import CPU_SCENES, GPU_CASES, _dpix, _gpu_case, far_and_needles, scene
from tests.test_raster_camera_grad import EXTRA_CASES, CamRun, _extra_case, _gradcheck_case, _model_inputs

OUT_LABELS = {"means3D": "dL_dmeans3D", "cov3D": "dL_dcov3D", "sh": "dL_dsh", "scales": "dL_dscales", "rots": "dL_drotations"}


# ---------------------------------------------------------------------------------------------------------------------
# scenes beyond CPU_SCENES / GPU_CASES: (g, cm, W, H, bg, degree, scale_modifier)
# ---------------------------------------------------------------------------------------------------------------------
def _quat_from_matrix(Rm):
    """(x, y, z, w) of a proper rotation matrix (Shepperd's method, float64)."""
    m = Rm
    tr = np.trace(m)
    if tr > 0:
        s = 2.0 * np.sqrt(1.0 + tr)
        return np.array([(m[2, 1] - m[1, 2]) / s, (m[0, 2] - m[2, 0]) / s, (m[1, 0] - m[0, 1]) / s, s / 4])
    i = int(np.argmax(np.diag(m)))
    j, k = (i + 1) % 3, (i + 2) % 3
    s = 2.0 * np.sqrt(1.0 + m[i, i] - m[j, j] - m[k, k])
    q = np.zeros(4)
    q[i], q[j], q[k], q[3] = s / 4, (m[j, i] + m[i, j]) / s, (m[k, i] + m[i, k]) / s, (m[k, j] - m[j, k]) / s
    return q


def wall_scene():
    """fb_20000 with 5 Gaussians whose two 1 km axes lie in the image plane, 3 m in front of the camera: at 320x240 their
    2D determinant is about 6e19 px^4, so denom^2 overflows float32 (threshold 1.8e19)."""
    g, cm = scene(20000, 2, (320, 240))
    view = cm["viewmatrix"].astype(np.float64)
    right, down, fwd = view[:3, 0], view[:3, 1], view[:3, 2]
    Rm = np.stack([right, down, fwd], 1)  # local x, y, z -> world right, down, forward
    q = _quat_from_matrix(Rm)
    cov = CM.cov3d(torch.tensor([[1.0, 1.0, 0.0]], dtype=torch.float64), torch.tensor(q[None]))[0].numpy()
    if fwd @ cov @ fwd > 1e-6:  # the other quaternion convention
        q = q * np.array([-1, -1, -1, 1])
    for k, (z, ox, oy) in enumerate([(3.0, 0.0, 0.0), (3.1, 0.3, -0.2), (3.2, -0.4, 0.1), (3.3, 0.2, 0.4), (3.4, -0.1, -0.3)]):
        g["means3D"][k] = cm["campos"] + z * fwd + ox * right + oy * down
        g["scales"][k] = [1000.0, 1000.0, 0.01]
        g["rotations"][k] = q
        g["opacities"][k] = 0.1
    return g, cm, 320, 240, np.array([0.1, 0.2, 0.3], np.float32), 0, 1.0


def tiny_scene():
    """fb_20000 with every Gaussian 1e-4 m wide: the 2D covariance is the 0.3 px^2 low-pass, denom < 0.1."""
    g, cm = scene(20000, 2, (320, 240))
    g["scales"][:] = 1e-4
    g["opacities"][:] = 0.9
    return g, cm, 320, 240, np.array([0.1, 0.2, 0.3], np.float32), 0, 1.0


def mod_scene():
    """scale_modifier 0.7, an SH table of degree 3 rendered at active degree 1; every 5th Gaussian's green is clamped at 0
    in most directions."""
    g, cm = scene(20000, 6, (320, 240), degree=3)
    g["shs"][::5, 0, 1] = -2.5
    return g, cm, 320, 240, np.array([0.1, 0.2, 0.3], np.float32), 1, PM.f32(0.7)


def needles_scene():
    g, cm = scene(3000, 17, (200, 152))
    return far_and_needles(g, cm), cm, 200, 152, np.array([0.3, 0.6, 0.9], np.float32), 0, 1.0


MORE_SCENES = {"wall": wall_scene, "tiny": tiny_scene, "mod0.7": mod_scene, "far_and_needles": needles_scene}


def _params(g, vis, degree, mod=1.0, cov=None, colors=None):
    d = lambda x: torch.as_tensor(np.asarray(x, np.float32)[vis], dtype=torch.float64)
    p = dict(means=d(g["means3D"]), degree=degree, scale_modifier=mod,
             sh=None if colors is not None else d(g["shs"]))
    if cov is not None:
        p["cov"] = d(cov)
    else:
        p.update(scales=d(g["scales"]), rots=d(g["rotations"]))
    return p


# ---------------------------------------------------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------------------------------------------------
def flagged(got, val, bnd):
    """Rows (Gaussians) where some component of some output lies outside the bound (NaN counts as outside)."""
    bad = np.zeros(len(got["means3D"]), bool)
    for k, v in val.items():
        if v is None:
            continue
        ok = np.abs(got[k].reshape(len(v), -1) - v.reshape(len(v), -1)) <= bnd[k].reshape(len(v), -1)
        bad |= ~ok.all(1)
    return np.flatnonzero(bad)


def ratios(got, val, bnd):
    r = []
    for k, v in val.items():
        if v is None:
            continue
        b = bnd[k].reshape(-1)
        e = np.abs(got[k].reshape(-1) - v.reshape(-1))
        keep = b > PM.FLOOR * 1.0001
        r.append(e[keep] / b[keep])
    r = np.concatenate(r)
    return (float(r.max()), float(np.median(r))) if r.size else (0.0, 0.0)


def describe(name, got, val, bnd, rows, k=6):
    out = []
    for g in rows[:k]:
        worst = (-1.0, None)
        for key, v in val.items():
            if v is None:
                continue
            e = np.abs(got[key][g].reshape(-1) - v[g].reshape(-1))
            r = np.nan_to_num(e / bnd[key][g].reshape(-1), nan=np.inf)
            i = int(r.argmax())
            worst = max(worst, (float(r[i]), (key, i, float(got[key][g].reshape(-1)[i]), float(v[g].reshape(-1)[i]),
                                              float(bnd[key][g].reshape(-1)[i]))), key=lambda t: t[0])
        key, i, a, b, B = worst[1]
        out.append(f"Gaussian {g} {OUT_LABELS[key]}[{i}]: got {a:.9g} ref {b:.9g} err {abs(a - b):.3g} bound {B:.3g}")
    return f"{name}: {len(rows)} Gaussians outside the bound:\n  " + "\n  ".join(out)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: structure (quirks off = autograd of the forward)
# ---------------------------------------------------------------------------------------------------------------------
def _structure(mu, V, Pm, cp, kw, rows, mod=1.0, seed=0):
    """chain(quirks=False) vs torch.func.vjp of camera_grad_model.project on the Gaussians `rows`, random cotangents."""
    mu = mu[rows]
    kw = {k: (v[rows] if k in ("cov", "scales", "rots", "sh", "colors") else v) for k, v in kw.items()}
    n = mu.shape[0]
    gen = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    g2, dc, czx, cyz, dep, rgb = r(n, 2), r(n, 3), r(n), r(n), r(n), r(n, 3)
    rg = dict(g2=(PM.RE(g2[:, 0]), PM.RE(g2[:, 1])), dc=tuple(PM.RE(dc[:, i]) for i in range(3)), covzx=PM.RE(czx),
              covyz=PM.RE(cyz), depth=PM.RE(dep), rgb=tuple(PM.RE(rgb[:, i]) for i in range(3)))
    cot = (g2, torch.stack([dc[:, 0], 2 * dc[:, 1], dc[:, 2]], 1), czx, cyz, dep, rgb)
    keys = ("ndc", "conic", "cov_zx", "cov_yz", "depth", "rgb")
    fixed = {k: v for k, v in kw.items() if k not in ("cov", "scales", "rots", "sh")}
    iu = [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]

    def f(mu_, cov_, sc_, rot_, sh_):
        extra = dict(cov=cov_) if cov_ is not None else dict(scales=sc_, rots=rot_, scale_modifier=mod)
        o = CM.project(mu_, V, Pm, cp, sh=sh_, **fixed, **extra)
        return tuple(o[k] for k in keys)

    sh = kw.get("sh")
    if "cov" in kw:
        _, vjp = torch.func.vjp(lambda m, c, s: f(m, c, None, None, s), mu, kw["cov"], sh if sh is not None else mu)
        ref = dict(zip(("means3D", "cov3D", "sh"), vjp(cot)))
    else:
        _, vjp = torch.func.vjp(lambda m, a, b, s: f(m, None, a, b, s), mu, kw["scales"], kw["rots"], sh if sh is not None else mu)
        ref = dict(zip(("means3D", "scales", "rots", "sh"), vjp(cot)))
        c6 = CM.cov3d(kw["scales"], kw["rots"], mod)[:, iu[0], iu[1]]
        _, vjp_c = torch.func.vjp(lambda m, c, s: f(m, c, None, None, s), mu, c6, sh if sh is not None else mu)
        ref["cov3D"] = vjp_c(cot)[1]
    if sh is None:
        ref.pop("sh")
    tanx, tany = kw["tanfovx"], kw["tanfovy"]
    cam = dict(view=V.reshape(-1).tolist(), proj=Pm.reshape(-1).tolist(), campos=cp.tolist(), tanfovx=tanx, tanfovy=tany,
               focal=kw["focal"], W=kw["W"], H=kw["H"])
    params = dict(means=mu, degree=kw.get("degree", 0), scale_modifier=mod, sh=sh, cov=kw.get("cov"), scales=kw.get("scales"),
                  rots=kw.get("rots"))
    out, dec = PM.chain(params, cam, rg, quirks=False)
    worst = 0.0
    for k, v in ref.items():
        a, b = out[k].v.reshape(n, -1), v.reshape(n, -1)
        scale = b.abs().amax(1, keepdim=True)
        err = ((a - b).abs() / torch.clamp(scale, min=1e-300)).max().item()
        assert err <= 1e-10, f"{k}: chain(quirks=False) differs from autograd by {err:.3g} of the row maximum"
        worst = max(worst, err)
    return worst, dec


def _visible_rows(mu, V, n=1500):
    """Up to n Gaussians in front of the near plane (every n-th), as a bool mask."""
    t = torch.cat([mu, torch.ones_like(mu[:, :1])], 1) @ V[:, 2]
    idx = torch.nonzero(t > 0.2).reshape(-1)
    idx = idx[:: max(1, len(idx) // n)]
    m = torch.zeros(len(mu), dtype=torch.bool)
    m[idx] = True
    return m


STRUCT_CASES = [f"cpu:{k}" for k in CPU_SCENES] + ["gradcheck", "gradcheck_clamped", "cov3D_precomp", "colors_precomp", "mod0.7"]


@pytest.mark.parametrize("case", STRUCT_CASES)
def test_quirks_off_is_the_forward_vjp(case):
    mod = 1.0
    if case.startswith("cpu:"):
        g, cm, W, H, bg, deg = CPU_SCENES[case[4:]]()
        mu, V, Pm, cp, kw = _model_inputs(g, cm, W, H, deg)
        rows = _visible_rows(mu, V)
    elif case.startswith("gradcheck"):
        mu, V, Pm, cp, kw = _gradcheck_case(case.endswith("clamped"))
        rows = torch.ones(len(mu), dtype=torch.bool)
    elif case == "mod0.7":
        g, cm, W, H, bg, deg, mod = mod_scene()
        mu, V, Pm, cp, kw = _model_inputs(g, cm, W, H, deg)
        rows = _visible_rows(mu, V)
    else:
        g, cm, W, H, bg, deg, gc, gd, cov, col = _extra_case(case)
        mu, V, Pm, cp, kw = _model_inputs(g, cm, W, H, deg, cov_pre=cov, colors=col)
        rows = _visible_rows(mu, V)
    worst, dec = _structure(mu, V, Pm, cp, kw, rows, mod=mod)
    n_cl = int(dec["clamp_x"][0].sum() + dec["clamp_y"][0].sum())
    if case == "gradcheck_clamped":
        assert n_cl >= 6
    print(f"\n[paramgrad] {case}: chain(quirks=False) = autograd of the forward on {int(rows.sum())} Gaussians "
          f"({n_cl} clamped axes), worst {worst:.3g} of the row maximum")


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the bound holds on the float32 oracle, and errors are caught
# ---------------------------------------------------------------------------------------------------------------------
SOUND_SCENES = list(CPU_SCENES) + list(MORE_SCENES)


def _scene(name):
    if name in CPU_SCENES:
        return CPU_SCENES[name]() + (1.0,)
    return MORE_SCENES[name]()


@pytest.fixture(scope="module")
def oracle_runs():
    """name -> (params, camera, render gradients, oracle outputs of the visible Gaussians, their ids)."""
    from oracle import raster_oracle as RO

    out = {}
    for name in SOUND_SCENES:
        g, cm, W, H, bg, deg, mod = _scene(name)
        st = RO.State(g, cm, H, W, bg, sh_degree=deg, scale_modifier=mod)
        try:
            gc, gd = _dpix(7, H, W)
            acc, outs = st.backward_acc(gc, gd, with_outputs=True)
            vis = st.radii > 0
        finally:
            st.free()
        got = dict(means3D=outs[3][vis], cov3D=outs[4][vis], sh=outs[5][vis], scales=outs[6][vis], rots=outs[7][vis])
        out[name] = (_params(g, vis, deg, mod), PM.camera(cm, W, H), PM.render_grads_from_acc(acc[vis]), got,
                     np.flatnonzero(vis))
    return out


@pytest.mark.parametrize("name", SOUND_SCENES)
def test_bound_holds_on_float32_oracle(oracle_runs, name):
    params, cam, rg, got, ids = oracle_runs[name]
    val, bnd, amb, dec = PM.reference(params, cam, rg)
    rows = flagged(got, val, bnd)
    assert len(rows) == 0, describe(name, got, val, bnd, rows)
    worst, med = ratios(got, val, bnd)
    n_ov = int(dec["overflow"][0].sum())
    print(f"\n[paramgrad] {name}: K = {PM.K_BOUND}, {len(ids)} Gaussians, |err|/B worst {worst:.3g} median {med:.3g}, "
          f"ambiguous {int(amb.sum())}, denom^2 overflows {n_ov}")
    assert worst >= 1e-3, "the bound is too loose to catch anything"
    if name == "wall":
        assert n_ov >= 1, "no visible Gaussian takes the overflow branch"


# the scene on which each departure of the kernel's chain from the true derivative must show
DEPARTURES = {"eps": "tiny", "overflow": "wall", "dropped_yz": "fb_320x240", "clamp_tz": "far_and_needles",
              "scale_mod": "mod0.7"}


@pytest.mark.parametrize("quirk", list(DEPARTURES))
def test_each_quirk_is_modelled_and_visible(oracle_runs, quirk):
    """The oracle copies the reference's chain: a reference without one quirk, or without all of them, flags Gaussians.

    The exception is 'eps' (1 / (denom^2 + 1e-7)): it changes dL_da, dL_db, dL_dc by at most 1e-7 / 0.09^2 = 1.2e-5
    relative (denom >= 0.09 by the 0.3 low-pass), while a tiny Gaussian's dL_da carries the cancellation of
    (denom - ca cc) dc_z, so its shadow is several times |dL_da| and K u S exceeds the departure.  There the check is
    that the reference without the quirk lies at least 10x further from the oracle, in units of the bound."""
    name = DEPARTURES[quirk]
    params, cam, rg, got, ids = oracle_runs[name]
    with_all = ratios(got, *PM.reference(params, cam, rg)[:2])[0]
    v1, b1 = PM.reference(params, cam, rg, quirks=set(PM.QUIRKS) - {quirk})[:2]
    v0, b0 = PM.reference(params, cam, rg, quirks=False)[:2]
    one, none = flagged(got, v1, b1), flagged(got, v0, b0)
    w1, w0 = ratios(got, v1, b1)[0], ratios(got, v0, b0)[0]
    print(f"\n[paramgrad] {name}: without '{quirk}' {len(one)} of {len(ids)} Gaussians flagged (|err|/B worst {w1:.3g}), "
          f"without any quirk {len(none)} ({w0:.3g}); with every quirk {with_all:.3g}")
    if quirk == "eps":
        assert w1 >= 10 * with_all and w0 >= 10 * with_all
    else:
        assert len(one) >= 1 and len(none) >= 1


def _median_pick(mag, cand):
    """The Gaussian of median magnitude among the candidates."""
    cand = cand[np.argsort(mag[cand], kind="stable")]
    return int(cand[len(cand) // 2])


def test_planted_errors_are_caught(oracle_runs):
    # two SH coefficient gradients of one Gaussian swapped (degree 3): bands 1 and 3 are -C1 y dRGB and -C1 x dRGB
    params, cam, rg, got, ids = oracle_runs["sh3_333x211"]
    val, bnd, amb, dec = PM.reference(params, cam, rg)
    sh = got["sh"]
    diff = np.abs(sh[:, 1] - sh[:, 3]).max(1)
    g = _median_pick(diff, np.flatnonzero((diff > 0) & ~amb))
    bad = dict(got, sh=sh.copy())
    bad["sh"][g, [1, 3]] = sh[g, [3, 1]]
    assert list(flagged(bad, val, bnd)) == [g], "swapped SH bands not caught"

    # one clamped channel's mask ignored: the coefficient-0 gradient of that channel is C0 dL/dRGB instead of 0
    params, cam, rg, got, ids = oracle_runs["mod0.7"]
    val, bnd, amb, dec = PM.reference(params, cam, rg)
    sh = got["sh"]
    taken, amb_c = dec["sh_clamp"]
    rgb = np.stack([r.v.numpy() for r in rg["rgb"]], 1)
    cand = np.argwhere(taken & ~amb_c & (rgb != 0))
    assert len(cand), "no clamped colour channel with a gradient"
    g, c = (int(x) for x in cand[len(cand) // 2])
    assert np.all(sh[g, :, c] == 0)
    bad = dict(got, sh=sh.copy())
    bad["sh"][g, 0, c] = np.float32(CM.SH_C0) * np.float32(rgb[g, c])
    assert list(flagged(bad, val, bnd)) == [g], "ignored clamp mask not caught"

    # the sign of one Gaussian's dq.w flipped
    params, cam, rg, got, ids = oracle_runs["fb_320x240"]
    val, bnd, amb, dec = PM.reference(params, cam, rg)
    w = np.abs(got["rots"][:, 3])
    g = _median_pick(w, np.flatnonzero((w > 0) & ~amb))
    bad = dict(got, rots=got["rots"].copy())
    bad["rots"][g, 3] *= -1
    assert list(flagged(bad, val, bnd)) == [g], "flipped dq.w not caught"


# ---------------------------------------------------------------------------------------------------------------------
# GPU: every visible Gaussian's five gradient arrays against the chain fed the kernel's own moments
# ---------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _scale_modifier(mod):
    """CamRun passes scale_modifier 1.0: substitute `mod` in the rasterizer calls it makes."""
    from gs_icp_slam_b200 import rasterizer as R

    names = ("rasterize_gaussians", "rasterize_gaussians_backward", "rasterize_gaussians_backward_camera")
    orig = {n: getattr(R, n) for n in names}

    def sub(f):
        return lambda *a: f(*a[:6], mod, *a[7:])

    try:
        for n in names:
            setattr(R, n, sub(orig[n]))
        yield
    finally:
        for n in names:
            setattr(R, n, orig[n])


class ModRun(CamRun):
    """CamRun at a scale modifier other than 1."""

    def __init__(self, cuda, mod, *a, **k):
        self.mod = mod
        with _scale_modifier(mod):
            super().__init__(cuda, *a, **k)

    def backward_camera(self, *a, **k):
        with _scale_modifier(self.mod):
            return super().backward_camera(*a, **k)


PARAM_CASES = GPU_CASES + EXTRA_CASES + ["mod0.7", "wall", "tiny", "fb_20000_deterministic"]


def _param_case(cuda, name):
    """(run, g, degree, scale_modifier, cov_pre, colors, dL/dpix colour, depth)."""
    cov, col, mod = None, None, 1.0
    if name in ("mod0.7", "wall", "tiny"):
        g, cm, W, H, bg, deg, mod = MORE_SCENES[name]()
        gc, gd = _dpix(7, H, W)
    elif name in EXTRA_CASES:
        g, cm, W, H, bg, deg, gc, gd, cov, col = _extra_case(name)
    else:
        g, cm, W, H, bg, deg, gc, gd = _gpu_case(name.replace("_deterministic", ""))
    if mod != 1.0:
        run = ModRun(cuda, mod, g, cm, W, H, bg, deg)
    else:
        run = CamRun(cuda, g, cm, W, H, bg, deg, cov_pre=cov, colors=col)
    return run, g, cm, deg, mod, cov, col, gc, gd


def _gpu_run(cuda, name):
    """(the five gradient arrays [P, ...], the visible rows of them in float64, the chain's inputs, vis, degree, cov)."""
    from tests.test_raster_deterministic import torch_deterministic

    run, g, cm, deg, mod, cov, col, gc, gd = _param_case(cuda, name)
    with torch_deterministic(name.endswith("_deterministic")):
        tap, grads, _ = run.backward_camera(gc, gd, camera=False)
    sp = run.state()[0]
    vis = run.radii.cpu().numpy() > 0
    P = len(vis)
    params = _params(g, vis, deg, mod, cov=cov, colors=col)
    rg = PM.render_grads(tap[vis], sp[vis], run.W, run.H)
    full = dict(means3D=grads[3].reshape(P, 3), cov3D=grads[4].reshape(P, 6), sh=grads[5].reshape(P, -1, 3) if col is None else None,
                scales=grads[6].reshape(P, 3), rots=grads[7].reshape(P, 4))
    got = {k: (None if v is None else v[vis].astype(np.float64)) for k, v in full.items()}
    return full, got, (params, PM.camera(cm, run.W, run.H), rg), vis, deg, cov


@pytest.mark.gpu
@pytest.mark.parametrize("name", PARAM_CASES)
def test_parameter_gradients_per_gaussian(cuda, name):
    full, got, inputs, vis, deg, cov = _gpu_run(cuda, name)
    val, bnd, amb, dec = PM.reference(*inputs)
    rows = flagged(got, val, bnd)
    assert len(rows) == 0, describe(name, got, val, bnd, rows)
    worst, med = ratios(got, val, bnd)
    # exact zeros the kernel writes by construction
    if full["sh"] is not None:
        assert not np.any(full["sh"][:, (deg + 1) ** 2:]), "a coefficient above the active degree has a gradient"
        taken, amb_c = dec["sh_clamp"]
        g_, c_ = np.nonzero(taken & ~amb_c)
        assert not np.any(got["sh"][g_, :, c_]), "a clamped colour channel has an SH gradient"
    if cov is not None:
        assert not np.any(full["scales"]) and not np.any(full["rots"]), "scale / rotation gradient under cov3D_precomp"
    n_ov = int(dec["overflow"][0].sum())
    if name == "wall":
        assert n_ov >= 1, "no visible Gaussian takes the overflow branch"
    if name == "mod0.7":
        assert int(dec["sh_clamp"][0].sum()) > 0
    print(f"\n[paramgrad] {name}: K = {PM.K_BOUND}, {int(vis.sum())} visible, |err|/B worst {worst:.3g} median {med:.3g}, "
          f"ambiguous {int(amb.sum())}, denom^2 overflows {n_ov}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tiny", "wall", "far_and_needles", "mod0.7"])
def test_gpu_negative_control(cuda, name):
    """The same tap against the true derivative (every quirk off): the kernel's chain is the reference's, so Gaussians
    must fall outside; on the tiny case (only 'eps' differs there) the worst |err|/B must grow at least tenfold."""
    full, got, inputs, vis, deg, cov = _gpu_run(cuda, name)
    val, bnd = PM.reference(*inputs, quirks=False)[:2]
    v1, b1 = PM.reference(*inputs)[:2]
    rows = flagged(got, val, bnd)
    w0, w1 = ratios(got, val, bnd)[0], ratios(got, v1, b1)[0]
    print(f"\n[paramgrad] {name}: true derivative flags {len(rows)} of {int(vis.sum())} Gaussians (|err|/B worst {w0:.3g}; "
          f"{w1:.3g} with every quirk)")
    if name == "tiny":
        assert w0 >= 10 * w1
    else:
        assert len(rows) >= 1
