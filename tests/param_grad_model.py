"""Float64 restatement of gaussian_backward_kernel (raster_backward.cu), the per-Gaussian parameter chain of the rasterizer
backward, with a running error bound.

The kernel turns the render gradients of a visible Gaussian (dL/dndc, dL/dconic, dL/dcov_zx, dL/dcov_yz, dL/ddepth,
dL/dRGB) into dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales and dL_drotations.  It copies the reference rasterizer's chain on
purpose, and that chain is not the derivative of the forward (tests/camera_grad_model.project).  `chain` restates the
kernel's expressions in the kernel's order; each departure from the true derivative is a switch (QUIRKS), and with all of
them off `chain` is the vector-Jacobian product of `project` (tests/test_raster_param_grad.py checks this against autograd):
    eps          denom2inv = 1 / (denom^2 + 1e-7) instead of 1 / denom^2
    overflow     denom * denom overflowing float32 makes denom2inv 0: dL_da, dL_db, dL_dc and dL_dcov3D are then 0
    dropped_yz   the cov_yz terms of dL_dT11 and dL_dT12 are dropped (a stray ';' in the reference)
    clamp_tz     a t_x (t_y) clamped at 1.3 tan_fov only zeroes dL/dt_x; the clamped value's dependence on t_z is ignored
    depth_mul    the depth path's view[3] * mul term (0 for a rigid view)
    scale_mod    dL_dscales is the derivative w.r.t. scale_modifier * scale (no modifier factor)
Two more departures sit in the render gradients the chain is fed (dL/dcov_yz lacks the conic_yy term, dL/dconic_xy enters
as 2 dc_y); render_grads forms them with the kernel's expressions, as camera_grad_model.render_grads does.  Quaternions
are not normalised on either side.

Error model.  Every quantity is an RE: a float64 value and a shadow S, vectorised over Gaussians.  A float32 input is exact
with S = |x|; + and - add shadows; a * b has S = min(S_a S_b, |a| S_b + S_a |b|); a / b has S = S_a / |b| + |a| S_b / b^2;
sqrt(a) has S = S_a / (2 sqrt a) + sqrt a.  S >= |value| throughout.  Without cancellation S is |value|; the first-order
forms take over where an operand has cancelled: the product of shadows alone would square the determinant's cancellation
in denom^2 (relative shadows of 1e9 on ordinary scenes) and leave no bound worth the name.  If every float32 step rounds
to within u = 2^-24 of its result, an expression whose operations lie n deep along any path from an input is within
n u S of the float64 value (to first order); the division rule carries the conditioning of the 2D covariance's
determinant through denom2inv without a hand-made kappa.  The bound is
    |float32 - ref| <= K u S + FLOOR,  K = 64.
Count of the longest path (dL_drotations; dL_dmeans3D is a few steps shorter): the render gradients from the moment tap, 5;
cov3 from scale and quaternion, 10; t, the clamp and J, 11; T = W J, 3; T^T V T, 6; +0.3 and denom, 3; denom^2 + eps and its
reciprocal, 3 (up to 4 more where denom2inv is subnormal: above det = 9e18 px^4 it is >= 2^-128 with an absolute error of
2^-150); dL_da, 4; dcov, 5; dL_dM, 3; the modifier product and dq, 6.  That is 59 <= K.  The float32 constants of the kernel
(0.3f, the SH constants, 1.3f) differ from the float64 ones used here by one rounding each, inside the same count.
FLOOR = K 2^-126 covers intermediates that fall below float32's normal range, where the relative guarantee does not hold.
Measured worst |err| / B per scene: 0.03, both on the float32 oracle and on an H100 (SXM, default power limit).

fp32 decisions.  Four branches depend on a float32 comparison that a float64 replay cannot know near its threshold: the
t_x / t_z (t_y / t_z) clamp against 1.3f tan_fov, each SH colour channel's clamp at 0, and float32 overflow of denom^2 + eps
(at 2^128 (1 - 2^-25)).  The depth quirk's view[3] * mul is an exact 0 for a rigid view, so no decision is taken there.
A decision whose operand lies within K u S of its threshold is ambiguous: `reference` evaluates the chain again with that
decision flipped for the ambiguous Gaussians and adds |branch A - branch B| to their bound, component by component.
"""
import numpy as np
import torch

from tests import camera_grad_model as CM

U24 = 2.0 ** -24
K_BOUND = 64
FLOOR = K_BOUND * 2.0 ** -126
OVERFLOW = 2.0 ** 128 * (1.0 - 2.0 ** -25)  # the smallest real that float32 round-to-nearest takes to +inf
QUIRKS = ("eps", "overflow", "dropped_yz", "clamp_tz", "depth_mul", "scale_mod")


def f32(x):
    return float(np.float32(x))


class RE:
    """A float64 value and its running-error shadow (both tensors, or broadcastable)."""
    __slots__ = ("v", "s")

    def __init__(self, v, s=None):
        self.v = torch.as_tensor(v, dtype=torch.float64)
        self.s = torch.abs(self.v) if s is None else s

    def __add__(self, o):
        o = _re(o)
        return RE(self.v + o.v, self.s + o.s)

    __radd__ = __add__

    def __sub__(self, o):
        o = _re(o)
        return RE(self.v - o.v, self.s + o.s)

    def __rsub__(self, o):
        return _re(o) - self

    def __mul__(self, o):
        o = _re(o)
        return RE(self.v * o.v, torch.minimum(self.s * o.s, torch.abs(self.v) * o.s + self.s * torch.abs(o.v)))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = _re(o)
        return RE(self.v / o.v, self.s / torch.abs(o.v) + torch.abs(self.v) * o.s / (o.v * o.v))

    def __rtruediv__(self, o):
        return _re(o) / self

    def __neg__(self):
        return RE(-self.v, self.s)


def _re(x):
    return x if isinstance(x, RE) else RE(x)


def sqrt(a):
    r = torch.sqrt(a.v)
    return RE(r, 0.5 * a.s / r + r)


def where(mask, a, b):
    a, b = _re(a), _re(b)
    return RE(torch.where(mask, a.v, b.v), torch.where(mask, a.s, b.s))


ZERO = RE(0.0)


def leaves(x):
    """The columns of a float tensor [P, k] as exact RE inputs."""
    x = torch.as_tensor(x, dtype=torch.float64)
    return [RE(x[:, i]) for i in range(x.shape[1])]


# column-major 3x3 (m[col][row]) like the kernel's M3
def m3_mul(a, b):
    return [[a[0][r] * b[c][0] + a[1][r] * b[c][1] + a[2][r] * b[c][2] for r in range(3)] for c in range(3)]


def m3_t(a):
    return [[a[r][c] for r in range(3)] for c in range(3)]


def quat_to_m3(x, y, z, w):
    return [[1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - w * z), 2.0 * (x * z + w * y)],
            [2.0 * (x * y + w * z), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - w * x)],
            [2.0 * (x * z - w * y), 2.0 * (y * z + w * x), 1.0 - 2.0 * (x * x + y * y)]]


def _near(x, thr, K=K_BOUND):
    return torch.abs(x.v - thr) <= K * U24 * x.s


# ---------------------------------------------------------------------------------------------------------------------
# render gradients
# ---------------------------------------------------------------------------------------------------------------------
def render_grads(tap, splats, W, H):
    """The render gradients gaussian_backward_kernel forms from the moment tap [P,12] and the splat records [P,12]
    (camera_grad_model.render_grads in RE): dict(g2 = (dL/dndc x, y), dc = (dL/dconic xx, dc_y, dL/dconic yy),
    covzx, covyz, depth, rgb = 3 channels before the clamp mask)."""
    m, s = leaves(tap), leaves(splats)
    cA, cB, cC, opac, czx, cyz = (s[k] for k in (2, 3, 4, 5, 6, 7))
    ux, uy, uxx, uxy, uyy = opac * m[1], opac * m[2], opac * m[3], opac * m[4], opac * m[5]
    v0, vx, vy = m[6], m[7], m[8]
    g2x = (-cA * ux - cB * uy - (czx * cA + cyz * cB) * v0) * (0.5 * W)
    g2y = (-cC * uy - cB * ux - (czx * cB + cyz * cC) * v0) * (0.5 * H)
    return dict(g2=(g2x, g2y), dc=(-0.5 * uxx - czx * vx, -0.5 * uxy - cyz * vx - czx * vy, -0.5 * uyy - cyz * vy),
                covzx=-cA * vx - cB * vy, covyz=-cB * vx, depth=v0, rgb=(m[9], m[10], m[11]))


def render_grads_from_acc(acc):
    """The render gradients the float32 oracle (raster_oracle.c, ro_backward_ex) reads: float32 of its double sums
    acc [P,12] = {colour r,g,b, depth, mean2D x,y, conic xx,xy,yy, cov_zx, cov_yz, opacity}, exact inputs."""
    a = leaves(np.asarray(acc, np.float32))
    return dict(g2=(a[4], a[5]), dc=(a[6], a[7], a[8]), covzx=a[9], covyz=a[10], depth=a[3], rgb=(a[0], a[1], a[2]))


# ---------------------------------------------------------------------------------------------------------------------
# the chain
# ---------------------------------------------------------------------------------------------------------------------
def camera(cm, W, H):
    """The chain's camera from a synthetic.camera_matrices dict: the float32 values the library works with."""
    tx, ty = f32(cm["tanfovx"]), f32(cm["tanfovy"])
    fx = f32(np.float32(W) / (np.float32(2.0) * np.float32(tx)))
    fy = f32(np.float32(H) / (np.float32(2.0) * np.float32(ty)))
    flat = lambda k: [float(v) for v in np.asarray(cm[k], np.float32).reshape(-1)]
    return dict(view=flat("viewmatrix"), proj=flat("projmatrix"), campos=flat("campos"), tanfovx=tx, tanfovy=ty,
                focal=(fx, fy), W=W, H=H)


def _sh_rgb(sh, D, x, y, z):
    """One channel's SH colour + 0.5 (the forward's clamp operand); sh: list of RE coefficients."""
    r = CM.SH_C0 * sh[0]
    if D > 0:
        r = r - CM.SH_C1 * y * sh[1] + CM.SH_C1 * z * sh[2] - CM.SH_C1 * x * sh[3]
        if D > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            C2 = CM.SH_C2
            r = (r + C2[0] * xy * sh[4] + C2[1] * yz * sh[5] + C2[2] * (2.0 * zz - xx - yy) * sh[6] + C2[3] * xz * sh[7]
                 + C2[4] * (xx - yy) * sh[8])
            if D > 2:
                C3 = CM.SH_C3
                r = (r + C3[0] * y * (3.0 * xx - yy) * sh[9] + C3[1] * xy * z * sh[10] + C3[2] * y * (4.0 * zz - xx - yy) * sh[11]
                     + C3[3] * z * (2.0 * zz - 3.0 * xx - 3.0 * yy) * sh[12] + C3[4] * x * (4.0 * zz - xx - yy) * sh[13]
                     + C3[5] * z * (xx - yy) * sh[14] + C3[6] * x * (xx - 3.0 * yy) * sh[15])
    return r + 0.5


def _sh_backward(sh, D, x, y, z, d):
    """sh_backward of one channel: (dL/dsh coefficients 0..(D+1)^2 - 1, dRGB/ddir (x, y, z)) for the masked dL/dRGB d."""
    C1, C2, C3 = CM.SH_C1, CM.SH_C2, CM.SH_C3
    dsh = [CM.SH_C0 * d]
    dx = dy = dz = ZERO
    if D > 0:
        dsh += [(-C1 * y) * d, (C1 * z) * d, (-C1 * x) * d]
        dx, dy, dz = -C1 * sh[3], -C1 * sh[1], C1 * sh[2]
        if D > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            dsh += [(C2[0] * xy) * d, (C2[1] * yz) * d, (C2[2] * (2.0 * zz - xx - yy)) * d, (C2[3] * xz) * d,
                    (C2[4] * (xx - yy)) * d]
            dx = dx + (C2[0] * y * sh[4] + C2[2] * 2.0 * -x * sh[6] + C2[3] * z * sh[7] + C2[4] * 2.0 * x * sh[8])
            dy = dy + (C2[0] * x * sh[4] + C2[1] * z * sh[5] + C2[2] * 2.0 * -y * sh[6] + C2[4] * 2.0 * -y * sh[8])
            dz = dz + (C2[1] * y * sh[5] + C2[2] * 2.0 * 2.0 * z * sh[6] + C2[3] * x * sh[7])
            if D > 2:
                dsh += [(C3[0] * y * (3.0 * xx - yy)) * d, (C3[1] * xy * z) * d, (C3[2] * y * (4.0 * zz - xx - yy)) * d,
                        (C3[3] * z * (2.0 * zz - 3.0 * xx - 3.0 * yy)) * d, (C3[4] * x * (4.0 * zz - xx - yy)) * d,
                        (C3[5] * z * (xx - yy)) * d, (C3[6] * x * (xx - 3.0 * yy)) * d]
                dx = dx + (C3[0] * sh[9] * 3.0 * 2.0 * xy + C3[1] * sh[10] * yz + C3[2] * sh[11] * -2.0 * xy
                           + C3[3] * sh[12] * -3.0 * 2.0 * xz + C3[4] * sh[13] * (-3.0 * xx + 4.0 * zz - yy)
                           + C3[5] * sh[14] * 2.0 * xz + C3[6] * sh[15] * 3.0 * (xx - yy))
                dy = dy + (C3[0] * sh[9] * 3.0 * (xx - yy) + C3[1] * sh[10] * xz + C3[2] * sh[11] * (-3.0 * yy + 4.0 * zz - xx)
                           + C3[3] * sh[12] * -3.0 * 2.0 * yz + C3[4] * sh[13] * -2.0 * xy + C3[5] * sh[14] * -2.0 * yz
                           + C3[6] * sh[15] * -3.0 * 2.0 * xy)
                dz = dz + (C3[1] * sh[10] * xy + C3[2] * sh[11] * 4.0 * 2.0 * yz + C3[3] * sh[12] * 3.0 * (2.0 * zz - xx - yy)
                           + C3[4] * sh[13] * 4.0 * 2.0 * xz + C3[5] * sh[14] * (xx - yy))
    return dsh, (dx, dy, dz)


def _dnormv(v, dv):
    sum2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2]
    inv = 1.0 / sqrt(sum2 * sum2 * sum2)
    return [((sum2 - v[0] * v[0]) * dv[0] - v[1] * v[0] * dv[1] - v[2] * v[0] * dv[2]) * inv,
            (-v[0] * v[1] * dv[0] + (sum2 - v[1] * v[1]) * dv[1] - v[2] * v[1] * dv[2]) * inv,
            (-v[0] * v[2] * dv[0] - v[1] * v[2] * dv[1] + (sum2 - v[2] * v[2]) * dv[2]) * inv]


def _quirk_set(quirks):
    if quirks is True:
        return set(QUIRKS)
    if quirks is False:
        return set()
    q = set(quirks)
    assert q <= set(QUIRKS), q - set(QUIRKS)
    return q


def chain(params, cam, rg, quirks=True, flip=None):
    """gaussian_backward_kernel for P visible Gaussians, in RE.

    params: dict(means [P,3], scales [P,3] and rots [P,4] (x, y, z, w), or cov [P,6]; sh [P,M,3] or None; degree;
    scale_modifier), float tensors.  cam: `camera`.  rg: the render gradients (render_grads / render_grads_from_acc).
    quirks: True (all of QUIRKS, the kernel), False (none: the true derivative) or the set of QUIRKS that are on.
    flip: {decision: bool mask} takes the other branch of a float32 decision for those Gaussians.
    Returns (out, decisions): out[k] = RE of means3D [P,3], cov3D [P,6], sh [P,M,3], scales [P,3], rots [P,4] (None where
    the kernel writes zero rows by construction: scales / rots under cov, sh without SH); decisions[k] = (taken [P] or
    [P,3] bool, ambiguous) for clamp_x, clamp_y, sh_clamp, overflow."""
    q = _quirk_set(quirks)
    flip = flip or {}
    mu = leaves(params["means"])
    P = params["means"].shape[0]
    vm, pm = cam["view"], cam["proj"]
    hx, hy = cam["focal"]
    mod = f32(params.get("scale_modifier", 1.0))
    dec = {}

    def decide(key, taken, amb):
        f = flip.get(key)
        dec[key] = (taken if f is None else taken ^ f, amb)
        return dec[key][0]

    # ---- 3D covariance ----
    if params.get("cov") is not None:
        cov3 = leaves(params["cov"])
    else:
        sc, qv = leaves(params["scales"]), leaves(params["rots"])
        s = [mod * sc[i] for i in range(3)]
        Rq = quat_to_m3(*qv)
        S = [[s[c] if c == r else ZERO for r in range(3)] for c in range(3)]
        Mx = m3_mul(S, Rq)
        Sg = m3_mul(m3_t(Mx), Mx)
        cov3 = [Sg[0][0], Sg[0][1], Sg[0][2], Sg[1][1], Sg[1][2], Sg[2][2]]

    # ---- render gradients ----
    g2x, g2y = rg["g2"]
    dc_x, dc_y, dc_z = rg["dc"]
    dL_dcovzx, dL_dcovyz, dL_ddepth = rg["covzx"], rg["covyz"], rg["depth"]

    # ---- ewa_project ----
    t = [vm[r] * mu[0] + vm[4 + r] * mu[1] + vm[8 + r] * mu[2] + vm[12 + r] for r in range(3)]
    ct = []
    for i, key in ((0, "clamp_x"), (1, "clamp_y")):
        tan = cam["tanfovx"] if i == 0 else cam["tanfovy"]
        lim32 = f32(np.float32(1.3) * np.float32(tan))  # the kernel's threshold
        lim = 1.3 * tan  # the value (camera_grad_model.project's)
        ratio = t[i] / t[2]
        taken = decide(key, (ratio.v < -lim32) | (ratio.v > lim32), _near(ratio, lim32) | _near(ratio, -lim32))
        sgn = torch.sign(ratio.v)
        ct.append((where(taken, RE(sgn * lim) * t[2], ratio * t[2]), taken, sgn * lim))
    (tx, clx, limx), (ty, cly, limy) = ct
    tz = t[2]
    J = [[hx / tz, ZERO, -(hx * tx) / (tz * tz)], [ZERO, hy / tz, -(hy * ty) / (tz * tz)], [ZERO, ZERO, RE(1.0)]]
    Wm = [[RE(vm[4 * r + c]) for r in range(3)] for c in range(3)]
    T = m3_mul(Wm, J)
    V = [[cov3[0], cov3[1], cov3[2]], [cov3[1], cov3[3], cov3[4]], [cov3[2], cov3[4], cov3[5]]]
    cov = m3_mul(m3_mul(m3_t(T), V), T)

    # ---- 2D covariance backward ----
    ca, cb, cc = cov[0][0] + 0.3, cov[0][1], cov[1][1] + 0.3
    denom = ca * cc - cb * cb
    d2 = denom * denom + CM.EPS_W if "eps" in q else denom * denom
    ov = torch.zeros(P, dtype=torch.bool)
    if "overflow" in q:
        ov = decide("overflow", d2.v >= OVERFLOW, _near(d2, OVERFLOW))
    denom2inv = 1.0 / d2
    dL_da = where(ov, 0.0, denom2inv * (-cc * cc * dc_x + 2.0 * cb * cc * dc_y + (denom - ca * cc) * dc_z))
    dL_dc = where(ov, 0.0, denom2inv * (-ca * ca * dc_z + 2.0 * ca * cb * dc_y + (denom - ca * cc) * dc_x))
    dL_db = where(ov, 0.0, denom2inv * 2.0 * (cb * cc * dc_x - (denom + 2.0 * cb * cb) * dc_y + ca * cb * dc_z))

    def Tm(c, r):
        return T[c][r]

    dcov = [
        Tm(0, 0) * Tm(0, 0) * dL_da + Tm(0, 0) * Tm(1, 0) * dL_db + Tm(0, 0) * Tm(2, 0) * dL_dcovzx + Tm(1, 0) * Tm(1, 0) * dL_dc
        + Tm(1, 0) * Tm(2, 0) * dL_dcovyz,
        2.0 * Tm(0, 0) * Tm(0, 1) * dL_da + (Tm(0, 0) * Tm(1, 1) + Tm(0, 1) * Tm(1, 0)) * dL_db
        + (Tm(0, 1) * Tm(2, 0) + Tm(0, 0) * Tm(2, 1)) * dL_dcovzx + (Tm(1, 1) * Tm(2, 0) + Tm(1, 0) * Tm(2, 1)) * dL_dcovyz
        + 2.0 * Tm(1, 0) * Tm(1, 1) * dL_dc,
        2.0 * Tm(0, 0) * Tm(0, 2) * dL_da + (Tm(0, 0) * Tm(1, 2) + Tm(0, 2) * Tm(1, 0)) * dL_db
        + (Tm(0, 2) * Tm(2, 0) + Tm(0, 0) * Tm(2, 2)) * dL_dcovzx + (Tm(1, 2) * Tm(2, 0) + Tm(1, 0) * Tm(2, 2)) * dL_dcovyz
        + 2.0 * Tm(1, 0) * Tm(1, 2) * dL_dc,
        Tm(0, 1) * Tm(0, 1) * dL_da + Tm(0, 1) * Tm(1, 1) * dL_db + Tm(0, 1) * Tm(2, 1) * dL_dcovzx + Tm(1, 1) * Tm(1, 1) * dL_dc
        + Tm(1, 1) * Tm(2, 1) * dL_dcovyz,
        2.0 * Tm(0, 2) * Tm(0, 1) * dL_da + (Tm(0, 1) * Tm(1, 2) + Tm(0, 2) * Tm(1, 1)) * dL_db
        + (Tm(0, 2) * Tm(2, 1) + Tm(0, 1) * Tm(2, 2)) * dL_dcovzx + (Tm(1, 2) * Tm(2, 1) + Tm(1, 1) * Tm(2, 2)) * dL_dcovyz
        + 2.0 * Tm(1, 1) * Tm(1, 2) * dL_dc,
        Tm(0, 2) * Tm(0, 2) * dL_da + Tm(0, 2) * Tm(1, 2) * dL_db + Tm(0, 2) * Tm(2, 2) * dL_dcovzx + Tm(1, 2) * Tm(1, 2) * dL_dc
        + Tm(1, 2) * Tm(2, 2) * dL_dcovyz,
    ]
    dcov = [where(ov, 0.0, x) for x in dcov]

    def TV(a, k):  # T.m[a][0] V.m[k][0] + T.m[a][1] V.m[k][1] + T.m[a][2] V.m[k][2]
        return Tm(a, 0) * V[k][0] + Tm(a, 1) * V[k][1] + Tm(a, 2) * V[k][2]

    dT0 = [2.0 * TV(0, k) * dL_da + TV(1, k) * dL_db + TV(2, k) * dL_dcovzx for k in range(3)]
    dT1 = [2.0 * TV(1, k) * dL_dc + TV(0, k) * dL_db for k in range(3)]
    dT1[0] = dT1[0] + TV(2, 0) * dL_dcovyz
    if "dropped_yz" not in q:
        dT1[1] = dT1[1] + TV(2, 1) * dL_dcovyz
        dT1[2] = dT1[2] + TV(2, 2) * dL_dcovyz
    dJ00 = Wm[0][0] * dT0[0] + Wm[0][1] * dT0[1] + Wm[0][2] * dT0[2]
    dJ02 = Wm[2][0] * dT0[0] + Wm[2][1] * dT0[1] + Wm[2][2] * dT0[2]
    dJ11 = Wm[1][0] * dT1[0] + Wm[1][1] * dT1[1] + Wm[1][2] * dT1[2]
    dJ12 = Wm[2][0] * dT1[0] + Wm[2][1] * dT1[1] + Wm[2][2] * dT1[2]

    itz = 1.0 / tz
    tz2 = itz * itz
    tz3 = tz2 * itz
    dtx_c, dty_c = -hx * tz2 * dJ02, -hy * tz2 * dJ12  # dL/d(clamped t_x), dL/d(clamped t_y)
    dL_dtx = where(clx, 0.0, dtx_c)
    dL_dty = where(cly, 0.0, dty_c)
    dL_dtz = -hx * tz2 * dJ00 - hy * tz2 * dJ11 + (2.0 * hx * tx) * tz3 * dJ02 + (2.0 * hy * ty) * tz3 * dJ12
    if "clamp_tz" not in q:  # a clamped t_x is +-lim t_z
        dL_dtz = dL_dtz + where(clx, dtx_c * RE(limx), 0.0) + where(cly, dty_c * RE(limy), 0.0)
    dmean = [vm[0] * dL_dtx + vm[1] * dL_dty + vm[2] * dL_dtz, vm[4] * dL_dtx + vm[5] * dL_dty + vm[6] * dL_dtz,
             vm[8] * dL_dtx + vm[9] * dL_dty + vm[10] * dL_dtz]

    # ---- depth and 2D-mean paths ----
    mw_h = pm[3] * mu[0] + pm[7] * mu[1] + pm[11] * mu[2] + pm[15]
    m_w = 1.0 / (mw_h + CM.EPS_W)
    mul = vm[2] * mu[0] + vm[6] * mu[1] + vm[10] * mu[2] + vm[14]
    for i in range(3):
        dd = (vm[4 * i + 2] - vm[4 * i + 3] * mul) if "depth_mul" in q else RE(vm[4 * i + 2])
        dmean[i] = dmean[i] + dL_ddepth * dd
    mul1 = (pm[0] * mu[0] + pm[4] * mu[1] + pm[8] * mu[2] + pm[12]) * m_w * m_w
    mul2 = (pm[1] * mu[0] + pm[5] * mu[1] + pm[9] * mu[2] + pm[13]) * m_w * m_w
    for i in range(3):
        dmean[i] = dmean[i] + (pm[4 * i] * m_w - pm[4 * i + 3] * mul1) * g2x + (pm[4 * i + 1] * m_w - pm[4 * i + 3] * mul2) * g2y

    out = dict(cov3D=dcov, sh=None, scales=None, rots=None)

    # ---- SH path ----
    if params.get("sh") is not None:
        shp = torch.as_tensor(params["sh"], dtype=torch.float64)
        M, D = shp.shape[1], params["degree"]
        dir_orig = [mu[i] - cam["campos"][i] for i in range(3)]
        ln = sqrt(dir_orig[0] * dir_orig[0] + dir_orig[1] * dir_orig[1] + dir_orig[2] * dir_orig[2])
        x, y, z = (dir_orig[i] / ln for i in range(3))
        res = []
        for c in range(3):
            res.append(_sh_rgb([RE(shp[:, k, c]) for k in range(M)], D, x, y, z))
        taken = decide("sh_clamp", torch.stack([r.v < 0 for r in res], 1), torch.stack([_near(r, 0.0) for r in res], 1))
        dsh_all = [[ZERO] * 3 for _ in range(M)]
        ddir = [ZERO, ZERO, ZERO]
        for c in range(3):
            d = where(taken[:, c], 0.0, rg["rgb"][c])
            dsh, dr = _sh_backward([RE(shp[:, k, c]) for k in range(M)], D, x, y, z, d)
            for k, v in enumerate(dsh):
                dsh_all[k][c] = v
            ddir = [ddir[i] + dr[i] * d for i in range(3)]
        dm = _dnormv(dir_orig, ddir)
        dmean = [dmean[i] + dm[i] for i in range(3)]
        out["sh"] = dsh_all
    out["means3D"] = dmean

    # ---- scale / rotation ----
    if params.get("cov") is None:
        qx, qy, qz, qw = qv
        dSig = [[dcov[0], 0.5 * dcov[1], 0.5 * dcov[2]], [0.5 * dcov[1], dcov[3], 0.5 * dcov[4]],
                [0.5 * dcov[2], 0.5 * dcov[4], dcov[5]]]
        M2 = [[2.0 * Mx[c][r] for r in range(3)] for c in range(3)]
        dL_dM = m3_mul(M2, dSig)
        Rt = m3_t(Rq)
        dMt = m3_t(dL_dM)
        dscale = [Rt[k][0] * dMt[k][0] + Rt[k][1] * dMt[k][1] + Rt[k][2] * dMt[k][2] for k in range(3)]
        if "scale_mod" not in q:
            dscale = [mod * v for v in dscale]
        dMt = [[dMt[c][r] * s[c] for r in range(3)] for c in range(3)]
        dq = [2.0 * qy * (dMt[1][0] + dMt[0][1]) + 2.0 * qz * (dMt[2][0] + dMt[0][2]) + 2.0 * qw * (dMt[1][2] - dMt[2][1])
              - 4.0 * qx * (dMt[2][2] + dMt[1][1]),
              2.0 * qx * (dMt[1][0] + dMt[0][1]) + 2.0 * qw * (dMt[2][0] - dMt[0][2]) + 2.0 * qz * (dMt[1][2] + dMt[2][1])
              - 4.0 * qy * (dMt[2][2] + dMt[0][0]),
              2.0 * qw * (dMt[0][1] - dMt[1][0]) + 2.0 * qx * (dMt[2][0] + dMt[0][2]) + 2.0 * qy * (dMt[1][2] + dMt[2][1])
              - 4.0 * qz * (dMt[1][1] + dMt[0][0]),
              2.0 * qz * (dMt[0][1] - dMt[1][0]) + 2.0 * qy * (dMt[2][0] - dMt[0][2]) + 2.0 * qx * (dMt[1][2] - dMt[2][1])]
        out["scales"], out["rots"] = dscale, dq
    return {k: _stack(v, P) for k, v in out.items()}, dec


def _stack(v, P):
    """RE lists -> RE of stacked tensors ([P,k] or [P,M,3])."""
    if v is None:
        return None
    ex = lambda x: x.expand(P) if x.dim() == 0 else x
    if isinstance(v[0], list):
        return RE(torch.stack([torch.stack([ex(c.v) for c in row], 1) for row in v], 1),
                  torch.stack([torch.stack([ex(c.s) for c in row], 1) for row in v], 1))
    return RE(torch.stack([ex(c.v) for c in v], 1), torch.stack([ex(c.s) for c in v], 1))


def reference(params, cam, rg, quirks=True, K=K_BOUND):
    """(value, bound, ambiguous [P] bool, decisions) of the chain: value[k] and bound[k] are float64 numpy arrays of the
    five outputs (None where the kernel writes zeros by construction); bound = K u S + FLOOR plus, for every ambiguous
    float32 decision, |this branch - the other| on the Gaussians concerned."""
    out, dec = chain(params, cam, rg, quirks)
    val = {k: (None if v is None else v.v.numpy()) for k, v in out.items()}
    bnd = {k: (None if v is None else K * U24 * v.s.numpy() + FLOOR) for k, v in out.items()}
    P = params["means"].shape[0]
    amb_any = np.zeros(P, bool)
    for key, (_, amb) in dec.items():
        if not bool(amb.any()):
            continue
        alt, _ = chain(params, cam, rg, quirks, flip={key: amb})
        for k, v in alt.items():
            if v is not None:
                bnd[k] = bnd[k] + np.abs(v.v.numpy() - val[k])
        amb_any |= amb.reshape(P, -1).any(1).numpy()
    return val, bnd, amb_any, {k: (d.numpy(), a.numpy()) for k, (d, a) in dec.items()}
