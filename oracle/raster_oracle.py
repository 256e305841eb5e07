"""ctypes binding of oracle/libraster_oracle.so (raster_oracle.c) — numpy in, numpy out.  Test infrastructure."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_PATH = os.path.join(_HERE, "libraster_oracle.so")


class _Args(C.Structure):
    _fields_ = [("P", C.c_int), ("D", C.c_int), ("M", C.c_int), ("W", C.c_int), ("H", C.c_int),
                ("tan_fovx", C.c_float), ("tan_fovy", C.c_float), ("scale_modifier", C.c_float)] + \
               [(n, C.c_void_p) for n in ("bg", "means3D", "shs", "colors", "opac", "scales", "rots", "cov_pre", "view",
                                          "proj", "campos")]


def _load():
    if not os.path.exists(_PATH):
        raise ImportError(f"{_PATH} missing: run `make -C oracle libraster_oracle.so`")
    lib = C.CDLL(_PATH)
    lib.ro_forward.restype = C.c_void_p
    lib.ro_forward.argtypes = [C.POINTER(_Args), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.ro_backward.restype = C.c_int
    lib.ro_backward.argtypes = [C.POINTER(_Args), C.c_void_p, C.c_void_p] + [C.c_void_p] * 10
    lib.ro_backward_ex.restype = C.c_int
    lib.ro_backward_ex.argtypes = [C.POINTER(_Args), C.c_void_p, C.c_void_p] + [C.c_void_p] * 12
    lib.ro_num_rendered.restype = C.c_int
    lib.ro_num_rendered.argtypes = [C.c_void_p]
    for n in ("ro_point_list", "ro_ranges", "ro_n_contrib", "ro_final_T", "ro_means2D", "ro_conic_op", "ro_rgb", "ro_depths"):
        getattr(lib, n).restype = C.c_void_p
        getattr(lib, n).argtypes = [C.c_void_p]
    lib.ro_free.argtypes = [C.c_void_p]
    lib.ro_moment_reference.restype = C.c_int
    lib.ro_moment_reference.argtypes = [C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 13
    return lib


_lib = None


def _f32(x):
    return None if x is None else np.ascontiguousarray(x, dtype=np.float32)


def _p(x):
    return None if x is None else x.ctypes.data


class Result:
    pass


def forward_backward(scene, cam, H, W, bg, sh_degree=0, scale_modifier=1.0, colors_precomp=None, cov3D_precomp=None,
                     dL_dcolor=None, dL_ddepth=None):
    """Run the CPU restatement.  scene: dict(means3D, shs, opacities, scales, rotations); cam: dict(viewmatrix,
    projmatrix, campos, tanfovx, tanfovy).  Returns an object with color, depth, radii, is_used, num_rendered,
    point_list, ranges, n_contrib, final_T and (when gradients are given) the 8 gradient arrays."""
    global _lib
    if _lib is None:
        _lib = _load()
    means = _f32(scene["means3D"])
    P = means.shape[0]
    shs = None if colors_precomp is not None else _f32(scene["shs"])
    M = 0 if shs is None else shs.shape[1]
    cols = _f32(colors_precomp)
    opac = _f32(scene["opacities"]).reshape(-1)
    scales = None if cov3D_precomp is not None else _f32(scene["scales"])
    rots = None if cov3D_precomp is not None else _f32(scene["rotations"])
    covp = _f32(cov3D_precomp)
    view, proj, campos, bgc = _f32(cam["viewmatrix"]), _f32(cam["projmatrix"]), _f32(cam["campos"]), _f32(bg)
    a = _Args(P, sh_degree, M, W, H, cam["tanfovx"], cam["tanfovy"], scale_modifier, _p(bgc), _p(means), _p(shs),
              _p(cols), _p(opac), _p(scales), _p(rots), _p(covp), _p(view), _p(proj), _p(campos))
    r = Result()
    r.color = np.zeros((3, H, W), np.float32)
    r.depth = np.zeros((1, H, W), np.float32)
    r.radii = np.zeros(P, np.int32)
    r.is_used = np.zeros(P, np.uint8)
    st = _lib.ro_forward(C.byref(a), r.color.ctypes.data, r.depth.ctypes.data, r.radii.ctypes.data, r.is_used.ctypes.data)
    try:
        R = _lib.ro_num_rendered(st)
        r.num_rendered = R
        tiles = ((W + 15) // 16) * ((H + 15) // 16)
        if P > 0:
            r.point_list = np.ctypeslib.as_array(C.cast(_lib.ro_point_list(st), C.POINTER(C.c_uint32)), (max(R, 1),))[:R].astype(np.int64)
            r.ranges = np.ctypeslib.as_array(C.cast(_lib.ro_ranges(st), C.POINTER(C.c_uint32)), (tiles * 2,)).reshape(tiles, 2).astype(np.int64)
            r.n_contrib = np.ctypeslib.as_array(C.cast(_lib.ro_n_contrib(st), C.POINTER(C.c_uint32)), (H * W,)).reshape(H, W).astype(np.int64)
            r.final_T = np.ctypeslib.as_array(C.cast(_lib.ro_final_T(st), C.POINTER(C.c_float)), (H * W,)).reshape(H, W).copy()
        else:
            r.point_list = np.zeros(0, np.int64)
            r.ranges = np.zeros((tiles, 2), np.int64)
        if dL_dcolor is not None:
            gc, gd = _f32(dL_dcolor), _f32(dL_ddepth)
            z = lambda *s: np.zeros(s, np.float32)
            r.dL_dmeans2D, r.dL_dcolors, r.dL_dopacity = z(P, 3), z(P, 3), z(P, 1)
            r.dL_dmeans3D, r.dL_dcov3D, r.dL_dsh = z(P, 3), z(P, 6), z(P, max(M, 1), 3)
            r.dL_dscales, r.dL_drotations = z(P, 3), z(P, 4)
            _lib.ro_backward(C.byref(a), st, r.radii.ctypes.data, gc.ctypes.data, gd.ctypes.data,
                             r.dL_dmeans2D.ctypes.data, r.dL_dcolors.ctypes.data, r.dL_dopacity.ctypes.data,
                             r.dL_dmeans3D.ctypes.data, r.dL_dcov3D.ctypes.data, r.dL_dsh.ctypes.data,
                             r.dL_dscales.ctypes.data, r.dL_drotations.ctypes.data)
            if M == 0:
                r.dL_dsh = z(P, 0, 3)
    finally:
        _lib.ro_free(st)
    r.is_used = r.is_used.astype(bool)
    return r


def _view(ptr, ctype, shape):
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ctype)), shape)


class State:
    """A forward state of the CPU restatement kept alive for backward replays: the float32 splat records, instance list,
    tile ranges and per-pixel n_contrib / final_T the backward reads.  `final_T` is a writable view of the state itself.
    Call free() when done."""

    def __init__(self, scene, cam, H, W, bg, sh_degree=0, scale_modifier=1.0):
        global _lib
        if _lib is None:
            _lib = _load()
        self.keep = [_f32(scene["means3D"]), _f32(scene["shs"]), _f32(scene["opacities"]).reshape(-1),
                     _f32(scene["scales"]), _f32(scene["rotations"]), _f32(cam["viewmatrix"]), _f32(cam["projmatrix"]),
                     _f32(cam["campos"]), _f32(bg)]
        means, shs, opac, scales, rots, view, proj, campos, bgc = self.keep
        P = self.P = means.shape[0]
        self.H, self.W, self.bg = H, W, bgc
        self.args = _Args(P, sh_degree, shs.shape[1], W, H, cam["tanfovx"], cam["tanfovy"], scale_modifier, _p(bgc),
                          _p(means),
                          _p(shs), None, _p(opac), _p(scales), _p(rots), None, _p(view), _p(proj), _p(campos))
        self.color = np.zeros((3, H, W), np.float32)
        self.depth = np.zeros((1, H, W), np.float32)
        self.radii = np.zeros(P, np.int32)
        is_used = np.zeros(P, np.uint8)
        self.st = _lib.ro_forward(C.byref(self.args), self.color.ctypes.data, self.depth.ctypes.data,
                                  self.radii.ctypes.data, is_used.ctypes.data)
        R = _lib.ro_num_rendered(self.st)
        tiles = ((W + 15) // 16) * ((H + 15) // 16)
        self.point_list = _view(_lib.ro_point_list(self.st), C.c_uint32, (max(R, 1),))[:R]
        self.ranges = _view(_lib.ro_ranges(self.st), C.c_uint32, (tiles, 2))
        self.n_contrib = _view(_lib.ro_n_contrib(self.st), C.c_uint32, (H, W))
        self.final_T = _view(_lib.ro_final_T(self.st), C.c_float, (H, W))
        m2 = _view(_lib.ro_means2D(self.st), C.c_float, (P, 2))
        co = _view(_lib.ro_conic_op(self.st), C.c_float, (P, 6))
        rgb = _view(_lib.ro_rgb(self.st), C.c_float, (P, 3))
        dep = _view(_lib.ro_depths(self.st), C.c_float, (P,))
        # the GPU's record layout: {px, py, conic xx, xy, yy, opacity, cov_zx, cov_yz, r, g, b, depth}
        self.splats = np.ascontiguousarray(np.concatenate([m2, co, rgb, dep[:, None]], 1), np.float32)

    def backward_acc(self, dL_dcolor, dL_ddepth, shift=None, with_outputs=False):
        """The render-stage sums of ro_backward in float64, [P][12] = {colour r,g,b, depth, mean2D x,y, conic xx,xy,yy,
        cov_zx, cov_yz, opacity}.  shift=(g, x0, y0) plants a one-column offset for Gaussian g in the 8x4 sub-tile at
        (x0, y0).  with_outputs: (acc, the eight float32 gradient arrays of ro_backward computed from float32(acc))."""
        P = self.P
        gc, gd = _f32(dL_dcolor), _f32(dL_ddepth)
        z = lambda *s: np.zeros(s, np.float32)
        outs = [z(P, 3), z(P, 3), z(P, 1), z(P, 3), z(P, 6), z(P, max(self.args.M, 1), 3), z(P, 3), z(P, 4)]
        acc = np.zeros((P, 12), np.float64)
        sh = None if shift is None else np.asarray(shift, np.int32)
        _lib.ro_backward_ex(C.byref(self.args), self.st, self.radii.ctypes.data, gc.ctypes.data, gd.ctypes.data,
                            *[o.ctypes.data for o in outs], acc.ctypes.data, _p(sh))
        return (acc, outs) if with_outputs else acc

    def free(self):
        if self.st:
            _lib.ro_free(self.st)
            self.st = None


MOMENTS = ["t", "t dx", "t dy", "t dx2", "t dxdy", "t dy2", "v", "v dx", "v dy", "w r", "w g", "w b"]
RENDER_GRADS = ["colour r", "colour g", "colour b", "depth", "mean2D x", "mean2D y", "conic xx", "conic xy", "conic yy",
                "cov_zx", "cov_yz", "opacity"]


def moment_reference(splats, point_list, ranges, n_contrib, W, H, bg, dL_dcolor, dL_ddepth):
    """Float64 replay of the render backward from a saved forward state, with a per-Gaussian error bound
    (ro_moment_reference in raster_oracle.c).  Returns an object with mom, mom_bound, grad, grad_bound ([P][12] float64),
    n_pairs, S_g, deepest, n_amb ([P] int) and pairs, ambiguous, max_contrib (ints)."""
    global _lib
    if _lib is None:
        _lib = _load()
    sp = _f32(splats).reshape(-1, 12)
    P = sp.shape[0]
    pl = np.ascontiguousarray(point_list, np.uint32).reshape(-1)
    rg = np.ascontiguousarray(ranges, np.uint32).reshape(-1, 2)
    nc = np.ascontiguousarray(n_contrib, np.uint32).reshape(-1)
    assert nc.size == W * H and rg.shape[0] == ((W + 15) // 16) * ((H + 15) // 16)
    gc, gd, bgc = _f32(dL_dcolor).reshape(3, H * W), _f32(dL_ddepth).reshape(H * W), _f32(bg).reshape(3)
    r = Result()
    r.mom, r.mom_bound, r.grad, r.grad_bound = (np.zeros((P, 12), np.float64) for _ in range(4))
    diag = np.zeros((P, 4), np.int32)
    tot = np.zeros(3, np.int64)
    _lib.ro_moment_reference(P, W, H, sp.ctypes.data, pl.ctypes.data if pl.size else None, rg.ctypes.data,
                             nc.ctypes.data, bgc.ctypes.data, gc.ctypes.data, gd.ctypes.data, r.mom.ctypes.data,
                             r.mom_bound.ctypes.data, r.grad.ctypes.data, r.grad_bound.ctypes.data, diag.ctypes.data,
                             tot.ctypes.data)
    r.n_pairs, r.S_g, r.deepest, r.n_amb = (diag[:, k].copy() for k in range(4))
    r.pairs, r.ambiguous, r.max_contrib = (int(v) for v in tot)
    return r
