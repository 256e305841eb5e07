"""ctypes binding of oracle/_ref/libref_cuda.so — the REFERENCE's own CUDA rasterizer / simple-knn compiled
unmodified for sm_90a (oracle/Makefile, oracle/ref_shim.cu).  GPU only.  Test infrastructure (golden generation) and
the "reference kernels on the same GPU" timing leg of the tools."""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(_HERE, "_ref", "libref_cuda.so")
_lib = None


def available():
    return os.path.exists(PATH)


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(PATH)
        vp, i, f = C.c_void_p, C.c_int, C.c_float
        lib.ref_raster_forward.restype = vp
        lib.ref_raster_forward.argtypes = [i, i, i, vp, i, i, vp, vp, vp, vp, vp, f, vp, vp, vp, vp, vp, f, f, i, vp, vp, vp,
                                           vp, C.POINTER(C.c_int)]
        lib.ref_raster_backward.restype = i
        lib.ref_raster_backward.argtypes = [vp, i, i, vp, vp, vp, vp, vp, f, vp, vp, vp, vp, vp, f, f, vp, vp, vp] + [vp] * 10
        lib.ref_raster_export.restype = i
        lib.ref_raster_export.argtypes = [vp, vp, vp]
        lib.ref_raster_free.argtypes = [vp]
        lib.ref_dist2.restype = i
        lib.ref_dist2.argtypes = [i, vp, vp]
        lib.ref_mark_visible.restype = i
        lib.ref_mark_visible.argtypes = [i, vp, vp, vp, vp]
        _lib = lib
    return _lib


def _p(t):
    return None if t is None or t.numel() == 0 else t.data_ptr()


class RefRaster:
    """One forward (+ optional backward) of the reference rasterizer on CUDA tensors."""

    def __init__(self, bg, means3D, shs, colors, opacities, scales, rotations, cov_pre, view, proj, campos, tanx, tany,
                 H, W, degree, scale_modifier=1.0):
        lib = _load()
        dev = means3D.device
        self.a = dict(bg=bg, means3D=means3D, shs=shs, colors=colors, scales=scales, rotations=rotations, cov_pre=cov_pre,
                      view=view, proj=proj, campos=campos)
        self.P, self.H, self.W, self.D = means3D.shape[0], H, W, degree
        self.M = 0 if shs is None or shs.numel() == 0 else shs.shape[1]
        self.tanx, self.tany, self.sm = tanx, tany, scale_modifier
        self.depth = torch.zeros((1, H, W), device=dev)
        self.color = torch.zeros((3, H, W), device=dev)
        self.radii = torch.zeros(self.P, dtype=torch.int32, device=dev)
        self.is_used = torch.zeros(self.P, dtype=torch.bool, device=dev)
        n = C.c_int(0)
        torch.cuda.synchronize()
        self.h = lib.ref_raster_forward(self.P, degree, self.M, _p(bg), W, H, _p(means3D), _p(shs), _p(colors),
                                        _p(opacities), _p(scales), scale_modifier, _p(rotations), _p(cov_pre), _p(view),
                                        _p(proj), _p(campos), tanx, tany, 0, _p(self.depth), _p(self.color),
                                        _p(self.radii), _p(self.is_used), C.byref(n))
        self.num_rendered = n.value

    def export(self):
        lib = _load()
        dev = self.depth.device
        tiles = ((self.W + 15) // 16) * ((self.H + 15) // 16)
        pl = torch.zeros(max(self.num_rendered, 1), dtype=torch.int32, device=dev)
        rg = torch.zeros(tiles * 2, dtype=torch.int32, device=dev)
        lib.ref_raster_export(self.h, _p(pl), _p(rg))
        return pl[: self.num_rendered].to(torch.int64), rg.view(tiles, 2).to(torch.int64)

    def backward(self, dL_dcolor, dL_ddepth):
        lib = _load()
        dev, P, M = self.depth.device, self.P, self.M
        z = lambda *s: torch.zeros(s, device=dev)
        g = dict(means2D=z(P, 3), conic=z(P, 6), opacity=z(P, 1), depths=z(P, 1), colors=z(P, 3), means3D=z(P, 3),
                 cov3D=z(P, 6), sh=z(P, max(M, 1), 3), scales=z(P, 3), rotations=z(P, 4))
        a = self.a
        torch.cuda.synchronize()
        rc = lib.ref_raster_backward(self.h, self.D, M, _p(a["bg"]), _p(a["means3D"]), _p(a["shs"]), _p(a["colors"]),
                                     _p(a["scales"]), self.sm, _p(a["rotations"]), _p(a["cov_pre"]), _p(a["view"]),
                                     _p(a["proj"]), _p(a["campos"]), self.tanx, self.tany, _p(self.radii),
                                     _p(dL_ddepth.contiguous()), _p(dL_dcolor.contiguous()), _p(g["means2D"]),
                                     _p(g["conic"]), _p(g["opacity"]), _p(g["depths"]), _p(g["colors"]), _p(g["means3D"]),
                                     _p(g["cov3D"]), _p(g["sh"]), _p(g["scales"]), _p(g["rotations"]))
        if rc != 0:
            raise RuntimeError(f"reference backward failed: cuda error {rc}")
        if M == 0:
            g["sh"] = z(P, 0, 3)
        return g

    def free(self):
        if self.h:
            _load().ref_raster_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def ref_dist2(points):
    lib = _load()
    out = torch.zeros(points.shape[0], device=points.device)
    p = points.contiguous().float()
    torch.cuda.synchronize()
    rc = lib.ref_dist2(p.shape[0], _p(p), _p(out))
    if rc != 0:
        raise RuntimeError(f"reference distCUDA2 failed: cuda error {rc}")
    return out
