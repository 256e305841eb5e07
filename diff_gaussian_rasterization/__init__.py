"""Drop-in `diff_gaussian_rasterization` backed by libgsicp_b200.so (sm_90a).

Public surface = the reference package's
(submodules/diff-gaussian-rasterization/diff_gaussian_rasterization/__init__.py:44-222):
`GaussianRasterizationSettings` (NamedTuple, same field order), `GaussianRasterizer` (nn.Module whose
forward returns `(depth[1,H,W], color[3,H,W], radii[P], is_used[P])`), `rasterize_gaussians`,
`_RasterizeGaussians`, and a `_C` namespace with `rasterize_gaussians`, `rasterize_gaussians_backward`,
`mark_visible`, so gaussian_renderer/__init__.py and mp_Mapper.py of the reference run unmodified.
"""
from types import SimpleNamespace
from typing import NamedTuple

import torch
from torch import nn

from gs_icp_slam_b200 import rasterizer as _impl

_C = SimpleNamespace(
    rasterize_gaussians=_impl.rasterize_gaussians,
    rasterize_gaussians_backward=_impl.rasterize_gaussians_backward,
    mark_visible=_impl.mark_visible,
)


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


def _snapshot(values, path):
    """debug=True behaviour of the reference: dump the call's inputs when the kernel call raises."""
    torch.save(tuple(v.detach().cpu().clone() if isinstance(v, torch.Tensor) else v for v in values), path)


class _RasterizeGaussians(torch.autograd.Function):
    """Autograd wiring: 8 differentiable-slot inputs + settings -> (depth, color, radii, is_used)."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings):
        rs = raster_settings
        call = (rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier, cov3Ds_precomp,
                rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width, sh, rs.sh_degree,
                rs.campos, rs.prefiltered, rs.debug)
        try:
            n, depth, color, radii, is_used, geom, binning, img = _C.rasterize_gaussians(*call)
        except Exception:
            if rs.debug:
                _snapshot(call, "snapshot_fw.dump")
                print("\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.")
            raise
        ctx.raster_settings = rs
        ctx.num_rendered = n
        ctx.set_materialize_grads(False)  # no zero tensors for the radii / is_used slots (backward handles None)
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geom, binning, img)
        ctx.mark_non_differentiable(radii, is_used)
        return depth, color, radii, is_used

    @staticmethod
    def backward(ctx, grad_depth, grad_color, _grad_radii, _grad_is_used):
        rs = ctx.raster_settings
        colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geom, binning, img = ctx.saved_tensors
        if grad_depth is None:
            grad_depth = torch.zeros((1, rs.image_height, rs.image_width), device=means3D.device)
        if grad_color is None:
            grad_color = torch.zeros((3, rs.image_height, rs.image_width), device=means3D.device)
        call = (rs.bg, means3D, radii, colors_precomp, scales, rotations, rs.scale_modifier, cov3Ds_precomp,
                rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, grad_depth, grad_color, sh, rs.sh_degree,
                rs.campos, geom, ctx.num_rendered, binning, img, rs.debug)
        try:
            g_means2D, g_colors, g_opac, g_means3D, g_cov3D, g_sh, g_scales, g_rots = _C.rasterize_gaussians_backward(*call)
        except Exception:
            if rs.debug:
                _snapshot(call, "snapshot_bw.dump")
                print("\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n")
            raise
        # order of forward's inputs: means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds, settings
        return g_means3D, g_means2D, g_sh, g_colors, g_opac, g_scales, g_rots, g_cov3D, None


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings)


def _absent():
    return torch.Tensor([])  # the reference's marker for "argument not provided"


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        rs = self.raster_settings
        with torch.no_grad():
            return _C.mark_visible(positions, rs.viewmatrix, rs.projmatrix)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        if (shs is None) == (colors_precomp is None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        has_sr = scales is not None or rotations is not None
        if ((scales is None or rotations is None) and cov3D_precomp is None) or (has_sr and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        opt = lambda t: _absent() if t is None else t
        return rasterize_gaussians(means3D, means2D, opt(shs), opt(colors_precomp), opacities, opt(scales),
                                   opt(rotations), opt(cov3D_precomp), self.raster_settings)
