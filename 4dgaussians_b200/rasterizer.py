"""Drop-in for the ``diff_gaussian_rasterization`` module the reference imports
(/root/reference/gaussian_renderer/__init__.py:14; merge_many_4dgs.py:33; scene/dataset_readers.py:485).

Same names, argument meaning and error behaviour as the upstream Python surface (SURVEY.md §8b, App. A.5);
behind it the hand-written sm_90a kernels of libg4d.so through the C-ABI (include/g4d.h).  PyTorch is only
plumbing here: device memory, the current stream, autograd bookkeeping.
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional

import torch
import torch.nn as nn

from . import _lib


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


def _dev_f32(t: torch.Tensor, numel: int, what: str) -> torch.Tensor:
    if not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor (the g4d path has no CPU fallback)" % what)
    t = t.detach()
    if t.dtype != torch.float32 or not t.is_contiguous():
        t = t.float().contiguous()
    if t.numel() != numel:
        raise RuntimeError("%s has %d elements, expected %d" % (what, t.numel(), numel))
    return t


def camera_from_settings(rs: GaussianRasterizationSettings, time: float = 0.0, keep=None) -> _lib.Camera:
    """Build the C-ABI camera.  Matrices given as CUDA tensors stay on the device (no D2H sync);
    CPU tensors are copied into the struct."""
    cam = _lib.Camera()
    cam.image_height, cam.image_width = int(rs.image_height), int(rs.image_width)
    cam.sh_degree, cam.debug = int(rs.sh_degree), int(bool(rs.debug))
    cam.tanfovx, cam.tanfovy, cam.scale_modifier, cam.time = float(rs.tanfovx), float(rs.tanfovy), \
        float(rs.scale_modifier), float(time)
    for name, field, dfield, n in (("viewmatrix", "viewmatrix", "d_viewmatrix", 16), ("projmatrix", "projmatrix", "d_projmatrix", 16),
                                   ("campos", "campos", "d_campos", 3), ("bg", "bg", "d_bg", 3)):
        t = getattr(rs, name)
        if not torch.is_tensor(t):
            t = torch.as_tensor(t, dtype=torch.float32)
        if t.is_cuda:
            t = _dev_f32(t, n, name)
            if keep is not None:
                keep.append(t)
            setattr(cam, dfield, t.data_ptr())
        else:
            flat = t.detach().float().reshape(-1)
            if flat.numel() != n:
                raise RuntimeError("%s has %d elements, expected %d" % (name, flat.numel(), n))
            getattr(cam, field)[:] = flat.tolist()
    return cam


class _ContextLease:
    """Returns the context to the workspace pool when the autograd node dies."""

    def __init__(self, ws: _lib.Workspace):
        self.ws = ws
        self.ctx = ws.acquire_context()

    def release(self):
        if self.ctx is not None:
            self.ws.release_context(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


def _stream_ptr(device) -> int:
    return int(torch.cuda.current_stream(device).cuda_stream)


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, opacities, scales, rotations, raster_settings):
        lib = _lib.load()
        dev = means3D.device
        n = means3D.shape[0]
        m3 = _dev_f32(means3D, n * 3, "means3D")
        shc = _dev_f32(sh, n * 48, "shs")
        op = _dev_f32(opacities, n, "opacities")
        sc = _dev_f32(scales, n * 3, "scales")
        ro = _dev_f32(rotations, n * 4, "rotations")
        H, W = int(raster_settings.image_height), int(raster_settings.image_width)
        color = torch.empty(3, H, W, device=dev, dtype=torch.float32)
        depth = torch.empty(1, H, W, device=dev, dtype=torch.float32)
        radii = torch.empty(n, device=dev, dtype=torch.int32)
        keep = []
        cam = camera_from_settings(raster_settings, keep=keep)
        with torch.cuda.device(dev):
            lease = _ContextLease(_lib.Workspace.get(dev.index if dev.index is not None else torch.cuda.current_device()))
            _lib.check(lib.g4d_rasterize_forward(lease.ctx.handle, C.byref(cam), n, m3.data_ptr(), shc.data_ptr(), op.data_ptr(),
                                                 sc.data_ptr(), ro.data_ptr(), color.data_ptr(), depth.data_ptr(),
                                                 radii.data_ptr(), _stream_ptr(dev)), "g4d_rasterize_forward")
        ctx.raster_settings = raster_settings
        ctx.lease = lease
        ctx.n = n
        ctx.save_for_backward(m3, shc, op, sc, ro)
        ctx.mark_non_differentiable(radii, depth)
        return color, radii, depth

    @staticmethod
    def backward(ctx, grad_color, _grad_radii, _grad_depth):
        lib = _lib.load()
        m3, shc, op, sc, ro = ctx.saved_tensors
        dev = m3.device
        n = ctx.n
        rs = ctx.raster_settings
        gcol = _dev_f32(grad_color, 3 * int(rs.image_height) * int(rs.image_width), "grad_out_color")
        g_means3D = torch.empty(n, 3, device=dev)
        g_means2D = torch.empty(n, 3, device=dev)
        g_sh = torch.empty(n, 16, 3, device=dev)
        g_op = torch.empty(n, 1, device=dev)
        g_sc = torch.empty(n, 3, device=dev)
        g_ro = torch.empty(n, 4, device=dev)
        keep = []
        cam = camera_from_settings(rs, keep=keep)
        lease = ctx.lease
        if lease is None or lease.ctx is None:
            raise RuntimeError("rasterizer backward called twice (context already released)")
        with torch.cuda.device(dev):
            _lib.check(lib.g4d_rasterize_backward(lease.ctx.handle, C.byref(cam), n, m3.data_ptr(), shc.data_ptr(), op.data_ptr(),
                                                  sc.data_ptr(), ro.data_ptr(), gcol.data_ptr(), g_means3D.data_ptr(),
                                                  g_means2D.data_ptr(), g_sh.data_ptr(), g_op.data_ptr(), g_sc.data_ptr(),
                                                  g_ro.data_ptr(), _stream_ptr(dev)), "g4d_rasterize_backward")
        lease.release()
        ctx.lease = None
        return g_means3D, g_means2D, g_sh, g_op, g_sc, g_ro, None


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings: GaussianRasterizationSettings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        raise NotImplementedError("markVisible is not used by 4DGaussians (SURVEY.md §8b) and is not part of the g4d path")

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        rs = self.raster_settings
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        if colors_precomp is not None or cov3D_precomp is not None:
            raise NotImplementedError("colors_precomp / cov3D_precomp are dead paths in the reference "
                                      "(gaussian_renderer/__init__.py:74-78,105-116) and are not provided")
        return _RasterizeGaussians.apply(means3D, means2D, shs, opacities, scales, rotations, rs)
