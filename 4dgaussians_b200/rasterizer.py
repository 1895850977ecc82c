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


def camera_from_settings(rs: GaussianRasterizationSettings, time: float = 0.0, keep=None, sh_coeffs: int = 16) -> _lib.Camera:
    """Build the C-ABI camera; sh_coeffs: M, the SH coefficients per Gaussian of the tensors it renders.  Matrices given as
    CUDA tensors stay on the device (no D2H sync); CPU tensors are copied into the struct."""
    cam = _lib.Camera()
    cam.image_height, cam.image_width = int(rs.image_height), int(rs.image_width)
    cam.sh_degree, cam.debug, cam.sh_coeffs = int(rs.sh_degree), int(bool(rs.debug)), int(sh_coeffs)
    cam.tanfovx, cam.tanfovy, cam.scale_modifier, cam.time = float(rs.tanfovx), float(rs.tanfovy), \
        float(rs.scale_modifier), float(time)
    for name, field, dfield, n in (("viewmatrix", "viewmatrix", "d_viewmatrix", 16), ("projmatrix", "projmatrix", "d_projmatrix", 16),
                                   ("campos", "campos", "d_campos", 3), ("bg", "bg", "d_bg", 3)):
        t = getattr(rs, name)
        if not torch.is_tensor(t):
            t = torch.as_tensor(t, dtype=torch.float32)
        if t.is_cuda:
            t = _lib.cuda_f32(t, name, n)
            if keep is not None:
                keep.append(t)
            setattr(cam, dfield, t.data_ptr())
        else:
            flat = t.detach().float().reshape(-1)
            if flat.numel() != n:
                raise RuntimeError("%s has %d elements, expected %d" % (name, flat.numel(), n))
            getattr(cam, field)[:] = flat.tolist()
    return cam


# the camera tensors a backward can differentiate: name in the settings, offset in the C-ABI's 35-float camera gradient
# (g4d_context_set_camera_grad), element count
_CAM_FIELDS = (("viewmatrix", 0, 16), ("projmatrix", 16, 16), ("campos", 32, 3))


def camera_grad_leaves(rss):
    """The camera tensors of the settings ``rss`` that take a gradient (grad mode on, ``requires_grad``): ``spec``, one
    (camera, field) pair per tensor, and the tensors.  Both are empty when there is none."""
    if not torch.is_grad_enabled():
        return (), ()
    spec, leaves = [], []
    for i, rs in enumerate(rss):
        for f, (name, _, _) in enumerate(_CAM_FIELDS):
            t = getattr(rs, name)
            if torch.is_tensor(t) and t.requires_grad:
                spec.append((i, f))
                leaves.append(t)
    return tuple(spec), tuple(leaves)


class CameraGradSinks:
    """One [k, 35] float32 device buffer whose row i the backward on context ``ctxs[i]`` overwrites with its camera's
    gradient, for the cameras named in ``spec``; with ``time``, one device float that the backward on ``ctxs[0]``
    overwrites with dL/d(time) (g4d_context_set_time_grad); ``depths[i]``, when given and not None, the gradient of camera
    i's depth image (contiguous fp32 CUDA, [H*W]) that the backward on ``ctxs[i]`` takes (g4d_context_set_depth_grad).  The
    contexts' pointers are cleared again on exit (they return to a pool)."""

    def __init__(self, spec, ctxs, dev, time=False, depths=()):
        self.cams = sorted({i for i, _ in spec})
        self.ctxs = ctxs
        self.buf = torch.empty(len(ctxs), 35, device=dev, dtype=torch.float32) if spec else None
        self.tbuf = torch.empty(1, device=dev, dtype=torch.float32) if time else None
        self.depths = [(i, d) for i, d in enumerate(depths) if d is not None]

    def __enter__(self):
        for i in self.cams:
            self.ctxs[i].set_camera_grad(self.buf[i].data_ptr())
        if self.tbuf is not None:
            self.ctxs[0].set_time_grad(self.tbuf.data_ptr())
        for i, d in self.depths:
            self.ctxs[i].set_depth_grad(d.data_ptr())
        return self

    def __exit__(self, *exc):
        for i in self.cams:
            self.ctxs[i].set_camera_grad(None)
        if self.tbuf is not None:
            self.ctxs[0].set_time_grad(None)
        for i, _ in self.depths:
            self.ctxs[i].set_depth_grad(None)
        return False

    def grads(self, spec, metas):
        """The gradient of each camera tensor of ``spec`` in its (shape, dtype, device), ``metas`` (``tensor_meta``)."""
        return tuple(self.buf[i, off:off + n].reshape(shape).to(device=device, dtype=dtype)
                     for (i, f), (shape, dtype, device) in zip(spec, metas) for _, off, n in (_CAM_FIELDS[f],))

    def time_grad(self, meta):
        """dL/d(time) in the time tensor's (shape, dtype, device), ``meta`` (one entry of ``tensor_meta``)."""
        shape, dtype, device = meta
        return self.tbuf.reshape(shape).to(device=device, dtype=dtype)


def tensor_meta(tensors):
    return tuple((t.shape, t.dtype, t.device) for t in tensors)


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


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, opacities, scales, rotations, raster_settings, differentiable_depth, cam_spec,
                *cam_leaves):
        lib = _lib.load()
        dev = means3D.device
        n = means3D.shape[0]
        m3 = _lib.cuda_f32(means3D, "means3D", n * 3)
        m = _lib.sh_coeffs(sh, n, "shs")
        _lib.check_sh_degree(m, int(raster_settings.sh_degree))
        shc = _lib.cuda_f32(sh, "shs", n * 3 * m)
        op = _lib.cuda_f32(opacities, "opacities", n)
        sc = _lib.cuda_f32(scales, "scales", n * 3)
        ro = _lib.cuda_f32(rotations, "rotations", n * 4)
        H, W = int(raster_settings.image_height), int(raster_settings.image_width)
        color = torch.empty(3, H, W, device=dev, dtype=torch.float32)
        depth = torch.empty(1, H, W, device=dev, dtype=torch.float32)
        radii = torch.empty(n, device=dev, dtype=torch.int32)
        keep = []
        cam = camera_from_settings(raster_settings, keep=keep, sh_coeffs=m)
        with torch.cuda.device(dev):
            lease = _ContextLease(_lib.workspace_of(dev))
            _lib.check(lib.g4d_rasterize_forward(lease.ctx.handle, C.byref(cam), n, m3.data_ptr(), shc.data_ptr(), op.data_ptr(),
                                                 sc.data_ptr(), ro.data_ptr(), color.data_ptr(), depth.data_ptr(),
                                                 radii.data_ptr(), _lib.stream_of(dev)), "g4d_rasterize_forward")
        ctx.raster_settings = raster_settings
        ctx.cam_spec, ctx.cam_meta = cam_spec, tensor_meta(cam_leaves)
        ctx.lease = lease
        ctx.n, ctx.m = n, m
        ctx.save_for_backward(m3, shc, op, sc, ro)
        ctx.mark_non_differentiable(*((radii,) if differentiable_depth else (radii, depth)))
        ctx.set_materialize_grads(False)         # a depth image outside the loss arrives as None: no depth gradient is set
        return color, radii, depth

    @staticmethod
    def backward(ctx, grad_color, _grad_radii, grad_depth):
        lib = _lib.load()
        m3, shc, op, sc, ro = ctx.saved_tensors
        dev = m3.device
        n = ctx.n
        rs = ctx.raster_settings
        hw = int(rs.image_height) * int(rs.image_width)
        if grad_color is None:      # a depth-only loss: the backward takes an image gradient
            grad_color = torch.zeros(3 * hw, device=dev)
        gcol = _lib.cuda_f32(grad_color, "grad_out_color", 3 * hw)
        gdep = _lib.cuda_f32(grad_depth, "grad_out_depth", hw)
        g_means3D = torch.empty(n, 3, device=dev)
        g_means2D = torch.empty(n, 3, device=dev)
        g_sh = torch.empty(n, ctx.m, 3, device=dev)
        g_op = torch.empty(n, 1, device=dev)
        g_sc = torch.empty(n, 3, device=dev)
        g_ro = torch.empty(n, 4, device=dev)
        keep = []
        cam = camera_from_settings(rs, keep=keep, sh_coeffs=ctx.m)
        lease = ctx.lease
        if lease is None or lease.ctx is None:
            raise RuntimeError("rasterizer backward called twice (context already released)")
        sinks = CameraGradSinks(ctx.cam_spec, [lease.ctx], dev, depths=(gdep,))
        with torch.cuda.device(dev), sinks:
            _lib.check(lib.g4d_rasterize_backward(lease.ctx.handle, C.byref(cam), n, m3.data_ptr(), shc.data_ptr(), op.data_ptr(),
                                                  sc.data_ptr(), ro.data_ptr(), gcol.data_ptr(), g_means3D.data_ptr(),
                                                  g_means2D.data_ptr(), g_sh.data_ptr(), g_op.data_ptr(), g_sc.data_ptr(),
                                                  g_ro.data_ptr(), _lib.stream_of(dev)), "g4d_rasterize_backward")
        lease.release()
        ctx.lease = None
        cam_grads = sinks.grads(ctx.cam_spec, ctx.cam_meta) if ctx.cam_spec else ()
        return (g_means3D, g_means2D, g_sh, g_op, g_sc, g_ro, None, None, None) + cam_grads


class GaussianRasterizer(nn.Module):
    """differentiable_depth: the depth image it returns takes a gradient too (render() and render_cameras() render theirs
    so).  Off by default the depth is a tensor without grad, as diff_gaussian_rasterization's callers read it (a tensor
    that requires grad refuses .numpy())."""

    def __init__(self, raster_settings: GaussianRasterizationSettings, differentiable_depth: bool = False):
        super().__init__()
        self.raster_settings = raster_settings
        self.differentiable_depth = bool(differentiable_depth)

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
        # the settings' viewmatrix / projmatrix / campos that require grad join the autograd graph as extra inputs
        cam_spec, cam_leaves = camera_grad_leaves((rs,))
        return _RasterizeGaussians.apply(means3D, means2D, shs, opacities, scales, rotations, rs, self.differentiable_depth,
                                         cam_spec, *cam_leaves)
