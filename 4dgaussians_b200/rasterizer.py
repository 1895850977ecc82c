"""Drop-in for the ``diff_gaussian_rasterization`` module the reference imports
(/root/reference/gaussian_renderer/__init__.py:14; merge_many_4dgs.py:33; scene/dataset_readers.py:485).

Same names, argument meaning and error behaviour as the upstream Python surface (SURVEY.md §8b, App. A.5);
behind it the hand-written sm_90a kernels of libg4d.so through the C-ABI (include/g4d.h).  PyTorch is only
plumbing here: device memory, the current stream, autograd bookkeeping.
"""
from __future__ import annotations

import contextlib
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


def per_view(seq, k):
    """The outputs of a render of k views, or their incoming gradients, in the order its autograd Function returns them:
    (colour images, radii, depth images, alpha images), k of each, and no alpha images unless they are rendered."""
    return seq[:k], seq[k:2 * k], seq[2 * k:3 * k], seq[3 * k:]


@contextlib.contextmanager
def _bound(terms):
    """``terms``: (context, name of its ``set_*`` method, tensor or None).  Inside the block each context points at its
    tensor; on exit, on an exception too, the pointers are cleared again: the contexts return to a pool and must not keep
    reading or writing a tensor that may be freed."""
    done = []
    try:
        for c, setter, t in terms:
            if t is not None:
                getattr(c, setter)(t.data_ptr())
                done.append((c, setter))
        yield
    finally:
        for c, setter in done:
            getattr(c, setter)(None)


class ViewTerms:
    """What the views of one render call, the settings ``rss``, take and give beyond their colour images, and its binding to
    the contexts leased for the call, ``ctxs[i]`` for view i, for the one C-ABI call made inside ``forward`` or ``backward``.

    Forward: each view's depth image and, with ``alpha``, its alpha image (g4d_context_set_alpha_out).  Backward: the depth
    and alpha images' incoming gradients (g4d_context_set_depth_grad / _alpha_grad), the gradient of each camera tensor that
    takes one (``camera_grad_leaves``; g4d_context_set_camera_grad) and, with ``time_leaf``, dL/d(time), which the backward
    on ``ctxs[0]`` writes (g4d_context_set_time_grad).  ``leaves``: the camera tensors, then the time, that the caller
    passes to its autograd Function as inputs."""

    def __init__(self, rss, alpha=False, time_leaf=None):
        self.rss, self.k, self.alpha, self.timed = rss, len(rss), bool(alpha), time_leaf is not None
        self.cam_spec, cam_leaves = camera_grad_leaves(rss)
        self.leaves = cam_leaves + ((time_leaf,) if self.timed else ())
        self.metas = tuple((t.shape, t.dtype, t.device) for t in self.leaves)
        self.cam_sink = self.time_sink = None

    def outputs(self, dev, n):
        """The fp32 images and the int32 radii of n Gaussians of every view, in ``per_view`` order."""
        def images(c):
            return [torch.empty(c, int(rs.image_height), int(rs.image_width), device=dev, dtype=torch.float32) for rs in self.rss]
        return images(3), [torch.empty(n, device=dev, dtype=torch.int32) for _ in self.rss], images(1), \
            images(1) if self.alpha else []

    def forward(self, ctxs, alphas):
        """``with``: the forward on ``ctxs[i]`` also writes view i's alpha image into ``alphas[i]``."""
        return _bound([(c, "set_alpha_out", a) for c, a in zip(ctxs, alphas)])

    def gradients(self, grads, dev):
        """The incoming gradients ``grads`` (``per_view`` order) as contiguous fp32 CUDA buffers: per view its colour, depth
        and alpha gradient, None for one outside the loss -- but with one view the colour gradient is zeros then, since the
        single-camera backward entry points take an image gradient."""
        gcol, _, gdep, galpha = per_view(grads, self.k)
        hw = [int(rs.image_height) * int(rs.image_width) for rs in self.rss]
        gcols = [_lib.cuda_f32(g, "grad_out_color", 3 * p) for g, p in zip(gcol, hw)]
        if self.k == 1 and gcols[0] is None:
            gcols[0] = torch.zeros(3 * hw[0], device=dev, dtype=torch.float32)
        return gcols, [_lib.cuda_f32(g, "grad_out_depth", p) for g, p in zip(gdep, hw)], \
            [_lib.cuda_f32(g, "grad_out_alpha", p) for g, p in zip(galpha, hw)]

    def backward(self, ctxs, dev, depths=(), alphas=()):
        """``with``: the backward on ``ctxs[i]`` takes ``depths[i]`` and ``alphas[i]`` (None: outside the loss) and writes the
        sinks ``leaf_grads`` reads."""
        cams = sorted({i for i, _ in self.cam_spec})
        self.cam_sink = torch.empty(len(ctxs), 35, device=dev, dtype=torch.float32) if cams else None
        self.time_sink = torch.empty(1, device=dev, dtype=torch.float32) if self.timed else None
        return _bound([(ctxs[i], "set_camera_grad", self.cam_sink[i]) for i in cams] +
                      [(ctxs[0], "set_time_grad", self.time_sink)] +
                      [(c, "set_depth_grad", d) for c, d in zip(ctxs, depths)] +
                      [(c, "set_alpha_grad", a) for c, a in zip(ctxs, alphas)])

    def leaf_grads(self):
        """The gradient of each tensor of ``leaves`` in its shape, dtype and device, from the last ``backward``'s sinks."""
        rows = [self.cam_sink[i, off:off + n] for i, f in self.cam_spec for _, off, n in (_CAM_FIELDS[f],)]
        if self.timed:
            rows.append(self.time_sink)
        return tuple(r.reshape(shape).to(device=device, dtype=dtype) for r, (shape, dtype, device) in zip(rows, self.metas))


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
    def forward(ctx, means3D, means2D, sh, opacities, scales, rotations, terms, differentiable_depth, *cam_leaves):
        lib = _lib.load()
        dev = means3D.device
        n = means3D.shape[0]
        rs = terms.rss[0]
        m3 = _lib.cuda_f32(means3D, "means3D", n * 3)
        m = _lib.sh_coeffs(sh, n, "shs")
        _lib.check_sh_degree(m, int(rs.sh_degree))
        shc = _lib.cuda_f32(sh, "shs", n * 3 * m)
        op = _lib.cuda_f32(opacities, "opacities", n)
        sc = _lib.cuda_f32(scales, "scales", n * 3)
        ro = _lib.cuda_f32(rotations, "rotations", n * 4)
        (color,), (radii,), (depth,), alphas = terms.outputs(dev, n)
        keep = []
        cam = camera_from_settings(rs, keep=keep, sh_coeffs=m)
        with torch.cuda.device(dev):
            lease = _ContextLease(_lib.workspace_of(dev))
            with terms.forward([lease.ctx], alphas):
                _lib.check(lib.g4d_rasterize_forward(lease.ctx.handle, C.byref(cam), n, m3.data_ptr(), shc.data_ptr(),
                                                     op.data_ptr(), sc.data_ptr(), ro.data_ptr(), color.data_ptr(),
                                                     depth.data_ptr(), radii.data_ptr(), _lib.stream_of(dev)),
                           "g4d_rasterize_forward")
        ctx.terms, ctx.lease = terms, lease
        ctx.n, ctx.m = n, m
        ctx.save_for_backward(m3, shc, op, sc, ro)
        ctx.mark_non_differentiable(*((radii,) if differentiable_depth else (radii, depth)))
        # a depth or alpha image outside the loss arrives as None: no depth or alpha gradient is set
        ctx.set_materialize_grads(False)
        return (color, radii, depth, *alphas)

    @staticmethod
    def backward(ctx, *grads):
        lib = _lib.load()
        m3, shc, op, sc, ro = ctx.saved_tensors
        dev = m3.device
        n, terms = ctx.n, ctx.terms
        gcols, gdeps, galphas = terms.gradients(grads, dev)
        g_means3D = torch.empty(n, 3, device=dev)
        g_means2D = torch.empty(n, 3, device=dev)
        g_sh = torch.empty(n, ctx.m, 3, device=dev)
        g_op = torch.empty(n, 1, device=dev)
        g_sc = torch.empty(n, 3, device=dev)
        g_ro = torch.empty(n, 4, device=dev)
        keep = []
        cam = camera_from_settings(terms.rss[0], keep=keep, sh_coeffs=ctx.m)
        lease = ctx.lease
        if lease is None or lease.ctx is None:
            raise RuntimeError("rasterizer backward called twice (context already released)")
        with torch.cuda.device(dev), terms.backward([lease.ctx], dev, gdeps, galphas):
            _lib.check(lib.g4d_rasterize_backward(lease.ctx.handle, C.byref(cam), n, m3.data_ptr(), shc.data_ptr(), op.data_ptr(),
                                                  sc.data_ptr(), ro.data_ptr(), gcols[0].data_ptr(), g_means3D.data_ptr(),
                                                  g_means2D.data_ptr(), g_sh.data_ptr(), g_op.data_ptr(), g_sc.data_ptr(),
                                                  g_ro.data_ptr(), _lib.stream_of(dev)), "g4d_rasterize_backward")
        lease.release()
        ctx.lease = None
        return (g_means3D, g_means2D, g_sh, g_op, g_sc, g_ro, None, None) + terms.leaf_grads()


class GaussianRasterizer(nn.Module):
    """differentiable_depth: the depth image it returns takes a gradient too (render() and render_cameras() render theirs
    so).  Off by default the depth is a tensor without grad, as diff_gaussian_rasterization's callers read it (a tensor
    that requires grad refuses .numpy()).
    return_alpha: return (color, radii, depth, alpha), alpha [1,H,W] the accumulated opacity 1 - T of each pixel, which
    takes a gradient; off by default the result is diff_gaussian_rasterization's (color, radii, depth)."""

    def __init__(self, raster_settings: GaussianRasterizationSettings, differentiable_depth: bool = False,
                 return_alpha: bool = False):
        super().__init__()
        self.raster_settings = raster_settings
        self.differentiable_depth = bool(differentiable_depth)
        self.return_alpha = bool(return_alpha)

    def markVisible(self, positions):
        raise NotImplementedError("markVisible is not used by 4DGaussians (SURVEY.md §8b) and is not part of the g4d path")

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None):
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        if colors_precomp is not None or cov3D_precomp is not None:
            raise NotImplementedError("colors_precomp / cov3D_precomp are dead paths in the reference "
                                      "(gaussian_renderer/__init__.py:74-78,105-116) and are not provided")
        # the settings' viewmatrix / projmatrix / campos that require grad join the autograd graph as extra inputs
        terms = ViewTerms((self.raster_settings,), self.return_alpha)
        return _RasterizeGaussians.apply(means3D, means2D, shs, opacities, scales, rotations, terms, self.differentiable_depth,
                                         *terms.leaves)
