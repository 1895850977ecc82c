"""Loss terms either side of the render path (SURVEY.md 8f N2), same names and argument meaning as the reference:

    l1_loss(network_output, gt)                    <- utils/loss_utils.py:20-21
    ssim(img1, img2, window_size=11, size_average=True)   <- utils/loss_utils.py:37-66
    compute_regulation(deformation, time_smoothness_weight, l1_time_planes_weight, plane_tv_weight)
                                                   <- GaussianModel.compute_regulation, scene/gaussian_model.py:538-577

Each is ONE kernel for the value and ONE for the gradient (the reference: ~8 / ~25 / ~60 ATen launches), through the
C-ABI of libg4d.so.  CUDA tensors only; there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib


class _L1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, out, gt):
        if out.shape != gt.shape:
            raise RuntimeError("l1_loss: shapes differ: %s vs %s" % (tuple(out.shape), tuple(gt.shape)))
        a, b = _lib.cuda_f32(out, "network_output"), _lib.cuda_f32(gt, "gt")
        n = a.numel()
        loss = torch.zeros((), device=a.device, dtype=torch.float32)
        with torch.cuda.device(a.device):
            _lib.check(_lib.load().g4d_l1_loss(_lib.workspace_of(a.device).handle, a.data_ptr(), b.data_ptr(), n,
                                               1.0 / max(n, 1), loss.data_ptr(), _lib.stream_of(a.device)), "g4d_l1_loss")
        ctx.save_for_backward(a, b)
        ctx.needs_gt = ctx.needs_input_grad[1]
        return loss

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        n = a.numel()
        up = _lib.cuda_f32(g, "grad_output")
        grad = torch.empty_like(a)
        with torch.cuda.device(a.device):
            _lib.check(_lib.load().g4d_l1_loss_backward(_lib.workspace_of(a.device).handle, a.data_ptr(), b.data_ptr(), n,
                                                        1.0 / max(n, 1), up.data_ptr(), grad.data_ptr(), _lib.stream_of(a.device)),
                       "g4d_l1_loss_backward")
        return grad, (-grad if ctx.needs_gt else None)


def l1_loss(network_output: torch.Tensor, gt: torch.Tensor) -> torch.Tensor:
    return _L1.apply(network_output, gt)


class _SSIM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img1, img2):
        a, b = _lib.cuda_f32(img1, "img1"), _lib.cuda_f32(img2, "img2")
        if a.shape != b.shape or a.dim() < 3:
            raise RuntimeError("ssim: expects two [..., C, H, W] tensors of the same shape")
        H, W = int(a.shape[-2]), int(a.shape[-1])
        ch = a.numel() // (H * W)
        need = any(ctx.needs_input_grad)
        saved = torch.empty(3 * a.numel(), device=a.device, dtype=torch.float32) if need else None
        val = torch.zeros((), device=a.device, dtype=torch.float32)
        with torch.cuda.device(a.device):
            _lib.check(_lib.load().g4d_ssim(_lib.workspace_of(a.device).handle, a.data_ptr(), b.data_ptr(), ch, H, W,
                                            1.0 / max(a.numel(), 1), val.data_ptr(), saved.data_ptr() if saved is not None else None,
                                            _lib.stream_of(a.device)), "g4d_ssim")
        ctx.save_for_backward(a, b, saved)
        return val

    @staticmethod
    def backward(ctx, g):
        a, b, saved = ctx.saved_tensors
        if ctx.needs_input_grad[1]:
            raise NotImplementedError("ssim: gradient w.r.t. the second image (the ground truth) is not provided")
        H, W = int(a.shape[-2]), int(a.shape[-1])
        ch = a.numel() // (H * W)
        up = _lib.cuda_f32(g, "grad_output")
        grad = torch.empty_like(a)
        with torch.cuda.device(a.device):
            _lib.check(_lib.load().g4d_ssim_backward(_lib.workspace_of(a.device).handle, a.data_ptr(), b.data_ptr(), ch, H, W,
                                                     1.0 / max(a.numel(), 1), up.data_ptr(), saved.data_ptr(), grad.data_ptr(),
                                                     _lib.stream_of(a.device)), "g4d_ssim_backward")
        return grad, None


def ssim(img1: torch.Tensor, img2: torch.Tensor, window_size: int = 11, size_average: bool = True) -> torch.Tensor:
    if window_size != 11 or not size_average:
        raise NotImplementedError("ssim: only window_size=11, size_average=True (the reference's only call: train.py:211)")
    return _SSIM.apply(img1, img2)


class _Regulation(torch.autograd.Function):
    """inputs: the plane parameters (level-major); weights are python floats"""

    @staticmethod
    def forward(ctx, module, w_ts, w_l1, w_tv, *planes):
        keep = []
        prm = module.c_params(keep)
        dev = planes[0].device
        need = any(ctx.needs_input_grad)
        loss = torch.zeros((), device=dev, dtype=torch.float32)
        grads = module.alloc_plane_grads() if need else None
        cg = module.c_plane_grads(grads) if grads is not None else None
        with torch.cuda.device(dev):
            _lib.check(_lib.load().g4d_plane_regulation(_lib.workspace_of(dev).handle, C.byref(prm),
                                                        C.byref(cg) if cg is not None else None, float(w_tv), float(w_ts),
                                                        float(w_l1), None, loss.data_ptr(), _lib.stream_of(dev)),
                       "g4d_plane_regulation")
        ctx.grads = grads
        return loss

    @staticmethod
    def backward(ctx, g):
        grads = ctx.grads
        ctx.grads = None
        # the unit gradients were produced together with the value; scale by the upstream scalar (1 in train.py:210)
        base = grads[0]._base if grads[0]._base is not None else None
        if base is not None:
            base.mul_(g)
        else:
            grads = [x * g for x in grads]
        return (None, None, None, None) + tuple(grads)


def compute_regulation(deformation, time_smoothness_weight: float, l1_time_planes_weight: float, plane_tv_weight: float):
    """plane_tv_weight * _plane_regulation() + time_smoothness_weight * _time_regulation() + l1_time_planes_weight *
    _l1_regulation()  (scene/gaussian_model.py:576-577) for a g4d ``deform_network``."""
    planes = [p for lvl in deformation.deformation_net.grid.grids for p in lvl]
    return _Regulation.apply(deformation, float(time_smoothness_weight), float(l1_time_planes_weight), float(plane_tv_weight),
                             *planes)


def accumulate_regulation(deformation, time_smoothness_weight: float, l1_time_planes_weight: float, plane_tv_weight: float,
                          loss_accum: torch.Tensor | None = None):
    """Training-harness shortcut (no autograd node): adds the regulariser's plane gradients straight into the parameters'
    ``.grad`` (e.g. views of a dp.FlatGradBucket) and its value into ``loss_accum`` -- one launch, no staging buffer."""
    keep = []
    prm = deformation.c_params(keep)
    planes = [p for lvl in deformation.deformation_net.grid.grids for p in lvl]
    for i, p in enumerate(planes):
        if p.grad is None or p.grad.stride() != p.stride() or p.grad.dtype != torch.float32:
            raise RuntimeError("accumulate_regulation: plane %d has no .grad with the parameter's own layout" % i)
    cg = deformation.c_plane_grads([p.grad for p in planes])
    dev = planes[0].device
    with torch.cuda.device(dev):
        _lib.check(_lib.load().g4d_plane_regulation(_lib.workspace_of(dev).handle, C.byref(prm), C.byref(cg),
                                                    float(plane_tv_weight), float(time_smoothness_weight),
                                                    float(l1_time_planes_weight), None,
                                                    loss_accum.data_ptr() if loss_accum is not None else None, _lib.stream_of(dev)),
                   "g4d_plane_regulation")
