"""Helpers for the alpha-map tests: the fp64 dense oracle with a differentiable alpha image, and the C oracle's alpha image and
gradients of a loss on the colour, depth and alpha images.

The alpha image is A = 1 - T with T the transmittance the blend leaves behind the pixel's colour instances.  T is also the
first colour channel of the same scene with colour 0 and background (1, 0, 0), so both oracles get A from their colour path:
  * dense_alpha is 1 - final_T of oracle/dense_ref.py (fp64 autograd then differentiates A in the Gaussians and the camera);
  * oracle_backward runs the C oracle's hand-derived colour backward (oracle/raster_ref.c) with rgb = 0, bg = (1, 0, 0) and
    the cotangent -dL/dA on channel 0: its mean2D / conic / opacity gradients are the alpha image's, and the per-Gaussian
    backward carries them to the means, scales and rotations."""
import dataclasses

import numpy as np
import torch

from oracle import raster_ref as rr
from oracle.dense_ref import dense_render
import util_depth_grad as udg

NAMES = udg.NAMES


def oracle_alpha(fwd):
    """[1,H,W] float32 alpha image of a C-oracle forward (rr.rasterize_forward's dict)"""
    return (np.float32(1.0) - fwd["final_T"].astype(np.float32))[None]


def dense_alpha(cd, means3D, scales, rots, opac, pix_offset=None):
    """[1,H,W] fp64 alpha image of the dense oracle, differentiable; pix_offset: dense_render's screen-space leaf"""
    n = means3D.shape[0]
    shs = torch.zeros(n, 16, 3, dtype=means3D.dtype)
    return 1.0 - dense_render(cd, means3D, scales, rots, opac, shs, pix_offset=pix_offset)["final_T"][None]


def dense_grads(cd, ins, dL_dcolor, dL_ddepth, dL_dalpha, cam_keys=()):
    """fp64 gradients of <dL_dcolor, colour> + <dL_ddepth, depth> + <dL_dalpha, alpha> (any cotangent may be None) w.r.t. the
    five inputs (fp32 arrays or tensors), means2D (NDC units, [N,2]) and the camera tensors named in cam_keys"""
    x = [torch.as_tensor(np.asarray(a, np.float64)).clone().requires_grad_(True) for a in ins]
    leaves = {k: torch.as_tensor(np.asarray(cd[k], np.float64)).clone().requires_grad_(True) for k in cam_keys}
    c = dict(cd, **leaves)
    off = torch.zeros(len(x[0]), 2, dtype=torch.float64, requires_grad=True)
    loss = torch.zeros((), dtype=torch.float64)
    if dL_dcolor is not None:
        loss = loss + (dense_render(c, *x, pix_offset=off)["color"] * torch.as_tensor(dL_dcolor).double()).sum()
    if dL_ddepth is not None:
        d = udg.dense_depth(c, *x[:4], pix_offset=off)
        loss = loss + (d * torch.as_tensor(dL_ddepth).double().reshape(d.shape)).sum()
    if dL_dalpha is not None:
        a = dense_alpha(c, *x[:4], pix_offset=off)
        loss = loss + (a * torch.as_tensor(dL_dalpha).double().reshape(a.shape)).sum()
    loss.backward()
    zero = lambda t: torch.zeros_like(t) if t.grad is None else t.grad
    g = {nm: zero(t).numpy() for nm, t in zip(NAMES, x)}
    g["means2D"] = zero(off).numpy() * np.array([0.5 * cd["W"], 0.5 * cd["H"]])
    for k, t in leaves.items():
        g[k] = zero(t).numpy().reshape(-1)
    return g


def _transmittance_cam(rc):
    z = rr.RefCam.from_buffer_copy(rc)
    z.bg[:] = [1.0, 0.0, 0.0]
    return z


def oracle_backward(rc, ins, fwd, dL_dcolor, dL_ddepth, dL_dalpha):
    """The C oracle's gradients (rr.rasterize_backward's dict, fp32 arithmetic) of <dL_dcolor, colour> + <dL_ddepth, depth>
    + <dL_dalpha, alpha>; a None cotangent is a term outside the loss.  Key "depth": dL/dz [N] (util_depth_grad)."""
    H, W = rc.H, rc.W
    g = udg.oracle_backward(rc, ins, fwd, dL_dcolor, dL_ddepth)
    if dL_dalpha is None:
        return g
    ins = [np.ascontiguousarray(np.asarray(a, np.float32)) for a in ins]
    m3, sc, ro, op, sh = ins
    n = len(m3)
    pr, bn = fwd["proj"], fwd["bin"]
    prt = dataclasses.replace(pr, rgb=np.zeros((n, 3), np.float32))
    cot = np.zeros((3, H, W), np.float32)
    cot[0] = -np.asarray(dL_dalpha, np.float32).reshape(H, W)
    gm2, gcon, gop, _ = rr.blend_backward(_transmittance_cam(rc), prt, bn, fwd["final_T"], fwd["n_contrib"], cot)
    gm3, gsc, gro, _ = rr.preprocess_backward(rc, m3, sc, ro, sh, pr, gm2, gcon, np.zeros((n, 3), np.float32))
    g["means3D"] += gm3
    g["scales"] += gsc
    g["rots"] += gro
    g["opacities"] += gop.reshape(n, 1)
    g["means2D"][:, :2] += gm2
    g["conic"] += gcon
    return g


def oracle_time_grads(cfg, prm, scene, cd, t, dL_dcolor, dL_dalpha):
    """dL/d(t_g) [N] fp64 of L = <dL_dcolor, colour> + <dL_dalpha, alpha> for the chain deform_ref -> activations -> dense
    render, every Gaussian at its own copy t_g = t of the time: their sum is dL/dt"""
    from oracle import deform_ref as dr
    keys = ("xyz", "scaling", "rotation", "opacity", "features_dc", "features_rest")
    p64 = prm.to(torch.float64)
    lv = {k: scene[k].detach().double().cpu() for k in keys}
    n = lv["xyz"].shape[0]
    tt = torch.full((n,), float(t), dtype=torch.float64, requires_grad=True)
    shs = torch.cat([lv["features_dc"], lv["features_rest"]], dim=1)
    pts, sc, rot, op, sh = dr.deform_forward(cfg, p64, lv["xyz"], lv["scaling"], lv["rotation"], lv["opacity"], shs, tt)
    s, r, o = dr.activate(sc, rot, op)
    loss = (dense_alpha(cd, pts, s, r, o) * torch.as_tensor(dL_dalpha).double()).sum()
    if dL_dcolor is not None:
        loss = loss + (dense_render(cd, pts, s, r, o, sh)["color"] * torch.as_tensor(dL_dcolor).double()).sum()
    loss.backward()
    return tt.grad
