"""Helpers for the depth-gradient tests: the fp64 dense oracle with a differentiable depth image, and the C oracle's gradients
of a loss on the colour image and the depth image.

The depth image is D = sum_i w_i z_i with the colour's weights w_i = alpha_i T_i and z_i the Gaussian's view-space depth (no
background term).  That is the first colour channel of the same scene with colour z_i and a black background, so both oracles
get it from their colour path:
  * dense_depth renders, with oracle/dense_ref.py, a scene of SH degree 0 whose coefficient makes the colour exactly z (fp64
    autograd then differentiates D in the Gaussians and in the view matrix);
  * oracle_backward runs the C oracle's hand-derived colour backward (oracle/raster_ref.c) with rgb = (z, 0, 0), bg = 0 and the
    depth cotangent on channel 0: its rgb gradient is dL/dz_i, its mean2D / conic / opacity gradients are the depth's; the
    per-Gaussian backward adds dL/dz_i (view[2], view[6], view[10]) to the mean (z is row 2 of the view transform)."""
import dataclasses

import numpy as np
import torch

from oracle import raster_ref as rr
from oracle.dense_ref import C0, dense_render

NAMES = ("means3D", "scales", "rots", "opacities", "shs")


def view_depth(view, means3D):
    """z of every Gaussian: row 2 of the view transform (xform4x3), differentiable in both"""
    v = torch.as_tensor(view, dtype=means3D.dtype).reshape(16)
    return v[2] * means3D[:, 0] + v[6] * means3D[:, 1] + v[10] * means3D[:, 2] + v[14]


def dense_depth(cd, means3D, scales, rots, opac, pix_offset=None, detach_z=False):
    """[1,H,W] fp64 depth image of the dense oracle, differentiable; pix_offset: dense_render's screen-space leaf; detach_z:
    z as a constant (only the weights move)"""
    z = view_depth(cd["view"], means3D)
    if detach_z:
        z = z.detach()
    n = means3D.shape[0]
    dc = torch.stack([(z - 0.5) / C0, torch.zeros_like(z), torch.zeros_like(z)], dim=-1).reshape(n, 1, 3)
    shs = torch.cat([dc, torch.zeros(n, 15, 3, dtype=means3D.dtype)], dim=1)
    return dense_render(dict(cd, sh_degree=0, bg=[0.0, 0.0, 0.0]), means3D, scales, rots, opac, shs,
                        pix_offset=pix_offset)["color"][0:1]


def dense_grads(cd, ins, dL_dcolor, dL_ddepth, cam_keys=()):
    """fp64 gradients of <dL_dcolor, colour> + <dL_ddepth, depth> (either cotangent may be None) w.r.t. the five inputs (ins:
    fp32 arrays or tensors), means2D (NDC units, [N,2]) and the camera tensors named in cam_keys ("view", "proj", "campos")"""
    x = [torch.as_tensor(np.asarray(a, np.float64)).clone().requires_grad_(True) for a in ins]
    leaves = {k: torch.as_tensor(np.asarray(cd[k], np.float64)).clone().requires_grad_(True) for k in cam_keys}
    c = dict(cd, **leaves)
    off = torch.zeros(len(x[0]), 2, dtype=torch.float64, requires_grad=True)
    loss = torch.zeros((), dtype=torch.float64)
    if dL_dcolor is not None:
        loss = loss + (dense_render(c, *x, pix_offset=off)["color"] * torch.as_tensor(dL_dcolor).double()).sum()
    if dL_ddepth is not None:
        d = dense_depth(c, *x[:4], pix_offset=off)
        loss = loss + (d * torch.as_tensor(dL_ddepth).double().reshape(d.shape)).sum()
    loss.backward()
    zero = lambda t: torch.zeros_like(t) if t.grad is None else t.grad
    g = {nm: zero(t).numpy() for nm, t in zip(NAMES, x)}
    g["means2D"] = zero(off).numpy() * np.array([0.5 * cd["W"], 0.5 * cd["H"]])
    for k, t in leaves.items():
        g[k] = zero(t).numpy().reshape(-1)
    return g


def _black(rc):
    z = rr.RefCam.from_buffer_copy(rc)
    z.bg[:] = [0.0, 0.0, 0.0]
    return z


def oracle_backward(rc, ins, fwd, dL_dcolor, dL_ddepth):
    """The C oracle's gradients (rr.rasterize_backward's dict, fp32 arithmetic) of <dL_dcolor, colour> + <dL_ddepth, depth>;
    dL_dcolor None: a depth-only loss.  Extra key "depth": dL/dz [N]."""
    H, W = rc.H, rc.W
    ins = [np.ascontiguousarray(np.asarray(a, np.float32)) for a in ins]
    m3, sc, ro, op, sh = ins
    dc = np.zeros((3, H, W), np.float32) if dL_dcolor is None else np.asarray(dL_dcolor, np.float32)
    g = rr.rasterize_backward(rc, *ins, fwd, dc)
    n = len(m3)
    g = {k: v.astype(np.float64) for k, v in g.items()}
    g["depth"] = np.zeros(n)
    if dL_ddepth is None:
        return g
    pr, bn = fwd["proj"], fwd["bin"]
    zero = np.zeros(n, np.float32)
    prz = dataclasses.replace(pr, rgb=np.ascontiguousarray(np.stack([pr.depth, zero, zero], axis=1)))
    cot = np.zeros((3, H, W), np.float32)
    cot[0] = np.asarray(dL_ddepth, np.float32).reshape(H, W)
    gm2, gcon, gop, grgb = rr.blend_backward(_black(rc), prz, bn, fwd["final_T"], fwd["n_contrib"], cot)
    g_z = np.where(pr.radii > 0, grgb[:, 0], 0.0).astype(np.float32)
    gm3, gsc, gro, _ = rr.preprocess_backward(rc, m3, sc, ro, sh, pr, gm2, gcon, np.zeros((n, 3), np.float32))
    v = np.asarray(rc.view, np.float64)
    gm3 = gm3.astype(np.float64) + g_z[:, None].astype(np.float64) * v[[2, 6, 10]][None, :]
    g["means3D"] += gm3
    g["scales"] += gsc
    g["rots"] += gro
    g["opacities"] += gop.reshape(n, 1)
    g["means2D"][:, :2] += gm2
    g["conic"] += gcon
    g["depth"] = g_z.astype(np.float64)
    return g


def view_depth_terms(means3D, g_z):
    """[16] the part of dL/d view that reaches it through z directly: view[2, 6, 10, 14] get sum_i g_z_i (x_i, y_i, z_i, 1)"""
    m = np.asarray(means3D, np.float64)
    g = np.zeros(16)
    g[[2, 6, 10]] = (np.asarray(g_z, np.float64)[:, None] * m).sum(axis=0)
    g[14] = float(np.sum(g_z))
    return g


def oracle_time_grads(cfg, prm, scene, cd, t, dL_dcolor, dL_ddepth):
    """dL/d(t_g) [N] fp64 of L = <dL_dcolor, colour> + <dL_ddepth, depth> for the chain deform_ref -> activations -> dense
    render, every Gaussian at its own copy t_g = t of the time (as util_time_grad.oracle_time_grads): their sum is dL/dt"""
    from oracle import deform_ref as dr
    keys = ("xyz", "scaling", "rotation", "opacity", "features_dc", "features_rest")
    p64 = prm.to(torch.float64)
    lv = {k: scene[k].detach().double().cpu() for k in keys}
    n = lv["xyz"].shape[0]
    tt = torch.full((n,), float(t), dtype=torch.float64, requires_grad=True)
    shs = torch.cat([lv["features_dc"], lv["features_rest"]], dim=1)
    pts, sc, rot, op, sh = dr.deform_forward(cfg, p64, lv["xyz"], lv["scaling"], lv["rotation"], lv["opacity"], shs, tt)
    s, r, o = dr.activate(sc, rot, op)
    loss = (dense_depth(cd, pts, s, r, o) * torch.as_tensor(dL_ddepth).double()).sum()
    if dL_dcolor is not None:
        loss = loss + (dense_render(cd, pts, s, r, o, sh)["color"] * torch.as_tensor(dL_dcolor).double()).sum()
    loss.backward()
    return tt.grad
