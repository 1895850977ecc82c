"""Helpers for the time-gradient tests: the fp64 chain oracle deform_ref -> dense render with the time as a leaf, per
Gaussian, and a numpy restatement of the kernel's formula for dL/dt from the gradients of the collapsed time rows
(DESIGN.md §4.11)."""
import numpy as np
import torch

from oracle import deform_ref as dr
from oracle.dense_ref import dense_render

SCENE_LEAVES = ("xyz", "scaling", "rotation", "opacity", "features_dc", "features_rest")


def texel_row_fraction(t, T):
    """fractional part of t's position on the time axis of T rows, (t + 1) / 2 * (T - 1)"""
    x = (t + 1.0) / 2.0 * (T - 1)
    return x - np.floor(x)


def oracle_time_grads(cfg, prm, scene, cd, t, cot):
    """dL/d(t_g) [N] fp64 of L = sum(cot * colour) for the chain deform_ref -> activations -> dense render, every Gaussian
    at its own copy t_g = t of the time: their sum is dL/dt, the sum of their magnitudes the scale a comparison of dL/dt
    is judged against (cancellation cannot make it small)."""
    p64 = prm.to(torch.float64)
    lv = {k: scene[k].detach().double().cpu() for k in SCENE_LEAVES}
    n = lv["xyz"].shape[0]
    tt = torch.full((n,), float(t), dtype=torch.float64, requires_grad=True)
    shs = torch.cat([lv["features_dc"], lv["features_rest"]], dim=1)
    pts, sc, rot, op, sh = dr.deform_forward(cfg, p64, lv["xyz"], lv["scaling"], lv["rotation"], lv["opacity"], shs, tt)
    s, r, o = dr.activate(sc, rot, op)
    out = dense_render(cd, pts, s, r, o, sh)
    (out["color"] * cot.double()).sum().backward()
    return tt.grad


def time_grad_from_rows(planes, row_grads, t, T):
    """The kernel's formula: dL/dt = gmul * sum over (level l, time axis a, x, channel e) of the collapsed row's gradient
    times (P[i1] - P[i0]), P the (a, t) plane of level l ([C, T, W] numpy), row_grads[l][a] its row's gradient [C, W].  i0
    = floor of the row coordinate (a time on a texel row takes the row above it), gmul = 0 at and past the border."""
    hi = T - 1
    x = (t + 1.0) / 2.0 * hi
    gmul = 0.5 * hi if 0.0 < x < hi else 0.0
    x = min(max(x, 0.0), hi)
    i0 = int(np.floor(x))
    i1 = min(i0 + 1, T - 1)
    total = 0.0
    for lvl_p, lvl_g in zip(planes, row_grads):
        for P, g in zip(lvl_p, lvl_g):
            total += float((g * (P[:, i1, :] - P[:, i0, :])).sum())
    return gmul * total
