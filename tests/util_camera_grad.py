"""Helpers for the camera-gradient tests: the fp64 dense oracle with the camera tensors as leaves, a torch restatement of
the reference's pose -> matrices chain, central differences, and the threshold-pixel rule fixed before any comparison."""
import math

import numpy as np
import torch

from oracle.dense_ref import NEAR_CULL, dense_render

CAM_KEYS = ("view", "proj", "campos")
# elements of view / proj the forward reads (xform4x3 rows 0..2; clip rows x, y, w): the others have zero gradient
VIEW_READ = [i for i in range(16) if i % 4 != 3]
PROJ_READ = [i for i in range(16) if i % 4 != 2]


def dense_camera_grads(cd, inputs, cot):
    """(color [3,H,W], {view, proj, campos: fp64 gradient of sum(cot * color)}) of the dense oracle; cd: a dense_ref camera
    dict, inputs: (means3D, scales, rots, opac, shs) in fp64."""
    leaves = {k: torch.as_tensor(np.asarray(cd[k], np.float64)).clone().requires_grad_(True) for k in CAM_KEYS}
    c = dict(cd, **leaves)
    out = dense_render(c, *[t.detach().double() for t in inputs])
    (out["color"] * cot.double()).sum().backward()
    # (at SH degree 0 the colour does not read campos: no gradient reaches it)
    return out, {k: torch.zeros(leaves[k].numel(), dtype=torch.float64) if leaves[k].grad is None else leaves[k].grad.reshape(-1)
                 for k in CAM_KEYS}


def central_differences(f, x, eps):
    """d f / d x for every element of the fp64 vector x (f: x -> scalar), by central differences of step eps."""
    g = torch.zeros_like(x)
    for i in range(x.numel()):
        xp, xm = x.clone(), x.clone()
        xp[i] += eps
        xm[i] -= eps
        g[i] = (f(xp) - f(xm)) / (2 * eps)
    return g


def world_view(R, T):
    """getWorld2View2(R, T) of utils/graphics_utils.py (translate 0, scale 1), transposed as scene/cameras.py stores it:
    Rt = [[R^T, T], [0, 1]], world_view_transform = Rt^T."""
    top = torch.cat([R.t(), T.reshape(3, 1)], dim=1)
    bottom = torch.cat([torch.zeros(1, 3, dtype=R.dtype, device=R.device), torch.ones(1, 1, dtype=R.dtype, device=R.device)], 1)
    return torch.cat([top, bottom], dim=0).t()


def projection(znear, zfar, fovx, fovy, dtype=torch.float64, device="cpu"):
    """getProjectionMatrix of utils/graphics_utils.py (z_sign = 1), transposed as scene/cameras.py stores it."""
    tanx, tany = math.tan(fovx / 2), math.tan(fovy / 2)
    P = torch.zeros(4, 4, dtype=dtype, device=device)
    P[0, 0] = 1.0 / tanx
    P[1, 1] = 1.0 / tany
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P.t()


def camera_tensors(R, T, fovx, fovy, znear=0.01, zfar=100.0):
    """(world_view_transform, full_proj_transform, camera_center) from R, T as scene/cameras.py builds them."""
    wv = world_view(R, T)
    full = wv @ projection(znear, zfar, fovx, fovy, dtype=R.dtype, device=R.device)
    return wv, full, torch.linalg.inv(wv)[3, :3]


def rodrigues(w):
    """exp of the skew matrix of the axis-angle vector w [3] (differentiable, also at w = 0 to first order)."""
    th2 = (w * w).sum()
    K = torch.zeros(3, 3, dtype=w.dtype, device=w.device)
    K[0, 1], K[0, 2], K[1, 0], K[1, 2], K[2, 0], K[2, 1] = -w[2], w[1], w[2], -w[0], -w[1], w[0]
    th = torch.sqrt(th2 + 1e-30)
    a = torch.where(th2 > 1e-12, torch.sin(th) / th, 1.0 - th2 / 6.0)
    b = torch.where(th2 > 1e-12, (1.0 - torch.cos(th)) / (th2 + 1e-30), 0.5 - th2 / 24.0)
    return torch.eye(3, dtype=w.dtype, device=w.device) + a * K + b * (K @ K)


def pose_of(camera):
    """(R, T) of a synth camera, fp64: world_view_transform = [[R^T, T], [0, 1]]^T."""
    wv = camera.world_view_transform.double().cpu()
    return wv[:3, :3].clone(), wv[3, :3].clone()


def threshold_pixel_mask(cd, inputs, d_alpha=1e-4, d_T=2e-3, d_power=1e-6):
    """[H,W] bool, the rule of DESIGN.md §2.2 fixed before comparing: pixels where a Gaussian whose tile rect covers the
    pixel sits within rounding of a discrete decision of the compositing loop (alpha = 1/255, alpha = 0.99, T = 1e-4,
    power = 0), from the fp64 oracle forward.  A superset of the pixels whose list position matters: every covering
    Gaussian is tested, not only those before the pixel's stop."""
    with torch.no_grad():
        means3D, scales, rots, opac, shs = [t.detach().double() for t in inputs]
        f = dense_render(cd, means3D, scales, rots, opac, shs)
    H, W = cd["H"], cd["W"]
    v = torch.as_tensor(np.asarray(cd["view"], np.float64)).reshape(16)
    tz = v[2] * means3D[:, 0] + v[6] * means3D[:, 1] + v[10] * means3D[:, 2] + v[14]
    order = torch.argsort(tz.float(), stable=True)
    rect, pix, con = f["rect"][order], f["pix"][order], f["conic"][order]
    ok = (f["radii"][order] > 0) & (tz[order] > NEAR_CULL)
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    px, py = xs.reshape(-1).double(), ys.reshape(-1).double()
    tx, ty = xs.reshape(-1) // 16, ys.reshape(-1) // 16
    cover = ok[None, :] & (tx[:, None] >= rect[None, :, 0]) & (tx[:, None] < rect[None, :, 2]) & \
        (ty[:, None] >= rect[None, :, 1]) & (ty[:, None] < rect[None, :, 3])
    dx, dy = pix[None, :, 0] - px[:, None], pix[None, :, 1] - py[:, None]
    power = -0.5 * (con[None, :, 0] * dx * dx + con[None, :, 2] * dy * dy) - con[None, :, 1] * dx * dy
    a = opac.reshape(-1)[order][None, :] * torch.exp(torch.clamp(power, max=0.0))
    alpha = torch.clamp(a, max=0.99)
    valid = cover & (power <= 0) & (alpha >= 1.0 / 255.0)
    T = torch.cumprod(torch.where(valid, 1.0 - alpha, torch.ones_like(alpha)), dim=1)
    near = ((a * 255.0 - 1.0).abs() < d_alpha) | ((a - 0.99).abs() < d_alpha) | ((T / 1e-4 - 1.0).abs() < d_T) | \
        (power.abs() < d_power)
    return (near & cover).any(dim=1).reshape(H, W)


def assert_close_to_max(got, ref, tol, what):
    """|got - ref| <= tol * max|ref| element-wise (DESIGN.md §2.2's bound for a gradient tensor)."""
    got, ref = np.asarray(got, np.float64).reshape(-1), np.asarray(ref, np.float64).reshape(-1)
    scale = max(np.abs(ref).max(), 1e-12)
    err = np.abs(got - ref).max()
    assert err <= tol * scale, "%s: max |err| %.3e > %.1e * max |ref| %.3e\ngot %s\nref %s" % (what, err, tol, scale, got, ref)
