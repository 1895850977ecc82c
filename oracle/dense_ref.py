"""Dense, differentiable fp64 formulation of the rasterizer (torch autograd) -- an INDEPENDENT check of
oracle/raster_ref.c (forward values and, above all, its hand-derived backward).

TEST INFRASTRUCTURE ONLY.  O(pixels x Gaussians) memory: tiny scenes only.

Follows SURVEY.md Appendix A.1/A.3 (see raster_ref.c for the provenance note: the rasterizer source is
absent from /root/reference, parity unpinned).  The discrete decisions (cull, radius, tile rect, skip,
early stop) are evaluated without gradient; the quirks of the published backward are encoded as
straight-through / detach constructs:
  * alpha = min(0.99, o*G): gradient passes as if unclamped;
  * the 1.3*tanfov guard band: a clamped t.x / t.y is a constant;
  * max(rgb, 0): zero gradient where clamped;
  * depth image: no gradient.
(The published backward uses 1/(det^2+1e-7) where autograd uses 1/det^2: relative difference <= 1.3e-5
because the +0.3 dilation keeps det >= 0.09.)
"""
from __future__ import annotations

import math
from typing import Dict

import torch

C0 = 0.28209479177387814
NEAR_CULL = 0.20000000298023224     # the fp32 constant 0.2f of the kernels' `depth <= 0.2f` cull, exactly
C1 = 0.4886025119029199
C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435]


def _sh_color(deg, sh, d):
    x, y, z = d[:, 0:1], d[:, 1:2], d[:, 2:3]
    res = C0 * sh[:, 0]
    if deg > 0:
        res = res - C1 * y * sh[:, 1] + C1 * z * sh[:, 2] - C1 * x * sh[:, 3]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        res = (res + C2[0] * xy * sh[:, 4] + C2[1] * yz * sh[:, 5] + C2[2] * (2 * zz - xx - yy) * sh[:, 6]
               + C2[3] * xz * sh[:, 7] + C2[4] * (xx - yy) * sh[:, 8])
    if deg > 2:
        res = (res + C3[0] * y * (3 * xx - yy) * sh[:, 9] + C3[1] * xy * z * sh[:, 10]
               + C3[2] * y * (4 * zz - xx - yy) * sh[:, 11] + C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[:, 12]
               + C3[4] * x * (4 * zz - xx - yy) * sh[:, 13] + C3[5] * z * (xx - yy) * sh[:, 14]
               + C3[6] * x * (xx - 3 * yy) * sh[:, 15])
    return res


def dense_render(cam: Dict, means3D, scales, rots, opac, shs, pix_offset=None, guard_band_grad=False, alpha_clamp=True):
    """cam: dict(H,W,tanfovx,tanfovy,view[16],proj[16],campos[3],bg[3],sh_degree,scale_modifier).
    All tensors fp64.  Returns dict(color[3,H,W], depth[1,H,W], radii[N], rect[N,4], n_contrib[H,W]).
    Two opt-in departures from the published algorithm, for tests that show a check would catch a kernel that made them:
    guard_band_grad passes the gradient straight through a guard-band-clamped t.x / t.y (as if the clamp were not there in
    the backward); alpha_clamp=False drops the 0.99 clamp of alpha in the forward and the backward."""
    dt = means3D.dtype
    H, W = cam["H"], cam["W"]
    v = torch.as_tensor(cam["view"], dtype=dt).reshape(16)
    pm = torch.as_tensor(cam["proj"], dtype=dt).reshape(16)
    campos = torch.as_tensor(cam["campos"], dtype=dt)
    bg = torch.as_tensor(cam["bg"], dtype=dt)
    mod = cam.get("scale_modifier", 1.0)
    N = means3D.shape[0]
    px_, py_, pz_ = means3D[:, 0], means3D[:, 1], means3D[:, 2]

    def xf(m, row):
        return m[row] * px_ + m[4 + row] * py_ + m[8 + row] * pz_ + m[12 + row]

    tx, ty, tz = xf(v, 0), xf(v, 1), xf(v, 2)
    hw = xf(pm, 3)
    pw = 1.0 / (hw + 0.0000001)
    ndcx, ndcy = xf(pm, 0) * pw, xf(pm, 1) * pw
    visible = tz.detach() > NEAR_CULL

    r, x, y, z = rots[:, 0], rots[:, 1], rots[:, 2], rots[:, 3]
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], dim=-1).reshape(N, 3, 3)
    S = torch.diag_embed(mod * scales)
    L = R @ S
    Sigma = L @ L.transpose(1, 2)

    fx, fy = W / (2.0 * cam["tanfovx"]), H / (2.0 * cam["tanfovy"])
    limx, limy = 1.3 * cam["tanfovx"], 1.3 * cam["tanfovy"]
    tzs = torch.where(visible, tz, torch.ones_like(tz))
    txtz, tytz = tx / tzs, ty / tzs
    cxm = (txtz.detach() < -limx) | (txtz.detach() > limx)
    cym = (tytz.detach() < -limy) | (tytz.detach() > limy)
    txc = torch.where(cxm, (txtz.clamp(-limx, limx) * tzs).detach(), tx)
    tyc = torch.where(cym, (tytz.clamp(-limy, limy) * tzs).detach(), ty)
    if guard_band_grad:
        txc = tx + (txc - tx).detach()
        tyc = ty + (tyc - ty).detach()
    zero = torch.zeros_like(tzs)
    J = torch.stack([fx / tzs, zero, -(fx * txc) / (tzs * tzs), zero, fy / tzs, -(fy * tyc) / (tzs * tzs)],
                    dim=-1).reshape(N, 2, 3)
    Wm = torch.stack([v[0], v[4], v[8], v[1], v[5], v[9], v[2], v[6], v[10]]).reshape(3, 3)
    T = J @ Wm
    cov2 = T @ Sigma @ T.transpose(1, 2)
    a, b, c = cov2[:, 0, 0] + 0.3, cov2[:, 0, 1], cov2[:, 1, 1] + 0.3
    det = a * c - b * b
    ok = visible & (det.detach() != 0)
    dets = torch.where(ok, det, torch.ones_like(det))
    conx, cony, conz = c / dets, -b / dets, a / dets
    mid = 0.5 * (a + c)
    lam = mid + torch.sqrt(torch.clamp(mid * mid - det, min=0.1))
    rad = torch.ceil(3.0 * torch.sqrt(lam)).detach()
    pix_x = ((ndcx + 1.0) * W - 1.0) * 0.5
    pix_y = ((ndcy + 1.0) * H - 1.0) * 0.5
    if pix_offset is not None:      # leaf whose gradient is the screen-space (pixel-unit) gradient
        pix_x = pix_x + pix_offset[:, 0]
        pix_y = pix_y + pix_offset[:, 1]
    gx, gy = (W + 15) // 16, (H + 15) // 16

    def tile(vv, g):
        return torch.clamp(torch.trunc(vv / 16.0), 0, g).long()

    rminx, rminy = tile(pix_x.detach() - rad, gx), tile(pix_y.detach() - rad, gy)
    rmaxx, rmaxy = tile(pix_x.detach() + rad + 15.0, gx), tile(pix_y.detach() + rad + 15.0, gy)
    area = (rmaxx - rminx) * (rmaxy - rminy)
    ok = ok & (area > 0)
    radii = torch.where(ok, rad, torch.zeros_like(rad)).long()

    d = means3D - campos
    dirn = d / d.norm(dim=-1, keepdim=True)
    rgb = torch.clamp_min(_sh_color(cam["sh_degree"], shs, dirn) + 0.5, 0.0)

    # depth-ascending order with fp32 depth bits, ties by index (A.2)
    depth32 = tz.detach().float()
    order = sorted(range(N), key=lambda i: (depth32[i].item(), i))
    order = torch.tensor(order, dtype=torch.long)

    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    pxf, pyf = xs.reshape(-1).to(dt), ys.reshape(-1).to(dt)
    ptx, pty = (xs.reshape(-1) // 16), (ys.reshape(-1) // 16)
    o = order
    member = (ok[o][None, :] & (ptx[:, None] >= rminx[o][None, :]) & (ptx[:, None] < rmaxx[o][None, :])
              & (pty[:, None] >= rminy[o][None, :]) & (pty[:, None] < rmaxy[o][None, :]))
    dx = pix_x[o][None, :] - pxf[:, None]
    dy = pix_y[o][None, :] - pyf[:, None]
    power = -0.5 * (conx[o][None, :] * dx * dx + conz[o][None, :] * dy * dy) - cony[o][None, :] * dx * dy
    G = torch.exp(torch.clamp(power, max=0.0))
    a_raw = opac.reshape(-1)[o][None, :] * G
    alpha = a_raw + (torch.clamp(a_raw, max=0.99) - a_raw).detach() if alpha_clamp else a_raw
    valid = member & (power.detach() <= 0) & (alpha.detach() >= 1.0 / 255.0)
    om = torch.where(valid, 1.0 - alpha, torch.ones_like(alpha))
    t_incl = torch.cumprod(om, dim=1)
    stop = valid & (t_incl.detach() < 0.0001)
    stopped = torch.cummax(stop.to(torch.int8), dim=1).values.bool()
    contrib = valid & ~stopped
    t_before = torch.cat([torch.ones_like(t_incl[:, :1]), t_incl[:, :-1]], dim=1)
    w = torch.where(contrib, alpha * t_before, torch.zeros_like(alpha))
    color = w @ rgb[o]                                              # [P,3]
    t_final = torch.prod(torch.where(contrib, om, torch.ones_like(om)), dim=1)
    color = color + t_final[:, None] * bg[None, :]
    depth_img = (w.detach() @ tz.detach()[o][:, None]).reshape(1, H, W)
    # n_contrib: 1-based position (within the tile list) of the last contributing entry
    pos = torch.cumsum(member.long(), dim=1)
    n_contrib = torch.where(contrib, pos, torch.zeros_like(pos)).max(dim=1).values.reshape(H, W)
    return {"color": color.t().reshape(3, H, W), "depth": depth_img, "radii": radii,
            "rect": torch.stack([rminx, rminy, rmaxx, rmaxy], dim=-1) * ok[:, None].long(),
            "n_contrib": n_contrib, "final_T": t_final.reshape(H, W), "pix": torch.stack([pix_x, pix_y], -1),
            "conic": torch.stack([conx, cony, conz], -1), "rgb": rgb}


def cam_dict_from(camera, bg, sh_degree=3, scale_modifier=1.0) -> Dict:
    """camera: an object with the reference Camera fields (see 4dgaussians_b200/synth.py::SynthCamera)."""
    return {"H": int(camera.image_height), "W": int(camera.image_width),
            "tanfovx": math.tan(camera.FoVx * 0.5), "tanfovy": math.tan(camera.FoVy * 0.5),
            "view": camera.world_view_transform.reshape(-1).tolist(),
            "proj": camera.full_proj_transform.reshape(-1).tolist(),
            "campos": camera.camera_center.tolist(), "bg": list(bg), "sh_degree": sh_degree,
            "scale_modifier": scale_modifier}
