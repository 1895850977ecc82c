"""Shared helpers for tests: small synthetic scenes in the rasterizer's post-activation input space."""
import math
from importlib import import_module

import numpy as np
import torch

synth = import_module("4dgaussians_b200.synth")


def raster_inputs(n, seed, scale_mean=0.08, sh_scale=0.3):
    """(means3D, scales, rots[normalised], opac, shs) as fp64 torch tensors that are exactly fp32-representable."""
    sc = synth.make_scene(n, seed=seed, scale_mean=scale_mean)
    g = torch.Generator().manual_seed(seed + 77)
    means3D = sc["xyz"].double()
    scales = torch.exp(sc["scaling"]).float().double()
    rots = torch.nn.functional.normalize(sc["rotation"], dim=-1).float().double()
    opac = torch.sigmoid(sc["opacity"]).float().double()
    shs = torch.cat([sc["features_dc"], torch.randn(n, 15, 3, generator=g) * sh_scale], dim=1).float().double()
    return means3D, scales, rots, opac, shs


def cam_tuple(camera, bg, sh_degree=3, scale_modifier=1.0):
    from oracle import raster_ref as rr
    from oracle.dense_ref import cam_dict_from
    cd = cam_dict_from(camera, bg, sh_degree, scale_modifier)
    rc = rr.make_cam(cd["H"], cd["W"], cd["tanfovx"], cd["tanfovy"], cd["view"], cd["proj"], cd["campos"], cd["bg"],
                     sh_degree, scale_modifier)
    # use the fp32-rounded tangents in the dense path too
    cd["tanfovx"] = float(np.float32(cd["tanfovx"])); cd["tanfovy"] = float(np.float32(cd["tanfovy"]))
    return rc, cd


# ---------------------------------------------------------------------------------------------------
# helpers for the GPU parity tests: oracle-side composition of the whole render() path
# ---------------------------------------------------------------------------------------------------
import importlib

g4d = importlib.import_module("4dgaussians_b200")


class OracleRaster(torch.autograd.Function):
    """CPU autograd wrapper around the C rasterizer oracle (forward + hand-derived backward)."""

    @staticmethod
    def forward(ctx, means3D, shs, opac, scales, rots, rc):
        from oracle import raster_ref as rr
        arrs = [t.detach().numpy().astype(np.float32) for t in (means3D, scales, rots, opac, shs)]
        f = rr.rasterize_forward(rc, *arrs)
        ctx.rc, ctx.f, ctx.arrs = rc, f, arrs
        return torch.from_numpy(f["color"].copy()), torch.from_numpy(f["depth"].copy()), torch.from_numpy(f["radii"].copy())

    @staticmethod
    def backward(ctx, g_color, _gd, _gr):
        from oracle import raster_ref as rr
        g = rr.rasterize_backward(ctx.rc, *ctx.arrs, ctx.f, g_color.numpy().astype(np.float32))
        ctx.means2D_grad = g["means2D"]
        OracleRaster.last_means2D_grad = g["means2D"]
        return (torch.from_numpy(g["means3D"]), torch.from_numpy(g["shs"]), torch.from_numpy(g["opacities"]),
                torch.from_numpy(g["scales"]), torch.from_numpy(g["rots"]), None)


def oracle_params_from_module(module):
    """DeformConfig + DeformParams (CPU fp32 leaves with requires_grad) mirroring a g4d deform_network."""
    from oracle import deform_ref as dr
    a = module.args
    kc = a.kplanes_config
    cfg = dr.DeformConfig(channels=kc["output_coordinate_dim"], resolution=tuple(kc["resolution"]), multires=tuple(a.multires),
                          net_width=a.net_width, no_dx=a.no_dx, no_ds=a.no_ds, no_dr=a.no_dr, no_do=a.no_do, no_dshs=a.no_dshs)
    sd = {k: v.detach().cpu().contiguous().clone() for k, v in module.state_dict().items()}
    prm = dr.params_from_state_dict(sd, cfg.levels)
    for t in prm.leaves():
        t.requires_grad_(True)
    return cfg, prm


def oracle_render(cfg, prm, scene_cpu, camera, t, bg, sh_degree=3, stage="fine", scale_modifier=1.0):
    """Reference composition (gaussian_renderer/__init__.py:80-128) on the oracle: deform -> activations -> rasterize.
    scene_cpu: dict of CPU tensors (leaves may require grad).  Returns (color, depth, radii, rc)."""
    from oracle import deform_ref as dr
    shs = torch.cat([scene_cpu["features_dc"], scene_cpu["features_rest"]], dim=1)
    if stage == "fine":
        pts, sc, rot, op, sh = dr.deform_forward(cfg, prm, scene_cpu["xyz"], scene_cpu["scaling"], scene_cpu["rotation"],
                                                 scene_cpu["opacity"], shs, float(t))
    else:
        pts, sc, rot, op, sh = scene_cpu["xyz"], scene_cpu["scaling"], scene_cpu["rotation"], scene_cpu["opacity"], shs
    s, r, o = dr.activate(sc, rot, op)
    rc, _ = cam_tuple(camera, bg, sh_degree=sh_degree, scale_modifier=scale_modifier)
    color, depth, radii = OracleRaster.apply(pts, sh, o, s, r, rc)
    return color, depth, radii, rc, (pts, s, r, o, sh)


def make_module(net: str, seed: int = 0, device="cuda", aabb=None):
    torch.manual_seed(1234 + seed)          # nn.Linear / plane initialisation draws from the global generator
    m = g4d.deform_network(synth.hidden_args(net))
    synth.perturb_deformation(m, seed)
    if aabb is not None:
        m.deformation_net.set_aabb(aabb[0].tolist(), aabb[1].tolist())
    return m.to(device)


def _assert_index_data_bit_exact(ctx, radii_gpu, ref, colour_exact=True):
    """The GPU context's projected records and instance list against the oracle forward `ref` (rr.rasterize_forward on the
    same fp32 inputs): bit for bit.  Returns the instance count R."""
    pr, bn = ref["proj"], ref["bin"]
    assert np.array_equal(radii_gpu, ref["radii"])
    for name, want in (("depth", pr.depth), ("rect", pr.rect), ("tiles_touched", pr.tiles_touched), ("xy", pr.xy),
                       ("conic_opacity", pr.conic_op), ("rgb", pr.rgb), ("clamped", pr.clamped)):
        got = ctx.read(name)
        assert got.shape == want.shape, name
        if name in ("rgb", "clamped") and not colour_exact:
            # the fused tensor-core kernel evaluates the SH polynomial with all 16 basis values in registers (a different
            # association order from the standalone preprocess kernel) and also for culled Gaussians (whose colour nobody
            # reads): colours of the VISIBLE Gaussians agree to fp32 rounding, not bit for bit
            vis = ref["radii"] > 0
            if name == "rgb":
                assert float(np.abs(got[vis] - want[vis]).max(initial=0.0)) <= 2e-6, name
            else:
                assert float((got[vis] != want[vis]).mean()) <= 1e-4 if vis.any() else True, name
            continue
        assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), name
    st = ctx.stats()
    assert st.num_rendered == bn.R and st.num_visible == int((ref["radii"] > 0).sum())
    assert np.array_equal(ctx.read("sorted_ids"), bn.ids)
    assert np.array_equal(ctx.read("ranges"), bn.ranges)
    assert np.array_equal(ctx.read("sorted_keys"), bn.keys)
    return bn.R


def _assert_pixel_outliers_are_threshold_flips(img_gpu, ref, W, max_outliers_frac=2e-5, max_err=6e-3, tol=1e-4):
    """Pixels where the GPU image is off by more than tol (1e-4) must be pixels where a DISCRETE decision of the compositing
    loop (A.3) sits within fp32 rounding of its threshold for one of the pixel's instances: alpha >= 1/255 (a skipped / kept
    contribution changes the pixel by up to alpha * T * colour ~ 4e-3), the alpha clamp at 0.99, or the T < 1e-4 stop.  The
    blend kernel's ex2-based exponential and the oracle's libm expf differ in the last ulp, so either side may take the
    other branch there.  Everything else must agree to tol.  Evaluated in fp64 from the oracle's own projected records."""
    err = np.abs(img_gpu - ref["color"]).max(axis=0)
    ys, xs = np.nonzero(err > tol)
    assert len(ys) <= max_outliers_frac * err.size + 2, (len(ys), float(err.max()))
    assert float(err.max()) <= max_err, float(err.max())
    pr, bn = ref["proj"], ref["bin"]
    gx = (W + 15) // 16
    for y, x in zip(ys, xs):
        lo, hi = bn.ranges[(y // 16) * gx + (x // 16)]
        ids = bn.ids[lo:hi]
        xy = pr.xy[ids].astype(np.float64); co = pr.conic_op[ids].astype(np.float64)
        dx, dy = xy[:, 0] - x, xy[:, 1] - y
        power = -0.5 * (co[:, 0] * dx * dx + co[:, 2] * dy * dy) - co[:, 1] * dx * dy
        alpha = np.minimum(0.99, co[:, 3] * np.exp(power))
        ok = (power <= 0) & (alpha >= 1.0 / 255.0)
        T = np.cumprod(np.where(ok, 1.0 - alpha, 1.0))
        near = (np.abs(co[:, 3] * np.exp(power) * 255.0 - 1.0) < 2e-5) | (np.abs(co[:, 3] * np.exp(power) - 0.99) < 2e-5) | \
               (np.abs(T / 1e-4 - 1.0) < 2e-3) | (np.abs(power) < 1e-6)
        assert near.any(), ("unexplained pixel", int(x), int(y), float(err[y, x]))
    return len(ys), float(err.max())


def rel_err(got, ref, floor=1e-3):
    got = np.asarray(got, dtype=np.float64); ref = np.asarray(ref, dtype=np.float64)
    return float(np.abs(got - ref).max() / max(floor, np.abs(ref).max()))


def row_errors(got, ref, floor=1e-4):
    """[rows] e_i = max_k |got_ik - ref_ik| / max(max_k |ref_ik|, floor * max|ref|), rows = the leading axis."""
    ref = np.asarray(ref, dtype=np.float64)
    rows = ref.shape[0]
    r = ref.reshape(rows, -1)
    g = np.asarray(got, dtype=np.float64).reshape(rows, -1)
    d = np.abs(g - r).max(axis=1, initial=0.0)
    scale = np.maximum(np.abs(r).max(axis=1, initial=0.0), floor * np.abs(r).max(initial=0.0))
    e = np.where(d > 0, np.inf, 0.0)            # a row of an all-zero reference must be exactly zero
    np.divide(d, scale, out=e, where=scale > 0)
    return e


def row_err(got, ref, floor=1e-4):
    """Per-row relative error: (max_i e_i, the worst five rows as (index, got row, ref row)), e_i as in row_errors.  Every row
    is measured against its own magnitude (down to floor x the tensor's max), so a row that is wrong by 100 % fails even when
    it is tiny next to the largest row -- strictly stronger than rel_err at the same tolerance."""
    e = row_errors(got, ref, floor)
    rows = e.shape[0]
    g = np.asarray(got, dtype=np.float64).reshape(rows, -1)
    r = np.asarray(ref, dtype=np.float64).reshape(rows, -1)
    worst = np.argsort(-e, kind="stable")[:5]
    return (float(e.max()) if rows else 0.0), [(int(i), g[i].tolist(), r[i].tolist()) for i in worst]


def rel_err_bulk(got, ref, floor=1e-3, q=99.9):
    """(q-th percentile, max) of |got - ref| relative to max|ref|.  For gradients that pass through ReLU / floor()
    decisions: an input sitting within fp32 rounding of a kink may legitimately land on the other side on the GPU."""
    got = np.asarray(got, dtype=np.float64); ref = np.asarray(ref, dtype=np.float64)
    e = np.abs(got - ref).reshape(-1) / max(floor, np.abs(ref).max())
    return float(np.percentile(e, q)), float(e.max())


def kink_rows(cfg, prm, xyz, t, delta_act=2e-6, delta_grid=2e-4):
    """[N] bool: Gaussians sitting within rounding distance of a NON-DIFFERENTIABLE point of the deformation network,
    evaluated in fp64 on the oracle: a pre-activation of an active ReLU within delta_act of 0, or a HexPlane sample
    coordinate within delta_grid (in texels) of a grid line, where floor() picks the bilinear cell.  On such rows an fp32
    implementation may legitimately take the other branch, and the gradient is then the (equally valid) one-sided
    derivative of the neighbouring piece.  Everywhere else gradients must agree to the stated tolerance."""
    from oracle import deform_ref as dr
    with torch.no_grad():
        x64 = xyz.detach().double().cpu()
        n = x64.shape[0]
        planes = [[p.detach().double() for p in lvl] for lvl in prm.planes]
        aabb = prm.aabb.detach().double()
        tt = torch.full((n,), float(t), dtype=torch.float64)
        p = dr.normalize(x64, aabb)
        q = torch.cat([p, tt.reshape(-1, 1)], dim=-1)
        mask = torch.zeros(n, dtype=torch.bool)
        for l, lvl in enumerate(planes):
            for k, (c0, c1) in enumerate(dr.PLANE_AXES):
                _, _, H, W = lvl[k].shape
                for coord, size in ((q[:, c0], W), (q[:, c1], H)):
                    g = (coord + 1.0) / 2.0 * (size - 1)          # unclamped: far outside the aabb the border rule is smooth
                    mask |= ((g - torch.round(g)).abs() < delta_grid) & (g > -delta_grid) & (g < size - 1 + delta_grid)
        feat = dr.hexplane_features(planes, x64, aabb, tt)
        hidden = feat @ prm.w0.detach().double().t() + prm.b0.detach().double()
        mask |= (hidden.abs() < delta_act).any(dim=1)
        active = {"pos": not cfg.no_dx, "scales": not cfg.no_ds, "rotations": not cfg.no_dr, "opacity": not cfg.no_do,
                  "shs": not cfg.no_dshs}
        a = torch.relu(hidden)
        for name, on in active.items():
            if not on:
                continue
            w1, b1, _, _ = prm.heads[name]
            z = a @ w1.detach().double().t() + b1.detach().double()
            mask |= (z.abs() < delta_act).any(dim=1)
    return mask


# ---------------------------------------------------------------------------------------------------
# decomposed fp64 oracle of the fused backward: raster oracle on the GPU's own deformed tensors, then an fp64 chain
# ---------------------------------------------------------------------------------------------------
SCENE_LEAVES = ("xyz", "scaling", "rotation", "opacity", "features_dc", "features_rest")


def params_fp64(prm):
    """fp64 copies of the oracle parameters as fresh leaves that collect gradients."""
    p = prm.to(torch.float64)
    p.aabb = p.aabb.detach()
    p.planes = [[q.detach().requires_grad_(True) for q in lvl] for lvl in p.planes]
    p.w0, p.b0 = p.w0.detach().requires_grad_(True), p.b0.detach().requires_grad_(True)
    p.heads = {k: tuple(q.detach().requires_grad_(True) for q in v) for k, v in p.heads.items()}
    return p


def _deform_activate(cfg, prm, leaves, t):
    shs = torch.cat([leaves["features_dc"], leaves["features_rest"]], dim=1)
    from oracle import deform_ref as dr
    pts, sc, rot, op, sh = dr.deform_forward(cfg, prm, leaves["xyz"], leaves["scaling"], leaves["rotation"], leaves["opacity"],
                                             shs, float(t))
    s, r, o = dr.activate(sc, rot, op)
    return pts, s, r, o, sh


def deformed_fp64(cfg, prm, scene, t, chunk=65536):
    """(means3D [N,3], shs [N,16,3]) of the fine stage in fp64, without gradients."""
    p64 = prm.to(torch.float64)
    n = scene["xyz"].shape[0]
    pts, shs = [], []
    with torch.no_grad():
        for a in range(0, n, chunk):
            lv = {k: scene[k][a:a + chunk].detach().double() for k in SCENE_LEAVES}
            p, _, _, _, sh = _deform_activate(cfg, p64, lv, t)
            pts.append(p); shs.append(sh)
    return torch.cat(pts), torch.cat(shs)


def colour_kink_rows(means3D, shs, cameras, sh_degree, delta=1e-5):
    """[N] bool: Gaussians in front of one of the cameras (view depth > 0.2, the projection's cull) with an SH colour channel
    within delta of the clamp max(colour + 0.5, 0).  Inputs in fp64.  The fused kernels evaluate the SH polynomial in
    another association order than the oracle, so on such a row the clamp decision (and with it the colour gradient) may
    legitimately differ."""
    from oracle.dense_ref import _sh_color
    x = means3D.double()
    mask = torch.zeros(x.shape[0], dtype=torch.bool)
    for cam in cameras:
        v = cam.world_view_transform.double().reshape(16)
        tz = v[2] * x[:, 0] + v[6] * x[:, 1] + v[10] * x[:, 2] + v[14]
        d = x - cam.camera_center.double()
        c = _sh_color(sh_degree, shs.double(), d / d.norm(dim=-1, keepdim=True)) + 0.5
        mask |= (tz > 0.2) & (c.abs() < delta).any(dim=1)
    return mask


def raster_oracle_inputs(deformed, shs):
    """The raster oracle's (means3D, scales, rots, opacities, shs) from the post-activation tensors deformed [N,11]
    (means3D | scales | rots | opacity, the layout of the context's "deformed" buffer) and shs [N,16,3]."""
    d = np.asarray(deformed, np.float32)
    return (np.ascontiguousarray(d[:, 0:3]), np.ascontiguousarray(d[:, 3:6]), np.ascontiguousarray(d[:, 6:10]),
            np.ascontiguousarray(d[:, 10:11]), np.ascontiguousarray(np.asarray(shs, np.float32).reshape(-1, 16, 3)))


def threshold_pixels(fwd, W, H, d_alpha=2e-5, d_T=2e-3, d_power=1e-6, include_stop=False):
    """[H,W] bool: pixels where an instance before the pixel's stop (list position < n_contrib) sits within rounding of a
    discrete decision of the compositing loop (A.3): alpha = 1/255, the clamp alpha = 0.99, T = 1e-4 or power = 0.
    include_stop: also the instance at position n_contrib, whose T < 1e-4 stopped the pixel if it stopped (a flip there
    changes n_contrib, which a comparison of two fp32 runs sees; a comparison with fp64 needs it here).  This is
    the predicate (same margins) of test_gpu_fullsize._assert_pixel_outliers_are_threshold_flips, evaluated in fp64 from the
    oracle's projected records for every pixel.  The blend kernels' ex2-based exponential and libm expf differ in the last
    ulp, so either side may take the other branch there; when the instance is not the pixel's last contributor and T is
    small the image moves by less than 1e-4, but that instance's gradient from the pixel appears on one side only."""
    pr, bn = fwd["proj"], fwd["bin"]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    xy = pr.xy.astype(np.float64); co = pr.conic_op.astype(np.float64)
    nc = fwd["n_contrib"].reshape(H, W)
    ly, lx = np.divmod(np.arange(256), 16)
    out = np.zeros((H, W), dtype=bool)
    for tile in range(gx * gy):
        ty, tx = divmod(tile, gx)
        px, py = tx * 16 + lx, ty * 16 + ly
        inside = (px < W) & (py < H)
        px, py = px[inside], py[inside]
        last = nc[py, px].astype(np.int64)
        m = int(last.max())
        if m == 0:
            continue
        lo, hi = (int(v) for v in bn.ranges[tile])
        ids = bn.ids[lo:min(hi, lo + m + int(include_stop))].astype(np.int64)
        dx = xy[ids, 0][:, None] - px[None, :]
        dy = xy[ids, 1][:, None] - py[None, :]
        power = -0.5 * (co[ids, 0][:, None] * dx * dx + co[ids, 2][:, None] * dy * dy) - co[ids, 1][:, None] * dx * dy
        a = co[ids, 3][:, None] * np.exp(np.minimum(power, 0.0))
        alpha = np.minimum(0.99, a)
        T = np.cumprod(np.where((power <= 0) & (alpha >= 1.0 / 255.0), 1.0 - alpha, 1.0), axis=0)
        near = (np.abs(a * 255.0 - 1.0) < d_alpha) | (np.abs(a - 0.99) < d_alpha) | (np.abs(T / 1e-4 - 1.0) < d_T) | \
               (np.abs(power) < d_power)
        near &= np.arange(len(ids))[:, None] < last[None, :] + int(include_stop)
        out[py, px] = near.any(axis=0)
    return out


def oracle_chain_backward(cfg, prm, scene, t, cot, chunk=65536):
    """fp64 chain of the fine stage: gradients of sum <cot, activate(deform(scene))> for the six Gaussian leaves and for every
    network parameter.  cot: post-activation cotangents as returned by rr.rasterize_backward (means3D, scales, rots,
    opacities, shs; summed over cameras for a multi-camera loss).  Rows are independent, so the chain runs in chunks of
    Gaussians; the parameter gradients add up across chunks.  Returns ({leaf: fp64 ndarray}, fp64 DeformParams with .grad)."""
    p64 = params_fp64(prm)
    n = scene["xyz"].shape[0]
    grads = {k: np.zeros(tuple(scene[k].shape), np.float64) for k in SCENE_LEAVES}
    names = ("means3D", "scales", "rots", "opacities", "shs")
    for a in range(0, n, chunk):
        lv = {k: scene[k][a:a + chunk].detach().double().requires_grad_(True) for k in SCENE_LEAVES}
        outs = _deform_activate(cfg, p64, lv, t)
        cts = [torch.from_numpy(np.asarray(cot[nm][a:a + chunk], np.float64)).reshape(o.shape) for nm, o in zip(names, outs)]
        torch.autograd.backward(list(outs), cts)
        for k in SCENE_LEAVES:
            grads[k][a:a + chunk] = lv[k].grad.numpy()
    return grads, p64
