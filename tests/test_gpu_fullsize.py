"""Full-size GPU parity: BASELINE.json configs C1 (70k, 800x800, dnerf net -> FFMA kernels), C2 (200k, 536x960, hypernerf
net, L=3) and C3 (300k, 1352x1014, dynerf net, 5 heads) against the CPU oracle -- the sizes at which the persistent tile
loops (132 CTAs x 18 tiles on an H100), the 85 x 64 tile grid, ~3 M tile instances and the chunked counting placement actually run.

Structure of the proof for the fused path (SURVEY 7 "bit-exact ... given identical post-deformation inputs"):
  (i)   the deformed + activated tensors the fused kernel produced are within fp32 rounding of the oracle's deformation;
  (ii)  the oracle rasterizer fed with EXACTLY those tensors reproduces the GPU's index data bit for bit (radii, rects, depth
        bits, sorted keys / ids, tile ranges) and its image within 1e-4 L-inf at every pixel EXCEPT a handful (< 2e-5 of
        the pixels) that are each shown to hold an instance whose alpha / T sits on a compositing threshold (A.3);
  (iii) the end-to-end image against the full oracle composition differs only where (i)'s rounding moved a Gaussian across
        a discrete decision (ceil of the radius, alpha = 1/255, T = 1e-4): bulk within tolerance, isolated flips bounded.
Measured statistics are written to gpurun_out/parity_fullsize.json (quoted in DESIGN.md).
"""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import deform_ref as dr
from oracle import raster_ref as rr
from util_scene import cam_tuple, g4d, make_module, oracle_params_from_module, oracle_render, raster_inputs, rel_err, synth

pytestmark = pytest.mark.gpu
IMG_TOL = 1e-4
GRAD_TOL = 2e-3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATS = os.path.join(ROOT, "gpurun_out", "parity_fullsize.json")


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


def _record(key, val):
    try:
        os.makedirs(os.path.dirname(STATS), exist_ok=True)
        cur = json.load(open(STATS)) if os.path.isfile(STATS) else {}
        cur[key] = val
        json.dump(cur, open(STATS, "w"), indent=1, sort_keys=True)
    except Exception:
        pass


def _settings(cam, bg, sh_degree=3, dev="cuda"):
    return g4d.GaussianRasterizationSettings(
        image_height=cam.image_height, image_width=cam.image_width, tanfovx=math.tan(cam.FoVx * 0.5),
        tanfovy=math.tan(cam.FoVy * 0.5), bg=torch.tensor(bg, dtype=torch.float32, device=dev), scale_modifier=1.0,
        viewmatrix=cam.world_view_transform.to(dev), projmatrix=cam.full_proj_transform.to(dev), sh_degree=sh_degree,
        campos=cam.camera_center.to(dev), prefiltered=False, debug=False)


def _assert_index_data_bit_exact(ctx, radii_gpu, ref, colour_exact=True):
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
                assert float(np.abs(got[vis] - want[vis]).max()) <= 2e-6, name
            else:
                assert float((got[vis] != want[vis]).mean()) <= 1e-4, name
            continue
        assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), name
    st = ctx.stats()
    assert st.num_rendered == bn.R and st.num_visible == int((ref["radii"] > 0).sum())
    assert np.array_equal(ctx.read("sorted_ids"), bn.ids)
    assert np.array_equal(ctx.read("ranges"), bn.ranges)
    assert np.array_equal(ctx.read("sorted_keys"), bn.keys)
    return bn.R


def _assert_pixel_outliers_are_threshold_flips(img_gpu, ref, W, max_outliers_frac=2e-5, max_err=6e-3):
    """Pixels where the GPU image is off by more than 1e-4 must be pixels where a DISCRETE decision of the compositing loop
    (A.3) sits within fp32 rounding of its threshold for one of the pixel's instances: alpha >= 1/255 (a skipped / kept
    contribution changes the pixel by up to alpha * T * colour ~ 4e-3), the alpha clamp at 0.99, or the T < 1e-4 stop.  The
    blend kernel's ex2-based exponential and the oracle's libm expf differ in the last ulp, so either side may take the
    other branch there.  Everything else must agree to 1e-4.  Evaluated in fp64 from the oracle's own projected records."""
    err = np.abs(img_gpu - ref["color"]).max(axis=0)
    ys, xs = np.nonzero(err > IMG_TOL)
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


@pytest.mark.parametrize("wl", ["C1", "C2", "C3"])
@pytest.mark.parametrize("sync_mode", [1, 0])
def test_full_size_rasterizer_forward_vs_oracle(wl, sync_mode):
    """Drop-in GaussianRasterizer at BASELINE sizes: every index array bit-exact, image L-inf <= 1e-4.  sync_mode 0 = the
    capacity-bounded device-side binning the bench uses (second forward on the context; the first one learns the capacity)."""
    w = synth.WORKLOADS[wl]
    cam = synth.make_camera(-40.0, w["width"], w["height"], radius=w["radius"], focal=w["focal"])
    ins = [t.float() for t in raster_inputs(w["n"], 1, scale_mean=w["scale_mean"])]
    m3, sc, ro, op, sh = [t.cuda() for t in ins]
    rc, _ = cam_tuple(cam, w["bg"], sh_degree=3)
    rast = g4d.GaussianRasterizer(_settings(cam, w["bg"]))
    ws = g4d._lib.Workspace.get(0)
    ws._free_contexts.clear()            # fresh context: the no-sync capacity is learnt from THIS scene's first forward
    color = radii = depth = ctx = None
    try:
        ws.set_option(g4d._lib.OPT_SYNC_MODE, sync_mode)
        for _ in range(2 if sync_mode == 0 else 1):
            color = radii = depth = ctx = None       # hand the context back to the pool before the next forward
            m3r = m3.clone().requires_grad_(True)
            color, radii, depth = rast(means3D=m3r, means2D=torch.zeros_like(m3), shs=sh, colors_precomp=None, opacities=op,
                                       scales=sc, rotations=ro, cov3D_precomp=None)
            torch.cuda.synchronize()
            ctx = color.grad_fn.lease.ctx
            if sync_mode == 0:
                ctx.stats()          # consumes the asynchronous R (and would raise on overflow)
        ref = rr.rasterize_forward(rc, *[t.numpy() for t in ins])
        R = _assert_index_data_bit_exact(ctx, radii.cpu().numpy(), ref)
        img = color.detach().cpu().numpy()
        err = np.abs(img - ref["color"])
        derr = float(np.abs(depth.cpu().numpy() - ref["depth"]).max())
        nc = float((ctx.read("n_contrib").reshape(cam.image_height, -1) != ref["n_contrib"]).mean())
        n_out, emax = _assert_pixel_outliers_are_threshold_flips(img, ref, cam.image_width)
        _record("raster_fwd_%s_sync%d" % (wl, sync_mode), {"R": int(R), "image_linf": emax, "pixels_gt_1e-4": n_out,
                                                             "image_p99999": float(np.quantile(err, 0.99999)),
                                                             "depth_linf": derr, "n_contrib_mismatch": nc})
        assert nc < 1e-4 and derr <= 5e-2, (derr, nc)
    finally:
        ws.set_option(g4d._lib.OPT_SYNC_MODE, 1)
        ws.set_option(g4d._lib.OPT_INSTANCE_CAPACITY, 0)
        color = radii = depth = ctx = None
        ws._free_contexts.clear()


def test_full_size_rasterizer_backward_C3_vs_oracle():
    w = synth.WORKLOADS["C3"]
    cam = synth.make_camera(25.0, w["width"], w["height"], radius=w["radius"], focal=w["focal"])
    ins = [t.float() for t in raster_inputs(w["n"], 2, scale_mean=w["scale_mean"])]
    rc, _ = cam_tuple(cam, w["bg"], sh_degree=3)
    dev_ins = [t.cuda().requires_grad_(True) for t in ins]
    m3, sc, ro, op, sh = dev_ins
    m2 = torch.zeros_like(m3, requires_grad=True)
    rast = g4d.GaussianRasterizer(_settings(cam, w["bg"]))
    color, radii, depth = rast(means3D=m3, means2D=m2, shs=sh, colors_precomp=None, opacities=op, scales=sc, rotations=ro,
                               cov3D_precomp=None)
    g = torch.Generator().manual_seed(7)
    dL = torch.randn(color.shape, generator=g)
    color.backward(dL.cuda())
    ref = rr.rasterize_forward(rc, *[t.numpy() for t in ins])
    want = rr.rasterize_backward(rc, *[t.numpy() for t in ins], ref, dL.numpy())
    stats = {}
    for t, nm in ((m3, "means3D"), (m2, "means2D"), (sh, "shs"), (op, "opacities"), (sc, "scales"), (ro, "rots")):
        stats[nm] = rel_err(t.grad.cpu().numpy().reshape(want[nm].shape), want[nm])
    _record("raster_bwd_C3", stats)
    for nm, e in stats.items():
        assert e <= GRAD_TOL, (nm, e)


@pytest.mark.parametrize("wl", ["C1", "C2", "C3"])
def test_full_size_fused_forward_vs_oracle(wl):
    w = synth.WORKLOADS[wl]
    scene = synth.make_scene(w["n"], seed=0, scale_mean=w["scale_mean"])
    mod = make_module(w["net"], seed=0, aabb=scene["aabb"])
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3)
    t = 0.4
    cam = synth.make_camera(30.0, w["width"], w["height"], radius=w["radius"], focal=w["focal"], time=t)
    bg = torch.tensor(w["bg"], dtype=torch.float32, device="cuda")
    ws = g4d._lib.Workspace.get(0)
    ws._free_contexts.clear()
    ws.set_option(g4d._lib.OPT_KEEP_DEFORMED, 1)                 # (a no-grad render skips the stores of these tensors by default)
    try:
        with torch.no_grad():
            out = g4d.render(cam, pc, _Pipe(), bg)
        torch.cuda.synchronize()
    finally:
        ws.set_option(g4d._lib.OPT_KEEP_DEFORMED, 0)
    ctx = ws._free_contexts[-1]
    dfm = ctx.read("deformed")                                   # [N,11] what the fused kernel handed to its projection stage
    has_sh = not mod.args.no_dshs
    shs_gpu = ctx.read("deformed_shs") if has_sh else torch.cat([scene["features_dc"], scene["features_rest"]], dim=1).numpy()
    cfg, prm = oracle_params_from_module(mod)
    for p_ in prm.leaves():
        p_.requires_grad_(False)
    with torch.no_grad():
        color, depth, radii, rc, (pts, s, r, o, sh) = oracle_render(cfg, prm, scene, cam, t, w["bg"], sh_degree=3)
    # ---- (i) deformation + activations within fp32 rounding of the oracle
    d_xyz = float(np.abs(dfm[:, 0:3] - pts.numpy()).max())
    d_sc = float((np.abs(dfm[:, 3:6] - s.numpy()) / s.numpy()).max())
    d_rot = float(np.abs(dfm[:, 6:10] - r.numpy()).max())
    d_op = float(np.abs(dfm[:, 10] - o.numpy().reshape(-1)).max())
    d_sh = float(np.abs(shs_gpu.reshape(-1, 48) - sh.numpy().reshape(-1, 48)).max())
    assert d_xyz <= 3e-5 and d_sc <= 3e-5 and d_rot <= 3e-5 and d_op <= 3e-5 and d_sh <= 3e-5, (d_xyz, d_sc, d_rot, d_op, d_sh)
    # ---- (ii) identical post-deformation inputs -> bit-exact indices, image within 1e-4 at EVERY pixel
    ref = rr.rasterize_forward(rc, np.ascontiguousarray(dfm[:, 0:3]), np.ascontiguousarray(dfm[:, 3:6]),
                               np.ascontiguousarray(dfm[:, 6:10]), np.ascontiguousarray(dfm[:, 10:11]),
                               np.ascontiguousarray(shs_gpu.reshape(-1, 16, 3)))
    R = _assert_index_data_bit_exact(ctx, out["radii"].cpu().numpy(), ref, colour_exact=False)
    n_out, e2 = _assert_pixel_outliers_are_threshold_flips(out["render"].cpu().numpy(), ref, cam.image_width)
    assert float(np.abs(out["depth"].cpu().numpy() - ref["depth"]).max()) <= 5e-2
    # ---- (iii) end to end against the full oracle composition
    err = (out["render"].cpu() - color).abs()
    mism = float((out["radii"].cpu().numpy() != radii.numpy()).mean())
    stats = {"R": int(R), "deform_linf": {"xyz": d_xyz, "scale_rel": d_sc, "rot": d_rot, "opacity": d_op, "sh": d_sh},
             "image_linf_same_inputs": e2, "pixels_gt_1e-4_same_inputs": n_out, "image_linf_end_to_end": float(err.max()), "image_median_err": float(err.median()),
             "frac_pixels_gt_1e-4": float((err > IMG_TOL).float().mean()), "radii_mismatch_frac": mism,
             "depth_linf_end_to_end": float((out["depth"].cpu() - depth).abs().max())}
    _record("fused_fwd_%s" % wl, stats)
    assert mism <= 2e-3, mism
    assert float((err > IMG_TOL).float().mean()) <= 1e-3 and float(err.max()) <= 1e-2, stats
    assert float(err.median()) <= 1e-6
