"""Projection (g4d_math.cuh, geom_finish.cuh) and blending (g4d_raster.cu) on the scenes of util_raster_edges.py, against the
oracle: clamped opacities, 255-1100 instances per tile, the guard band, the near plane, rects clamped at every grid side,
the SH colour clamp, degenerate covariances and images of 1-33 pixels a side.

Forward on the drop-in GaussianRasterizer (preprocess_kernel), render() fine on the FFMA and both tensor-core deform kernels,
the coarse stage (activate_preprocess_kernel) and render_cameras with three cameras (project_cameras_kernel); backward on
the rasterizer (blend_backward_kernel, preprocess_backward_kernel), render() (plus the activation and network backward)
and render_cameras (preprocess_backward_cameras_kernel).  The fused paths zero the position head's last Linear, so the
deformed means are the scene's means bit for bit and every boundary of the scene survives the network; opacities are
reached through logits (6, 10 and 20, which rounds to 1.0f).  The oracle runs on the GPU's own deformed tensors.

Every case asserts on the GPU's own records that it reached its condition (Scene.claim), index data bit for bit, the image
within 1e-4 except at explained threshold flips, and -- where every instance up to a pixel's stop is clamped -- n_contrib and
final_T bit for bit (no exp is involved there).  Gradients are compared per row (e_i <= 2e-3, floor 1e-4) with the upstream
gradient zeroed on both sides at flip pixels and at threshold pixels other than those all-clamped ones; on the fused paths
Gaussians at a kink of the network or of the colour clamp are silenced (logit -40) and must get exactly zero gradients, as
must Gaussians no camera sees.
"""
import math

import numpy as np
import pytest
import torch

from oracle import raster_ref as rr
import util_raster_edges as ue
from test_gpu_binning_edges import FUSED_PATHS
from util_scene import (SCENE_LEAVES, _assert_index_data_bit_exact, _assert_pixel_outliers_are_threshold_flips, cam_tuple,
                        colour_kink_rows, deformed_fp64, g4d, kink_rows, make_module, oracle_chain_backward,
                        oracle_params_from_module, raster_oracle_inputs, row_errors, synth, threshold_pixels)

pytestmark = pytest.mark.gpu
ROW_TOL = 2e-3
FLOOR = 1e-4
IMG_TOL = 1e-4
SILENCED_LOGIT = -40.0
T = 0.4
WORST = {}


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


def _settings(sc):
    cam = sc.cam
    return g4d.GaussianRasterizationSettings(
        image_height=cam.image_height, image_width=cam.image_width, tanfovx=math.tan(cam.FoVx * 0.5),
        tanfovy=math.tan(cam.FoVy * 0.5), bg=torch.tensor(sc.bg, dtype=torch.float32, device="cuda"), scale_modifier=1.0,
        viewmatrix=cam.world_view_transform.cuda(), projmatrix=cam.full_proj_transform.cuda(), sh_degree=sc.deg,
        campos=cam.camera_center.cuda(), prefiltered=False, debug=False)


def _check_forward(sc, ctx, radii, img, ref, colour_exact=True, fused=False):
    """index data, image, the scene's condition on the GPU's records, and bit-equal n_contrib / final_T where every instance
    up to the stop is clamped.  Returns the upstream mask: pixels whose gradient is compared."""
    W, H = sc.W, sc.H
    _assert_index_data_bit_exact(ctx, radii, ref, colour_exact=colour_exact)
    _assert_pixel_outliers_are_threshold_flips(img, ref, W)
    rec = ue.gpu_record(ctx, radii, W, H)
    if sc.fused_claim or not fused:
        sc.claim(sc, rec, fused=fused)
    clamped = ue.all_clamped_pixels(ue.oracle_record(ref), W, H)
    if sc.group == "opaque" and not len(sc.rows["thin"]):
        assert clamped.any()
    assert np.array_equal(rec["n_contrib"][clamped], ref["n_contrib"][clamped])
    assert np.array_equal(rec["final_T"][clamped].view(np.uint32), ref["final_T"][clamped].view(np.uint32))
    err = np.abs(img - ref["color"]).max(axis=0)
    flip = (rec["n_contrib"] != ref["n_contrib"]) | (err > IMG_TOL)
    near = threshold_pixels(ref, W, H) & ~clamped
    return ~(flip | near)


def _record(group, key, e):
    WORST[(group, key)] = max(WORST.get((group, key), 0.0), e)


def _compare_rows(sc, got, want, rows=None, tag=""):
    failures = []
    for k in want:
        g, w = np.asarray(got[k]), np.asarray(want[k])
        if rows is not None:
            g, w = g[rows], w[rows]
        e = row_errors(g.reshape(len(g), -1), w.reshape(len(w), -1), FLOOR)
        emax = float(e.max(initial=0.0))
        _record(sc.group, tag + k, emax)
        if emax > ROW_TOL:
            failures.append((k, emax, int(np.argmax(e))))
    assert not failures, (sc.name, tag, failures)


# ------------------------------------------------------------------------------------------------------------- rasterizer
@pytest.mark.parametrize("name", ue.names())
def test_rasterizer(name):
    sc = ue.scene(name)
    rc, _ = cam_tuple(sc.cam, sc.bg, sh_degree=sc.deg)
    ref = rr.rasterize_forward(rc, *sc.ins)
    dev = [torch.from_numpy(a).cuda().requires_grad_(True) for a in sc.ins]
    m3, s, r, o, sh = dev
    m2 = torch.zeros_like(m3, requires_grad=True)
    color, radii, _ = g4d.GaussianRasterizer(_settings(sc))(
        means3D=m3, means2D=m2, shs=sh, colors_precomp=None, opacities=o, scales=s, rotations=r, cov3D_precomp=None)
    torch.cuda.synchronize()
    ctx = color.grad_fn.lease.ctx
    keep = _check_forward(sc, ctx, radii.cpu().numpy(), color.detach().cpu().numpy(), ref)
    dL = torch.randn(3, sc.H, sc.W, generator=torch.Generator().manual_seed(sum(map(ord, name))))
    dL[:, torch.from_numpy(~keep)] = 0.0
    color.backward(dL.cuda())
    torch.cuda.synchronize()
    want = rr.rasterize_backward(rc, *sc.ins, ref, dL.numpy())
    got = {"means3D": m3.grad, "means2D": m2.grad, "scales": s.grad, "rots": r.grad, "opacities": o.grad, "shs": sh.grad}
    got = {k: v.cpu().numpy() for k, v in got.items()}
    unseen = ref["radii"] == 0
    for k, v in got.items():
        assert not v[unseen].any(), k
    _compare_rows(sc, got, {k: want[k] for k in got})
    if sc.group == "colour":                  # kept at an exact zero: the colour gradient flows; one float below: it does not
        for ch in range(3):
            z, b = sc.rows["zero"][ch], sc.rows["below"][ch]
            assert got["shs"][z, 0, ch] != 0 and got["shs"][b, :, ch].tolist() == [0.0] * 16


# ------------------------------------------------------------------------------------------------------------- fused paths
_MODULES = {}


def _module(net, aabb):
    if net not in _MODULES:
        mod = make_module(net, seed=2)
        with torch.no_grad():
            last = mod.deformation_net.pos_deform[3]
            last.weight.zero_(); last.bias.zero_()
        _MODULES[net] = mod
    mod = _MODULES[net]
    mod.deformation_net.set_aabb(aabb[0].tolist(), aabb[1].tolist())
    return mod


def _leaves(sc):
    """pre-activation leaves whose activation is the scene (opacities through logits; the clamped ones through 6, 10, 20)"""
    m, s, r, o, sh = sc.ins
    o64 = o.astype(np.float64).reshape(-1)
    logit = np.log(o64 / np.maximum(1.0 - o64, 1e-300))
    for val, lg in ue.OPAQUE_LOGITS.items():
        logit[o.reshape(-1) == np.float32(val)] = lg
    return {"xyz": torch.from_numpy(m.copy()), "scaling": torch.from_numpy(np.log(s.astype(np.float64)).astype(np.float32)),
            "rotation": torch.from_numpy(r.copy()), "opacity": torch.from_numpy(logit.astype(np.float32).reshape(-1, 1)),
            "features_dc": torch.from_numpy(sh[:, :1].copy()), "features_rest": torch.from_numpy(sh[:, 1:].copy())}


@pytest.mark.parametrize("path", list(FUSED_PATHS))
@pytest.mark.parametrize("name", ue.names())
def test_fused_paths(name, path):
    p = FUSED_PATHS[path]
    stage = p.get("stage", "fine")
    sc = ue.scene(name)
    scene = _leaves(sc)
    x = scene["xyz"]
    # unequal margins: a point on a symmetric box's centre plane would sit on a grid line of every odd-sized plane
    pad = 0.01 * (x.max(0).values - x.min(0).values) + 0.01
    aabb = torch.stack([x.max(0).values + 1.37 * pad, x.min(0).values - 2.91 * pad])
    mod = _module(p["net"], aabb)
    cfg, prm = oracle_params_from_module(mod)
    for q in prm.leaves():
        q.requires_grad_(False)
    has_sh = stage == "fine" and not mod.args.no_dshs
    k = p.get("cameras", 1)
    cams = [ue.origin_camera(sc.W, sc.H) for _ in range(k)]
    for c in cams:
        c.time = T
    t = float(np.float32(T))
    silenced = np.zeros(len(x), bool)
    if stage == "fine":
        silenced |= kink_rows(cfg, prm, x, t).numpy()
        pts, shs64 = deformed_fp64(cfg, prm, scene, t)
        silenced |= colour_kink_rows(pts, shs64, cams[:1], sh_degree=sc.deg).numpy()
    else:
        shs0 = torch.cat([scene["features_dc"], scene["features_rest"]], 1).double()
        silenced |= colour_kink_rows(x.double(), shs0, cams[:1], sh_degree=sc.deg).numpy()
    scene["opacity"][torch.from_numpy(silenced)] = SILENCED_LOGIT
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=sc.deg, requires_grad=True)
    bg = torch.tensor(sc.bg, dtype=torch.float32, device="cuda")
    ws = g4d._lib.Workspace.get(0)
    mod.zero_grad(set_to_none=True)
    try:
        ws.set_option(g4d._lib.OPT_TENSOR_CORES, p["tc"])
        if k > 1:
            outs = g4d.render_cameras(cams, pc, _Pipe, bg, stage=stage)
            ctxs = [lease.ctx for lease in outs[0]["render"].grad_fn.leases]
        else:
            outs = [g4d.render(cams[0], pc, _Pipe, bg, stage=stage)]
            ctxs = [outs[0]["render"].grad_fn.lease.ctx]
        torch.cuda.synchronize()
        dfm = ctxs[0].read("deformed")
        assert np.array_equal(dfm[:, 0:3], sc.ins[0])                 # the zeroed position head keeps every mean exact
        shs = ctxs[0].read("deformed_shs") if has_sh else torch.cat([scene["features_dc"], scene["features_rest"]], 1).numpy()
        ins = raster_oracle_inputs(dfm, shs)
        refs, dLs = [], []
        for i, (c, ctx, o) in enumerate(zip(cams, ctxs, outs)):
            rc, _ = cam_tuple(c, sc.bg, sh_degree=sc.deg)
            ref = rr.rasterize_forward(rc, *ins)
            keep = _check_forward(sc, ctx, o["radii"].cpu().numpy(), o["render"].detach().cpu().numpy(), ref,
                                  colour_exact=False, fused=True)
            dL = torch.randn(3, sc.H, sc.W, generator=torch.Generator().manual_seed(sum(map(ord, name)) + i))
            dL[:, torch.from_numpy(~keep)] = 0.0
            refs.append((rc, ref)); dLs.append(dL)
        if stage == "coarse":
            return
        sum((o["render"] * dL.cuda()).sum() for o, dL in zip(outs, dLs)).backward()
        torch.cuda.synchronize()
    finally:
        ws.set_option(g4d._lib.OPT_TENSOR_CORES, 2)
    cots = [rr.rasterize_backward(rc, *ins, ref, dL.numpy()) for (rc, ref), dL in zip(refs, dLs)]
    cot = {nm: sum(g[nm].astype(np.float64) for g in cots) for nm in ("means3D", "scales", "rots", "opacities", "shs")}
    want, _ = oracle_chain_backward(cfg, prm, scene, t, cot)
    got = {kk: getattr(pc, "_" + kk).grad.cpu().numpy().reshape(want[kk].shape) for kk in SCENE_LEAVES}
    unseen = np.logical_and.reduce([o["radii"].cpu().numpy() == 0 for o in outs])
    for kk in SCENE_LEAVES:
        for rows in (silenced, unseen):
            assert not got[kk][rows].any(), kk
    # a logit whose fp32 sigmoid is 1.0f (20) has 1 - sigmoid = 0: its opacity gradient is exactly zero in fp32, not the
    # fp64 chain's ~1e-9 of the cotangent
    sat = dfm[:, 10] == 1.0
    assert not got["opacity"][sat].any()
    want["opacity"][sat] = 0.0
    _compare_rows(sc, got, want, tag=path + ":")
    for o, g in zip(outs, cots):
        _compare_rows(sc, {"means2D": o["viewspace_points"].grad.cpu().numpy()}, {"means2D": g["means2D"]}, tag=path + ":")


def test_report_worst_row_errors():
    """prints the worst row error per scene group (quoted in DESIGN.md)"""
    for (g, k), e in sorted(WORST.items()):
        print("worst row error %-10s %-24s %.3g" % (g, k, e))
