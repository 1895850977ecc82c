"""The decomposed fp64 oracle of the fused training backward (tests/test_gpu_fullsize_backward.py), checked on the CPU.

That oracle splits the composition deform -> activations -> rasterize at the post-activation tensors: the raster oracle runs
on the deformed tensors the GPU produced, and its cotangents are chained back through the deformation in fp64.  Here:
  * the split changes nothing: fed the oracle's own deformed tensors it reproduces oracle_render + autograd;
  * the per-row comparator flags a small row that is off by 1 %, where the max-normalised metric cannot;
  * the colour-clamp silencing picks exactly the Gaussians at the clamp.
"""
import numpy as np
import pytest
import torch

from oracle import deform_ref as dr
from oracle import raster_ref as rr
from util_scene import (SCENE_LEAVES, OracleRaster, cam_tuple, colour_kink_rows, deformed_fp64, kink_rows, make_module,
                        oracle_chain_backward, oracle_params_from_module, oracle_render, params_fp64, raster_inputs,
                        raster_oracle_inputs, rel_err, row_err, synth)

# the shapes of test_gpu_parity.FUSED_CASES[2]: dynerf network (all five heads), 2,500 Gaussians, 203 x 152
CASE = dict(net="dynerf", n=2500, wh=(203, 152), theta=100.0, radius=2.2, t=0.5, deg=3, bg=(0.0, 0.0, 0.0), scale=0.04)
CHAIN_TOL = 1e-9         # per row: the two fp64 chains differ only in summation order


def _case(modifier):
    c = CASE
    scene = synth.make_scene(c["n"], seed=11, scale_mean=c["scale"])
    mod = make_module(c["net"], seed=2, device="cpu", aabb=scene["aabb"])
    cfg, prm = oracle_params_from_module(mod)
    cam = synth.make_camera(c["theta"], c["wh"][0], c["wh"][1], radius=c["radius"], time=c["t"])
    t = float(np.float32(c["t"]))
    # silence the Gaussians at a kink of the network: there an fp32 and an fp64 chain may take different branches
    kink = kink_rows(cfg, prm, scene["xyz"], t)
    scene = {k: v.clone() for k, v in scene.items()}
    scene["opacity"][kink] = -40.0
    return scene, cfg, prm, cam, t, kink


@pytest.mark.parametrize("modifier", [1.0, 0.7])
def test_decomposed_chain_equals_composed_oracle(modifier):
    """oracle_render + autograd with the deformation in fp64 (the raster oracle takes fp32 inputs either way) against the
    raster oracle on that composition's deformed tensors followed by oracle_chain_backward.  (An fp32 composition differs from
    both by its own rounding: up to ~2e-3 of a row on plane texels where many Gaussians' contributions cancel.)"""
    scene, cfg, prm, cam, t, kink = _case(modifier)
    assert 0 < int(kink.sum()) <= 0.05 * CASE["n"]
    tol = CHAIN_TOL
    prm = params_fp64(prm)
    leaves = {k: scene[k].clone().double().requires_grad_(True) for k in SCENE_LEAVES}
    color, _, radii, rc, (pts, s, r, o, sh) = oracle_render(cfg, prm, leaves, cam, t, CASE["bg"], sh_degree=CASE["deg"],
                                                           scale_modifier=modifier)
    dL = torch.randn(color.shape, generator=torch.Generator().manual_seed(5))
    (color * dL).sum().backward()
    # decomposed: the raster oracle on the composition's own deformed tensors, then the fp64 chain in several chunks
    deformed = torch.cat([pts, s, r, o], dim=1).detach().float().numpy()
    ins = raster_oracle_inputs(deformed, sh.detach().float().numpy())
    fwd = rr.rasterize_forward(rc, *ins)
    assert np.array_equal(fwd["color"], color.detach().numpy()) and np.array_equal(fwd["radii"], radii.numpy())
    cot = rr.rasterize_backward(rc, *ins, fwd, dL.numpy())
    assert np.array_equal(cot["means2D"], OracleRaster.last_means2D_grad)
    grads, p64 = oracle_chain_backward(cfg, prm, scene, t, cot, chunk=1000)
    for k in SCENE_LEAVES:
        assert float(np.abs(grads[k]).max()) > 0, k
        assert np.all(grads[k][kink.numpy()] == 0), k          # silenced rows carry no gradient at all
        e, worst = row_err(leaves[k].grad.numpy(), grads[k])
        assert e <= tol, (k, e, worst)
    osd_c, osd64 = dr.params_to_state_dict(prm), dr.params_to_state_dict(p64)
    n_checked = 0
    for key, p in osd64.items():
        if p.grad is None:
            continue
        n_checked += 1
        got = osd_c[key].grad.numpy()
        if key.startswith("deformation_net.grid.grids."):
            C = got.shape[1]
            e, worst = row_err(got[0].transpose(1, 2, 0).reshape(-1, C), p.grad.numpy()[0].transpose(1, 2, 0).reshape(-1, C))
        else:
            e, worst = rel_err(got, p.grad.numpy()), None
        assert e <= tol, (key, e, worst)
    assert n_checked == 2 * 6 + 2 + 4 * 5          # planes, feature_out, five active heads


def _visible_row_gradient():
    cam = synth.make_camera(30.0, 96, 64, radius=4.0)
    ins = [t.float().numpy() for t in raster_inputs(600, 3, scale_mean=0.08)]
    rc, _ = cam_tuple(cam, (0.0, 0.0, 0.0))
    fwd = rr.rasterize_forward(rc, *ins)
    dL = np.random.default_rng(0).standard_normal((3, 64, 96)).astype(np.float32)
    return rr.rasterize_backward(rc, *ins, fwd, dL)["means3D"].astype(np.float64), fwd["radii"]


def test_row_err_flags_a_small_row_that_rel_err_misses():
    ref, radii = _visible_row_gradient()
    mag = np.abs(ref).max(axis=1) / np.abs(ref).max()
    cand = np.nonzero((radii > 0) & (mag > 1e-3) & (mag < 0.05))[0]
    assert cand.size > 0
    got = ref.copy()
    got[cand[0]] *= 1.01
    e, worst = row_err(got, ref)
    assert e > 2e-3 and worst[0][0] == int(cand[0]), (e, worst[0][0])
    assert rel_err(got, ref) <= 2e-3
    assert row_err(ref, ref)[0] == 0.0
    # an all-zero reference must be matched exactly
    assert row_err(np.full((2, 3), 1e-30), np.zeros((2, 3)))[0] == np.inf


def test_colour_kink_selection():
    """Three Gaussians on the camera's axis: one with its red channel 1e-7 above the clamp, one with a clear colour, one at the
    clamp but behind the camera (culled: its colour is never evaluated)."""
    cam = synth.make_camera(0.0, 64, 64, radius=4.0)
    C0 = 0.28209479177387814
    centre = cam.camera_center.double()
    fwd = -centre / centre.norm()                        # the camera looks at the origin
    xyz = torch.stack([torch.zeros(3, dtype=torch.float64), 0.3 * centre / centre.norm(), centre - fwd])
    shs = torch.zeros(3, 16, 3, dtype=torch.float64)
    shs[0, 0, 0] = (-0.5 + 1e-7) / C0
    shs[1, 0] = 0.2
    shs[2, 0, 1] = -0.5 / C0
    mask = colour_kink_rows(xyz, shs, [cam], sh_degree=3)
    assert mask.tolist() == [True, False, False]
    # a clamp 2e-5 away is clear; a second camera that has the third Gaussian in front of it selects that one too
    shs[0, 0, 0] = (-0.5 + 2e-5) / C0
    assert colour_kink_rows(xyz, shs, [cam], sh_degree=3).tolist() == [False, False, False]
    assert colour_kink_rows(xyz, shs, [cam, synth.make_camera(90.0, 64, 64)], sh_degree=3).tolist() == [False, False, True]


def test_silenced_gaussians_never_contribute():
    """Opacity logit -40 keeps alpha below 1/255 at every pixel: the raster oracle gives the silenced rows no gradient, and
    dropping them from the scene changes no pixel."""
    scene, cfg, prm, cam, t, kink = _case(1.0)
    pts, sh = deformed_fp64(cfg, prm, scene, t, chunk=700)
    with torch.no_grad():
        _, _, _, rc, (p32, s, r, o, sh32) = oracle_render(cfg, prm, scene, cam, t, CASE["bg"], sh_degree=CASE["deg"])
    assert float((pts - p32.double()).abs().max()) <= 1e-5 and float((sh - sh32.double()).abs().max()) <= 1e-5
    assert float(o[kink].max()) < 1e-9
    ins = raster_oracle_inputs(torch.cat([p32, s, r, o], dim=1).numpy(), sh32.numpy())
    fwd = rr.rasterize_forward(rc, *ins)
    dL = np.ones((3,) + fwd["color"].shape[1:], np.float32)
    cot = rr.rasterize_backward(rc, *ins, fwd, dL)
    assert int((fwd["radii"][kink.numpy()] > 0).sum()) > 0          # (some are on screen: the statement is not vacuous)
    for nm in ("means3D", "means2D", "shs", "opacities", "scales", "rots"):
        assert np.all(cot[nm][kink.numpy()] == 0), nm
    keep = ~kink.numpy()
    fwd2 = rr.rasterize_forward(rc, *[a[keep] for a in ins])
    assert np.array_equal(fwd2["color"], fwd["color"])
