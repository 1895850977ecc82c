"""CPU companion of test_gpu_depth_grad.py: the depth gradient of the oracles the GPU is checked against.

* The C oracle's depth backward (util_depth_grad.oracle_backward), for a depth-only and a mixed colour + depth cotangent,
  equals fp64 autograd of the dense formulation on every scene of util_raster_edges.py, per row.
* On two Gaussians centred on one pixel, D = z1 a1 + z2 a2 (1 - a1): the oracle's opacity and mean gradients match the
  closed form's central differences.
* The part of the view matrix's gradient that reaches it through z directly is sum_i dL/dz_i (x_i, y_i, z_i, 1) on
  view[2, 6, 10, 14], with the oracle's dL/dz.
* The host rules that need no device: the symbol is declared and exported, and the autograd plumbing points a context at a
  depth gradient only for the call and only when one arrived.

Pixels with an instance within rounding of a compositing threshold get no upstream gradient (as test_raster_edge_scenes)."""
import importlib
import os
import re

import numpy as np
import pytest
import torch

from oracle import raster_ref as rr
from oracle.dense_ref import dense_render
import util_depth_grad as udg
import util_raster_edges as ue
from util_camera_grad import central_differences
from util_scene import cam_tuple, row_errors, threshold_pixels

ROW_TOL = 2e-3
LONG_ROW_TOL = 5e-3
FLOOR = 1e-4
# the long scenes stack 255-1400 layers 5e-4 apart in depth: a depth-only loss gives the back layers a dL/dalpha that is a
# difference of nearly equal depths, z_i - aD' ~ 1e-3 z, where the fp32 rounding of the back-to-front accumulator is amplified
# a thousandfold.  Relative to the tensor's max the oracle stays within 5e-5 of fp64; rows below 1 % of it are measured
# against that 1 %.
LONG_DEPTH_FLOOR = 1e-2
_lib = importlib.import_module("4dgaussians_b200._lib")
rasterizer = importlib.import_module("4dgaussians_b200.rasterizer")


def _cotangents(sc, fwd, mode):
    g = torch.Generator().manual_seed(sum(map(ord, sc.name)) + 7)
    near = torch.from_numpy(threshold_pixels(fwd, sc.W, sc.H, include_stop=True))
    dD = torch.randn(1, sc.H, sc.W, generator=g).double()
    dD[:, near] = 0.0
    dC = None
    if mode == "mixed":
        dC = torch.randn(3, sc.H, sc.W, generator=g).double()
        dC[:, near] = 0.0
    return dC, dD, near


def test_dense_depth_is_the_dense_depth_image():
    sc = ue.scene("shape_17x17")
    _, cd = cam_tuple(sc.cam, sc.bg, sh_degree=sc.deg)
    ins = [torch.from_numpy(a.astype(np.float64)) for a in sc.ins]
    ref = dense_render(cd, *ins)["depth"]
    got = udg.dense_depth(cd, *ins[:4])
    assert float(ref.abs().max()) > 1.0
    assert float((got - ref).abs().max()) <= 1e-12 * float(ref.abs().max())


@pytest.mark.parametrize("mode", ["depth", "mixed"])
@pytest.mark.parametrize("name", ue.names())
def test_oracle_depth_backward_matches_dense_fp64(name, mode):
    sc = ue.scene(name)
    rc, cd = cam_tuple(sc.cam, sc.bg, sh_degree=sc.deg)
    fwd = rr.rasterize_forward(rc, *sc.ins)
    dC, dD, near = _cotangents(sc, fwd, mode)
    assert (~near).float().mean() >= 0.25
    want = udg.dense_grads(cd, sc.ins, dC, dD)
    got = udg.oracle_backward(rc, sc.ins, fwd, None if dC is None else dC.numpy(), dD.numpy())
    # as test_raster_edge_scenes: the colour-clamp rows may clamp differently in fp64 (a depth-only loss reads no colour)
    rows = np.arange(len(sc.ins[0]))
    if mode == "mixed":
        rows = np.setdiff1d(rows, np.concatenate([sc.rows.get("zero", []), sc.rows.get("below", [])]))
    tol = LONG_ROW_TOL if sc.group == "long" else ROW_TOL
    floor = LONG_DEPTH_FLOOR if sc.group == "long" and mode == "depth" else FLOOR
    for nm in udg.NAMES + ("means2D",):
        g = got[nm][:, :2] if nm == "means2D" else got[nm]
        e = row_errors(g[rows], want[nm][rows], floor)
        assert float(e.max()) <= tol, (nm, float(e.max()), int(rows[np.argmax(e)]))
    vis = fwd["radii"] > 0
    assert np.abs(got["depth"][vis]).max() > 0 and not got["depth"][~vis].any()
    if mode == "depth":
        assert not got["shs"].any()         # the depth reads no colour


def _two_on_a_pixel(o1, o2, z1, z2, W=16, H=16, px=7, py=9):
    """two small Gaussians centred on pixel (px, py), at view depths z1 < z2, opacities o1, o2 (fp32 inputs)"""
    cam = ue.origin_camera(W, H)
    pv = ue.pixel_view(cam, np.array([px, px], np.float64), np.array([py, py], np.float64), np.array([z1, z2]))
    means = ue.world_of(cam, pv).astype(np.float32)
    scales = np.full((2, 3), 0.01, np.float32)
    rots = np.tile(np.array([1.0, 0.0, 0.0, 0.0], np.float32), (2, 1))
    opac = np.array([[o1], [o2]], np.float32)
    shs = np.zeros((2, 16, 3), np.float32)
    return cam, [means, scales, rots, opac, shs]


def test_two_gaussians_closed_form():
    """At the pixel both are centred on, G = 1 and dG/d(position) = 0: D = z1 o1 + z2 o2 (1 - o1) with z = row 2 of the view
    transform.  The oracle's gradients of D at that pixel match the closed form's central differences."""
    o1, o2, z1, z2 = 0.6, 0.7, 2.0, 3.5
    cam, ins = _two_on_a_pixel(o1, o2, z1, z2)
    rc, cd = cam_tuple(cam, (0.0, 0.0, 0.0), sh_degree=0)
    fwd = rr.rasterize_forward(rc, *ins)
    m, op = ins[0].astype(np.float64), ins[3].astype(np.float64).reshape(-1)
    v = np.asarray(rc.view, np.float64)
    z = v[2] * m[:, 0] + v[6] * m[:, 1] + v[10] * m[:, 2] + v[14]
    assert abs(fwd["depth"][0, 9, 7] - (z[0] * op[0] + z[1] * op[1] * (1 - op[0]))) < 1e-5
    dD = np.zeros((1, 16, 16), np.float32)
    dD[0, 9, 7] = 1.0
    got = udg.oracle_backward(rc, ins, fwd, None, dD)

    def D(x):       # x = (o1, o2, m1[3], m2[3])
        zz = [v[2] * x[2 + 3 * i] + v[6] * x[3 + 3 * i] + v[10] * x[4 + 3 * i] + v[14] for i in range(2)]
        return zz[0] * x[0] + zz[1] * x[1] * (1 - x[0])

    x0 = torch.tensor([op[0], op[1], *m[0], *m[1]], dtype=torch.float64)
    fd = central_differences(D, x0, 1e-6).numpy()
    np.testing.assert_allclose(got["opacities"].reshape(-1), fd[:2], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(got["means3D"].reshape(-1), fd[2:], rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(got["depth"], [op[0], op[1] * (1 - op[0])], rtol=1e-5)


@pytest.mark.parametrize("name", ["shape_17x17", "guard_band", "colour_deg3"])
def test_view_row_terms(name):
    """dense fp64 dL/d view of a depth loss = the same with z held constant (the weights' part) + sum_i dL/dz_i (x, y, z, 1)
    on view[2, 6, 10, 14], with dL/dz from the C oracle"""
    sc = ue.scene(name)
    rc, cd = cam_tuple(sc.cam, sc.bg, sh_degree=sc.deg)
    fwd = rr.rasterize_forward(rc, *sc.ins)
    _, dD, _ = _cotangents(sc, fwd, "depth")
    ins = [torch.from_numpy(a.astype(np.float64)) for a in sc.ins]

    def view_grad(detach_z):
        view = torch.as_tensor(np.asarray(cd["view"], np.float64)).clone().requires_grad_(True)
        (udg.dense_depth(dict(cd, view=view), *ins[:4], detach_z=detach_z) * dD).sum().backward()
        return view.grad.numpy().reshape(-1)

    full, weights = view_grad(False), view_grad(True)
    got = udg.oracle_backward(rc, sc.ins, fwd, None, dD.numpy())
    direct = udg.view_depth_terms(sc.ins[0], got["depth"])
    scale = np.abs(full).max()
    assert np.abs(direct).max() > 1e-3 * scale
    np.testing.assert_allclose(weights + direct, full, rtol=0, atol=2e-3 * scale)


# ---- host rules ----------------------------------------------------------------------------------------------------------
def test_setter_is_declared_and_bound():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "g4d.h")).read()
    assert re.search(r"int g4d_context_set_depth_grad\(G4DContext \*ctx, const float \*d_dL_ddepth\);", header)
    assert "g4d_context_set_depth_grad" in _lib.ABI_SYMBOLS
    assert _lib.ABI_VERSION == 3


class _FakeContext:
    def __init__(self, log, i):
        self.log, self.i = log, i

    def set_camera_grad(self, p):
        self.log.append(("camera", self.i, p))

    def set_time_grad(self, p):
        self.log.append(("time", self.i, p))

    def set_depth_grad(self, p):
        self.log.append(("depth", self.i, p))


def test_depth_gradient_is_set_for_the_call_only():
    log = []
    ctxs = [_FakeContext(log, i) for i in range(3)]
    d1 = torch.zeros(12)
    with rasterizer.CameraGradSinks((), ctxs, torch.device("cpu"), depths=(None, d1, None)):
        assert log == [("depth", 1, d1.data_ptr())]
    assert log == [("depth", 1, d1.data_ptr()), ("depth", 1, None)]


def test_no_depth_gradient_sets_nothing():
    log = []
    ctxs = [_FakeContext(log, i) for i in range(2)]
    for depths in ((), (None, None)):
        with rasterizer.CameraGradSinks((), ctxs, torch.device("cpu"), depths=depths):
            pass
    assert log == []
