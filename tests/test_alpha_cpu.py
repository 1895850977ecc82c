"""CPU companion of test_gpu_alpha.py: the alpha image and its gradient in the oracles the GPU is checked against.

* The C oracle's alpha (1 - final_T) is the dense fp64 alpha image within fp32 rounding, and the colour it composites is
  C_fg + (1 - A) bg: the colour on two backgrounds differs by (1 - A) (bg1 - bg2).
* The C oracle's alpha backward (util_alpha.oracle_backward), for an alpha-only and a mixed colour + depth + alpha cotangent,
  equals fp64 autograd of the dense formulation on every scene of util_raster_edges.py, per row.
* On two Gaussians centred on one pixel, A = 1 - (1 - a1)(1 - a2): the oracle's opacity gradients match the closed form.
* The host rules that need no device: the setters are declared and bound, and the autograd plumbing points a context at an
  alpha gradient only for the call and only when one arrived.

Pixels with an instance within rounding of a compositing threshold get no upstream gradient (as test_raster_edge_scenes)."""
import importlib
import os
import re

import numpy as np
import pytest
import torch

from oracle import raster_ref as rr
import util_alpha as ua
import util_raster_edges as ue
from util_scene import cam_tuple, row_errors, threshold_pixels

ROW_TOL = 2e-3
LONG_ROW_TOL = 5e-3
FLOOR = 1e-4
_lib = importlib.import_module("4dgaussians_b200._lib")
rasterizer = importlib.import_module("4dgaussians_b200.rasterizer")


def _cotangents(sc, fwd, mode):
    g = torch.Generator().manual_seed(sum(map(ord, sc.name)) + 11)
    near = torch.from_numpy(threshold_pixels(fwd, sc.W, sc.H, include_stop=True))
    dA = torch.randn(1, sc.H, sc.W, generator=g).double()
    dA[:, near] = 0.0
    dC = dD = None
    if mode == "mixed":
        dC = torch.randn(3, sc.H, sc.W, generator=g).double()
        dD = torch.randn(1, sc.H, sc.W, generator=g).double()
        dC[:, near] = 0.0
        dD[:, near] = 0.0
    return dC, dD, dA, near


@pytest.mark.parametrize("name", ["shape_17x17", "guard_band", "colour_deg3"])
def test_oracle_alpha_is_the_dense_alpha(name):
    sc = ue.scene(name)
    rc, cd = cam_tuple(sc.cam, sc.bg, sh_degree=sc.deg)
    fwd = rr.rasterize_forward(rc, *sc.ins)
    got = ua.oracle_alpha(fwd)
    assert got.dtype == np.float32 and np.array_equal(got[0], np.float32(1.0) - fwd["final_T"])
    ins = [torch.from_numpy(a.astype(np.float64)) for a in sc.ins]
    want = ua.dense_alpha(cd, *ins[:4]).detach().numpy()
    assert float(want.max()) > 0.5
    far = ~threshold_pixels(fwd, sc.W, sc.H, include_stop=True)
    assert float(np.abs(got - want)[:, far].max()) <= 1e-4


def test_colour_is_foreground_plus_transmitted_background():
    sc = ue.scene("shape_17x17")
    bgs = ((0.0, 0.0, 0.0), (0.9, 0.5, 0.2))
    fwds = [rr.rasterize_forward(cam_tuple(sc.cam, bg, sh_degree=sc.deg)[0], *sc.ins) for bg in bgs]
    a = ua.oracle_alpha(fwds[0]).astype(np.float64)
    assert np.array_equal(a, ua.oracle_alpha(fwds[1]))
    diff = fwds[1]["color"].astype(np.float64) - fwds[0]["color"].astype(np.float64)
    want = (1.0 - a) * np.asarray(bgs[1])[:, None, None]
    assert float(np.abs(diff - want).max()) <= 1e-6


@pytest.mark.parametrize("mode", ["alpha", "mixed"])
@pytest.mark.parametrize("name", ue.names())
def test_oracle_alpha_backward_matches_dense_fp64(name, mode):
    sc = ue.scene(name)
    rc, cd = cam_tuple(sc.cam, sc.bg, sh_degree=sc.deg)
    fwd = rr.rasterize_forward(rc, *sc.ins)
    dC, dD, dA, near = _cotangents(sc, fwd, mode)
    assert (~near).float().mean() >= 0.25
    want = ua.dense_grads(cd, sc.ins, dC, dD, dA)
    np_ = lambda t: None if t is None else t.numpy()
    got = ua.oracle_backward(rc, sc.ins, fwd, np_(dC), np_(dD), dA.numpy())
    # as test_raster_edge_scenes: the colour-clamp rows may clamp differently in fp64 (an alpha-only loss reads no colour)
    rows = np.arange(len(sc.ins[0]))
    if mode == "mixed":
        rows = np.setdiff1d(rows, np.concatenate([sc.rows.get("zero", []), sc.rows.get("below", [])]))
    tol = LONG_ROW_TOL if sc.group == "long" else ROW_TOL
    # as test_depth_grad_cpu: a depth term on the long scenes' stacked layers is ill-conditioned in fp32
    floor = 1e-2 if sc.group == "long" and mode == "mixed" else FLOOR
    for nm in ua.NAMES + ("means2D",):
        g = got[nm][:, :2] if nm == "means2D" else got[nm]
        e = row_errors(g[rows], want[nm][rows], floor)
        assert float(e.max()) <= tol, (nm, float(e.max()), int(rows[np.argmax(e)]))
    unseen = fwd["radii"] == 0
    assert not got["opacities"][unseen].any() and np.abs(got["opacities"]).max() > 0
    if mode == "alpha":
        assert not got["shs"].any()         # the alpha reads no colour


def test_two_gaussians_closed_form():
    """At the pixel both are centred on, G = 1: A = 1 - (1 - o1)(1 - o2), so dA/do1 = 1 - o2 and dA/do2 = 1 - o1."""
    o1, o2 = 0.6, 0.7
    cam = ue.origin_camera(16, 16)
    pv = ue.pixel_view(cam, np.array([7.0, 7.0]), np.array([9.0, 9.0]), np.array([2.0, 3.5]))
    ins = [ue.world_of(cam, pv).astype(np.float32), np.full((2, 3), 0.01, np.float32),
           np.tile(np.array([1.0, 0.0, 0.0, 0.0], np.float32), (2, 1)), np.array([[o1], [o2]], np.float32),
           np.zeros((2, 16, 3), np.float32)]
    rc, _ = cam_tuple(cam, (0.0, 0.0, 0.0), sh_degree=0)
    fwd = rr.rasterize_forward(rc, *ins)
    assert abs(float(ua.oracle_alpha(fwd)[0, 9, 7]) - (1 - (1 - o1) * (1 - o2))) < 1e-6
    dA = np.zeros((1, 16, 16), np.float32)
    dA[0, 9, 7] = 1.0
    got = ua.oracle_backward(rc, ins, fwd, None, None, dA)
    np.testing.assert_allclose(got["opacities"].reshape(-1), [1 - o2, 1 - o1], rtol=1e-5)
    assert not got["shs"].any()


# ---- host rules ----------------------------------------------------------------------------------------------------------
def test_setters_are_declared_and_bound():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "g4d.h")).read()
    assert re.search(r"int g4d_context_set_alpha_out\(G4DContext \*ctx, float \*d_out\);", header)
    assert re.search(r"int g4d_context_set_alpha_grad\(G4DContext \*ctx, const float \*d_dL_dalpha\);", header)
    for name in ("g4d_context_set_alpha_out", "g4d_context_set_alpha_grad"):
        assert name in _lib.ABI_SYMBOLS
    assert callable(_lib.Context.set_alpha_out) and callable(_lib.Context.set_alpha_grad)
    assert _lib.ABI_VERSION == 3


class _FakeContext:
    def __init__(self, log, i):
        self.log, self.i = log, i

    def set_depth_grad(self, p):
        self.log.append(("depth", self.i, p))

    def set_alpha_grad(self, p):
        self.log.append(("alpha", self.i, p))

    def set_alpha_out(self, p):
        self.log.append(("out", self.i, p))


def _views(k):
    rs = rasterizer.GaussianRasterizationSettings(4, 3, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0,
                                                  torch.zeros(3), False, False)
    return [rs] * k


def test_view_terms_set_the_alpha_gradient_for_the_call_only():
    log = []
    ctxs = [_FakeContext(log, i) for i in range(3)]
    a2, d0 = torch.zeros(12), torch.zeros(12)
    with rasterizer.ViewTerms(_views(3)).backward(ctxs, torch.device("cpu"), depths=(d0,), alphas=(None, None, a2)):
        assert log == [("depth", 0, d0.data_ptr()), ("alpha", 2, a2.data_ptr())]
    assert log[2:] == [("depth", 0, None), ("alpha", 2, None)]


def test_view_terms_without_an_alpha_gradient_set_nothing():
    log = []
    ctxs = [_FakeContext(log, i) for i in range(2)]
    for alphas in ((), (None, None)):
        with rasterizer.ViewTerms(_views(2)).backward(ctxs, torch.device("cpu"), alphas=alphas):
            pass
    assert log == []


def test_view_terms_set_the_alpha_output_for_the_forward_only():
    log = []
    ctxs = [_FakeContext(log, i) for i in range(2)]
    terms = rasterizer.ViewTerms(_views(2), alpha=True)
    outs = terms.outputs(torch.device("cpu"), 5)[3]
    assert [tuple(a.shape) for a in outs] == [(1, 4, 3), (1, 4, 3)]
    with pytest.raises(RuntimeError):
        with terms.forward(ctxs, outs):
            assert log == [("out", 0, outs[0].data_ptr()), ("out", 1, outs[1].data_ptr())]
            raise RuntimeError("a failed forward")
    assert log[2:] == [("out", 0, None), ("out", 1, None)]
    log.clear()
    no_alpha = rasterizer.ViewTerms(_views(2))
    assert no_alpha.outputs(torch.device("cpu"), 5)[3] == []
    with no_alpha.forward(ctxs, []):
        pass
    assert log == []
