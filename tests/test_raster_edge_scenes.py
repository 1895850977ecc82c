"""CPU companion of test_gpu_raster_edges.py: every scene it renders (util_raster_edges.py) reaches its condition on the oracle,
the oracle equals the dense fp64 autograd formulation (oracle/dense_ref.py) on it, forward and backward per row, and the
checks that matter would catch a kernel that lost the guard-band clamp of the backward or the 0.99 clamp of alpha.

Pixels with an instance within rounding of a compositing threshold (util_scene.threshold_pixels) are left out of the image
comparison and get no upstream gradient: there fp64 may take the other branch.  Two clamped layers sit on one of them by
construction: (1 - 0.99f)^2 = 9.999981e-5 stops the pixel in fp32, (1 - 0.99)^2 = 1.0000000000000018e-4 does not in fp64."""
import numpy as np
import pytest
import torch

from oracle import raster_ref as rr
from oracle.dense_ref import dense_render
import util_raster_edges as ue
from util_scene import cam_tuple, row_errors, threshold_pixels

ROW_TOL = 2e-3
LONG_ROW_TOL = 5e-3     # 257-1100 layers: the fp32 backward recovers T by dividing by (1 - alpha) once per layer
FLOOR = 1e-4
NAMES = ("means3D", "scales", "rots", "opacities", "shs")


def _oracle(sc):
    rc, cd = cam_tuple(sc.cam, sc.bg, sh_degree=sc.deg)
    return rc, cd, rr.rasterize_forward(rc, *sc.ins)


def _upstream(sc, fwd):
    g = torch.Generator().manual_seed(sum(map(ord, sc.name)))
    dL = torch.randn(3, sc.H, sc.W, generator=g).double()
    near = threshold_pixels(fwd, sc.W, sc.H, include_stop=True)
    dL[:, torch.from_numpy(near)] = 0.0
    return dL, near


def _dense(sc, cd, dL, **flags):
    ins = [torch.from_numpy(a.astype(np.float64)).requires_grad_(True) for a in sc.ins]
    off = torch.zeros(len(sc.ins[0]), 2, dtype=torch.float64, requires_grad=True)
    d = dense_render(cd, *ins, pix_offset=off, **flags)
    (d["color"] * dL).sum().backward()
    g = {nm: t.grad.numpy().reshape(a.shape) for nm, t, a in zip(NAMES, ins, sc.ins)}
    g["means2D"] = off.grad.numpy() * np.array([0.5 * sc.W, 0.5 * sc.H])       # means2D gradients are in NDC units
    return d, g


@pytest.mark.parametrize("name", ue.names())
def test_scene_reaches_its_condition(name):
    sc = ue.scene(name)
    _, _, fwd = _oracle(sc)
    sc.claim(sc, ue.oracle_record(fwd))


@pytest.mark.parametrize("name", ue.names())
def test_oracle_matches_dense_fp64(name):
    sc = ue.scene(name)
    rc, cd, fwd = _oracle(sc)
    dL, near = _upstream(sc, fwd)
    d, want = _dense(sc, cd, dL)
    # radii of hundreds of pixels are the ceiling of an fp32 square root: a few land one pixel apart from fp64 (rects agree)
    dr = np.abs(fwd["radii"].astype(np.int64) - d["radii"].numpy())
    assert dr.max() <= 1 and (dr > 0).mean() <= 0.01 and (fwd["radii"][dr > 0] > 100).all()
    assert np.array_equal(fwd["proj"].rect, d["rect"].numpy())
    keep = ~near
    assert keep.mean() >= 0.25, keep.mean()
    err = np.abs(fwd["color"] - d["color"].detach().numpy()).max(axis=0)
    assert float(err[keep].max()) < 2e-5, float(err[keep].max())
    assert np.array_equal(fwd["n_contrib"][keep], d["n_contrib"].numpy()[keep])
    got = rr.rasterize_backward(rc, *sc.ins, fwd, dL.numpy().astype(np.float32))
    # the colour-clamp rows sit on max(colour + 0.5, 0) in fp32; fp64 evaluates the SH sum to another rounding and may
    # clamp where fp32 does not (they are compared bit for bit with the oracle on the host build and the GPU)
    rows = np.setdiff1d(np.arange(len(sc.ins[0])), np.concatenate([sc.rows.get("zero", []), sc.rows.get("below", [])]))
    tol = LONG_ROW_TOL if sc.group == "long" else ROW_TOL
    for nm in NAMES + ("means2D",):
        g = got[nm][:, :2] if nm == "means2D" else got[nm]
        e = row_errors(g[rows], want[nm][rows], FLOOR)
        assert float(e.max()) <= tol, (nm, float(e.max()), int(rows[np.argmax(e)]))
    vis = fwd["radii"] > 0
    assert np.abs(want["means3D"][vis]).max() > 0


def _guard_rows(sc, fwd):
    cx, cy = ue.guard_flags(sc.cam, sc.ins[0])
    return np.nonzero((cx | cy) & (fwd["radii"] > 0))[0]


def test_guard_band_gradient_check_is_sensitive():
    """passing the gradient through a clamped t.x / t.y (a kernel without `clampx ? 0.f :`) moves every guard-band-clamped row
    of the means3D gradient by more than 5 ROW_TOL of the row, and some by more than 10 %"""
    sc = ue.scene("guard_band")
    rc, cd, fwd = _oracle(sc)
    dL, _ = _upstream(sc, fwd)
    _, ref = _dense(sc, cd, dL)
    _, alt = _dense(sc, cd, dL, guard_band_grad=True)
    rows = _guard_rows(sc, fwd)
    assert len(rows) >= 4
    e = row_errors(alt["means3D"][rows], ref["means3D"][rows], 0.0)
    assert (e > 5 * ROW_TOL).all() and e.max() > 0.1, e
    others = np.setdiff1d(np.arange(len(sc.ins[0])), rows)
    assert np.array_equal(alt["means3D"][others], ref["means3D"][others])


@pytest.mark.parametrize("opacity", ue.OPAQUE_OPACITIES)
@pytest.mark.parametrize("layers,thin", [(1, 0), (2, 0), (2, 3)])
def test_alpha_clamp_gradient_check_is_sensitive(opacity, layers, thin):
    """a blend kernel without fminf(0.99, ...) changes the image on the clamped core by far more than the 1e-4 the GPU test
    allows, and, with a second clamped layer, the gradient of a clamped layer by more than 5 ROW_TOL of its row.
    (A single layer over the background has d colour / d alpha = colour - bg whatever alpha is: only the image shows it.)"""
    sc = ue.scene("opaque_o%g_l%d_t%d" % (opacity, layers, thin))
    rc, cd, fwd = _oracle(sc)
    dL, _ = _upstream(sc, fwd)
    d_ref, ref = _dense(sc, cd, dL)
    d_alt, alt = _dense(sc, cd, dL, alpha_clamp=False)
    core = ue.all_clamped_pixels(ue.oracle_record(fwd), sc.W, sc.H) if thin == 0 else np.ones((sc.H, sc.W), bool)
    diff = np.abs(d_alt["color"].detach().numpy() - d_ref["color"].detach().numpy()).max(axis=0)
    assert float(diff[core].max()) > 1e-3, float(diff[core].max())
    if layers > 1 and thin == 0:
        rows = sc.rows["opaque"]
        e = max(float(row_errors(alt[nm][rows], ref[nm][rows], 0.0).max()) for nm in ("opacities", "means2D", "means3D"))
        assert e > 5 * ROW_TOL, e
