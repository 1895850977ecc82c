"""CPU: the fp64 dense oracle with the camera tensors as leaves (util_camera_grad) pinned by central differences on all 35
entries -- view [16], proj [16], campos [3] -- on scenes of 1-3 Gaussians where no discrete decision flips within the step;
the chain through a pose (R, T -> getWorld2View2 / getProjectionMatrix -> dense render); and the host side of the Python
surface: which camera tensors join the autograd graph, and the refusals raised before any launch."""
import importlib
import math

import numpy as np
import pytest
import torch

import util_camera_grad as ucg
from oracle.dense_ref import cam_dict_from, dense_render
from util_scene import synth

rasterizer = importlib.import_module("4dgaussians_b200.rasterizer")
_lib = importlib.import_module("4dgaussians_b200._lib")


def _tiny(n, seed, deg, W=24, H=20, theta=25.0, radius=3.0):
    """n Gaussians well inside the view (off the guard band, in front of the near plane), large enough to cover pixels"""
    cam = synth.make_camera(theta, W, H, radius=radius)
    g = torch.Generator().manual_seed(seed)
    wv = cam.world_view_transform.double()
    inv = torch.linalg.inv(wv)
    pv = torch.stack([(torch.rand(n, generator=g, dtype=torch.float64) - 0.5) * 0.6,
                      (torch.rand(n, generator=g, dtype=torch.float64) - 0.5) * 0.5,
                      2.5 + torch.rand(n, generator=g, dtype=torch.float64)], dim=1)
    means = (torch.cat([pv, torch.ones(n, 1, dtype=torch.float64)], 1) @ inv)[:, :3]
    scales = 0.15 + 0.1 * torch.rand(n, 3, generator=g, dtype=torch.float64)
    rots = torch.nn.functional.normalize(torch.randn(n, 4, generator=g, dtype=torch.float64), dim=1)
    opac = 0.3 + 0.4 * torch.rand(n, 1, generator=g, dtype=torch.float64)
    shs = torch.randn(n, 16, 3, generator=g, dtype=torch.float64) * 0.3
    cd = cam_dict_from(cam, (0.1, 0.2, 0.3), deg)
    cot = torch.randn(3, H, W, generator=g, dtype=torch.float64)
    return cam, cd, (means, scales, rots, opac, shs), cot


def _decisions(out):
    return out["radii"], out["rect"], out["n_contrib"]


def _loss(cd, inputs, cot, centre, **cam):
    """the loss at a perturbed camera, after checking that no discrete decision moved from the centre's (radii, tile
    rects, per-pixel contributor counts): central differences only mean something where the forward is smooth"""
    out = dense_render(dict(cd, **cam), *inputs)
    for a, b in zip(_decisions(out), centre):
        assert torch.equal(a, b), "a discrete decision flipped within the step"
    return float((out["color"] * cot).sum())


@pytest.mark.parametrize("n,deg,seed", [(1, 0, 0), (2, 3, 1), (3, 3, 2), (3, 1, 3)])
def test_dense_camera_grads_vs_central_differences(n, deg, seed):
    _, cd, inputs, cot = _tiny(n, seed, deg)
    out, got = ucg.dense_camera_grads(cd, inputs, cot)
    assert (out["radii"] > 0).all()
    for key, eps in (("view", 1e-6), ("proj", 1e-6), ("campos", 1e-6)):
        x0 = torch.as_tensor(np.asarray(cd[key], np.float64)).reshape(-1)
        fd = ucg.central_differences(lambda x: _loss(cd, inputs, cot, _decisions(out), **{key: x}), x0, eps)
        err = (got[key] - fd).abs().max()
        assert err <= 1e-5 * max(1.0, float(fd.abs().max())), (key, got[key], fd)
    for i in range(16):
        if i not in ucg.VIEW_READ:
            assert float(got["view"][i]) == 0.0
        if i not in ucg.PROJ_READ:
            assert float(got["proj"][i]) == 0.0
    if deg == 0:
        assert float(got["campos"].abs().max()) == 0.0
    else:
        assert float(got["campos"].abs().max()) > 0.0


def test_pose_chain_vs_central_differences():
    cam, cd, inputs, cot = _tiny(3, 7, 3)
    R0, T0 = ucg.pose_of(cam)
    wv, full, centre = ucg.camera_tensors(R0, T0, cam.FoVx, cam.FoVy)
    # the restated chain rebuilds the camera the synth module made (to fp32 rounding)
    assert torch.allclose(wv, cam.world_view_transform.double(), atol=1e-6)
    assert torch.allclose(full, cam.full_proj_transform.double(), atol=1e-5)
    assert torch.allclose(centre, cam.camera_center.double(), atol=1e-5)

    base = _decisions(dense_render(cd, *inputs))

    def loss(R, T):
        wv, full, centre = ucg.camera_tensors(R, T, cam.FoVx, cam.FoVy)
        out = dense_render(dict(cd, view=wv.reshape(-1), proj=full.reshape(-1), campos=centre), *inputs)
        for a, b in zip(_decisions(out), base):
            assert torch.equal(a, b), "a discrete decision flipped within the step"
        return (out["color"] * cot).sum()

    R, T = R0.clone().requires_grad_(True), T0.clone().requires_grad_(True)
    loss(R, T).backward()
    fd_R = ucg.central_differences(lambda x: float(loss(x.reshape(3, 3), T0)), R0.reshape(-1), 1e-6).reshape(3, 3)
    fd_T = ucg.central_differences(lambda x: float(loss(R0, x)), T0, 1e-6)
    assert (R.grad - fd_R).abs().max() <= 1e-5 * max(1.0, float(fd_R.abs().max()))
    assert (T.grad - fd_T).abs().max() <= 1e-5 * max(1.0, float(fd_T.abs().max()))
    assert float(T.grad.abs().max()) > 0


def _settings(view, proj, campos):
    return rasterizer.GaussianRasterizationSettings(8, 8, 0.5, 0.5, torch.zeros(3), 1.0, view, proj, 3, campos, False, False)


def test_camera_grad_leaves():
    v, p, c = torch.eye(4), torch.eye(4), torch.zeros(3)
    assert rasterizer.camera_grad_leaves([_settings(v, p, c)]) == ((), ())
    vl, cl = v.clone().requires_grad_(True), c.clone().requires_grad_(True)
    spec, leaves = rasterizer.camera_grad_leaves([_settings(v, p, c), _settings(vl, p, cl)])
    assert spec == ((1, 0), (1, 2)) and leaves[0] is vl and leaves[1] is cl
    with torch.no_grad():
        assert rasterizer.camera_grad_leaves([_settings(vl, p, cl)]) == ((), ())


class _FakeContext:
    def __init__(self, log, i):
        self.log, self.i = log, i

    def set_camera_grad(self, p):
        self.log.append(("camera", self.i, p))


def test_view_terms_return_camera_grads_in_the_callers_layout():
    v, p, c = torch.eye(4), torch.eye(4), torch.zeros(3)
    leaves = (torch.zeros(4, 4, dtype=torch.float64, requires_grad=True), torch.zeros(16, requires_grad=True),
              torch.zeros(1, 3, dtype=torch.float16, requires_grad=True))
    terms = rasterizer.ViewTerms([_settings(v, p, c), _settings(*leaves)])
    assert terms.cam_spec == ((1, 0), (1, 1), (1, 2)) and all(a is b for a, b in zip(terms.leaves, leaves))
    log = []
    with terms.backward([_FakeContext(log, 0), _FakeContext(log, 1)], "cpu"):
        assert log == [("camera", 1, terms.cam_sink[1].data_ptr())]
        terms.cam_sink[1].copy_(torch.arange(35, dtype=torch.float32))
    assert log[1:] == [("camera", 1, None)]
    gv, gp, gc = terms.leaf_grads()
    assert gv.shape == (4, 4) and gv.dtype == torch.float64 and gv.reshape(-1).tolist() == list(range(16))
    assert gp.shape == (16,) and gp.tolist() == list(range(16, 32))
    assert gc.shape == (1, 3) and gc.dtype == torch.float16 and gc.reshape(-1).tolist() == [32, 33, 34]


@pytest.mark.parametrize("field,n", [("viewmatrix", 12), ("projmatrix", 9), ("campos", 4)])
def test_refuses_wrong_sized_cpu_camera_tensors(field, n):
    kw = dict(view=torch.eye(4), proj=torch.eye(4), campos=torch.zeros(3))
    kw[{"viewmatrix": "view", "projmatrix": "proj", "campos": "campos"}[field]] = torch.zeros(n, requires_grad=True)
    with pytest.raises(RuntimeError, match="%s has %d elements, expected" % (field, n)):
        rasterizer.camera_from_settings(_settings(**kw))


def test_set_camera_grad_null_context():
    assert _lib.load().g4d_context_set_camera_grad(None, None) == -2
