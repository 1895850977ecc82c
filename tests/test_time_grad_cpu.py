"""CPU: the time gradient's oracle -- the reference's own deform_network with one time leaf for every row, then the fp64
dense render -- pinned by central differences; the kernel's formula for dL/dt from the collapsed time rows' gradients
(util_time_grad.time_grad_from_rows) against that oracle's autograd, the border included; and the host rules: which
camera times take a gradient, the render_cameras refusal raised before anything runs, the C-ABI's NULL-context refusal."""
import importlib
import math

import pytest
import torch

import util_time_grad as utg
from util_camera_grad import central_differences
from oracle import deform_ref as dr
from oracle import ref_loader
from oracle.dense_ref import cam_dict_from, dense_render
from util_deep_network import reference_module
from util_scene import synth

renderer = importlib.import_module("4dgaussians_b200.renderer")
rasterizer = importlib.import_module("4dgaussians_b200.rasterizer")
_lib = importlib.import_module("4dgaussians_b200._lib")

needs_reference = pytest.mark.skipif(not ref_loader.reference_available(), reason="reference module not available")
AABB = torch.tensor([[1.31, 1.27, 1.3], [-1.29, -1.3, -1.22]])
CFG = dr.CONFIGS["tiny"]        # T = 7 time rows, channels 4, every head active
T = CFG.resolution[3]


def _scene(n=4, seed=0, W=24, H=20):
    """n Gaussians near the origin in front of a camera at radius 3, pre-activation tensors in fp64; a random cotangent"""
    cam = synth.make_camera(25.0, W, H, radius=3.0)
    g = torch.Generator().manual_seed(seed)
    xyz = (torch.rand(n, 3, generator=g, dtype=torch.float64) - 0.5) * 0.6
    scales = torch.log(0.15 + 0.1 * torch.rand(n, 3, generator=g, dtype=torch.float64))
    rots = torch.nn.functional.normalize(torch.randn(n, 4, generator=g, dtype=torch.float64), dim=1)
    opac = torch.randn(n, 1, generator=g, dtype=torch.float64) * 0.3
    shs = torch.randn(n, 16, 3, generator=g, dtype=torch.float64) * 0.3
    cot = torch.randn(3, H, W, generator=g, dtype=torch.float64)
    return cam_dict_from(cam, (0.1, 0.2, 0.3), 3), (xyz, scales, rots, opac, shs), cot


def _reference_net(seed=3):
    prm = dr.random_params(CFG, seed=seed, aabb=AABB, dtype=torch.float64)
    net = reference_module(CFG, 1).double()
    sd = net.state_dict()
    sd.update(dr.params_to_state_dict(prm))
    net.load_state_dict(sd)
    return net, prm


def _render_ref(net, cd, inputs, t):
    """the dense render of the reference module's deformation at time t ([1, 1] fp64), every row at t"""
    xyz, scales, rots, opac, shs = inputs
    pts, sc, rot, op, sh = net(xyz, scales, rots, opac, shs, t.expand(xyz.shape[0], 1))
    s, r, o = dr.activate(sc, rot, op)
    return dense_render(cd, pts, s, r, o, sh)


def _decisions(out):
    return out["radii"], out["rect"], out["n_contrib"]


@needs_reference
@pytest.mark.parametrize("t0,seed", [(1.0 / 6.0, 0), (-0.55, 1), (0.55, 2)])
def test_reference_time_grad_vs_central_differences(t0, seed):
    assert 0.2 <= utg.texel_row_fraction(t0, T) <= 0.8        # no texel row within the step
    net, _ = _reference_net(seed + 3)
    cd, inputs, cot = _scene(seed=seed)
    t = torch.tensor([[t0]], dtype=torch.float64, requires_grad=True)
    out = _render_ref(net, cd, inputs, t)
    assert (out["radii"] > 0).sum() >= 2
    (out["color"] * cot).sum().backward()
    centre = _decisions(out)

    def loss(x):
        o = _render_ref(net, cd, inputs, x.reshape(1, 1))
        for a, b in zip(_decisions(o), centre):
            assert torch.equal(a, b), "a discrete decision flipped within the step"
        return float((o["color"] * cot).sum())

    with torch.no_grad():
        fd = central_differences(loss, torch.tensor([t0], dtype=torch.float64), 1e-6)
    got = float(t.grad)
    assert abs(got) > 1e-6
    assert abs(got - float(fd)) <= 1e-6 * max(1.0, abs(float(fd))), (got, float(fd))


def _row_grads(prm, cd, inputs, cot, t0):
    """the gradients of the collapsed time rows r = w0 P[i0] + w1 P[i1] at t0: each (axis, t) plane replaced by its row
    (two equal copies, so that any t inside (-1, 1) samples exactly the row), fp64 autograd through the dense render"""
    hi = T - 1
    x = min(max((t0 + 1.0) / 2.0 * hi, 0.0), hi)
    i0 = int(math.floor(x))
    i1 = min(i0 + 1, T - 1)
    w1 = x - i0
    planes, rows = [], []
    for lvl in prm.planes:
        lp, lr = [], []
        for k, (c0, c1) in enumerate(dr.PLANE_AXES):
            P = lvl[k].detach()
            if c1 == 3:
                r = ((1.0 - w1) * P[:, :, i0:i0 + 1, :] + w1 * P[:, :, i1:i1 + 1, :]).clone().requires_grad_(True)
                lr.append(r)
                P = torch.cat([r, r], dim=2)
            lp.append(P)
        planes.append(lp)
        rows.append(lr)
    p = dr.DeformParams(aabb=prm.aabb, planes=planes, w0=prm.w0, b0=prm.b0, heads=prm.heads)
    xyz, scales, rots, opac, shs = inputs
    pts, sc, rot, op, sh = dr.deform_forward(CFG, p, xyz, scales, rots, opac, shs, 0.0)
    s, r, o = dr.activate(sc, rot, op)
    (dense_render(cd, pts, s, r, o, sh)["color"] * cot).sum().backward()
    return [[q.grad[0, :, 0, :].numpy() for q in lr] for lr in rows]


@needs_reference
@pytest.mark.parametrize("t0", [1.0 / 6.0, -0.55, 1.0, 1.5, -1.0])
def test_kernel_formula_matches_reference_autograd(t0):
    net, prm = _reference_net(7)
    cd, inputs, cot = _scene(n=5, seed=4)
    t = torch.tensor([[t0]], dtype=torch.float64, requires_grad=True)
    (_render_ref(net, cd, inputs, t)["color"] * cot).sum().backward()
    ref = float(t.grad)
    row_grads = _row_grads(prm, cd, inputs, cot, t0)
    planes = [[prm.planes[l][k][0].detach().numpy() for k in (2, 4, 5)] for l in range(CFG.levels)]
    got = utg.time_grad_from_rows(planes, row_grads, t0, T)
    if abs(t0) >= 1.0:
        assert ref == 0.0 and got == 0.0
    else:
        assert abs(ref) > 1e-6
        assert abs(got - ref) <= 1e-9 * max(1.0, abs(ref)), (got, ref)


# ---- host rules ----------------------------------------------------------------------------------------------------------
class _Cam:
    def __init__(self, time):
        self.time = time


def test_which_times_take_a_gradient():
    leaf0 = torch.tensor(0.25, requires_grad=True)
    leaf1 = torch.tensor([0.25], requires_grad=True)
    assert renderer.time_grad_leaf([_Cam(0.25)]) is None
    assert renderer.time_grad_leaf([_Cam(0)]) is None
    assert renderer.time_grad_leaf([_Cam(torch.tensor(0.25))]) is None
    assert renderer.time_grad_leaf([_Cam(leaf0)]) is leaf0
    assert renderer.time_grad_leaf([_Cam(leaf1), _Cam(leaf1)]) is leaf1
    assert renderer.time_grad_leaf([{"time": leaf0, "camera": None}], cam_type="PanopticSports") is leaf0
    with torch.no_grad():
        assert renderer.time_grad_leaf([_Cam(leaf0)]) is None
    with pytest.raises(ValueError, match="one element"):
        renderer.time_grad_leaf([_Cam(torch.zeros(3, 1, requires_grad=True))])


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


@pytest.mark.parametrize("times", ["distinct", "mixed"])
def test_render_cameras_refuses_distinct_time_tensors(times):
    a = torch.tensor(0.25, requires_grad=True)
    b = torch.tensor(0.25, requires_grad=True) if times == "distinct" else 0.25
    # refused before the model, the settings or the device are looked at: no model is needed
    with pytest.raises(ValueError, match="render\\(\\) per camera"):
        renderer.render_cameras([_Cam(a), _Cam(b)], None, _Pipe, None)


class _FakeContext:
    def __init__(self, log, i):
        self.log, self.i = log, i

    def set_time_grad(self, p):
        self.log.append(("time", self.i, p))


def test_view_terms_return_the_time_grad_of_camera_0_in_the_callers_layout():
    rs = rasterizer.GaussianRasterizationSettings(4, 3, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0,
                                                  torch.zeros(3), False, False)
    for leaf in (torch.tensor(0.0, dtype=torch.float64), torch.zeros(1, 1, dtype=torch.float16), torch.zeros(1)):
        log = []
        terms = rasterizer.ViewTerms([rs, rs], time_leaf=leaf)
        assert terms.leaves[0] is leaf
        with terms.backward([_FakeContext(log, 0), _FakeContext(log, 1)], "cpu"):
            assert log == [("time", 0, terms.time_sink.data_ptr())]
            terms.time_sink.fill_(2.5)
        assert log[1:] == [("time", 0, None)]
        (g,) = terms.leaf_grads()
        assert g.shape == leaf.shape and g.dtype == leaf.dtype and float(g.reshape(-1)[0]) == 2.5


def test_set_time_grad_null_context():
    assert _lib.load().g4d_context_set_time_grad(None, None) == -2
