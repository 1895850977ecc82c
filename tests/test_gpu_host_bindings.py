"""Which C-ABI entry points each Python binding calls, and in which order.

A recorder replaces every g4d_* function of the loaded library with one that notes the name and forwards the call
unchanged.  Each case runs once unrecorded, so that the workspace, the context pool and the packed weight images exist,
and then once recorded: the recorded names are the whole host-to-library traffic of that call.  A one-camera
render_cameras() runs the single-camera entry points, as render() does.
"""
import importlib

import pytest
import torch

from util_scene import g4d, make_module, synth

_lib = importlib.import_module("4dgaussians_b200._lib")
losses = importlib.import_module("4dgaussians_b200.losses")
renderer = importlib.import_module("4dgaussians_b200.renderer")
simple_knn = importlib.import_module("4dgaussians_b200.simple_knn")
train_dp = importlib.import_module("4dgaussians_b200.train_dp")

pytestmark = pytest.mark.gpu

W, H, T = 64, 48, 0.4
FWD, BWD = "g4d_render_forward", "g4d_render_backward"
FWD_CAMS, BWD_CAMS = "g4d_render_forward_cameras", "g4d_render_backward_cameras"


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


def _cameras(k):
    return [synth.make_camera(20.0 + 50.0 * i, W, H, radius=3.0, time=T) for i in range(k)]


@pytest.fixture(scope="module")
def scene():
    return synth.make_scene(600, seed=5, scale_mean=0.06)


@pytest.fixture
def pc(scene):
    return synth.SyntheticGaussianModel(scene, make_module("small64", seed=1, aabb=scene["aabb"]), sh_degree=3,
                                        requires_grad=True)


@pytest.fixture
def bg():
    return torch.tensor([0.1, 0.2, 0.3], device="cuda")


@pytest.fixture
def recorded(monkeypatch):
    lib = _lib.load()
    calls = []

    def recorder(name, fn):
        def call(*args):
            calls.append(name)
            return fn(*args)
        return call
    for name in _lib.ABI_SYMBOLS:
        monkeypatch.setattr(lib, name, recorder(name, getattr(lib, name)))

    def run(fn):
        fn()
        torch.cuda.synchronize()
        calls.clear()
        fn()
        torch.cuda.synchronize()
        return list(calls)
    return run


@pytest.mark.parametrize("grad", [True, False])
@pytest.mark.parametrize("stage", ["fine", "coarse"])
def test_render(recorded, pc, bg, stage, grad):
    cam = _cameras(1)[0]

    def run():
        with torch.set_grad_enabled(grad):
            out = g4d.render(cam, pc, _Pipe, bg, stage=stage)
        if grad:
            out["render"].sum().backward()
    assert recorded(run) == ([FWD, BWD] if grad else [FWD])


@pytest.mark.parametrize("grad", [True, False])
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("stage", ["fine", "coarse"])
def test_render_cameras(recorded, pc, bg, stage, k, grad):
    cams = _cameras(k)

    def run():
        with torch.set_grad_enabled(grad):
            outs = g4d.render_cameras(cams, pc, _Pipe, bg, stage=stage)
        if grad:
            sum(o["render"].sum() for o in outs).backward()
    fwd, bwd = (FWD, BWD) if k == 1 else (FWD_CAMS, BWD_CAMS)
    assert recorded(run) == ([fwd, bwd] if grad else [fwd])


def test_rasterizer(recorded, scene, pc, bg):
    rs, _ = renderer.settings_from_camera(_cameras(1)[0], pc, _Pipe, bg)
    n = scene["xyz"].shape[0]
    leaf = lambda t: t.detach().float().cuda().requires_grad_(True)
    m3, m2 = leaf(scene["xyz"]), leaf(torch.zeros(n, 3))
    shs = leaf(torch.cat([scene["features_dc"], scene["features_rest"]], dim=1))
    op, sc = leaf(torch.sigmoid(scene["opacity"])), leaf(torch.exp(scene["scaling"]))
    ro = leaf(torch.nn.functional.normalize(scene["rotation"], dim=-1))

    def run():
        img, _, _ = g4d.GaussianRasterizer(rs)(means3D=m3, means2D=m2, shs=shs, colors_precomp=None, opacities=op, scales=sc,
                                               rotations=ro, cov3D_precomp=None)
        img.sum().backward()
    assert recorded(run) == ["g4d_rasterize_forward", "g4d_rasterize_backward"]


def test_deform_network(recorded, scene, pc):
    leaf = lambda t: t.detach().float().cuda().requires_grad_(True)
    x, s, r, o = leaf(scene["xyz"]), leaf(scene["scaling"]), leaf(scene["rotation"]), leaf(scene["opacity"])
    sh = leaf(torch.cat([scene["features_dc"], scene["features_rest"]], dim=1))

    def run():
        outs = pc._deformation(x, s, r, o, sh, torch.full((x.shape[0], 1), T, device="cuda"))
        sum(t.sum() for t in outs).backward()
    assert recorded(run) == ["g4d_deform_forward", "g4d_deform_backward"]


def test_losses_and_knn(recorded, scene, pc):
    gen = torch.Generator(device="cuda").manual_seed(3)
    img = torch.rand(3, H, W, device="cuda", generator=gen).requires_grad_(True)
    gt = torch.rand(3, H, W, device="cuda", generator=gen)
    mod = pc._deformation

    def l1():
        losses.l1_loss(img, gt).backward()

    def ssim():
        losses.ssim(img, gt).backward()

    def regulation():
        losses.compute_regulation(mod, 0.001, 0.0001, 0.0002).backward()

    def accumulate():
        for lvl in mod.deformation_net.grid.grids:
            for p in lvl:
                p.grad = torch.zeros_like(p)
        losses.accumulate_regulation(mod, 0.001, 0.0001, 0.0002, loss_accum=torch.zeros((), device="cuda"))

    def knn():
        simple_knn.distCUDA2(scene["xyz"].cuda())
    assert recorded(l1) == ["g4d_l1_loss", "g4d_l1_loss_backward"]
    assert recorded(ssim) == ["g4d_ssim", "g4d_ssim_backward"]
    assert recorded(regulation) == ["g4d_plane_regulation"]
    assert recorded(accumulate) == ["g4d_plane_regulation"]
    assert recorded(knn) == ["g4d_dist2_knn3"]


def test_dp_trainer_step(recorded, scene, bg):
    gs = train_dp.GaussianSet(scene, make_module("small64", seed=1, aabb=scene["aabb"]), device="cuda", sh_degree=3)
    tr = train_dp.DPTrainer(gs, train_dp.default_opt(), cameras_extent=2.6)
    cams = _cameras(2)
    target = torch.rand(3, H, W, device="cuda")

    def run():
        tr.step(cams, [target] * 2, bg, _Pipe)
    view = [FWD, "g4d_l1_loss", "g4d_l1_loss_backward", BWD]
    assert recorded(run) == view * 2 + ["g4d_plane_regulation", "g4d_adam_step"]
