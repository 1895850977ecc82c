"""render_cameras: one timestamp seen by several cameras in one call (g4d_render_forward_cameras / _backward_cameras).

The deformation runs once; every extra camera is projected from camera 0's stored deformed tensors, which are the very
floats the fused kernels project from, so each camera's records must equal those of its own render() bit for bit and its
image within 1e-6.  Gradients are sums over the cameras and must equal the sum of separate render() backward passes to the
2e-5 x max bound of test_batched_views_single_backward_matches_per_view_backward (fp32 atomics in another order).
"""
import ctypes as C
import importlib

import numpy as np
import pytest
import torch

from util_scene import g4d, make_module, oracle_params_from_module, oracle_render, rel_err, synth

_lib = importlib.import_module("4dgaussians_b200._lib")
build = importlib.import_module("4dgaussians_b200.build")
renderer = importlib.import_module("4dgaussians_b200.renderer")

IMG_TOL = 1e-4
GRAD_TOL = 2e-3
SUM_TOL = 2e-5


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


# FFMA path (small64), tensor-core path (small128, dynerf with the SHS head, c32w128sh)
CASES = [dict(net="small64", n=900, wh=(96, 64), theta=20.0, radius=4.0, t=0.3, deg=3, bg=(1.0, 1.0, 1.0), scale=0.08),
         dict(net="small128", n=1100, wh=(80, 112), theta=-50.0, radius=2.0, t=0.8, deg=2, bg=(0.0, 0.0, 0.0), scale=0.05),
         dict(net="dynerf", n=2500, wh=(203, 152), theta=100.0, radius=2.2, t=0.5, deg=3, bg=(0.0, 0.0, 0.0), scale=0.04),
         dict(net="c32w128sh", n=1300, wh=(120, 90), theta=30.0, radius=2.4, t=0.6, deg=3, bg=(0.2, 0.1, 0.0), scale=0.05)]


def _setup(c, grad):
    scene = synth.make_scene(c["n"], seed=11, scale_mean=c["scale"])
    mod = make_module(c["net"], seed=2, aabb=scene["aabb"])
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=c["deg"], requires_grad=grad)
    return scene, mod, pc


def _cameras(c, extra=()):
    """three cameras at the case's time, the third with another image size"""
    W, H = c["wh"]
    cams = [synth.make_camera(c["theta"], W, H, radius=c["radius"], time=c["t"]),
            synth.make_camera(c["theta"] + 55.0, W, H, radius=c["radius"] * 1.1, time=c["t"]),
            synth.make_camera(c["theta"] - 80.0, W + 37, H - 11, radius=c["radius"], time=c["t"])]
    return cams + list(extra)


def _blind_camera(c):
    """a camera every Gaussian is behind: it sees nothing"""
    cam = synth.make_camera(c["theta"], c["wh"][0], c["wh"][1], radius=c["radius"], time=c["t"])
    proj = torch.linalg.inv(cam.world_view_transform) @ cam.full_proj_transform
    cam.world_view_transform = cam.world_view_transform.clone()
    cam.world_view_transform[3, 2] -= 100.0
    cam.full_proj_transform = (cam.world_view_transform @ proj).contiguous()
    return cam


def _ctx_reads(ctx):
    return ctx.read("rect"), ctx.read("depth")


# ----------------------------------------------------------------------------------------------------------- no GPU
def _cpu_model(n=16):
    return synth.SyntheticGaussianModel(synth.make_scene(n, seed=1), None, device="cpu")


def test_mismatched_times_raise_value_error():
    pc = _cpu_model()
    cams = [synth.make_camera(0.0, 32, 32, time=0.5), synth.make_camera(40.0, 32, 32, time=0.5000001)]
    with pytest.raises(ValueError, match="times differ"):
        g4d.render_cameras(cams, pc, _Pipe, torch.zeros(3))


def test_camera_count_is_bounded():
    pc = _cpu_model()
    with pytest.raises(ValueError, match="at most 32"):
        g4d.render_cameras([synth.make_camera(10.0 * i, 16, 16) for i in range(_lib.MAX_CAMERAS + 1)], pc, _Pipe, torch.zeros(3))
    with pytest.raises(ValueError, match="at least one"):
        g4d.render_cameras([], pc, _Pipe, torch.zeros(3))


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def _c_cameras(times, wh=(32, 24)):
    cams = (_lib.Camera * len(times))()
    for i, t in enumerate(times):
        cams[i].image_width, cams[i].image_height = wh
        cams[i].tanfovx = cams[i].tanfovy = 0.5
        cams[i].scale_modifier = 1.0
        cams[i].time = t
    return cams


def test_c_abi_refuses_bad_camera_groups_before_touching_a_device(lib):
    """The camera checks come first: they need neither contexts nor a device."""
    cams = _c_cameras([0.25, 0.25, 0.5])
    rc =lib.g4d_render_forward_cameras(None, 3, cams, None, None, None, None, None, None)
    assert rc == -2 and b"time" in lib.g4d_last_error()
    rc = lib.g4d_render_backward_cameras(None, 3, cams, None, None, None, None, None, None, None)
    assert rc == -2 and b"time" in lib.g4d_last_error()
    for k in (0, _lib.MAX_CAMERAS + 1):
        assert lib.g4d_render_forward_cameras(None, k, _c_cameras([0.0]), None, None, None, None, None, None) == -2
        assert lib.g4d_render_backward_cameras(None, k, _c_cameras([0.0]), None, None, None, None, None, None, None) == -2
    assert lib.g4d_render_forward_cameras(None, 2, _c_cameras([0.0, 0.0]), None, None, None, None, None, None) == -2   # no contexts


# ----------------------------------------------------------------------------------------------------------- GPU
def _check_forward(outs, singles, ctxs_multi=None, ctxs_single=None):
    for i, (o, s) in enumerate(zip(outs, singles)):
        assert o["render"].shape == s["render"].shape and o["depth"].shape == s["depth"].shape
        assert torch.equal(o["radii"], s["radii"]), i
        assert torch.equal(o["visibility_filter"], s["visibility_filter"]), i
        if i == 0:
            assert torch.equal(o["render"], s["render"]) and torch.equal(o["depth"], s["depth"])
        else:
            assert float((o["render"] - s["render"]).abs().max()) <= 1e-6, i
            assert float((o["depth"] - s["depth"]).abs().max()) <= 1e-6, i
    if ctxs_multi is not None:
        for i, (a, b) in enumerate(zip(ctxs_multi, ctxs_single)):
            for x, y in zip(_ctx_reads(a), _ctx_reads(b)):
                assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), i


@pytest.mark.gpu
@pytest.mark.parametrize("ci,stage", [(0, "fine"), (1, "fine"), (2, "fine"), (3, "fine"), (2, "coarse")])
def test_same_images_as_separate_renders(ci, stage):
    c = CASES[ci]
    bg = torch.tensor(c["bg"], device="cuda")
    cams = _cameras(c)
    # grad mode keeps every camera's context (records for the bit-exact comparison)
    scene, mod, pc = _setup(c, grad=True)
    outs = g4d.render_cameras(cams, pc, _Pipe, bg, stage=stage)
    singles = [g4d.render(cam, pc, _Pipe, bg, stage=stage) for cam in cams]
    torch.cuda.synchronize()
    node = outs[0]["render"].grad_fn
    _check_forward(outs, singles, [lease.ctx for lease in node.leases], [s["render"].grad_fn.lease.ctx for s in singles])
    # no-grad calls (nothing saved for a backward; camera 0 still stores the tensors the other cameras read)
    with torch.no_grad():
        outs_ng = g4d.render_cameras(cams, pc, _Pipe, bg, stage=stage)
        singles_ng = [g4d.render(cam, pc, _Pipe, bg, stage=stage) for cam in cams]
    _check_forward(outs_ng, singles_ng)
    for a, b in zip(outs_ng, outs):
        assert torch.equal(a["render"], b["render"].detach()) and torch.equal(a["radii"], b["radii"])


def _grads(pc, mod, points=()):
    return ([p.grad.clone() for p in pc.gaussian_parameters()] + [p.grad.clone() for p in mod.flat_parameters() if p.grad is not None],
            [None if p.grad is None else p.grad.clone() for p in points])


@pytest.mark.gpu
@pytest.mark.parametrize("ci,stage", [(0, "fine"), (2, "fine"), (3, "fine"), (1, "coarse")])
def test_same_gradients_as_separate_renders(ci, stage):
    """sum_i <w_i, image_i> with one backward == the sum of separate render() backward passes; camera 2 is left out of the
    loss (its blend backward is skipped, its screen-space gradient is zero), camera 3 sees no Gaussian."""
    c = CASES[ci]
    bg = torch.tensor(c["bg"], device="cuda")
    cams = _cameras(c, extra=[_blind_camera(c)])
    in_loss = [0, 1, 3]
    gen = torch.Generator().manual_seed(ci)
    weights = [torch.rand(3, cam.image_height, cam.image_width, generator=gen).cuda() for cam in cams]
    res = []
    for mode in ("group", "separate"):
        scene, mod, pc = _setup(c, grad=True)
        if mode == "group":
            outs = g4d.render_cameras(cams, pc, _Pipe, bg, stage=stage)
            assert int(outs[3]["radii"].max()) == 0
            sum((outs[i]["render"] * weights[i]).sum() for i in in_loss).backward()
            points = [o["viewspace_points"] for o in outs]
        else:
            points = []
            for i in in_loss:
                o = g4d.render(cams[i], pc, _Pipe, bg, stage=stage)
                (o["render"] * weights[i]).sum().backward()
                points.append(o["viewspace_points"])
        res.append(_grads(pc, mod, points))
    (ga, pa), (gb, pb) = res
    assert len(ga) == len(gb)
    for a, b in zip(ga, gb):
        assert float((a - b).abs().max()) <= SUM_TOL * max(1e-3, float(b.abs().max())), float((a - b).abs().max())
    for j, i in enumerate(in_loss):
        assert float((pa[i] - pb[j]).abs().max()) <= SUM_TOL * max(1e-3, float(pb[j].abs().max())), i
    assert pa[2] is None or float(pa[2].abs().max()) == 0.0
    assert float(pa[3].abs().max()) == 0.0
    if stage == "coarse":
        assert all(p.grad is None for p in mod.parameters())


@pytest.mark.gpu
def test_each_camera_against_the_oracle():
    c = CASES[1]
    bg = torch.tensor(c["bg"], device="cuda")
    cams = _cameras(c)
    scene, mod, pc = _setup(c, grad=True)
    outs = g4d.render_cameras(cams, pc, _Pipe, bg)
    gen = torch.Generator().manual_seed(7)
    dLs = [torch.randn(o["render"].shape, generator=gen) for o in outs]
    sum((o["render"] * d.cuda()).sum() for o, d in zip(outs, dLs)).backward()
    cfg, prm = oracle_params_from_module(mod)
    leaves = {k: v.clone().requires_grad_(True) for k, v in scene.items() if k != "aabb"}
    loss = 0.0
    for o, cam, d in zip(outs, cams, dLs):
        color, depth, radii, rc, _ = oracle_render(cfg, prm, leaves, cam, c["t"], c["bg"], sh_degree=c["deg"])
        err = (o["render"].detach().cpu() - color.detach()).abs()
        assert float((err > IMG_TOL).float().mean()) <= 1e-3 and float(err.max()) <= 1e-2 and float(err.median()) <= 1e-6
        assert (o["radii"].cpu().numpy() != radii.numpy()).mean() <= 2e-3
        loss = loss + (color * d).sum()
    loss.backward()
    pairs = (("xyz", pc._xyz), ("scaling", pc._scaling), ("rotation", pc._rotation), ("opacity", pc._opacity),
             ("features_dc", pc._features_dc), ("features_rest", pc._features_rest))
    for nm, p in pairs:
        e = rel_err(p.grad.cpu().numpy(), leaves[nm].grad.numpy())
        assert e <= 3 * GRAD_TOL, (nm, e)
    from oracle import deform_ref as dr
    osd = dr.params_to_state_dict(prm)
    for k, p in mod.named_parameters():
        if k in osd and p.requires_grad and osd[k].grad is not None:
            e = rel_err(p.grad.cpu().numpy(), osd[k].grad.numpy())
            assert e <= 3 * GRAD_TOL, (k, e)


@pytest.mark.gpu
@pytest.mark.parametrize("ci", [0, 2])
def test_one_camera_is_render(ci):
    """k = 1 runs render()'s kernels: image and radii bit for bit; gradients bit for bit whenever render() itself repeats
    bit for bit (the blend backward adds with atomics, whose order may vary from run to run)."""
    c = CASES[ci]
    bg = torch.tensor(c["bg"], device="cuda")
    cam = _cameras(c)[0]
    w = torch.rand(3, cam.image_height, cam.image_width, generator=torch.Generator().manual_seed(3)).cuda()
    runs = []
    for fn in (lambda pc: g4d.render_cameras([cam], pc, _Pipe, bg)[0], lambda pc: g4d.render(cam, pc, _Pipe, bg),
               lambda pc: g4d.render(cam, pc, _Pipe, bg)):
        scene, mod, pc = _setup(c, grad=True)
        o = fn(pc)
        (o["render"] * w).sum().backward()
        g, p = _grads(pc, mod, [o["viewspace_points"]])
        runs.append((o["render"].detach().clone(), o["radii"].clone(), g + p))
    (img, rad, gm), (img1, rad1, g1), (_, _, g2) = runs
    assert torch.equal(img, img1) and torch.equal(rad, rad1)
    repeatable = all(torch.equal(a, b) for a, b in zip(g1, g2))
    for a, b, b2 in zip(gm, g1, g2):
        if repeatable:
            assert torch.equal(a, b)
        else:
            assert float((a - b).abs().max()) <= SUM_TOL * max(1e-3, float(b.abs().max()))


@pytest.mark.gpu
def test_full_size_C3_four_cameras():
    w = synth.WORKLOADS["C3"]
    scene = synth.make_scene(w["n"], seed=0, scale_mean=w["scale_mean"])
    mod = make_module(w["net"], seed=0, aabb=scene["aabb"])
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
    cams = synth.orbit_cameras(4, w["width"], w["height"], radius=w["radius"], focal=w["focal"])
    for cam in cams:
        cam.time = 0.4
    bg = torch.tensor([0.0, 0.0, 0.0], device="cuda")
    outs = g4d.render_cameras(cams, pc, _Pipe, bg)
    singles = [g4d.render(cam, pc, _Pipe, bg) for cam in cams]
    torch.cuda.synchronize()
    _check_forward(outs, singles, [lease.ctx for lease in outs[0]["render"].grad_fn.leases],
                   [s["render"].grad_fn.lease.ctx for s in singles])
    assert all(int((o["radii"] > 0).sum()) > 1000 for o in outs)


@pytest.mark.gpu
def test_launch_modes():
    """G4D_OPT_PDL 0 and 1 give identical results; no-sync mode works across repeated calls and matches sync mode."""
    c = CASES[2]
    bg = torch.tensor(c["bg"], device="cuda")
    cams = _cameras(c)
    scene, mod, pc = _setup(c, grad=False)
    ws = _lib.Workspace.get(0)

    def run():
        with torch.no_grad():
            outs = g4d.render_cameras(cams, pc, _Pipe, bg)
        return [(o["render"].clone(), o["depth"].clone(), o["radii"].clone()) for o in outs]
    try:
        ref = []
        for pdl in (0, 1, 0, 1):
            ws.set_option(_lib.OPT_PDL, pdl)
            ref.append(run())
        ws.set_option(_lib.OPT_PDL, 1)
        ws.set_option(_lib.OPT_SYNC_MODE, 0)
        nosync = [run() for _ in range(6)]
        torch.cuda.synchronize()
    finally:
        ws.set_option(_lib.OPT_PDL, 1)
        ws.set_option(_lib.OPT_SYNC_MODE, 1)
    for other in ref[1:] + nosync:
        for a, b in zip(ref[0], other):
            assert all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.gpu
def test_errors_and_context_pool():
    c = CASES[1]
    bg = torch.tensor(c["bg"], device="cuda")
    cams = _cameras(c)
    scene, mod, pc = _setup(c, grad=True)
    lib = _lib.load()
    # mismatched times: ValueError in Python, G4D_ERR_ARG through ctypes (before any launch)
    bad = _cameras(c)
    bad[1].time = c["t"] + 1e-3
    with pytest.raises(ValueError):
        g4d.render_cameras(bad, pc, _Pipe, bg)
    ws = _lib.Workspace.get(0)
    ctxs = [_lib.Context(ws), _lib.Context(ws)]
    handles = (C.c_void_p * 2)(ctxs[0].handle, ctxs[1].handle)
    rc = lib.g4d_render_forward_cameras(handles, 2, _c_cameras([0.1, 0.2]), None, None, None, None, None, None)
    assert rc == -2 and b"time" in lib.g4d_last_error()
    same = (C.c_void_p * 2)(ctxs[0].handle, ctxs[0].handle)
    assert lib.g4d_render_forward_cameras(same, 2, _c_cameras([0.1, 0.1]), None, None, None, None, None, None) == -2
    # another forward on a member context: the group backward returns G4D_ERR_STATE; render()'s backward refuses a member
    outs = g4d.render_cameras(cams, pc, _Pipe, bg)
    node = outs[0]["render"].grad_fn
    cams_c, prm, g, keep, version, hs = node.cstructs
    rc = lib.g4d_render_backward(hs[0], C.byref(cams_c[0]), C.byref(prm), None, C.byref(g), None, None, None)
    assert rc == -4 and b"g4d_render_backward_cameras" in lib.g4d_last_error()
    color = torch.empty(3, 8, 8, device="cuda"); depth = torch.empty(1, 8, 8, device="cuda")
    small = _c_cameras([0.0], wh=(8, 8))
    assert lib.g4d_rasterize_forward(hs[1], small, 0, None, None, None, None, None, color.data_ptr(), depth.data_ptr(), None, None) == 0
    with pytest.raises(_lib.G4DError, match=r"code -4"):
        sum(o["render"].sum() for o in outs).backward()
    # a second backward raises
    outs = g4d.render_cameras(cams, pc, _Pipe, bg)
    loss = sum(o["render"].sum() for o in outs)
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="twice"):
        loss.backward()
    # no-grad calls return every lease at once
    with torch.no_grad():
        g4d.render_cameras(cams, pc, _Pipe, bg)
        torch.cuda.synchronize()
        pool = sorted(x.handle for x in ws._free_contexts)
        for _ in range(3):
            g4d.render_cameras(cams, pc, _Pipe, bg)
        assert sorted(x.handle for x in ws._free_contexts) == pool


@pytest.mark.gpu
def test_foreign_module_and_panoptic_cameras():
    """A deformation module that is not g4d's is run once and its output rasterized per camera; PanopticSports dict
    cameras carry prebuilt settings, as in render()."""
    c = CASES[2]
    bg = torch.tensor(c["bg"], device="cuda")
    cams = _cameras(c)
    scene, mod, pc = _setup(c, grad=False)

    class Wrapped(torch.nn.Module):
        def __init__(self, m):
            super().__init__()
            self.m = m

        def forward(self, *a):
            return self.m(*a)
    with torch.no_grad():
        fused = g4d.render_cameras(cams, pc, _Pipe, bg)
        pc._deformation = Wrapped(mod)
        foreign = g4d.render_cameras(cams, pc, _Pipe, bg)
        singles = [g4d.render(cam, pc, _Pipe, bg) for cam in cams]
        pc._deformation = mod
        for a, b, f in zip(foreign, singles, fused):
            assert torch.equal(a["render"], b["render"]) and torch.equal(a["radii"], b["radii"])
            assert float((a["render"] - f["render"]).abs().max()) <= IMG_TOL
        dicts = []
        for cam in cams:
            rs, t = renderer.settings_from_camera(cam, pc, _Pipe, bg)
            dicts.append({"camera": rs, "time": t})
        pan = g4d.render_cameras(dicts, pc, _Pipe, bg, cam_type="PanopticSports")
        for a, f in zip(pan, fused):
            assert torch.equal(a["render"], f["render"]) and torch.equal(a["radii"], f["radii"])
