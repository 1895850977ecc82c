"""GPU: the alpha image A = 1 - T and its gradient through the GaussianRasterizer drop-in, render() on both network engines and
render_cameras, against the oracles of util_alpha (the C oracle's colour backward with colour 0 on a (1, 0, 0) background,
and fp64 autograd of the dense formulation), with the rules of test_gpu_depth_grad.  Also: with no alpha loss every output
and gradient is bit-identical to a run that never asked for alpha, the colour composites (1 - A) bg, the camera and time
leaves take the alpha term, GraphedRender's alpha, the pointer rules of the two setters, and an alpha mask fitted by Adam."""
import ctypes as C
import importlib
import math

import numpy as np
import pytest
import torch

from oracle import raster_ref as rr
from oracle.dense_ref import cam_dict_from
import util_alpha as ua
import util_camera_grad as ucg
import util_raster_edges as ue
from test_gpu_depth_grad import (FLOOR, LONG_ROW_TOL, ROW_TOL, CAM_TOL, SUM_TOL, TIME_TOL, _Pipe, _check_network, _coarse,
                                 _compare_rows, _engine, _grads, _keep, _leaf_camera, _own_workspace, _silenced_scene)
from test_gpu_raster_edges import _check_forward, _settings
from util_scene import (SCENE_LEAVES, make_module, oracle_chain_backward, oracle_params_from_module, params_fp64,
                        raster_inputs, raster_oracle_inputs, rel_err, synth, _deform_activate, cam_tuple)

pytestmark = pytest.mark.gpu
g4d = importlib.import_module("4dgaussians_b200")
_lib = importlib.import_module("4dgaussians_b200._lib")
rasterizer = importlib.import_module("4dgaussians_b200.rasterizer")
graphs = importlib.import_module("4dgaussians_b200.graphs")

T = 0.4
_ = _own_workspace      # (autouse: this module renders on a workspace of its own)


def _cots(H, W, seed, mode, mask):
    """(colour, depth, alpha) cotangents, zero where mask is False; mode "alpha": colour and depth are None"""
    g = torch.Generator().manual_seed(seed)
    dA = torch.randn(1, H, W, generator=g)
    dA[:, ~mask] = 0.0
    dC = dD = None
    if mode != "alpha":
        dC, dD = torch.randn(3, H, W, generator=g), torch.randn(1, H, W, generator=g)
        dC[:, ~mask] = 0.0
        dD[:, ~mask] = 0.0
    return dC, dD, dA


def _loss(img, dep, alp, dC, dD, dA):
    loss = torch.zeros((), device="cuda")
    for x, c in ((img, dC), (dep, dD), (alp, dA)):
        if c is not None:
            loss = loss + (x * c.cuda()).sum()
    return loss


def _np(t):
    return None if t is None else t.numpy()


# ---- 1. the rasterizer drop-in on the edge scenes -----------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["alpha", "mixed"])
@pytest.mark.parametrize("name", ue.names())
def test_rasterizer(name, mode):
    sc = ue.scene(name)
    rc, _ = cam_tuple(sc.cam, sc.bg, sh_degree=sc.deg)
    ref = rr.rasterize_forward(rc, *sc.ins)
    m3, s, r, o, sh = [torch.from_numpy(a).cuda().requires_grad_(True) for a in sc.ins]
    m2 = torch.zeros_like(m3, requires_grad=True)
    color, radii, depth, alpha = g4d.GaussianRasterizer(_settings(sc), differentiable_depth=True, return_alpha=True)(
        means3D=m3, means2D=m2, shs=sh, colors_precomp=None, opacities=o, scales=s, rotations=r, cov3D_precomp=None)
    torch.cuda.synchronize()
    ctx = color.grad_fn.lease.ctx
    keep = _check_forward(sc, ctx, radii.cpu().numpy(), color.detach().cpu().numpy(), ref)
    # A is 1 - T of the GPU's own transmittance, bit for bit, and the oracle's where the pixel did not flip
    fin = ctx.read("final_T").reshape(1, sc.H, sc.W)
    a = alpha.detach().cpu().numpy()
    assert alpha.requires_grad and np.array_equal(a, np.float32(1.0) - fin)
    assert float(np.abs(a - ua.oracle_alpha(ref))[:, keep].max(initial=0.0)) <= 1e-5
    dC, dD, dA = _cots(sc.H, sc.W, sum(map(ord, name)) + len(mode), mode, torch.from_numpy(keep))
    _loss(color, depth, alpha, dC, dD, dA).backward()
    torch.cuda.synchronize()
    want = ua.oracle_backward(rc, sc.ins, ref, _np(dC), _np(dD), dA.numpy())
    got = {"means3D": m3.grad, "means2D": m2.grad, "scales": s.grad, "rots": r.grad, "opacities": o.grad, "shs": sh.grad}
    got = {k: v.cpu().numpy() for k, v in got.items()}
    unseen = ref["radii"] == 0
    for k, v in got.items():
        assert not v[unseen].any(), k
    if mode == "alpha":
        assert not got["shs"].any()
    long = sc.group == "long"
    _compare_rows(got, {k: want[k] for k in got}, LONG_ROW_TOL if long else ROW_TOL,
                  1e-2 if long and mode == "mixed" else FLOOR, name)


# ---- 2. render() on both engines against the fp64 chain --------------------------------------------------------------------
@pytest.mark.parametrize("tc", [0, 2])
def test_render_vs_oracle_chain(tc):
    W, H = 61, 47
    cam = synth.make_camera(30.0, W, H, radius=3.0, time=T)
    scene, mod, cfg, prm, silenced = _silenced_scene(500, 5 + tc, "small128", [cam])
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
    bg = (0.0, 0.1, 0.2)
    with _engine(tc):
        out = g4d.render(cam, pc, _Pipe, torch.tensor(bg, device="cuda"), stage="fine", return_alpha=True)
        torch.cuda.synchronize()
        ctx = out["render"].grad_fn.lease.ctx
        shs = ctx.read("deformed_shs") if not mod.args.no_dshs else \
            torch.cat([scene["features_dc"], scene["features_rest"]], 1).numpy()
        ins = raster_oracle_inputs(ctx.read("deformed"), shs)
        rc, _ = cam_tuple(cam, bg, sh_degree=3)
        ref = rr.rasterize_forward(rc, *ins)
        keep = _keep(ctx, out["radii"].cpu().numpy(), out["render"].detach().cpu().numpy(), ref, W, H)
        assert np.array_equal(out["alpha"].detach().cpu().numpy(), np.float32(1.0) - ctx.read("final_T").reshape(1, H, W))
        _, _, dA = _cots(H, W, 31 + tc, "alpha", torch.from_numpy(keep))
        (out["alpha"] * dA.cuda()).sum().backward()
    cot = ua.oracle_backward(rc, ins, ref, None, None, dA.numpy())
    want, p64 = oracle_chain_backward(cfg, prm, scene, float(np.float32(T)), cot)
    got = {k: getattr(pc, "_" + k).grad.cpu().numpy().reshape(want[k].shape) for k in SCENE_LEAVES}
    for k in SCENE_LEAVES:
        assert not got[k][silenced].any(), k
    what = "render alpha tc=%d" % tc
    _compare_rows(got, want, what=what)
    _compare_rows({"means2D": out["viewspace_points"].grad.cpu().numpy()}, {"means2D": cot["means2D"]}, what=what)
    _check_network(mod, p64, tc, what)


# ---- 3. render_cameras, k = 3: colour only, alpha only, all three ---------------------------------------------------------
def test_render_cameras_matches_three_renders():
    cams = [synth.make_camera(th, 61 + 4 * i, 47, radius=3.0, time=T) for i, th in enumerate((10.0, 100.0, -120.0))]
    scene = synth.make_scene(500, seed=9, scale_mean=0.05)
    mod = make_module("small128", seed=9, aabb=scene["aabb"])
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
    bg = torch.tensor([0.2, 0.1, 0.0], device="cuda")
    cots = []
    for i, (c, mode) in enumerate(zip(cams, ("colour", "alpha", "mixed"))):
        g = torch.Generator().manual_seed(40 + i)
        H, W = c.image_height, c.image_width
        rnd = lambda ch: torch.randn(ch, H, W, generator=g).cuda()
        cots.append((None if mode == "alpha" else rnd(3), rnd(1) if mode == "mixed" else None,
                     None if mode == "colour" else rnd(1)))
    loss = lambda o, c: _loss(o["render"], o["depth"], o["alpha"], *c)

    outs = g4d.render_cameras(cams, pc, _Pipe, bg, stage="fine", return_alpha=True)
    sum(loss(o, c) for o, c in zip(outs, cots)).backward()
    group = _grads(pc, mod)
    views = [o["viewspace_points"].grad.clone() for o in outs]
    for p in list(pc.gaussian_parameters()) + list(mod.parameters()):
        p.grad = None
    singles, single_views = [], []
    for c, cot in zip(cams, cots):
        o = g4d.render(c, pc, _Pipe, bg, stage="fine", return_alpha=True)
        singles.append(o["alpha"].detach())
        loss(o, cot).backward()
        single_views.append(o["viewspace_points"].grad.clone())
    single = _grads(pc, mod)
    for o, a in zip(outs, singles):
        assert o["alpha"].shape == a.shape and torch.equal(o["alpha"].detach(), a)
    assert len(group) == len(single)
    for i, (a, b) in enumerate(zip(group, single)):
        a, b = a.cpu().numpy(), b.cpu().numpy()
        if a.ndim >= 2 and a.shape[0] == 500:
            _compare_rows({"g%d" % i: a}, {"g%d" % i: b}, what="render_cameras leaf %d" % i)
        else:
            assert rel_err(a, b) <= 5e-4, ("render_cameras parameter", i, rel_err(a, b))
    for i, (a, b) in enumerate(zip(views, single_views)):
        _compare_rows({"m": a.cpu().numpy()}, {"m": b.cpu().numpy()}, what="viewspace_points %d" % i)
    assert float(views[1].abs().max()) > 0        # the alpha-only camera is part of the loss


# ---- 4. camera and time leaves take the alpha term -----------------------------------------------------------------------
@pytest.mark.parametrize("tc", [0, 2])
def test_camera_and_time_leaves(tc):
    cam = synth.make_camera(30.0, 61, 47, radius=3.0)
    scene = synth.make_scene(400, seed=6, scale_mean=0.05)
    mod = make_module("small128", seed=6, aabb=scene["aabb"])
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
    t, bg = -1.0 + 2.0 * 4.5 / 7, (0.0, 0.1, 0.2)     # the middle of a time interval of the small128 network's 8 rows
    cfg, prm = oracle_params_from_module(mod)
    with torch.no_grad():
        inputs = _deform_activate(cfg, params_fp64(prm), {k: scene[k].double() for k in SCENE_LEAVES}, t)
    cd = cam_dict_from(cam, bg, 3)
    cd["tanfovx"], cd["tanfovy"] = float(np.float32(cd["tanfovx"])), float(np.float32(cd["tanfovy"]))
    mask = ~ucg.threshold_pixel_mask(cd, inputs)
    dC, _, dA = _cots(47, 61, 17, "mixed", mask)
    dA = dA * 4.0           # an alpha term the camera check sees (below)
    want = ua.dense_grads(cd, [x.numpy() for x in inputs], dC.double(), None, dA.double(), cam_keys=ucg.CAM_KEYS)
    colour_only = ua.dense_grads(cd, [x.numpy() for x in inputs], dC.double(), None, None, cam_keys=("view",))
    per = ua.oracle_time_grads(cfg, prm, scene, cd, t, dC.double(), dA.double())
    leaf_t = torch.tensor(t, device="cuda", dtype=torch.float32, requires_grad=True)
    lc = _leaf_camera(cam, leaf_t)
    with _engine(tc):
        out = g4d.render(lc, pc, _Pipe, torch.tensor(bg, device="cuda"), stage="fine", return_alpha=True)
        _loss(out["render"], out["depth"], out["alpha"], dC, None, dA).backward()
    got = {"view": lc.world_view_transform.grad, "proj": lc.full_proj_transform.grad, "campos": lc.camera_center.grad}
    for k in ucg.CAM_KEYS:
        ucg.assert_close_to_max(got[k].reshape(-1).cpu(), want[k], CAM_TOL, "tc=%d %s" % (tc, k))
    # the alpha term is large enough here that a backward without it would fail the view check
    assert np.abs(want["view"] - colour_only["view"]).max() > 10 * CAM_TOL * np.abs(want["view"]).max()
    ref, scale = float(per.sum()), float(per.abs().sum())
    assert abs(float(leaf_t.grad) - ref) <= TIME_TOL * scale, (float(leaf_t.grad), ref, scale)


# ---- 5. nothing else moves --------------------------------------------------------------------------------------------------
def _everything(path, alpha, k=1):
    """images, depths, radii and every gradient of a colour + depth loss; alpha: False (never asked for), "out" (returned,
    outside the loss), "zero" (a zero alpha cotangent) or "random"; the alpha maps are appended to the forward outputs"""
    scene = synth.make_scene(500, seed=13, scale_mean=0.05)
    mod = make_module("small128", seed=13, aabb=scene["aabb"])
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
    bg = torch.tensor([0.3, 0.2, 0.1], device="cuda")
    cams = [synth.make_camera(25.0 + 70 * i, 64, 48, radius=3.0, time=0.3) for i in range(k)]
    cot = torch.randn(3, 48, 64, generator=torch.Generator().manual_seed(3)).cuda()
    dD = torch.randn(1, 48, 64, generator=torch.Generator().manual_seed(4)).cuda()
    dA = torch.randn(1, 48, 64, generator=torch.Generator().manual_seed(5)).cuda()
    dA = dA * 0.0 if alpha == "zero" else dA

    def loss(img, dep, alp):
        return (img * cot).sum() + (dep * dD).sum() + ((alp * dA).sum() if alpha in ("zero", "random") else 0.0)

    want = bool(alpha)
    if path == "rasterizer":
        c = cams[0]
        inputs = [t.float().cuda().requires_grad_(True) for t in raster_inputs(500, 13, scale_mean=0.05)]
        rs = rasterizer.GaussianRasterizationSettings(48, 64, math.tan(c.FoVx * 0.5), math.tan(c.FoVy * 0.5), bg, 1.0,
                                                      c.world_view_transform.cuda(), c.full_proj_transform.cuda(), 3,
                                                      c.camera_center.cuda(), False, False)
        m2 = torch.zeros_like(inputs[0], requires_grad=True)
        r = rasterizer.GaussianRasterizer(rs, differentiable_depth=True, return_alpha=want)(
            means3D=inputs[0], means2D=m2, shs=inputs[4], opacities=inputs[3], scales=inputs[1], rotations=inputs[2])
        assert len(r) == (4 if want else 3)
        loss(r[0], r[2], r[3] if want else None).backward()
        return [r[0], r[2], r[1]] + list(r[3:]), [m2.grad] + [t.grad for t in inputs]
    outs = g4d.render_cameras(cams, pc, _Pipe, bg, stage="fine", return_alpha=want)
    assert all(("alpha" in o) == want for o in outs)
    sum(loss(o["render"], o["depth"], o.get("alpha")) for o in outs).backward()
    fwd = [x for o in outs for x in (o["render"], o["depth"], o["radii"])] + [o["alpha"] for o in outs if want]
    grads = [o["viewspace_points"].grad for o in outs]
    return fwd, grads + [p.grad for p in pc.gaussian_parameters()] + [p.grad for p in mod.parameters() if p.grad is not None]


@pytest.mark.parametrize("path,k", [("rasterizer", 1), ("render", 1), ("render", 3)])
@pytest.mark.parametrize("tc", [0, 2])
def test_no_alpha_loss_changes_nothing(path, k, tc):
    """Forward outputs byte-identical whether alpha is asked for or not.  With alpha returned but outside the loss, or with a
    zero alpha cotangent, the gradients are those of a run that never asked for alpha, within twice the spread of two such
    runs or SUM_TOL of the tensor's max (the blend backward sums with atomics, whose order varies); a real alpha loss moves
    them"""
    if path == "rasterizer" and tc == 2:
        pytest.skip("the rasterizer drop-in runs no network")
    with _engine(tc):
        (f0, g0), (f1, g1), (fo, go), (fz, gz), (fr, gr) = [_everything(path, a, k)
                                                            for a in (False, False, "out", "zero", "random")]
    n = len(f0)
    for i, x in enumerate(f0):
        assert torch.equal(x, f1[i])
    for f in (fo, fz, fr):
        assert len(f) == n + k
        for i, x in enumerate(f0):
            assert torch.equal(x, f[i]), "forward output %d moved" % i
        for i in range(k):
            assert torch.equal(f[n + i], fo[n + i])
    assert len(g0) == len(g1) == len(go) == len(gz) == len(gr)
    moved = 0
    for x, x1, o, z, w in zip(g0, g1, go, gz, gr):
        x, x1, o, z, w = x.double(), x1.double(), o.double(), z.double(), w.double()
        bound = max(2 * float((x - x1).abs().max()), SUM_TOL * max(1e-3, float(x.abs().max())))
        assert float((x - o).abs().max()) <= bound
        assert float((x - z).abs().max()) <= bound
        moved += float((x - w).abs().max()) > bound
    assert moved > 0


# ---- 6. the colour composites (1 - A) bg ----------------------------------------------------------------------------------
def test_foreground_is_the_same_on_two_backgrounds():
    cams = [synth.make_camera(th, 64, 48, radius=3.0, time=T) for th in (20.0, 150.0)]
    scene = synth.make_scene(800, seed=3, scale_mean=0.05)
    pc = synth.SyntheticGaussianModel(scene, make_module("small128", seed=3, aabb=scene["aabb"]), sh_degree=3)
    fgs = []
    for bg in ((0.0, 0.0, 0.0), (0.9, 0.4, 0.1)):
        b = torch.tensor(bg, device="cuda")
        with torch.no_grad():
            outs = g4d.render_cameras(cams, pc, _Pipe, b, stage="fine", return_alpha=True)
        fgs.append([o["render"] - (1.0 - o["alpha"]) * b[:, None, None] for o in outs])
        assert float(outs[0]["alpha"].max()) > 0.3 and bool((outs[0]["alpha"] < 0.99).any())
    for a, b in zip(*fgs):
        assert float((a - b).abs().max()) <= 1e-6


# ---- 7. GraphedRender ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 3])
def test_graphed_render_alpha_equals_eager(k):
    scene = synth.make_scene(600, seed=8, scale_mean=0.05)
    pc = synth.SyntheticGaussianModel(scene, make_module("small128", seed=8, aabb=scene["aabb"]), sh_degree=3)
    bg = torch.tensor([0.1, 0.2, 0.3], device="cuda")
    views = [synth.make_camera(30.0 + 40 * i, 64, 48, radius=3.0, time=0.25) for i in range(k)]
    template = views if k > 1 else views[0]
    gr = graphs.GraphedRender(pc, _Pipe, bg, template, return_alpha=True)
    for shift in (0.0, 15.0):
        cams = [synth.make_camera(30.0 + 40 * i + shift, 64, 48, radius=3.0, time=0.25) for i in range(k)]
        got = gr(cams if k > 1 else cams[0])
        got = got if k > 1 else [got]
        with torch.no_grad():
            want = g4d.render_cameras(cams, pc, _Pipe, bg, stage="fine", return_alpha=True) if k > 1 else \
                [g4d.render(cams[0], pc, _Pipe, bg, stage="fine", return_alpha=True)]
        gr.check()
        for g, w in zip(got, want):
            assert torch.equal(g["alpha"], w["alpha"]) and torch.equal(g["render"], w["render"])
    plain = graphs.GraphedRender(pc, _Pipe, bg, template)
    out = plain(template)
    assert all("alpha" not in o for o in (out if k > 1 else [out]))


# ---- 8. the setters' pointer rules ------------------------------------------------------------------------------------------
def test_alpha_pointer_rules():
    ws = _lib.workspace_of(torch.device("cuda"))
    ctx = _lib.Context(ws)
    n = 200
    dA = torch.randn(48 * 64, generator=torch.Generator().manual_seed(1)).cuda()
    try:
        # under stream capture, with the gradient set: refused before any launch (nothing is captured)
        bwd, sinks = _coarse(ctx, n)
        torch.cuda.synchronize()
        ctx.set_alpha_grad(dA.data_ptr())
        graph, stream = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            graph.capture_begin()
            rc = bwd()
            graph.capture_end()
        torch.cuda.synchronize()
        assert rc == -4 and "alpha gradient" in _lib.load().g4d_last_error().decode()
        assert all(torch.isnan(t).all() for t in sinks)
        # set: the alpha term is in the gradients
        bwd, with_alpha = _coarse(ctx, n)
        assert bwd() == 0
        # NULL turns it off: the gradients of a context that never had one
        ctx.set_alpha_grad(None)
        bwd, off = _coarse(ctx, n)
        assert bwd() == 0
        other = _lib.Context(ws)
        bwd, never = _coarse(other, n)
        assert bwd() == 0
        torch.cuda.synchronize()
        for a, b, c in zip(off, never, with_alpha):
            assert torch.isfinite(a).all() and torch.isfinite(c).all()
            assert float((a - b).abs().max()) <= SUM_TOL * max(1e-3, float(b.abs().max()))
        assert float((with_alpha[3] - never[3]).abs().max()) > 1e-3 * float(never[3].abs().max())
        # the output: written by every forward while set (no-grad ones included), untouched once cleared
        out = torch.full((1, 48, 64), float("nan"), device="cuda")
        ctx.set_alpha_out(out.data_ptr())
        _coarse(ctx, n, no_grad=True)
        torch.cuda.synchronize()
        assert torch.isfinite(out).all() and float(out.max()) > 0
        assert torch.equal(out.cpu().reshape(-1), torch.from_numpy(1.0 - ctx.read("final_T")))
        ctx.set_alpha_out(None)
        out.fill_(float("nan"))
        _coarse(ctx, n)
        torch.cuda.synchronize()
        assert torch.isnan(out).all()
    finally:
        ctx.set_alpha_grad(None)
        ctx.set_alpha_out(None)


# ---- 9. an alpha mask fitted by Adam ---------------------------------------------------------------------------------------
FIT_STEPS = 100
FIT_RATIO = 0.2


def test_adam_fits_an_alpha_mask():
    cam = synth.make_camera(40.0, 128, 96, radius=4.0)
    m3, sc, ro, op, sh = [t.float().cuda() for t in raster_inputs(3000, 21, scale_mean=0.04)]
    rs = rasterizer.GaussianRasterizationSettings(96, 128, math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5),
                                                  torch.zeros(3, device="cuda"), 1.0, cam.world_view_transform.cuda(),
                                                  cam.full_proj_transform.cuda(), 3, cam.camera_center.cuda(), False, False)
    g = torch.Generator().manual_seed(2)
    target_xyz = m3 + 0.05 * torch.randn(m3.shape, generator=g).cuda()

    def alpha(xyz):
        return rasterizer.GaussianRasterizer(rs, return_alpha=True)(
            means3D=xyz, means2D=torch.zeros_like(xyz), shs=sh, opacities=op, scales=sc, rotations=ro)[3]

    with torch.no_grad():
        target = alpha(target_xyz)
    xyz = m3.clone().requires_grad_(True)
    opt = torch.optim.Adam([xyz], lr=2e-3)
    losses = []
    for _ in range(FIT_STEPS):
        opt.zero_grad()
        loss = ((alpha(xyz) - target) ** 2).mean()
        loss.backward()
        assert xyz.grad is not None and torch.isfinite(xyz.grad).all()
        opt.step()
        losses.append(float(loss.detach()))
    print("alpha loss: initial %.5g final %.5g ratio %.3f" % (losses[0], losses[-1], losses[-1] / losses[0]))
    assert losses[-1] <= FIT_RATIO * losses[0], losses[::10]
