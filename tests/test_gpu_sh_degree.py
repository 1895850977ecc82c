"""Models of SH degree d < 3 (M = (d + 1)^2 coefficients per Gaussian) against the same model zero-padded to 16 coefficients.

The colour at active degree a reads only the coefficients k < (a + 1)^2 <= M, so the padded model renders the very same
floats: images, depth, radii and every g4d_context_read buffer must be bit-identical, and the gradients must equal the padded
run's first M coefficients -- bit for bit whenever a repeated padded run is bit for bit (the blend backward and the network's
scatter add with atomics, whose order may vary), otherwise within test_gpu_sh_layouts.py's 2e-5 x max, or, for a sum that two
padded runs already disagree on by more, within twice their disagreement.  Gradients of coefficients >= (a + 1)^2 are 0.
"""
import ctypes as C
import importlib

import numpy as np
import pytest
import torch

from oracle import raster_ref as rr
from util_scene import cam_tuple, make_module, raster_inputs, synth

pytestmark = pytest.mark.gpu
_lib = importlib.import_module("4dgaussians_b200._lib")
renderer = importlib.import_module("4dgaussians_b200.renderer")
rasterizer = importlib.import_module("4dgaussians_b200.rasterizer")
graphs = importlib.import_module("4dgaussians_b200.graphs")
td = importlib.import_module("4dgaussians_b200.train_dp")

SUM_TOL = 2e-5
IMG_TOL = 1e-4          # DESIGN.md §2.2: images against the CPU oracle
BUFFERS = [b for b in _lib.BUF if b != "bin_phases"]
ERR_ARG, ERR_STATE = -2, -4
DEGREES = [(d, a) for d in (0, 1, 2) for a in range(d + 1)]     # (max degree, active degree)


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


# small64: FFMA network; c32w128: tensor-core network without the SHS head; coarse: no network
CASES = {"ffma": dict(net="small64", stage="fine", n=900, wh=(96, 64), theta=20.0, radius=4.0, t=0.3),
         "tc": dict(net="c32w128", stage="fine", n=1100, wh=(80, 112), theta=-50.0, radius=2.0, t=0.8),
         "coarse": dict(net=None, stage="coarse", n=1000, wh=(88, 72), theta=75.0, radius=3.0, t=0.5)}


def _scene(c, d, padded):
    """the degree-d scene, or (padded) the same scene with features_rest zero-padded to 15 coefficients"""
    s = synth.make_scene(c["n"], seed=11, scale_mean=0.06, sh_degree=d)
    if padded:
        rest = s["features_rest"]
        s["features_rest"] = torch.cat([rest, rest.new_zeros(rest.shape[0], 15 - rest.shape[1], 3)], dim=1)
    return s


def _close(a, b, repeatable, b2=None):
    """a equals b (bit for bit when the padded runs b and b2 repeat, else within the tolerance the module docstring gives)"""
    if repeatable:
        return torch.equal(a, b)
    spread = 2 * float((b - b2).abs().max()) if b2 is not None else 0.0
    return float((a - b).abs().max()) <= max(SUM_TOL * max(1e-3, float(b.abs().max())), spread)


def _run(c, d, act, k, fused, padded, no_grad=False):
    """forward (+ backward unless no_grad) of k cameras through the C-ABI; returns (outputs, reads, gradients)"""
    lib = _lib.load()
    ws = _lib.Workspace(0)
    if no_grad:
        ws.set_option(_lib.OPT_KEEP_DEFORMED, 1)
    scene = _scene(c, d, padded)
    mod = make_module(c["net"], seed=2, aabb=scene["aabb"]) if c["net"] else None
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=act, requires_grad=False)
    n, m = c["n"], scene["features_rest"].shape[1] + 1
    W, H = c["wh"]
    views = [synth.make_camera(c["theta"] + 55.0 * i, W + 13 * i, H, radius=c["radius"], time=c["t"]) for i in range(k)]
    bg = torch.tensor([0.2, 0.1, 0.0], device="cuda")
    keep = []
    cams = (_lib.Camera * k)()
    for i, v in enumerate(views):
        rs, t = renderer.settings_from_camera(v, pc, _Pipe, bg)
        cams[i] = rasterizer.camera_from_settings(rs, time=t, keep=keep, sh_coeffs=m)
        if no_grad:
            cams[i].debug |= _lib.CAM_NO_GRAD
    prm = mod.c_params(keep, fresh=True) if mod is not None else None
    x, s, r, o = (p.detach().float().contiguous() for p in (pc._xyz, pc._scaling, pc._rotation, pc._opacity))
    if fused:
        dc, rest = torch.cat([pc._features_dc, pc._features_rest], dim=1).detach().contiguous(), None
    else:
        dc, rest = pc._features_dc.detach().contiguous(), pc._features_rest.detach().contiguous()
    ptr = lambda tt: None if tt is None else tt.data_ptr()
    g = _lib.Gaussians(n, ptr(x), ptr(s), ptr(r), ptr(o), ptr(dc), ptr(rest))
    colors = [torch.empty(3, cams[i].image_height, cams[i].image_width, device="cuda") for i in range(k)]
    depths = [torch.empty(1, cams[i].image_height, cams[i].image_width, device="cuda") for i in range(k)]
    radii = [torch.empty(n, device="cuda", dtype=torch.int32) for _ in range(k)]
    ctxs = [_lib.Context(ws) for _ in range(k)]
    pp = lambda ts: (C.c_void_p * k)(*[ptr(tt) for tt in ts])
    handles = (C.c_void_p * k)(*[cx.handle for cx in ctxs])
    prm_ref = C.byref(prm) if prm is not None else None
    if k == 1:
        _lib.check(lib.g4d_render_forward(ctxs[0].handle, C.byref(cams[0]), prm_ref, C.byref(g), ptr(colors[0]), ptr(depths[0]),
                                          ptr(radii[0]), None), "g4d_render_forward")
    else:
        _lib.check(lib.g4d_render_forward_cameras(handles, k, cams, prm_ref, C.byref(g), pp(colors), pp(depths), pp(radii), None),
                   "g4d_render_forward_cameras")
    torch.cuda.synchronize()
    reads = []
    for cx in ctxs:
        for b in BUFFERS:
            try:
                reads.append((b, cx.read(b).copy()))
            except _lib.G4DError:
                reads.append((b, None))
    if no_grad:
        return colors + depths + radii, reads, []
    gen = torch.Generator().manual_seed(5)
    dL = [torch.rand(cl.shape, generator=gen).cuda() for cl in colors]
    pgrads = mod.alloc_grads() if mod is not None else []
    cg = C.byref(mod.c_grads(pgrads)) if mod is not None else None
    gx, gs, gm2 = torch.empty(n, 3, device="cuda"), torch.empty(n, 3, device="cuda"), [torch.empty(n, 3, device="cuda") for _ in range(k)]
    gr, go = torch.empty(n, 4, device="cuda"), torch.empty(n, 1, device="cuda")
    gdc = torch.full((n, m if fused else 1, 3), float("nan"), device="cuda")
    grest = None if fused else torch.full((n, m - 1, 3), float("nan"), device="cuda")
    if k == 1:
        gg = _lib.GaussianGrads(ptr(gx), ptr(gs), ptr(gr), ptr(go), ptr(gdc), ptr(grest), ptr(gm2[0]))
        _lib.check(lib.g4d_render_backward(ctxs[0].handle, C.byref(cams[0]), prm_ref, cg, C.byref(g), ptr(dL[0]), C.byref(gg), None),
                   "g4d_render_backward")
    else:
        gg = _lib.GaussianGrads(ptr(gx), ptr(gs), ptr(gr), ptr(go), ptr(gdc), ptr(grest), None)
        _lib.check(lib.g4d_render_backward_cameras(handles, k, cams, prm_ref, cg, C.byref(g), pp(dL), C.byref(gg), pp(gm2), None),
                   "g4d_render_backward_cameras")
    torch.cuda.synchronize()
    sh = gdc if fused else torch.cat([gdc, grest], dim=1)
    return colors + depths + radii, reads, [t.clone() for t in [sh, gx, gs, gr, go] + gm2 + list(pgrads)]


def _compare(got, pad, pad2, m, act):
    outs, reads, grads = got
    outs_p, reads_p, grads_p = pad
    for a, b in zip(outs, outs_p):
        assert torch.equal(a, b)
    for (name, a), (_, b) in zip(reads, reads_p):
        assert (a is None) == (b is None), name
        if a is not None:
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), name
    if not grads:
        return
    repeatable = all(torch.equal(a, b) for a, b in zip(grads_p, pad2[2]))
    used = (act + 1) ** 2
    sh, sh_p = grads[0], grads_p[0]
    assert sh.shape[1] == m and not bool(sh.isnan().any())
    assert bool((sh[:, used:] == 0).all()) and bool((sh_p[:, used:] == 0).all())
    assert _close(sh, sh_p[:, :m], repeatable, pad2[2][0][:, :m])
    assert len(grads) == len(grads_p)
    for i, (a, b, b2) in enumerate(zip(grads[1:], grads_p[1:], pad2[2][1:])):
        assert _close(a, b, repeatable, b2), i


@pytest.mark.parametrize("d,act", DEGREES)
@pytest.mark.parametrize("case,k,fused", [("ffma", 1, False), ("tc", 1, False), ("coarse", 1, False), ("ffma", 3, False),
                                          ("tc", 3, False), ("coarse", 3, True), ("tc", 1, True), ("ffma", 3, True)])
def test_render_equals_padded_model(case, k, fused, d, act):
    c = CASES[case]
    m = (d + 1) ** 2
    got = _run(c, d, act, k, fused, padded=False)
    pad = _run(c, d, act, k, fused, padded=True)
    pad2 = _run(c, d, act, k, fused, padded=True)
    _compare(got, pad, pad2, m, act)


@pytest.mark.parametrize("d,act", DEGREES)
@pytest.mark.parametrize("case,k", [("ffma", 1), ("tc", 1), ("tc", 3), ("coarse", 3)])
def test_no_grad_keep_deformed_equals_padded_model(case, k, d, act):
    c = CASES[case]
    got = _run(c, d, act, k, False, padded=False, no_grad=True)
    pad = _run(c, d, act, k, False, padded=True, no_grad=True)
    assert any(name == "deformed" and a is not None for name, a in got[1])
    _compare(got, pad, None, (d + 1) ** 2, act)


@pytest.mark.parametrize("d,act", DEGREES)
def test_python_render_paths_equal_padded_model(d, act):
    """render() / render_cameras() with autograd, and GraphedRender"""
    c = CASES["tc"]
    res = []
    for padded in (False, True, True):
        scene = _scene(c, d, padded)
        mod = make_module(c["net"], seed=2, aabb=scene["aabb"])
        pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=act, requires_grad=True)
        views = [synth.make_camera(c["theta"] + 40.0 * i, 80, 64, radius=c["radius"], time=c["t"]) for i in range(3)]
        bg = torch.tensor([0.1, 0.2, 0.3], device="cuda")
        one = renderer.render(views[0], pc, _Pipe, bg)
        many = renderer.render_cameras(views, pc, _Pipe, bg)
        loss = (one["render"] * 0.7).sum() + sum((o["render"] * (i + 1)).sum() for i, o in enumerate(many))
        loss.backward()
        with torch.no_grad():
            gr = graphs.GraphedRender(pc, _Pipe, bg, views)
            graphed = [dict(o) for o in gr(views)]
            gr.check()
        outs = [one["render"], one["depth"], one["radii"]] + [o[key] for o in many for key in ("render", "depth", "radii")]
        outs += [o[key].clone() for o in graphed for key in ("render", "depth", "radii")]
        grads = [torch.cat([pc._features_dc.grad, pc._features_rest.grad], dim=1)] + \
            [p.grad.clone() for p in (pc._xyz, pc._scaling, pc._rotation, pc._opacity)] + \
            [p.grad.clone() for p in mod.parameters() if p.grad is not None]
        res.append((outs, [], grads))
        assert pc._features_rest.grad.shape == scene["features_rest"].shape
    _compare(*res, (d + 1) ** 2, act)


@pytest.mark.parametrize("d,act", DEGREES)
def test_rasterizer_equals_padded_model(d, act):
    m = (d + 1) ** 2
    m3, sc, ro, op, sh = [t.float().cuda() for t in raster_inputs(700, seed=4)]
    cam = synth.make_camera(30.0, 72, 56, radius=3.0)
    bg = torch.tensor([0.0, 0.3, 0.1], device="cuda")
    rs = rasterizer.GaussianRasterizationSettings(56, 72, *[float(np.tan(f * 0.5)) for f in (cam.FoVx, cam.FoVy)], bg, 1.0,
                                                  cam.world_view_transform.cuda(), cam.full_proj_transform.cuda(), act,
                                                  cam.camera_center.cuda(), False, False)
    gen = torch.Generator().manual_seed(3)
    dL = torch.rand(3, 56, 72, generator=gen).cuda()
    res = []
    for shs in (sh[:, :m].contiguous(), torch.cat([sh[:, :m], sh.new_zeros(700, 16 - m, 3)], 1), None):
        shs = res[1][3] if shs is None else shs
        leaves = [t.clone().requires_grad_(True) for t in (m3, shs, op, sc, ro)]
        m2 = torch.zeros_like(m3, requires_grad=True)
        color, radii, depth = rasterizer.GaussianRasterizer(rs)(means3D=leaves[0], means2D=m2, shs=leaves[1], opacities=leaves[2],
                                                                scales=leaves[3], rotations=leaves[4])
        (color * dL).sum().backward()
        grads = [leaves[1].grad] + [t.grad for t in (leaves[0], m2, leaves[2], leaves[3], leaves[4])]
        res.append(([color.detach(), depth, radii], [], grads, shs))
    _compare(res[0][:3], res[1][:3], res[2][:3], m, act)
    if (d, act) == (1, 1):      # the CPU raster oracle, fed the padded inputs
        rc, _ = cam_tuple(cam, (0.0, 0.3, 0.1), sh_degree=act)
        ref = rr.rasterize_forward(rc, *[t.cpu().numpy() for t in (m3, sc, ro, op, res[1][3])])
        assert np.array_equal(res[0][0][2].cpu().numpy(), ref["radii"])
        assert np.abs(res[0][0][0].cpu().numpy() - ref["color"]).max() <= IMG_TOL


def _call_refused(fn, outs):
    for o in outs:
        o.fill_(7.0)
    rc = fn()
    torch.cuda.synchronize()
    assert all(bool((o == 7.0).all()) for o in outs)
    return rc


def test_c_abi_refusals_before_any_launch():
    lib = _lib.load()
    ws = _lib.Workspace(0)
    n = 300
    scene = {k: v.cuda() for k, v in synth.make_scene(n, seed=6, scale_mean=0.05, sh_degree=2).items()}
    cam_v = synth.make_camera(10.0, 48, 40)
    pc = synth.SyntheticGaussianModel(scene, None, sh_degree=2)
    rs, t = renderer.settings_from_camera(cam_v, pc, _Pipe, torch.zeros(3, device="cuda"))
    keep = []

    def mk(sh_coeffs, deg=2):
        c = rasterizer.camera_from_settings(rs, time=t, keep=keep, sh_coeffs=sh_coeffs)
        c.sh_degree = deg
        return c
    shs = torch.cat([scene["features_dc"], scene["features_rest"]], 1).contiguous()
    g = _lib.Gaussians(n, *[scene[k].data_ptr() for k in ("xyz", "scaling", "rotation", "opacity", "features_dc", "features_rest")])
    col, dep, rad = torch.empty(3, 40, 48, device="cuda"), torch.empty(1, 40, 48, device="cuda"), torch.empty(n, device="cuda", dtype=torch.int32)
    outs = [col, dep, rad]
    ctx = _lib.Context(ws)
    act_sc = torch.exp(scene["scaling"]).contiguous()
    rot_n = torch.nn.functional.normalize(scene["rotation"]).contiguous()
    op_s = torch.sigmoid(scene["opacity"]).contiguous()
    fwd = lambda cam, prm=None: lambda: lib.g4d_render_forward(ctx.handle, C.byref(cam), prm, C.byref(g), col.data_ptr(),
                                                               dep.data_ptr(), rad.data_ptr(), None)
    rast = lambda cam: lambda: lib.g4d_rasterize_forward(ctx.handle, C.byref(cam), n, scene["xyz"].data_ptr(), shs.data_ptr(),
                                                         op_s.data_ptr(), act_sc.data_ptr(), rot_n.data_ptr(), col.data_ptr(),
                                                         dep.data_ptr(), rad.data_ptr(), None)
    for bad in (2, 5, 15, 17, 25, -1):
        assert _call_refused(fwd(mk(bad)), outs) == ERR_ARG, bad
        assert _call_refused(rast(mk(bad)), outs) == ERR_ARG, bad
    assert _call_refused(fwd(mk(4, deg=2)), outs) == ERR_ARG           # (2 + 1)^2 > 4
    assert _call_refused(rast(mk(1, deg=1)), outs) == ERR_ARG
    shmod = make_module("small128", seed=1, aabb=scene["aabb"])         # the SHS head at M = 9
    prm = shmod.c_params(keep, fresh=True)
    assert _call_refused(fwd(mk(9), C.byref(prm)), outs) == ERR_ARG
    # k cameras whose M differs
    cams = (_lib.Camera * 2)(mk(9), mk(16))
    outs2 = outs + [torch.empty(3, 40, 48, device="cuda"), torch.empty(1, 40, 48, device="cuda"), torch.empty(n, device="cuda", dtype=torch.int32)]
    ctx2 = _lib.Context(ws)
    hs = (C.c_void_p * 2)(ctx.handle, ctx2.handle)
    pp = lambda a, b: (C.c_void_p * 2)(a.data_ptr(), b.data_ptr())
    assert _call_refused(lambda: lib.g4d_render_forward_cameras(hs, 2, cams, None, C.byref(g), pp(outs2[0], outs2[3]),
                                                                pp(outs2[1], outs2[4]), pp(outs2[2], outs2[5]), None), outs2) == ERR_ARG
    # a backward whose M differs from its forward's
    _lib.check(fwd(mk(9))(), "g4d_render_forward")
    gx = [torch.full(sh_, 7.0, device="cuda") for sh_ in ((n, 3), (n, 3), (n, 4), (n, 1), (n, 1, 3), (n, 8, 3), (n, 3))]
    gg = _lib.GaussianGrads(*[t.data_ptr() for t in gx])
    dL = torch.ones(3 * 40 * 48, device="cuda")
    assert _call_refused(lambda: lib.g4d_render_backward(ctx.handle, C.byref(mk(16)), None, None, C.byref(g), dL.data_ptr(),
                                                         C.byref(gg), None), gx) == ERR_STATE
    _lib.check(rast(mk(9))(), "g4d_rasterize_forward")
    gsh = torch.full((n, 9, 3), 7.0, device="cuda")
    rb = lambda cam: lambda: lib.g4d_rasterize_backward(ctx.handle, C.byref(cam), n, scene["xyz"].data_ptr(), shs.data_ptr(),
                                                        op_s.data_ptr(), act_sc.data_ptr(), rot_n.data_ptr(), dL.data_ptr(),
                                                        gx[0].data_ptr(), gx[6].data_ptr(), gsh.data_ptr(), gx[3].data_ptr(),
                                                        gx[1].data_ptr(), gx[2].data_ptr(), None)
    assert _call_refused(rb(mk(4, deg=1)), gx + [gsh]) == ERR_STATE
    _lib.check(rb(mk(9))(), "g4d_rasterize_backward")      # the matching backward still runs
    # the SHS head at M = 9 on the other fused entry points, and the k-camera backward whose M differs from its forward's
    mod64 = make_module("small64", seed=1, aabb=scene["aabb"])
    prm64 = mod64.c_params(keep, fresh=True)
    cg = mod64.c_grads(mod64.alloc_grads())
    cams9 = (_lib.Camera * 2)(mk(9), mk(9))
    fwd_k = lambda prm_: lambda: lib.g4d_render_forward_cameras(hs, 2, cams9, prm_, C.byref(g), pp(outs2[0], outs2[3]),
                                                                pp(outs2[1], outs2[4]), pp(outs2[2], outs2[5]), None)
    assert _call_refused(fwd_k(C.byref(prm)), outs2) == ERR_ARG
    _lib.check(fwd(mk(9), C.byref(prm64))(), "g4d_render_forward")          # FFMA network without the SHS head, M = 9
    bwd = lambda cam, prm_: lambda: lib.g4d_render_backward(ctx.handle, C.byref(cam), prm_, C.byref(cg), C.byref(g), dL.data_ptr(),
                                                            C.byref(gg), None)
    assert _call_refused(bwd(mk(9), C.byref(prm)), gx) == ERR_ARG
    assert _call_refused(bwd(mk(16), C.byref(prm64)), gx) == ERR_STATE
    _lib.check(fwd_k(C.byref(prm64))(), "g4d_render_forward_cameras")
    gk = _lib.GaussianGrads(*[t.data_ptr() for t in gx[:6]], None)
    g2 = [torch.full((n, 3), 7.0, device="cuda") for _ in range(2)]
    dLs = (C.c_void_p * 2)(dL.data_ptr(), dL.data_ptr())
    bwd_k = lambda cams_, prm_: lambda: lib.g4d_render_backward_cameras(hs, 2, cams_, prm_, C.byref(cg), C.byref(g), dLs, C.byref(gk),
                                                                        pp(g2[0], g2[1]), None)
    assert _call_refused(bwd_k(cams9, C.byref(prm)), gx + g2) == ERR_ARG
    assert _call_refused(bwd_k((_lib.Camera * 2)(mk(16), mk(16)), C.byref(prm64)), gx + g2) == ERR_STATE
    _lib.check(bwd_k(cams9, C.byref(prm64))(), "g4d_render_backward_cameras")   # the matching backward still runs
    # Python raises before the library is called
    pc1 = synth.SyntheticGaussianModel(synth.make_scene(n, seed=6, sh_degree=1), shmod, sh_degree=1)
    with pytest.raises(ValueError, match="SH head"):
        renderer.render(cam_v, pc1, _Pipe, torch.zeros(3, device="cuda"))
    pc1.active_sh_degree = 2
    with pytest.raises(ValueError, match="active SH degree 2"):
        renderer.render(cam_v, pc1, _Pipe, torch.zeros(3, device="cuda"), stage="coarse")


def _trainer(padded, seed=0):
    scene = _scene(dict(n=1200), 1, padded)
    mod = make_module("small64", seed=2, aabb=scene["aabb"])
    gs = td.GaussianSet(scene, mod, sh_degree=1)
    opt = td.default_opt()
    opt.densify_from_iter, opt.pruning_from_iter, opt.min_gaussians_for_prune = 2, 2, 100
    opt.densification_interval = opt.pruning_interval = 3
    opt.densify_grad_threshold_fine_init = opt.densify_grad_threshold_after = 5e-6
    opt.opacity_threshold_fine_init = opt.opacity_threshold_fine_after = 0.2
    return td.DPTrainer(gs, opt, cameras_extent=2.6, seed=seed)


def test_trainer_at_degree_1():
    W, H = 80, 64
    cams = [synth.make_camera(th, W, H, radius=4.0, time=t) for th, t in ((0.0, 0.1), (60.0, 0.5), (120.0, 0.9), (200.0, 0.3))]
    bg = torch.zeros(3, device="cuda")
    gts = [torch.full((3, H, W), 0.25, device="cuda") for _ in cams]
    # one step against the padded model's (and a second padded run for repeatability)
    runs = []
    for padded in (False, True, True):
        tr = _trainer(padded)
        tr.step(cams[:2], gts[:2], bg, _Pipe)
        torch.cuda.synchronize()
        runs.append(tr)
    a, p, p2 = (dict(t.g.named()) for t in runs)
    grads = lambda t: {k: v.grad.clone() for k, v in t.g.named().items()}
    ga, gp, gp2 = (grads(t) for t in runs)
    repeatable = all(torch.equal(gp[k], gp2[k]) for k in gp) and torch.equal(runs[1].state.grad[runs[1].state.segments["grid"][0]:],
                                                                               runs[2].state.grad[runs[2].state.segments["grid"][0]:])
    assert a["f_rest"].shape == (1200, 3, 3) and p["f_rest"].shape == (1200, 15, 3)
    assert bool((gp["f_rest"][:, 3:] == 0).all()) and bool((p["f_rest"].data[:, 3:] == 0).all())
    ga["f_rest"], gp["f_rest"] = ga["f_rest"], gp["f_rest"][:, :3]
    pa = {k: v.data for k, v in a.items()}
    pp_ = {k: (v.data[:, :3] if k == "f_rest" else v.data) for k, v in p.items()}
    for k in ga:
        assert _close(ga[k], gp[k], repeatable), k
        if repeatable:
            assert torch.equal(pa[k], pp_[k]), k
        else:   # Adam's first step moves an entry by lr * sign(g): equal wherever the tolerance fixes the gradient's sign
            sure = gp[k].abs() > SUM_TOL * max(1e-3, float(gp[k].abs().max()))
            assert float((pa[k] - pp_[k]).abs()[sure].max()) <= SUM_TOL * max(1.0, float(pp_[k].abs().max())), k
    sa, sp = runs[0].state, runs[1].state
    ba, ea = sa.segments["grid"][0], sa.numel
    bp, ep = sp.segments["grid"][0], sp.numel
    assert _close(sa.grad[ba:ea], sp.grad[bp:ep], repeatable)
    # a few more steps with densification and pruning at degree 1
    tr = runs[0]
    n0, first = tr.g._xyz.shape[0], None
    for it in range(8):
        loss = float(tr.step(cams[(it % 2) * 2:(it % 2) * 2 + 2], gts[:2], bg, _Pipe))
        first = loss if first is None else first
    assert tr.rebuilds > 1 and tr.g._xyz.shape[0] != n0
    assert tr.g._features_rest.shape[1:] == (3, 3) and tr.g.max_sh_degree == 1
    assert tr.state.attached() and bool(torch.isfinite(tr.state.param).all()) and loss < first
