"""GPU: the gradient of the depth image through the GaussianRasterizer drop-in, render() on both network engines and
render_cameras, against the oracles of util_depth_grad (the C oracle's colour backward with colour z, and fp64 autograd of the
dense formulation), with DESIGN.md §2.2's rules: per-row 2e-3 (floor 1e-4 of the tensor's max), the upstream gradient zeroed
on both sides at flip and threshold pixels, Gaussians on a kink of the network or of the colour clamp silenced.  Also:
everything else a backward computes is unchanged by a depth gradient, the camera and time leaves take its terms, the pointer
rules of g4d_context_set_depth_grad, and a depth map fitted by Adam."""
import ctypes as C
import gc
import importlib
import math

import numpy as np
import pytest
import torch

from oracle import deform_ref as dr
from oracle import raster_ref as rr
from oracle.dense_ref import cam_dict_from
import util_camera_grad as ucg
import util_depth_grad as udg
import util_raster_edges as ue
from test_gpu_raster_edges import _check_forward, _settings
from util_scene import (SCENE_LEAVES, colour_kink_rows, deformed_fp64, kink_rows, make_module, oracle_chain_backward,
                        oracle_params_from_module, params_fp64, raster_inputs, raster_oracle_inputs, rel_err, row_errors, synth,
                        threshold_pixels, _deform_activate, cam_tuple)

pytestmark = pytest.mark.gpu
g4d = importlib.import_module("4dgaussians_b200")
_lib = importlib.import_module("4dgaussians_b200._lib")
rasterizer = importlib.import_module("4dgaussians_b200.rasterizer")

ROW_TOL = 2e-3
LONG_ROW_TOL = 5e-3
FLOOR = 1e-4
LONG_DEPTH_FLOOR = 1e-2     # as test_depth_grad_cpu: depth-only on 255-1400 layers 5e-4 apart is ill-conditioned in fp32
PLANE_FLOOR = 1e-2          # as test_gpu_fullsize_backward
MLP_TOL = {0: 2e-4, 2: 5e-4}
CAM_TOL = 2e-3              # as test_gpu_camera_grad: of the tensor's max
TIME_TOL = 5e-3             # as test_gpu_time_grad: of sum |dL/dt_g|
SUM_TOL = 2e-5              # atomic accumulation order (as test_gpu_camera_grad)
SILENCED_LOGIT = -40.0
T = 0.4


@pytest.fixture(autouse=True, scope="module")
def _own_workspace():
    """This module renders on a workspace of its own (as test_gpu_camera_grad): its contexts learn small capacities."""
    dev = torch.cuda.current_device()
    shared = _lib.Workspace._by_device.get(dev)
    _lib.Workspace._by_device[dev] = _lib.Workspace(dev)
    try:
        yield
    finally:
        torch.cuda.synchronize()
        if shared is None:
            del _lib.Workspace._by_device[dev]
        else:
            _lib.Workspace._by_device[dev] = shared
        gc.collect()


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


class _engine:
    def __init__(self, tc):
        self.ws, self.tc = _lib.workspace_of(torch.device("cuda")), tc

    def __enter__(self):
        self.ws.set_option(_lib.OPT_TENSOR_CORES, self.tc)

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.ws.set_option(_lib.OPT_TENSOR_CORES, 2)
        return False


def _cots(H, W, seed, mode, mask):
    """(colour cotangent or None, depth cotangent), zero where mask is False"""
    g = torch.Generator().manual_seed(seed)
    dD = torch.randn(1, H, W, generator=g)
    dD[:, ~mask] = 0.0
    dC = None
    if mode != "depth":
        dC = torch.randn(3, H, W, generator=g)
        dC[:, ~mask] = 0.0
    return dC, dD


def _loss(img, dep, dC, dD):
    loss = (dep * dD.cuda()).sum()
    return loss if dC is None else loss + (img * dC.cuda()).sum()


def _compare_rows(got, want, tol=ROW_TOL, floor=FLOOR, what=""):
    failures = []
    for k in want:
        g, w = np.asarray(got[k], np.float64), np.asarray(want[k], np.float64)
        e = row_errors(g.reshape(len(g), -1), w.reshape(len(w), -1), floor)
        if float(e.max(initial=0.0)) > tol:
            failures.append((k, float(e.max()), int(np.argmax(e))))
    assert not failures, (what, failures)


# ---- 1. the rasterizer drop-in on the edge scenes -----------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["depth", "mixed"])
@pytest.mark.parametrize("name", ue.names())
def test_rasterizer(name, mode):
    sc = ue.scene(name)
    rc, _ = cam_tuple(sc.cam, sc.bg, sh_degree=sc.deg)
    ref = rr.rasterize_forward(rc, *sc.ins)
    m3, s, r, o, sh = [torch.from_numpy(a).cuda().requires_grad_(True) for a in sc.ins]
    m2 = torch.zeros_like(m3, requires_grad=True)
    color, radii, depth = g4d.GaussianRasterizer(_settings(sc), differentiable_depth=True)(
        means3D=m3, means2D=m2, shs=sh, colors_precomp=None, opacities=o, scales=s, rotations=r, cov3D_precomp=None)
    torch.cuda.synchronize()
    keep = _check_forward(sc, color.grad_fn.lease.ctx, radii.cpu().numpy(), color.detach().cpu().numpy(), ref)
    dC, dD = _cots(sc.H, sc.W, sum(map(ord, name)) + len(mode), mode, torch.from_numpy(keep))
    _loss(color, depth, dC, dD).backward()
    torch.cuda.synchronize()
    want = udg.oracle_backward(rc, sc.ins, ref, None if dC is None else dC.numpy(), dD.numpy())
    got = {"means3D": m3.grad, "means2D": m2.grad, "scales": s.grad, "rots": r.grad, "opacities": o.grad, "shs": sh.grad}
    got = {k: v.cpu().numpy() for k, v in got.items()}
    unseen = ref["radii"] == 0
    for k, v in got.items():
        assert not v[unseen].any(), k
    if mode == "depth":
        assert not got["shs"].any()
    long = sc.group == "long"
    _compare_rows(got, {k: want[k] for k in got}, LONG_ROW_TOL if long else ROW_TOL,
                  LONG_DEPTH_FLOOR if long and mode == "depth" else FLOOR, name)


# ---- 2. render() on both engines against the fp64 chain --------------------------------------------------------------------
def _silenced_scene(n, seed, net, cams):
    """a scene and module whose Gaussians on a kink of the network or of the colour clamp are silenced (logit -40)"""
    scene = dict(synth.make_scene(n, seed=seed, scale_mean=0.05))
    mod = make_module(net, seed=seed, aabb=scene["aabb"])
    cfg, prm = oracle_params_from_module(mod)
    for p in prm.leaves():
        p.requires_grad_(False)
    t = float(np.float32(T))
    pts, shs = deformed_fp64(cfg, prm, scene, t)
    silenced = (kink_rows(cfg, prm, scene["xyz"], t) | colour_kink_rows(pts, shs, cams, sh_degree=3)).numpy()
    scene["opacity"] = scene["opacity"].clone()
    scene["opacity"][torch.from_numpy(silenced)] = SILENCED_LOGIT
    return scene, mod, cfg, prm, silenced


def _keep(ctx, radii, img, ref, W, H):
    """pixels compared: no flip of n_contrib or the image between GPU and oracle, no instance on a threshold"""
    rec = ue.gpu_record(ctx, radii, W, H)
    flip = (rec["n_contrib"] != ref["n_contrib"]) | (np.abs(img - ref["color"]).max(axis=0) > 1e-4)
    assert flip.mean() < 0.01
    return ~(flip | threshold_pixels(ref, W, H, include_stop=True))


def _plane_rows(a):
    a = np.asarray(a)
    return a[0].transpose(1, 2, 0).reshape(-1, a.shape[1])


def _check_network(mod, p64, tc, what):
    gp = {k: p.grad for k, p in mod.named_parameters()}
    seen = 0
    for key, p in dr.params_to_state_dict(p64).items():
        if key not in gp or p.grad is None:
            continue
        g = gp[key].cpu().numpy()
        if key.startswith("deformation_net.grid.grids."):
            _compare_rows({key: _plane_rows(g)}, {key: _plane_rows(p.grad.numpy())}, ROW_TOL, PLANE_FLOOR, what)
        else:
            assert rel_err(g, p.grad.numpy()) <= MLP_TOL[tc], (what, key, rel_err(g, p.grad.numpy()))
        seen += 1
    assert seen > 10


@pytest.mark.parametrize("mode", ["depth", "mixed"])
@pytest.mark.parametrize("tc", [0, 2])
def test_render_vs_oracle_chain(tc, mode):
    W, H = 61, 47
    cam = synth.make_camera(30.0, W, H, radius=3.0, time=T)
    scene, mod, cfg, prm, silenced = _silenced_scene(500, 5 + tc, "small128", [cam])
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
    bg = (0.0, 0.1, 0.2)
    with _engine(tc):
        out = g4d.render(cam, pc, _Pipe, torch.tensor(bg, device="cuda"), stage="fine")
        torch.cuda.synchronize()
        ctx = out["render"].grad_fn.lease.ctx
        shs = ctx.read("deformed_shs") if not mod.args.no_dshs else \
            torch.cat([scene["features_dc"], scene["features_rest"]], 1).numpy()
        ins = raster_oracle_inputs(ctx.read("deformed"), shs)
        rc, _ = cam_tuple(cam, bg, sh_degree=3)
        ref = rr.rasterize_forward(rc, *ins)
        keep = _keep(ctx, out["radii"].cpu().numpy(), out["render"].detach().cpu().numpy(), ref, W, H)
        dC, dD = _cots(H, W, 31 + tc, mode, torch.from_numpy(keep))
        _loss(out["render"], out["depth"], dC, dD).backward()
    cot = udg.oracle_backward(rc, ins, ref, None if dC is None else dC.numpy(), dD.numpy())
    want, p64 = oracle_chain_backward(cfg, prm, scene, float(np.float32(T)), cot)
    got = {k: getattr(pc, "_" + k).grad.cpu().numpy().reshape(want[k].shape) for k in SCENE_LEAVES}
    for k in SCENE_LEAVES:
        assert not got[k][silenced].any(), k
    what = "render tc=%d %s" % (tc, mode)
    _compare_rows(got, want, what=what)
    _compare_rows({"means2D": out["viewspace_points"].grad.cpu().numpy()}, {"means2D": cot["means2D"]}, what=what)
    _check_network(mod, p64, tc, what)


# ---- 3. render_cameras, k = 3: colour only, depth only, both ---------------------------------------------------------------
def _grads(pc, mod):
    return [p.grad.clone() for p in pc.gaussian_parameters()] + [p.grad.clone() for p in mod.parameters() if p.grad is not None]


def test_render_cameras_matches_three_renders():
    cams = [synth.make_camera(th, 61 + 4 * i, 47, radius=3.0, time=T) for i, th in enumerate((10.0, 100.0, -120.0))]
    scene = synth.make_scene(500, seed=9, scale_mean=0.05)
    mod = make_module("small128", seed=9, aabb=scene["aabb"])
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
    bg = torch.tensor([0.2, 0.1, 0.0], device="cuda")
    cots = []
    for i, (c, mode) in enumerate(zip(cams, ("colour", "depth", "mixed"))):
        g = torch.Generator().manual_seed(40 + i)
        H, W = c.image_height, c.image_width
        cots.append((None if mode == "depth" else torch.randn(3, H, W, generator=g).cuda(),
                     None if mode == "colour" else torch.randn(1, H, W, generator=g).cuda()))

    def loss(o, dC, dD):
        out = torch.zeros((), device="cuda")
        if dC is not None:
            out = out + (o["render"] * dC).sum()
        if dD is not None:
            out = out + (o["depth"] * dD).sum()
        return out

    outs = g4d.render_cameras(cams, pc, _Pipe, bg, stage="fine")
    sum(loss(o, *c) for o, c in zip(outs, cots)).backward()
    group = _grads(pc, mod)
    views = [o["viewspace_points"].grad.clone() for o in outs]
    for p in list(pc.gaussian_parameters()) + list(mod.parameters()):
        p.grad = None
    single_views = []
    for c, cot in zip(cams, cots):
        o = g4d.render(c, pc, _Pipe, bg, stage="fine")
        loss(o, *cot).backward()
        single_views.append(o["viewspace_points"].grad.clone())
    single = _grads(pc, mod)
    assert len(group) == len(single)
    for i, (a, b) in enumerate(zip(group, single)):
        a, b = a.cpu().numpy(), b.cpu().numpy()
        if a.ndim >= 2 and a.shape[0] == 500:
            _compare_rows({"g%d" % i: a}, {"g%d" % i: b}, what="render_cameras leaf %d" % i)
        else:
            assert rel_err(a, b) <= 5e-4, ("render_cameras parameter", i, rel_err(a, b))
    for i, (a, b) in enumerate(zip(views, single_views)):
        _compare_rows({"m": a.cpu().numpy()}, {"m": b.cpu().numpy()}, what="viewspace_points %d" % i)
    assert float(views[1].abs().max()) > 0        # the depth-only camera is part of the loss


# ---- 4. camera and time leaves take the depth term ----------------------------------------------------------------------------
def _leaf_camera(cam, t):
    f = lambda x: x.detach().float().cuda().clone().requires_grad_(True)
    return synth.SynthCamera(FoVx=cam.FoVx, FoVy=cam.FoVy, image_width=cam.image_width, image_height=cam.image_height,
                             world_view_transform=f(cam.world_view_transform), full_proj_transform=f(cam.full_proj_transform),
                             camera_center=f(cam.camera_center), time=t)


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
    dC, dD = _cots(47, 61, 17, "mixed", mask)
    want = udg.dense_grads(cd, [x.numpy() for x in inputs], dC.double(), dD.double(), cam_keys=ucg.CAM_KEYS)
    colour_only = udg.dense_grads(cd, [x.numpy() for x in inputs], dC.double(), None, cam_keys=("view",))
    per = udg.oracle_time_grads(cfg, prm, scene, cd, t, dC.double(), dD.double())
    leaf_t = torch.tensor(t, device="cuda", dtype=torch.float32, requires_grad=True)
    lc = _leaf_camera(cam, leaf_t)
    with _engine(tc):
        out = g4d.render(lc, pc, _Pipe, torch.tensor(bg, device="cuda"), stage="fine")
        _loss(out["render"], out["depth"], dC, dD).backward()
    got = {"view": lc.world_view_transform.grad, "proj": lc.full_proj_transform.grad, "campos": lc.camera_center.grad}
    for k in ucg.CAM_KEYS:
        ucg.assert_close_to_max(got[k].reshape(-1).cpu(), want[k], CAM_TOL, "tc=%d %s" % (tc, k))
    # the depth term is large enough here that a backward without it would fail the view check
    assert np.abs(want["view"] - colour_only["view"]).max() > 10 * CAM_TOL * np.abs(want["view"]).max()
    ref, scale = float(per.sum()), float(per.abs().sum())
    assert abs(float(leaf_t.grad) - ref) <= TIME_TOL * scale, (float(leaf_t.grad), ref, scale)


# ---- 5. nothing else moves ----------------------------------------------------------------------------------------------------
def _everything(path, depth, k=1):
    """images, depths, radii and every gradient of a colour loss plus <depth, dD> (depth: "none", "zero" or "random"; "plain":
    the rasterizer drop-in's default, a depth without grad, and a colour loss)"""
    torch.manual_seed(0)
    scene = synth.make_scene(500, seed=13, scale_mean=0.05)
    mod = make_module("small128", seed=13, aabb=scene["aabb"])
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
    bg = torch.tensor([0.3, 0.2, 0.1], device="cuda")
    cams = [synth.make_camera(25.0 + 70 * i, 64, 48, radius=3.0, time=0.3) for i in range(k)]
    cot = torch.randn(3, 48, 64, generator=torch.Generator().manual_seed(3)).cuda()
    dD = torch.randn(1, 48, 64, generator=torch.Generator().manual_seed(4)).cuda()
    dD = dD * 0.0 if depth == "zero" else dD

    def loss(img, dep):
        return (img * cot).sum() + ((dep * dD).sum() if depth in ("zero", "random") else 0.0)

    if path == "rasterizer":
        c = cams[0]
        inputs = [t.float().cuda().requires_grad_(True) for t in raster_inputs(500, 13, scale_mean=0.05)]
        rs = rasterizer.GaussianRasterizationSettings(48, 64, math.tan(c.FoVx * 0.5), math.tan(c.FoVy * 0.5), bg, 1.0,
                                                      c.world_view_transform.cuda(), c.full_proj_transform.cuda(), 3,
                                                      c.camera_center.cuda(), False, False)
        m2 = torch.zeros_like(inputs[0], requires_grad=True)
        img, rad, dep = rasterizer.GaussianRasterizer(rs, differentiable_depth=depth != "plain")(
            means3D=inputs[0], means2D=m2, shs=inputs[4], opacities=inputs[3], scales=inputs[1], rotations=inputs[2])
        assert dep.requires_grad == (depth != "plain")
        loss(img, dep).backward()
        return [img, dep, rad], [m2.grad] + [t.grad for t in inputs]
    outs = g4d.render_cameras(cams, pc, _Pipe, bg, stage="fine")
    sum(loss(o["render"], o["depth"]) for o in outs).backward()
    fwd = [x for o in outs for x in (o["render"], o["depth"], o["radii"])]
    grads = [o["viewspace_points"].grad for o in outs]
    return fwd, grads + [p.grad for p in pc.gaussian_parameters()] + [p.grad for p in mod.parameters() if p.grad is not None]


@pytest.mark.parametrize("path,k", [("rasterizer", 1), ("render", 1), ("render", 3)])
@pytest.mark.parametrize("tc", [0, 2])
def test_depth_gradient_leaves_everything_else_unchanged(path, k, tc):
    """Forward outputs byte-identical with and without a depth loss; a zero depth cotangent gives the gradients of no depth
    loss within twice the spread of two runs without one, or SUM_TOL of the tensor's max (atomic accumulation order)"""
    if path == "rasterizer" and tc == 2:
        pytest.skip("the rasterizer drop-in runs no network")
    arms = ("none", "zero", "none", "random") + (("plain",) if path == "rasterizer" else ())
    with _engine(tc):
        runs = [_everything(path, d, k) for d in arms]
    (fa, ga), (fz, gz), (fa2, ga2), (fr, gr) = runs[:4]
    for f, _ in runs[1:]:
        for i, x in enumerate(fa):
            assert torch.equal(x, f[i]), "forward output %d moved" % i
    assert len({len(g) for _, g in runs}) == 1
    moved = 0
    for j, (x, x2, w) in enumerate(zip(ga, ga2, gr)):
        x, x2, w = x.double(), x2.double(), w.double()
        spread = float((x - x2).abs().max())
        bound = max(2 * spread, SUM_TOL * max(1e-3, float(x.abs().max())))
        for _, g in runs[1:2] + runs[4:]:        # a zero depth cotangent, and the drop-in's default: as no depth loss
            assert float((x - g[j].double()).abs().max()) <= bound
        moved += float((x - w).abs().max()) > bound
    assert moved > 0            # a real depth loss does move the gradients


# ---- 6. the setter's pointer rules ------------------------------------------------------------------------------------------
def _coarse(ctx, n, no_grad=False):
    """a coarse-stage render forward on ctx and a closure running its backward into NaN-filled sinks"""
    lib = _lib.load()
    sc = synth.make_scene(n, seed=4, scale_mean=0.05)
    x, s, r, o, dc, rest = [sc[k].float().cuda().contiguous() for k in SCENE_LEAVES]
    g = _lib.Gaussians(n, x.data_ptr(), s.data_ptr(), r.data_ptr(), o.data_ptr(), dc.data_ptr(), rest.data_ptr())
    cam0 = synth.make_camera(15.0, 64, 48, radius=3.0)
    rs = rasterizer.GaussianRasterizationSettings(48, 64, math.tan(cam0.FoVx * 0.5), math.tan(cam0.FoVy * 0.5),
                                                  torch.zeros(3, device="cuda"), 1.0, cam0.world_view_transform.cuda(),
                                                  cam0.full_proj_transform.cuda(), 3, cam0.camera_center.cuda(), False, False)
    keep = [x, s, r, o, dc, rest]
    cam = rasterizer.camera_from_settings(rs, keep=keep, sh_coeffs=16)
    if no_grad:
        cam.debug |= _lib.CAM_NO_GRAD
    col, dep = torch.empty(3, 48, 64, device="cuda"), torch.empty(1, 48, 64, device="cuda")
    rad = torch.empty(n, device="cuda", dtype=torch.int32)
    st = _lib.stream_of(torch.device("cuda"))
    _lib.check(lib.g4d_render_forward(ctx.handle, C.byref(cam), None, C.byref(g), col.data_ptr(), dep.data_ptr(),
                                      rad.data_ptr(), st), "g4d_render_forward")
    sinks = [torch.full((n * w,), float("nan"), device="cuda") for w in (3, 3, 4, 1, 3, 45, 3)]
    gg = _lib.GaussianGrads(*[t.data_ptr() for t in sinks])
    gcol = torch.ones(3 * 48 * 64, device="cuda")

    def bwd():
        keep.append((cam, g, gg, gcol))
        return lib.g4d_render_backward(ctx.handle, C.byref(cam), None, None, C.byref(g), gcol.data_ptr(), C.byref(gg),
                                       _lib.stream_of(torch.device("cuda")))
    return bwd, sinks


def test_depth_grad_pointer_rules():
    ws = _lib.workspace_of(torch.device("cuda"))
    ctx = _lib.Context(ws)
    n = 200
    dD = torch.randn(48 * 64, generator=torch.Generator().manual_seed(1)).cuda()
    try:
        # a no-grad forward's context: the backward is refused before any launch, the sinks untouched
        bwd, sinks = _coarse(ctx, n, no_grad=True)
        ctx.set_depth_grad(dD.data_ptr())
        assert bwd() == -4
        torch.cuda.synchronize()
        assert all(torch.isnan(t).all() for t in sinks)
        # under stream capture, with the pointer set: refused before any launch (nothing is captured)
        bwd, sinks = _coarse(ctx, n)
        torch.cuda.synchronize()
        graph, stream = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            graph.capture_begin()
            rc = bwd()
            graph.capture_end()
        torch.cuda.synchronize()
        assert rc == -4 and "depth gradient" in _lib.load().g4d_last_error().decode()
        assert all(torch.isnan(t).all() for t in sinks)
        # set: the depth term is in the gradients
        bwd, with_depth = _coarse(ctx, n)
        assert bwd() == 0
        # NULL turns it off: the gradients of a context that never had one
        ctx.set_depth_grad(None)
        bwd, off = _coarse(ctx, n)
        assert bwd() == 0
        other = _lib.Context(ws)
        bwd, never = _coarse(other, n)
        assert bwd() == 0
        torch.cuda.synchronize()
        for a, b, c in zip(off, never, with_depth):
            assert torch.isfinite(a).all() and torch.isfinite(c).all()
            assert float((a - b).abs().max()) <= SUM_TOL * max(1e-3, float(b.abs().max()))
        assert float((with_depth[0] - never[0]).abs().max()) > 1e-3 * float(never[0].abs().max())
    finally:
        ctx.set_depth_grad(None)


# ---- 7. a depth map fitted by Adam ---------------------------------------------------------------------------------------------
# first H100 run (H100 80GB HBM3, 700 W): the loss fell from 0.102 to 0.0024, a ratio of 0.024, in 100 steps; the bound keeps
# an 8x margin over it
FIT_STEPS = 100
FIT_RATIO = 0.2


def test_adam_fits_a_depth_map():
    cam = synth.make_camera(40.0, 128, 96, radius=4.0)
    m3, sc, ro, op, sh = [t.float().cuda() for t in raster_inputs(3000, 21, scale_mean=0.04)]
    rs = rasterizer.GaussianRasterizationSettings(96, 128, math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5),
                                                  torch.zeros(3, device="cuda"), 1.0, cam.world_view_transform.cuda(),
                                                  cam.full_proj_transform.cuda(), 3, cam.camera_center.cuda(), False, False)
    g = torch.Generator().manual_seed(2)
    target_xyz = m3 + 0.05 * torch.randn(m3.shape, generator=g).cuda()

    def depth(xyz):
        return rasterizer.GaussianRasterizer(rs, differentiable_depth=True)(
            means3D=xyz, means2D=torch.zeros_like(xyz), shs=sh, opacities=op, scales=sc, rotations=ro)[2]

    with torch.no_grad():
        target = depth(target_xyz)
    xyz = m3.clone().requires_grad_(True)
    opt = torch.optim.Adam([xyz], lr=2e-3)
    losses = []
    for _ in range(FIT_STEPS):
        opt.zero_grad()
        loss = ((depth(xyz) - target) ** 2).mean()
        loss.backward()
        assert xyz.grad is not None and torch.isfinite(xyz.grad).all()
        opt.step()
        losses.append(float(loss.detach()))
    print("depth loss: initial %.5g final %.5g ratio %.3f" % (losses[0], losses[-1], losses[-1] / losses[0]))
    assert losses[-1] <= FIT_RATIO * losses[0], losses[::10]
