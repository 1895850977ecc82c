"""GPU: gradients w.r.t. the camera -- view matrix, projection matrix, camera centre -- through the rasterizer drop-in,
render() on both network engines, and render_cameras, against the fp64 dense oracle with the camera tensors as leaves
(util_camera_grad).  Tolerance: DESIGN.md §2.2's 2e-3 of the tensor's max; the cotangent is zero on the threshold pixels of
util_camera_grad.threshold_pixel_mask, fixed before comparing.  Also: everything else a backward computes is unchanged when
camera gradients are requested, a pose recovered by Adam through render(), and the refusals."""
import ctypes as C
import gc
import importlib
import math

import numpy as np
import pytest
import torch

import util_camera_grad as ucg
from oracle.dense_ref import cam_dict_from
from util_scene import _deform_activate, make_module, oracle_params_from_module, params_fp64, raster_inputs, synth

pytestmark = pytest.mark.gpu
g4d = importlib.import_module("4dgaussians_b200")
_lib = importlib.import_module("4dgaussians_b200._lib")
rasterizer = importlib.import_module("4dgaussians_b200.rasterizer")

TOL = 2e-3


@pytest.fixture(autouse=True, scope="module")
def _own_workspace():
    """This module renders on a workspace of its own: its contexts learn the instance capacities of these small images and
    must not return to the shared pool that later modules lease from (a no-sync forward there would overflow them)."""
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
SCENE_LEAVES = ("xyz", "scaling", "rotation", "opacity", "features_dc", "features_rest")


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


def _fp32_cd(cam, bg, deg):
    cd = cam_dict_from(cam, bg, deg)
    cd["tanfovx"], cd["tanfovy"] = float(np.float32(cd["tanfovx"])), float(np.float32(cd["tanfovy"]))
    return cd


def _leaf_camera(cam):
    """the camera with its three tensors replaced by CUDA fp32 leaves that require grad"""
    f = lambda t: t.detach().float().cuda().clone().requires_grad_(True)
    return synth.SynthCamera(FoVx=cam.FoVx, FoVy=cam.FoVy, image_width=cam.image_width, image_height=cam.image_height,
                             world_view_transform=f(cam.world_view_transform), full_proj_transform=f(cam.full_proj_transform),
                             camera_center=f(cam.camera_center), time=cam.time)


def _grads_of(cam):
    return {"view": cam.world_view_transform.grad.reshape(-1).cpu(), "proj": cam.full_proj_transform.grad.reshape(-1).cpu(),
            "campos": cam.camera_center.grad.reshape(-1).cpu()}


def _cot(H, W, seed, mask=None):
    cot = torch.randn(3, H, W, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)
    if mask is not None:
        cot[:, mask] = 0.0
    return cot


def _check(got, ref, what):
    for k in ucg.CAM_KEYS:
        ucg.assert_close_to_max(got[k], ref[k], TOL, "%s %s" % (what, k))
    for i in range(16):
        if i not in ucg.VIEW_READ:
            assert float(got["view"][i]) == 0.0
        if i not in ucg.PROJ_READ:
            assert float(got["proj"][i]) == 0.0


# ---- 2. the rasterizer drop-in ------------------------------------------------------------------------------------------
# radius 0.9: the camera sits inside the point cloud (extent 1.3): Gaussians behind the near plane and in the guard band
@pytest.mark.parametrize("deg,theta,radius,wh,seed", [(0, 20.0, 4.0, (61, 47), 0), (1, -70.0, 3.0, (64, 48), 1),
                                                       (2, 140.0, 2.0, (61, 47), 2), (3, 35.0, 0.9, (61, 47), 3),
                                                       (3, -15.0, 3.5, (47, 61), 4)])
def test_rasterizer_camera_grads_vs_oracle(deg, theta, radius, wh, seed):
    W, H = wh
    inputs = raster_inputs(300, seed, scale_mean=0.05)
    cam = synth.make_camera(theta, W, H, radius=radius)
    bg = (0.1, 0.2, 0.3)
    cd = _fp32_cd(cam, bg, deg)
    if radius < 1.3:        # the scene this case is for: some Gaussians behind the near plane, some in the guard band
        v = cam.world_view_transform.double().reshape(16)
        m = inputs[0]
        tz = v[2] * m[:, 0] + v[6] * m[:, 1] + v[10] * m[:, 2] + v[14]
        tx = v[0] * m[:, 0] + v[4] * m[:, 1] + v[8] * m[:, 2] + v[12]
        assert (tz < 0.2).any() and ((tx / tz).abs() > 1.3 * cd["tanfovx"])[tz > 0.2].any()
    cot = _cot(H, W, seed, ucg.threshold_pixel_mask(cd, inputs))
    _, ref = ucg.dense_camera_grads(cd, inputs, cot)
    lc = _leaf_camera(cam)
    rs = rasterizer.GaussianRasterizationSettings(
        image_height=H, image_width=W, tanfovx=math.tan(cam.FoVx * 0.5), tanfovy=math.tan(cam.FoVy * 0.5),
        bg=torch.tensor(bg, device="cuda"), scale_modifier=1.0, viewmatrix=lc.world_view_transform,
        projmatrix=lc.full_proj_transform, sh_degree=deg, campos=lc.camera_center, prefiltered=False, debug=False)
    m3, sc, ro, op, sh = [t.float().cuda() for t in inputs]
    sh = sh[:, :(deg + 1) ** 2].contiguous()
    img, _, _ = rasterizer.GaussianRasterizer(rs)(means3D=m3, means2D=torch.zeros_like(m3, requires_grad=True), shs=sh,
                                                  opacities=op, scales=sc, rotations=ro)
    (img * cot.float().cuda()).sum().backward()
    got = _grads_of(lc)
    _check(got, ref, "rasterizer deg %d" % deg)
    if deg == 0:
        assert torch.equal(got["campos"], torch.zeros(3))


# ---- 3. render() on both engines, vs the fp64 chain deform_ref -> dense render ---------------------------------------------
def _fused_setup(n, seed):
    scene = synth.make_scene(n, seed=seed, scale_mean=0.05)
    mod = make_module("small128", seed=seed, aabb=scene["aabb"])
    return scene, mod


def _chain_oracle(mod, scene, cam, t, bg, deg, cot_seed):
    cfg, prm = oracle_params_from_module(mod)
    with torch.no_grad():
        lv = {k: scene[k].double() for k in SCENE_LEAVES}
        inputs = _deform_activate(cfg, params_fp64(prm), lv, t)
    cd = _fp32_cd(cam, bg, deg)
    W, H = cd["W"], cd["H"]
    cot = _cot(H, W, cot_seed, ucg.threshold_pixel_mask(cd, inputs))
    return cot, ucg.dense_camera_grads(cd, inputs, cot)[1]


@pytest.mark.parametrize("tc", [0, 2])
@pytest.mark.parametrize("deg", [0, 3])
def test_render_camera_grads_vs_oracle_chain(tc, deg):
    ws = _lib.workspace_of(torch.device("cuda"))
    ws.set_option(_lib.OPT_TENSOR_CORES, tc)
    try:
        scene, mod = _fused_setup(400, 5 + deg)
        pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=deg, requires_grad=True)
        cam = synth.make_camera(30.0, 61, 47, radius=3.0, time=0.4)
        bg = (0.0, 0.1, 0.2)
        cot, ref = _chain_oracle(mod, scene, cam, 0.4, bg, deg, cot_seed=11)
        lc = _leaf_camera(cam)
        out = g4d.render(lc, pc, _Pipe, torch.tensor(bg, device="cuda"), stage="fine")
        (out["render"] * cot.float().cuda()).sum().backward()
        _check(_grads_of(lc), ref, "render tc=%d deg=%d" % (tc, deg))
    finally:
        torch.cuda.synchronize()
        ws.set_option(_lib.OPT_TENSOR_CORES, 2)


# ---- 4. render_cameras, k = 3 --------------------------------------------------------------------------------------------
def test_render_cameras_camera_grads():
    scene, mod = _fused_setup(400, 9)
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
    bg = (0.2, 0.1, 0.0)
    cams = [synth.make_camera(th, 61 + 4 * i, 47, radius=3.0, time=0.25) for i, th in enumerate((10.0, 100.0, -120.0))]
    cots = [_chain_oracle(mod, scene, c, 0.25, bg, 3, cot_seed=20 + i) for i, c in enumerate(cams)]
    # every camera in the loss: each camera's gradients match the oracle and a render() of that camera alone
    leaf = [_leaf_camera(c) for c in cams]
    outs = g4d.render_cameras(leaf, pc, _Pipe, torch.tensor(bg, device="cuda"), stage="fine")
    sum((o["render"] * cot.float().cuda()).sum() for o, (cot, _) in zip(outs, cots)).backward()
    for i, (lc, (cot, ref)) in enumerate(zip(leaf, cots)):
        got = _grads_of(lc)
        _check(got, ref, "render_cameras camera %d" % i)
        single = _leaf_camera(cams[i])
        (g4d.render(single, pc, _Pipe, torch.tensor(bg, device="cuda"), stage="fine")["render"] * cot.float().cuda()).sum().backward()
        _check(got, _grads_of(single), "render_cameras camera %d vs render()" % i)
    # camera 1 outside the loss: zeros
    leaf = [_leaf_camera(c) for c in cams]
    outs = g4d.render_cameras(leaf, pc, _Pipe, torch.tensor(bg, device="cuda"), stage="fine")
    ((outs[0]["render"] * cots[0][0].float().cuda()).sum() + (outs[2]["render"] * cots[2][0].float().cuda()).sum()).backward()
    for k, v in _grads_of(leaf[1]).items():
        assert torch.equal(v, torch.zeros_like(v)), k
    _check(_grads_of(leaf[0]), cots[0][1], "render_cameras camera 0 (camera 1 out of the loss)")


# ---- 5. nothing else moves -----------------------------------------------------------------------------------------------
def _sparse_inputs(cam, W, H):
    """Gaussians of about one pixel, each centred in its own 16 x 4 pixel band of a tile: the pixels one warp of the blend
    backward shades.  Each Gaussian's gradient then arrives in one atomic add onto zero, so the rasterizer's backward
    repeats bit for bit from run to run."""
    wv = cam.world_view_transform.detach().double().cpu()
    tanx, tany = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    centres = [(16 * tx + 6 + (tx + by) % 5, 4 * by + 1.5) for tx in range(W // 16) for by in range(0, H // 4, 2)]
    g = torch.Generator().manual_seed(8)
    pts = []
    for px, py in centres:
        z = 2.5 + float(torch.rand(1, generator=g))
        ndcx, ndcy = (2 * px + 1) / W - 1, (2 * py + 1) / H - 1
        pts.append([ndcx * tanx * z, ndcy * tany * z, z, 1.0])
    means = (torch.tensor(pts, dtype=torch.float64) @ torch.linalg.inv(wv))[:, :3]
    n = means.shape[0]
    scales = torch.full((n, 3), 1e-3, dtype=torch.float64)
    rots = torch.nn.functional.normalize(torch.randn(n, 4, generator=g, dtype=torch.float64), dim=1)
    opac = torch.full((n, 1), 0.8, dtype=torch.float64)
    shs = torch.randn(n, 16, 3, generator=g, dtype=torch.float64) * 0.3
    return [t.float().cuda().requires_grad_(True) for t in (means, scales, rots, opac, shs)]


def _everything(path, with_cam, k=1):
    """images, depths, radii and every gradient a backward computes, with or without camera leaves"""
    torch.manual_seed(0)
    scene, mod = _fused_setup(500, 13)
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
    bg = torch.tensor([0.3, 0.2, 0.1], device="cuda")
    cams = [synth.make_camera(25.0 + 70 * i, 64, 48, radius=3.0, time=0.3) for i in range(k)]
    cams = [_leaf_camera(c) if with_cam else c for c in cams]
    cot = torch.randn(3, 48, 64, generator=torch.Generator().manual_seed(3)).cuda()
    if path.startswith("rasterizer"):
        c = cams[0]
        inputs = _sparse_inputs(c, 64, 48) if path == "rasterizer_sparse" else \
            [t.float().cuda().requires_grad_(True) for t in raster_inputs(500, 13, scale_mean=0.05)]
        rs = rasterizer.GaussianRasterizationSettings(48, 64, math.tan(c.FoVx * 0.5), math.tan(c.FoVy * 0.5), bg, 1.0,
                                                      c.world_view_transform, c.full_proj_transform, 3, c.camera_center,
                                                      False, False)
        m2 = torch.zeros_like(inputs[0], requires_grad=True)
        img, rad, dep = rasterizer.GaussianRasterizer(rs)(means3D=inputs[0], means2D=m2, shs=inputs[4], opacities=inputs[3],
                                                         scales=inputs[1], rotations=inputs[2])
        (img * cot).sum().backward()
        return [img, dep, rad, m2.grad] + [t.grad for t in inputs]
    outs = g4d.render_cameras(cams, pc, _Pipe, bg, stage="fine")
    sum((o["render"] * cot).sum() for o in outs).backward()
    res = []
    for o in outs:
        res += [o["render"], o["depth"], o["radii"], o["viewspace_points"].grad]
    return res + [p.grad for p in pc.gaussian_parameters()] + [p.grad for p in mod.parameters() if p.grad is not None]


SUM_TOL = 2e-5      # atomic accumulation order (as in test_gpu_sh_degree)


@pytest.mark.parametrize("path,k", [("rasterizer", 1), ("rasterizer_sparse", 1), ("render", 1), ("render", 3)])
@pytest.mark.parametrize("tc", [0, 2])
def test_camera_grads_leave_everything_else_unchanged(path, k, tc):
    """Images, depths and radii bit-identical.  The gradients bit-identical too whenever the two runs without camera
    gradients repeat each other bit for bit (as test_gpu_sh_degree._close): the camera terms are extra outputs only.  When
    those two runs do not repeat -- the blend backward adds each Gaussian's gradient with atomics per warp, the network's
    weight gradients and the plane scatter accumulate with atomics too, and their order varies between runs -- within twice
    their spread or SUM_TOL of the tensor's max."""
    if path.startswith("rasterizer") and tc == 2:
        pytest.skip("the rasterizer drop-in runs no network")
    ws = _lib.workspace_of(torch.device("cuda"))
    ws.set_option(_lib.OPT_TENSOR_CORES, tc)
    try:
        a, b, a2 = _everything(path, False, k), _everything(path, True, k), _everything(path, False, k)
    finally:
        torch.cuda.synchronize()
        ws.set_option(_lib.OPT_TENSOR_CORES, 2)
    assert len(a) == len(b) == len(a2)
    forward_ids = [0, 1, 2] if path.startswith("rasterizer") else [4 * i + j for i in range(k) for j in range(3)]
    grads = [i for i in range(len(a)) if i not in forward_ids]
    repeatable = all(torch.equal(a[i], a2[i]) for i in grads)
    if path == "rasterizer_sparse":      # (built to repeat: the bit-for-bit comparison must be the one that runs)
        assert repeatable and int((a[2] > 0).sum()) == int(a[2].numel())
    for i in forward_ids:
        assert torch.equal(a[i], b[i]) and torch.equal(a[i], a2[i]), "forward output %d moved" % i
    for i in grads:
        x, y, x2 = a[i], b[i], a2[i]
        if repeatable:
            assert torch.equal(x, y), "gradient %d moved (the runs without camera gradients repeat bit for bit)" % i
            continue
        spread = float((x.double() - x2.double()).abs().max())
        bound = max(2 * spread, SUM_TOL * max(1e-3, float(x.double().abs().max())))
        assert float((x.double() - y.double()).abs().max()) <= bound, "gradient %d moved" % i
    print("%s k=%d tc=%d: gradients %s" % (path, k, tc, "bit-identical" if repeatable else "within the spread"))


# ---- 6. a pose recovered through render() ----------------------------------------------------------------------------------
# first H100 run (H100 80GB HBM3, 700 W): the error fell from 2.00 to 0.130, a ratio of 0.065, in 150 steps; the bound keeps a
# 3x margin over it
POSE_STEPS = 150
POSE_RATIO = 0.2


def test_pose_refinement_recovers_the_camera():
    scene = synth.make_scene(3000, seed=21, scale_mean=0.04)
    mod = make_module("small128", seed=21, aabb=scene["aabb"])
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=False)
    true_cam = synth.make_camera(40.0, 128, 96, radius=4.0, time=0.5)
    bg = torch.tensor([0.0, 0.0, 0.0], device="cuda")
    with torch.no_grad():
        target = g4d.render(true_cam, pc, _Pipe, bg, stage="fine")["render"].clone()
    R0, T0 = [t.cuda() for t in ucg.pose_of(true_cam)]
    g = torch.Generator().manual_seed(5)
    axis = torch.nn.functional.normalize(torch.randn(3, generator=g, dtype=torch.float64), dim=0)
    R1 = ucg.rodrigues((axis * math.radians(0.5)).cuda()) @ R0           # 0.5 degrees
    T1 = T0 + (torch.nn.functional.normalize(torch.randn(3, generator=g, dtype=torch.float64), dim=0) * 0.04).cuda()  # 1 % of 4
    delta = torch.zeros(6, dtype=torch.float64, device="cuda", requires_grad=True)
    opt = torch.optim.Adam([delta], lr=2e-4)

    def camera(d):
        R = ucg.rodrigues(d[:3]) @ R1
        wv, full, centre = ucg.camera_tensors(R, T1 + d[3:], true_cam.FoVx, true_cam.FoVy)
        return synth.SynthCamera(FoVx=true_cam.FoVx, FoVy=true_cam.FoVy, image_width=128, image_height=96,
                                 world_view_transform=wv.float(), full_proj_transform=full.float(),
                                 camera_center=centre.float(), time=0.5), R, T1 + d[3:]

    def error(R, T):
        rot = torch.arccos(torch.clamp((torch.trace(R.t() @ R0) - 1) / 2, -1, 1))
        return float(rot) / math.radians(0.5) + float((T - T0).norm()) / 0.04

    _, R, T = camera(delta.detach())
    e0 = error(R, T)
    for _ in range(POSE_STEPS):
        opt.zero_grad()
        cam, _, _ = camera(delta)
        loss = (g4d.render(cam, pc, _Pipe, bg, stage="fine")["render"] - target).abs().mean()
        loss.backward()
        assert delta.grad is not None and torch.isfinite(delta.grad).all()
        opt.step()
    _, R, T = camera(delta.detach())
    e1 = error(R, T)
    print("pose error: initial %.4f final %.4f ratio %.4f" % (e0, e1, e1 / e0))
    assert e1 <= POSE_RATIO * e0, (e0, e1)


# ---- 7. refusals ---------------------------------------------------------------------------------------------------------
def _coarse_call(ctx, cam, n, g_tensors, no_grad=False):
    lib = _lib.load()
    x, s, r, o, dc, rest = g_tensors
    g = _lib.Gaussians(n, x.data_ptr(), s.data_ptr(), r.data_ptr(), o.data_ptr(), dc.data_ptr(), rest.data_ptr())
    H, W = cam.image_height, cam.image_width
    col, dep = torch.empty(3, H, W, device="cuda"), torch.empty(1, H, W, device="cuda")
    rad = torch.empty(n, device="cuda", dtype=torch.int32)
    if no_grad:
        cam.debug |= _lib.CAM_NO_GRAD
    _lib.check(lib.g4d_render_forward(ctx.handle, C.byref(cam), None, C.byref(g), col.data_ptr(), dep.data_ptr(),
                                      rad.data_ptr(), _lib.stream_of(torch.device("cuda"))), "g4d_render_forward")
    grads = [torch.empty(n * w, device="cuda") for w in (3, 3, 4, 1, 3, 45, 3)]
    gg = _lib.GaussianGrads(*[t.data_ptr() for t in grads])
    gcol = torch.ones(3 * H * W, device="cuda")
    return lambda: lib.g4d_render_backward(ctx.handle, C.byref(cam), None, None, C.byref(g), gcol.data_ptr(), C.byref(gg),
                                           _lib.stream_of(torch.device("cuda")))


def _coarse_scene(n=200):
    sc = synth.make_scene(n, seed=4, scale_mean=0.05)
    return [sc[k].float().cuda().contiguous() for k in SCENE_LEAVES]


def _abi_camera(n_cam=None):
    cam = synth.make_camera(15.0, 64, 48, radius=3.0)
    rs = rasterizer.GaussianRasterizationSettings(48, 64, math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5),
                                                  torch.zeros(3, device="cuda"), 1.0, cam.world_view_transform.cuda(),
                                                  cam.full_proj_transform.cuda(), 3, cam.camera_center.cuda(), False, False)
    keep = []
    return rasterizer.camera_from_settings(rs, keep=keep, sh_coeffs=16), keep


def test_refuses_wrong_sized_camera_tensors():
    scene, mod = _fused_setup(100, 1)
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
    cam = _leaf_camera(synth.make_camera(10.0, 32, 24))
    bad = torch.zeros(12, device="cuda", requires_grad=True)
    for field in ("world_view_transform", "full_proj_transform", "camera_center"):
        c = synth.SynthCamera(**{**cam.__dict__, field: bad})
        with pytest.raises(RuntimeError, match="elements, expected"):
            g4d.render(c, pc, _Pipe, torch.zeros(3, device="cuda"), stage="fine")


def test_camera_grad_pointer_rules():
    ws = _lib.workspace_of(torch.device("cuda"))
    ctx = _lib.Context(ws)
    n = 200
    gt = _coarse_scene(n)
    sink = torch.full((35,), float("nan"), device="cuda")
    try:
        # a no-grad forward's context: the backward is refused before any launch, the sink untouched
        cam, keep = _abi_camera()
        bwd = _coarse_call(ctx, cam, n, gt, no_grad=True)
        ctx.set_camera_grad(sink.data_ptr())
        assert bwd() == -4
        torch.cuda.synchronize()
        assert torch.isnan(sink).all()
        # a grad forward: the backward overwrites the sink
        cam, keep = _abi_camera()
        bwd = _coarse_call(ctx, cam, n, gt)
        assert bwd() == 0
        torch.cuda.synchronize()
        assert torch.isfinite(sink).all() and sink.abs().max() > 0
        assert float(sink[[3, 7, 11, 15, 18, 22, 26, 30]].abs().max()) == 0.0
        # under stream capture, with the pointer set: refused before any launch (nothing is captured)
        cam, keep = _abi_camera()
        bwd = _coarse_call(ctx, cam, n, gt)
        torch.cuda.synchronize()
        sink.fill_(float("nan"))
        graph, stream = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            graph.capture_begin()
            rc = bwd()
            graph.capture_end()
        torch.cuda.synchronize()
        assert rc == -4 and "capture" in _lib.load().g4d_last_error().decode()
        assert torch.isnan(sink).all()
        # NULL turns it off: a backward leaves the sink alone
        ctx.set_camera_grad(None)
        cam, keep = _abi_camera()
        bwd = _coarse_call(ctx, cam, n, gt)
        assert bwd() == 0
        torch.cuda.synchronize()
        assert torch.isnan(sink).all()
    finally:
        ctx.set_camera_grad(None)
