"""GPU: dL/d(camera time) through render() on both network engines and render_cameras, against the fp64 chain oracle
deform_ref -> dense render (util_time_grad) and against the per-row time path of deform_network + the rasterizer drop-in;
everything else a backward computes unchanged with a time leaf; the edges that give exactly 0; the time source; the sink's
pointer rules; and a time offset recovered by Adam through render()."""
import ctypes as C
import gc
import importlib
import math

import numpy as np
import pytest
import torch

import util_camera_grad as ucg
import util_time_grad as utg
from oracle.dense_ref import cam_dict_from
from util_scene import _deform_activate, make_module, oracle_params_from_module, params_fp64, raster_inputs, synth

pytestmark = pytest.mark.gpu
g4d = importlib.import_module("4dgaussians_b200")
_lib = importlib.import_module("4dgaussians_b200._lib")
rasterizer = importlib.import_module("4dgaussians_b200.rasterizer")
renderer = importlib.import_module("4dgaussians_b200.renderer")

T_ROWS = 8          # time rows of the "small128" network
# Against the fp64 oracle, relative to sum_g |dL/dt_g| (the oracle's per-Gaussian contributions, so that cancellation in
# the sum cannot make the bound small).  Fixed before the first run: the FP16x2 tensor-core forward rounds its operands to
# 11 bits (4.9e-4) and every Gaussian's term passes two such layers, the FFMA engine is fp32 throughout, and a Gaussian whose
# ReLU pre-activation or alpha threshold sits within rounding of its kink takes the other branch in fp32; 5e-3 covers the
# first with a margin of 5 and bounds the last to a few Gaussians' worth of the total.
TOL = 5e-3
# The same dL/dt computed by two GPU paths from the same fp32 network outputs: only the summation order differs
# (atomics in the blend backward, the scatter and the time-row reduction).
SAME_TOL = 1e-3


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


SCENE_LEAVES = utg.SCENE_LEAVES


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


def _t_mid(k):
    """the middle of time interval k of the small128 network's rows"""
    return -1.0 + 2.0 * (k + 0.5) / (T_ROWS - 1)


def _setup(n, seed, deg=3, requires_grad=True):
    scene = synth.make_scene(n, seed=seed, scale_mean=0.05)
    mod = make_module("small128", seed=seed, aabb=scene["aabb"])
    return scene, mod, synth.SyntheticGaussianModel(scene, mod, sh_degree=deg, requires_grad=requires_grad)


def _timed(cam, t):
    return synth.SynthCamera(**{**cam.__dict__, "time": t})


def _leaf(t):
    return torch.tensor(t, device="cuda", dtype=torch.float32, requires_grad=True)


def _fp32_cd(cam, bg, deg):
    cd = cam_dict_from(cam, bg, deg)
    cd["tanfovx"], cd["tanfovy"] = float(np.float32(cd["tanfovx"])), float(np.float32(cd["tanfovy"]))
    return cd


def _oracle(mod, scene, cam, t, bg, deg, cot_seed):
    """(cotangent masked at the threshold pixels, the oracle's per-Gaussian dL/dt_g)"""
    cfg, prm = oracle_params_from_module(mod)
    with torch.no_grad():
        inputs = _deform_activate(cfg, params_fp64(prm), {k: scene[k].double() for k in SCENE_LEAVES}, t)
    cd = _fp32_cd(cam, bg, deg)
    cot = torch.randn(3, cd["H"], cd["W"], generator=torch.Generator().manual_seed(cot_seed), dtype=torch.float64)
    cot[:, ucg.threshold_pixel_mask(cd, inputs)] = 0.0
    return cot, utg.oracle_time_grads(cfg, prm, scene, cd, t, cot)


def _check(got, per, tol, what):
    ref, scale = float(per.sum()), float(per.abs().sum())
    assert scale > 0
    assert abs(got - ref) <= tol * scale, "%s: dL/dt %.6e vs %.6e (sum |dL/dt_g| %.3e)" % (what, got, ref, scale)


def _render_time_grad(pc, cam, t, bg, cot, stage="fine"):
    leaf = _leaf(t)
    out = g4d.render(_timed(cam, leaf), pc, _Pipe, torch.tensor(bg, device="cuda"), stage=stage)
    (out["render"] * cot.float().cuda()).sum().backward()
    return leaf.grad


# ---- 1. render() against the fp64 chain oracle -----------------------------------------------------------------------------
@pytest.mark.parametrize("tc", [0, 2])
@pytest.mark.parametrize("deg", [0, 3])
def test_render_time_grad_vs_oracle_chain(tc, deg):
    with _engine(tc):
        scene, mod, pc = _setup(400, 5 + deg, deg)
        t = _t_mid(4)
        cam = synth.make_camera(30.0, 61, 47, radius=3.0)
        bg = (0.0, 0.1, 0.2)
        cot, per = _oracle(mod, scene, cam, t, bg, deg, cot_seed=11)
        g = _render_time_grad(pc, cam, t, bg, cot)
        assert g.shape == () and g.dtype == torch.float32 and g.device.type == "cuda"
        _check(float(g), per, TOL, "render tc=%d deg=%d" % (tc, deg))


# ---- 2. the same dL/dt as the per-row path of deform_network -----------------------------------------------------------------
@pytest.mark.parametrize("tc", [0, 2])
@pytest.mark.parametrize("t", [_t_mid(1), -1.0 + 2.0 * 5 / (T_ROWS - 1), 0.9])     # (the second lies on a texel row)
def test_matches_the_per_row_path(tc, t):
    with _engine(tc):
        scene, mod, pc = _setup(500, 3)
        cam = synth.make_camera(20.0, 64, 48, radius=3.0)
        bg = torch.tensor([0.2, 0.1, 0.0], device="cuda")
        cot = torch.randn(3, 48, 64, generator=torch.Generator().manual_seed(5)).cuda()
        fused = _render_time_grad(pc, cam, t, (0.2, 0.1, 0.0), cot)
        n = pc.get_xyz.shape[0]
        times = torch.full((n, 1), t, device="cuda", dtype=torch.float32, requires_grad=True)
        m3, sc, rot, op, shs = mod(pc.get_xyz, pc._scaling, pc._rotation, pc._opacity, pc.get_features, times)
        rs, _ = renderer.settings_from_camera(cam, pc, _Pipe, bg)
        img, _, _ = rasterizer.GaussianRasterizer(rs)(means3D=m3, means2D=torch.zeros_like(m3, requires_grad=True), shs=shs,
                                                      opacities=pc.opacity_activation(op), scales=pc.scaling_activation(sc),
                                                      rotations=pc.rotation_activation(rot))
        (img * cot).sum().backward()
        per = times.grad.reshape(-1).double().cpu()
        _check(float(fused), per, SAME_TOL, "per-row path tc=%d t=%.4f" % (tc, t))


# ---- 3. render_cameras, k = 3, one shared time tensor ------------------------------------------------------------------------
def test_render_cameras_time_grad():
    scene, mod, pc = _setup(400, 9)
    t = _t_mid(3)
    bg = (0.2, 0.1, 0.0)
    cams = [synth.make_camera(th, 61 + 4 * i, 47, radius=3.0) for i, th in enumerate((10.0, 100.0, -120.0))]
    oracles = [_oracle(mod, scene, c, t, bg, 3, cot_seed=20 + i) for i, c in enumerate(cams)]
    singles = [float(_render_time_grad(pc, c, t, bg, cot)) for c, (cot, _) in zip(cams, oracles)]

    def group(in_loss):
        leaf = _leaf(t)
        outs = g4d.render_cameras([_timed(c, leaf) for c in cams], pc, _Pipe, torch.tensor(bg, device="cuda"), stage="fine")
        sum((outs[i]["render"] * oracles[i][0].float().cuda()).sum() for i in in_loss).backward()
        return float(leaf.grad)

    for in_loss in ((0, 1, 2), (0, 2)):          # (camera 1 outside the loss contributes nothing)
        got = group(in_loss)
        per = torch.cat([oracles[i][1] for i in in_loss])
        _check(got, per, TOL, "render_cameras %s vs oracle" % (in_loss,))
        assert abs(got - sum(singles[i] for i in in_loss)) <= SAME_TOL * float(per.abs().sum()), (got, singles)
    a, b = _leaf(t), _leaf(t)
    with pytest.raises(ValueError, match="same time tensor"):
        g4d.render_cameras([_timed(cams[0], a), _timed(cams[1], b)], pc, _Pipe, torch.tensor(bg, device="cuda"), stage="fine")


# ---- 4. nothing else moves ---------------------------------------------------------------------------------------------------
def _everything(with_time, k):
    """images, depths, radii and every gradient a backward computes, with or without a time leaf"""
    torch.manual_seed(0)
    scene, mod, pc = _setup(500, 13)
    bg = torch.tensor([0.3, 0.2, 0.1], device="cuda")
    t = _leaf(0.3) if with_time else 0.3
    cams = [_timed(synth.make_camera(25.0 + 70 * i, 64, 48, radius=3.0), t) for i in range(k)]
    cot = torch.randn(3, 48, 64, generator=torch.Generator().manual_seed(3)).cuda()
    outs = g4d.render_cameras(cams, pc, _Pipe, bg, stage="fine")
    sum((o["render"] * cot).sum() for o in outs).backward()
    if with_time:
        assert t.grad is not None
    res = []
    for o in outs:
        res += [o["render"], o["depth"], o["radii"], o["viewspace_points"].grad]
    return res + [p.grad for p in pc.gaussian_parameters()] + [p.grad for p in mod.parameters() if p.grad is not None]


SUM_TOL = 2e-5      # atomic accumulation order (as in test_gpu_camera_grad)


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("tc", [0, 2])
def test_time_grad_leaves_everything_else_unchanged(k, tc):
    """Images, depths and radii bit-identical; the gradients bit-identical whenever the two runs without a time leaf repeat
    each other bit for bit, else within twice their spread or SUM_TOL of the tensor's max (test_gpu_camera_grad §5)."""
    with _engine(tc):
        a, b, a2 = _everything(False, k), _everything(True, k), _everything(False, k)
    assert len(a) == len(b) == len(a2)
    forward_ids = [4 * i + j for i in range(k) for j in range(3)]
    grads = [i for i in range(len(a)) if i not in forward_ids]
    repeatable = all(torch.equal(a[i], a2[i]) for i in grads)
    for i in forward_ids:
        assert torch.equal(a[i], b[i]) and torch.equal(a[i], a2[i]), "forward output %d moved" % i
    for i in grads:
        x, y, x2 = a[i], b[i], a2[i]
        if repeatable:
            assert torch.equal(x, y), "gradient %d moved (the runs without a time leaf repeat bit for bit)" % i
            continue
        spread = float((x.double() - x2.double()).abs().max())
        bound = max(2 * spread, SUM_TOL * max(1e-3, float(x.double().abs().max())))
        assert float((x.double() - y.double()).abs().max()) <= bound, "gradient %d moved" % i
    print("k=%d tc=%d: gradients %s" % (k, tc, "bit-identical" if repeatable else "within the spread"))


# ---- 5. edges ----------------------------------------------------------------------------------------------------------------
def test_edges_give_zero():
    scene, mod, pc = _setup(300, 2)
    cam = synth.make_camera(15.0, 64, 48, radius=3.0)
    cot = torch.randn(3, 48, 64, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    for t in (1.0, -1.0):
        assert float(_render_time_grad(pc, cam, t, (0.0, 0.0, 0.0), cot)) == 0.0, t
    assert float(_render_time_grad(pc, cam, 0.3, (0.0, 0.0, 0.0), cot, stage="coarse")) == 0.0
    empty = dict({k: v[:0] for k, v in scene.items() if k != "aabb"}, aabb=scene["aabb"])
    pc0 = synth.SyntheticGaussianModel(empty, mod, sh_degree=3, requires_grad=True)
    assert float(_render_time_grad(pc0, cam, 0.3, (0.0, 0.0, 0.0), cot)) == 0.0


def _abi_camera(cam, t, keep):
    rs, _ = renderer.settings_from_camera(cam, _ModelShape, _Pipe, torch.zeros(3, device="cuda"))
    return rasterizer.camera_from_settings(rs, time=t, keep=keep, sh_coeffs=16)


class _ModelShape:
    active_sh_degree = 3


def _gaussians(pc):
    ts = [pc._xyz, pc._scaling, pc._rotation, pc._opacity, pc._features_dc, pc._features_rest]
    ts = [t.detach().contiguous() for t in ts]
    return _lib.Gaussians(ts[0].shape[0], *[t.data_ptr() for t in ts]), ts


def test_rasterizer_backward_writes_zero():
    ctx = _lib.Context(_lib.workspace_of(torch.device("cuda")))
    sink = torch.full((1,), float("nan"), device="cuda")
    lib, st = _lib.load(), _lib.stream_of(torch.device("cuda"))
    try:
        keep = []
        cam = _abi_camera(synth.make_camera(15.0, 64, 48, radius=3.0), 0.3, keep)
        m3, sc, ro, op, sh = [t.float().cuda().contiguous() for t in raster_inputs(300, 2, scale_mean=0.05)]
        n = m3.shape[0]
        col, dep = torch.empty(3, 48, 64, device="cuda"), torch.empty(1, 48, 64, device="cuda")
        rad = torch.empty(n, device="cuda", dtype=torch.int32)
        _lib.check(lib.g4d_rasterize_forward(ctx.handle, C.byref(cam), n, m3.data_ptr(), sh.data_ptr(), op.data_ptr(),
                                             sc.data_ptr(), ro.data_ptr(), col.data_ptr(), dep.data_ptr(), rad.data_ptr(), st),
                   "g4d_rasterize_forward")
        g = [torch.empty(n, w, device="cuda") for w in (3, 3, 48, 1, 3, 4)]
        gcol = torch.ones(3 * 48 * 64, device="cuda")
        ctx.set_time_grad(sink.data_ptr())
        _lib.check(lib.g4d_rasterize_backward(ctx.handle, C.byref(cam), n, m3.data_ptr(), sh.data_ptr(), op.data_ptr(),
                                              sc.data_ptr(), ro.data_ptr(), gcol.data_ptr(), *[t.data_ptr() for t in g], st),
                   "g4d_rasterize_backward")
        torch.cuda.synchronize()
        assert float(sink[0]) == 0.0
    finally:
        ctx.set_time_grad(None)


def _fused_abi(ctx, cam, mod, pc, sink):
    """g4d_render_forward + g4d_render_backward of pc under mod on ctx, the time sink set for the backward"""
    lib, st = _lib.load(), _lib.stream_of(torch.device("cuda"))
    keep = []
    prm = mod.c_params(keep, fresh=True)
    cg, _ = mod.c_grad_sinks()
    g, ts = _gaussians(pc)
    n = g.n
    H, W = cam.image_height, cam.image_width
    col, dep = torch.empty(3, H, W, device="cuda"), torch.empty(1, H, W, device="cuda")
    rad = torch.empty(n, device="cuda", dtype=torch.int32)
    _lib.check(lib.g4d_render_forward(ctx.handle, C.byref(cam), C.byref(prm), C.byref(g), col.data_ptr(), dep.data_ptr(),
                                      rad.data_ptr(), st), "g4d_render_forward")
    grads = [torch.empty(n * w, device="cuda") for w in (3, 3, 4, 1, 3, 45, 3)]
    gg = _lib.GaussianGrads(*[t.data_ptr() for t in grads])
    gcol = torch.linspace(-1, 1, 3 * H * W, device="cuda")
    ctx.set_time_grad(sink.data_ptr())
    try:
        _lib.check(lib.g4d_render_backward(ctx.handle, C.byref(cam), C.byref(prm), C.byref(cg), C.byref(g), gcol.data_ptr(),
                                           C.byref(gg), st), "g4d_render_backward")
        torch.cuda.synchronize()
    finally:
        ctx.set_time_grad(None)
    return float(sink[0])


def test_time_source_gives_the_same_time_grad():
    scene, mod, pc = _setup(400, 6)
    t = _t_mid(2)
    ctx = _lib.Context(_lib.workspace_of(torch.device("cuda")))
    sink = torch.full((1,), float("nan"), device="cuda")
    src = torch.tensor([t], device="cuda", dtype=torch.float32)
    keep = []
    view = synth.make_camera(35.0, 64, 48, radius=3.0)
    direct = _fused_abi(ctx, _abi_camera(view, t, keep), mod, pc, sink)
    ctx.set_time_source(src.data_ptr())
    try:
        sourced = _fused_abi(ctx, _abi_camera(view, -0.77, keep), mod, pc, sink)    # G4DCamera.time is not read
    finally:
        ctx.set_time_source(None)
    assert direct != 0.0 and math.isfinite(direct)
    assert abs(sourced - direct) <= SAME_TOL * abs(direct), (sourced, direct)


# ---- 6. pointer rules ----------------------------------------------------------------------------------------------------
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


def test_time_grad_pointer_rules():
    ctx = _lib.Context(_lib.workspace_of(torch.device("cuda")))
    n = 200
    sc = synth.make_scene(n, seed=4, scale_mean=0.05)
    gt = [sc[k].float().cuda().contiguous() for k in SCENE_LEAVES]
    view = synth.make_camera(15.0, 64, 48, radius=3.0)
    sink = torch.full((1,), float("nan"), device="cuda")
    try:
        # a no-grad forward's context: the backward is refused before any launch, the sink untouched
        keep = []
        bwd = _coarse_call(ctx, _abi_camera(view, 0.3, keep), n, gt, no_grad=True)
        ctx.set_time_grad(sink.data_ptr())
        assert bwd() == -4
        torch.cuda.synchronize()
        assert torch.isnan(sink).all()
        # a grad forward: the backward overwrites the sink (the coarse stage: with 0)
        bwd = _coarse_call(ctx, _abi_camera(view, 0.3, keep), n, gt)
        assert bwd() == 0
        torch.cuda.synchronize()
        assert float(sink[0]) == 0.0
        # under stream capture, with the pointer set: refused before any launch (nothing is captured)
        bwd = _coarse_call(ctx, _abi_camera(view, 0.3, keep), n, gt)
        torch.cuda.synchronize()
        sink.fill_(float("nan"))
        graph, stream = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            graph.capture_begin()
            rc = bwd()
            graph.capture_end()
        torch.cuda.synchronize()
        assert rc == -4 and "time gradient" in _lib.load().g4d_last_error().decode()
        assert torch.isnan(sink).all()
        # NULL turns it off: a backward leaves the sink alone
        ctx.set_time_grad(None)
        bwd = _coarse_call(ctx, _abi_camera(view, 0.3, keep), n, gt)
        assert bwd() == 0
        torch.cuda.synchronize()
        assert torch.isnan(sink).all()
    finally:
        ctx.set_time_grad(None)


# ---- 7. a time offset recovered through render() ---------------------------------------------------------------------------
# The synthetic time planes are random, so the scene moves independently in each interval between two time rows and the L1
# loss has a local minimum just past each row.  A scan on an H100 80GB HBM3 (700 W) found the basin around t* reaching to
# the rows either side of it, 0.675 texel below and 0.325 above, and a start one texel below stuck in the neighbouring
# interval (error 0.78 of the initial after 200 steps).  The start is therefore half a texel below t*, inside the basin.
TIME_STEPS = 200
TIME_RATIO = 0.2


def test_time_offset_refinement_recovers_the_time():
    scene, mod, pc = _setup(3000, 21, requires_grad=False)
    t_true = _t_mid(4) + 0.05
    cam = synth.make_camera(40.0, 128, 96, radius=4.0)
    bg = torch.tensor([0.0, 0.0, 0.0], device="cuda")
    with torch.no_grad():
        target = g4d.render(_timed(cam, t_true), pc, _Pipe, bg, stage="fine")["render"].clone()
    texel = 2.0 / (T_ROWS - 1)
    t = torch.tensor(t_true - 0.5 * texel, device="cuda", dtype=torch.float32, requires_grad=True)
    opt = torch.optim.Adam([t], lr=texel / 40)
    e0 = abs(float(t) - t_true)
    for _ in range(TIME_STEPS):
        opt.zero_grad()
        loss = (g4d.render(_timed(cam, t), pc, _Pipe, bg, stage="fine")["render"] - target).abs().mean()
        loss.backward()
        assert t.grad is not None and torch.isfinite(t.grad).all()
        opt.step()
    e1 = abs(float(t) - t_true)
    print("time error: initial %.4f final %.4f ratio %.4f" % (e0, e1, e1 / e0))
    assert e1 <= TIME_RATIO * e0, (e0, e1)
