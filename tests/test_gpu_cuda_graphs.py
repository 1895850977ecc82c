"""CUDA-graph capture of no-grad rendering (graphs.GraphedRender; g4d_context_set_time_source, g4d_workspace_freeze,
g4d_workspace_graph_status).

A replay runs the very kernels an eager no-sync render runs, on the same inputs -- only read from device memory instead of
kernel parameters -- so images, depth maps and radii must equal eager render() / render_cameras() bit for bit.
"""
import ctypes as C
import importlib
import warnings

import pytest
import torch

from util_scene import g4d, make_module, synth

_lib = importlib.import_module("4dgaussians_b200._lib")
build = importlib.import_module("4dgaussians_b200.build")
renderer = importlib.import_module("4dgaussians_b200.renderer")
rasterizer = importlib.import_module("4dgaussians_b200.rasterizer")
graphs = importlib.import_module("4dgaussians_b200.graphs")


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


# small64: the FFMA network of the dnerf config; small128: tensor cores with all five heads (dynerf)
CASES = {"ffma": dict(net="small64", n=1500, wh=(96, 72), radius=4.0, deg=3, bg=(1.0, 1.0, 1.0)),
         "tc": dict(net="small128", n=1800, wh=(112, 80), radius=2.4, deg=3, bg=(0.0, 0.0, 0.0))}


@pytest.fixture(scope="module", autouse=True)
def _built():
    build.build()
    _lib.load()


def _model(c, seed=11):
    scene = synth.make_scene(c["n"], seed=seed, scale_mean=0.05)
    mod = make_module(c["net"], seed=2, aabb=scene["aabb"])
    return synth.SyntheticGaussianModel(scene, mod, sh_degree=c["deg"])


def _orbit(c, count, t0=0.0, radius=None):
    W, H = c["wh"]
    cams = synth.orbit_cameras(count, W, H, radius=radius or c["radius"])
    for i, cam in enumerate(cams):
        cam.time = t0 + (i + 1) / (count + 1.0)
    return cams


class _NoSync:
    """eager renders on the shared workspace in no-sync mode (as a graph replays them)"""

    def __enter__(self):
        self.ws = _lib.Workspace.get(torch.cuda.current_device())
        self.ws.set_option(_lib.OPT_SYNC_MODE, 0)

    def __exit__(self, *a):
        torch.cuda.synchronize()
        self.ws.set_option(_lib.OPT_SYNC_MODE, 1)


def _assert_same(got, ref):
    for key in ("render", "depth", "radii", "visibility_filter"):
        assert torch.equal(got[key], ref[key]), key


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_replay_equals_eager_render(case):
    c = CASES[case]
    pc = _model(c)
    bg = torch.tensor(c["bg"], device="cuda")
    cams = _orbit(c, 8)
    with torch.no_grad(), _NoSync():
        gr = graphs.GraphedRender(pc, _Pipe, bg, cams[0])
        for cam in cams:
            got = {k: v.clone() for k, v in gr(cam).items()}
            ref = g4d.render(cam, pc, _Pipe, bg)
            _assert_same(got, ref)
            assert got["radii"].gt(0).sum() > 100
        gr.check()


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_replay_equals_eager_render_cameras(case):
    c = CASES[case]
    pc = _model(c)
    bg = torch.tensor(c["bg"], device="cuda")
    W, H = c["wh"]
    with torch.no_grad(), _NoSync():
        def rig(t, turn):
            return [synth.make_camera(turn, W, H, radius=c["radius"], time=t),
                    synth.make_camera(turn + 55.0, W, H, radius=c["radius"] * 1.1, time=t),
                    synth.make_camera(turn - 80.0, W + 37, H - 11, radius=c["radius"], time=t)]
        gr = graphs.GraphedRender(pc, _Pipe, bg, rig(0.5, 10.0))
        for i, t in enumerate((0.1, 0.35, 0.6, 0.9)):
            views = rig(t, 10.0 + 30.0 * i)
            got = [{k: v.clone() for k, v in d.items()} for d in gr(views)]
            ref = g4d.render_cameras(views, pc, _Pipe, bg)
            for a, b in zip(got, ref):
                _assert_same(a, b)
        gr.check()
        with pytest.raises(ValueError, match="times differ"):
            gr([synth.make_camera(0.0, W, H, time=0.2), synth.make_camera(9.0, W, H, time=0.3),
                synth.make_camera(-9.0, W + 37, H - 11, time=0.2)])


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_in_place_updates_are_seen_by_replays(case):
    c = CASES[case]
    pc = _model(c)
    bg = torch.tensor(c["bg"], device="cuda")
    cams = _orbit(c, 3)
    net = pc._deformation.deformation_net
    with torch.no_grad(), _NoSync():
        gr = graphs.GraphedRender(pc, _Pipe, bg, cams[0])
        before = gr(cams[1])["render"].clone()
        for p in net.grid.grids[0]:
            p.mul_(1.05)
        net.feature_out[0].weight.add_(0.01)
        pc._xyz.add_(0.02)
        got = {k: v.clone() for k, v in gr(cams[1]).items()}
        ref = g4d.render(cams[1], pc, _Pipe, bg)
        _assert_same(got, ref)
        assert not torch.equal(got["render"], before)


@pytest.mark.gpu
def test_template_mismatch_raises_before_a_replay():
    c = CASES["ffma"]
    pc = _model(c)
    bg = torch.tensor(c["bg"], device="cuda")
    W, H = c["wh"]
    with torch.no_grad():
        gr = graphs.GraphedRender(pc, _Pipe, bg, synth.make_camera(0.0, W, H, time=0.5))
        with pytest.raises(ValueError, match="image size or FoV"):
            gr(synth.make_camera(0.0, W + 1, H, time=0.5))
        with pytest.raises(ValueError, match="image size or FoV"):
            gr(synth.make_camera(0.0, W, H, fovx=0.9, time=0.5))
        with pytest.raises(ValueError, match="captured for render"):
            gr([synth.make_camera(0.0, W, H)])
        pc.active_sh_degree = 2
        with pytest.raises(ValueError, match="SH degree"):
            gr(synth.make_camera(0.0, W, H))
        pc.active_sh_degree = c["deg"]
        plane = pc._deformation.deformation_net.grid.grids[0][2]
        old = plane.data
        plane.data = old.clone(memory_format=torch.channels_last)
        with pytest.raises(ValueError, match="deformation network"):
            gr(synth.make_camera(0.0, W, H))
        plane.data = old
        gr(synth.make_camera(0.0, W, H))
        pc._xyz = torch.nn.Parameter(pc._xyz.detach().clone())
        with pytest.raises(ValueError, match="replaced"):
            gr(synth.make_camera(0.0, W, H))


# ---------------------------------------------------------------------------------------------------- refusals
class _Render:
    """one g4d_render_forward call of a model and camera on a given context"""

    def __init__(self, c, pc, cam):
        self.keep = []
        rs, t = renderer.settings_from_camera(cam, pc, _Pipe, torch.tensor(c["bg"], device="cuda"))
        self.cam = rasterizer.camera_from_settings(rs, time=t, keep=self.keep)
        self.cam.debug |= _lib.CAM_NO_GRAD
        self.prm = pc._deformation.c_params(self.keep, fresh=True)
        n = pc.get_xyz.shape[0]
        self.g = _lib.Gaussians(n, *(t.data_ptr() for t in (pc._xyz, pc._scaling, pc._rotation, pc._opacity, pc._features_dc,
                                                             pc._features_rest)))
        self.out = (torch.empty(3, rs.image_height, rs.image_width, device="cuda"),
                    torch.empty(1, rs.image_height, rs.image_width, device="cuda"), torch.empty(n, device="cuda", dtype=torch.int32))

    def __call__(self, ctx):
        stream = torch.cuda.current_stream().cuda_stream
        return _lib.load().g4d_render_forward(ctx.handle, C.byref(self.cam), C.byref(self.prm), C.byref(self.g),
                                              *(t.data_ptr() for t in self.out), stream)


def _refused_capture(call, match):
    """capture `call`: it must return G4D_ERR_STATE naming the cause, so the graph ends up with nothing in it"""
    g = torch.cuda.CUDAGraph()
    rc = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")      # (torch may warn that the graph is empty)
        with torch.cuda.graph(g):
            rc.append(call())
    assert rc == [-4], rc
    assert match in _lib.load().g4d_last_error().decode()


@pytest.mark.gpu
def test_capture_refusals_launch_nothing():
    c = CASES["tc"]
    pc = _model(c)
    W, H = c["wh"]
    small = _Render(c, pc, synth.make_camera(20.0, W, H, radius=c["radius"], time=0.3))
    large = _Render(c, pc, synth.make_camera(20.0, 2 * W, 2 * H, radius=c["radius"], time=0.3))
    with torch.no_grad():
        ws = _lib.Workspace(torch.cuda.current_device())
        ctx = _lib.Context(ws)
        # exact sync mode (the default): the forward reads R back on the host
        assert small(ctx) == 0
        _refused_capture(lambda: small(ctx), "exact sync mode")
        ws.set_option(_lib.OPT_SYNC_MODE, 0)
        # a context that never ran a forward has no capacity to bound the placement with
        fresh = _lib.Context(ws)
        _refused_capture(lambda: small(fresh), "not learnt")
        # G4D_CAM_DEBUG synchronises after every stage
        small.cam.debug |= _lib.CAM_DEBUG
        _refused_capture(lambda: small(ctx), "G4D_CAM_DEBUG")
        small.cam.debug &= ~_lib.CAM_DEBUG
        # stage timing records host-managed events
        ws.set_option(_lib.OPT_STAGE_TIMING, 1)
        _refused_capture(lambda: small(ctx), "STAGE_TIMING")
        ws.set_option(_lib.OPT_STAGE_TIMING, 0)
        # the image buffers of ctx would have to grow for the larger view
        _refused_capture(lambda: large(ctx), "would have to grow")
        # the refusals left the context usable: an eager forward still matches a fresh workspace's
        assert small(ctx) == 0
        img = small.out[0].clone()
        ref_ws = _lib.Workspace(torch.cuda.current_device())
        assert small(_lib.Context(ref_ws)) == 0
        assert torch.equal(img, small.out[0])
        # a frozen workspace refuses to grow eagerly too, and keeps running what fits
        ws.freeze(True)
        assert large(ctx) == -4 and b"would have to grow" in _lib.load().g4d_last_error()
        assert small(ctx) == 0
        ws.freeze(False)
        assert large(ctx) == 0
        torch.cuda.synchronize()


@pytest.mark.gpu
def test_overflowing_replay_is_reported():
    """Captured with a far camera that sees few instances, replayed with a near one that needs many more than the capacity
    learnt: the placement clamps (the designed no-sync path), the status records it and check() raises G4D_ERR_OVERFLOW."""
    c = dict(CASES["ffma"], n=6000, wh=(320, 240))
    pc = _model(c)
    bg = torch.tensor(c["bg"], device="cuda")
    W, H = c["wh"]
    far = synth.make_camera(30.0, W, H, radius=60.0, time=0.4)
    near = synth.make_camera(30.0, W, H, radius=1.6, time=0.4)
    with torch.no_grad():
        gr = graphs.GraphedRender(pc, _Pipe, bg, far)
        gr(far)
        gr.check()
        # (the near view does need more than the capacity: an eager exact render counts its instances)
        ctx = _lib.Context(_lib.Workspace(torch.cuda.current_device()))
        assert _Render(c, pc, near)(ctx) == 0
        assert ctx.stats().num_rendered > gr.ctxs[0].stats().instance_capacity
        gr(near)
        with pytest.raises(_lib.G4DError, match=r"code -5.*tile instances"):
            gr.check()
        gr(far)
        gr.check()          # (read and cleared)
        st = gr.ws.graph_status()
        assert st.overflows == 0 and st.max_instances == 0


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_time_source_drives_forward_and_backward(case):
    """A context with a time source renders and differentiates at the device timestamp, whatever G4DCamera.time says: the
    same image bit for bit and the same gradients (fp32 atomics: to 1e-5 of their max) as a camera that carries the time."""
    c = CASES[case]
    pc = _model(c)
    W, H = c["wh"]
    lib = _lib.load()
    n = c["n"]
    stream = lambda: torch.cuda.current_stream().cuda_stream

    def run(time_src):
        r = _Render(c, pc, synth.make_camera(40.0, W, H, radius=c["radius"], time=0.3))
        r.cam.debug = 0
        ws = _lib.Workspace(torch.cuda.current_device())
        ctx = _lib.Context(ws)
        if time_src is not None:
            ctx.set_time_source(time_src.data_ptr())
            r.cam.time = 0.9
        assert r(ctx) == 0
        pg = pc._deformation.alloc_grads()
        cg = pc._deformation.c_grads(pg)
        gbuf = [torch.zeros(n, w, device="cuda") for w in (3, 3, 4, 1, 3, 45, 3)]
        gg = _lib.GaussianGrads(*(t.data_ptr() for t in gbuf))
        dl = torch.linspace(-1, 1, 3 * H * W, device="cuda")
        assert lib.g4d_render_backward(ctx.handle, C.byref(r.cam), C.byref(r.prm), C.byref(cg), C.byref(r.g), dl.data_ptr(),
                                       C.byref(gg), stream()) == 0, lib.g4d_last_error()
        torch.cuda.synchronize()
        return r.out[0].clone(), pg, gbuf

    with torch.no_grad():
        img_a, pg_a, g_a = run(None)
        img_b, pg_b, g_b = run(torch.tensor([0.3], device="cuda"))
    assert torch.equal(img_a, img_b)
    for x, y in zip(list(pg_a) + g_a, list(pg_b) + g_b):
        if x is None:
            continue
        assert float((x - y).abs().max()) <= 1e-5 * max(1e-6, float(y.abs().max()))


@pytest.mark.gpu
def test_adam_step_device_equals_adam_step_and_replays_each_steps_scalars():
    """g4d_adam_step_device with g4d_adam_scalars' block gives the bits of g4d_adam_step, step by step, eagerly and from one
    captured launch replayed with a new block per step."""
    lib = _lib.load()
    ws = _lib.Workspace(torch.cuda.current_device())
    numel = 4 * 3001
    gen = torch.Generator(device="cuda").manual_seed(5)
    p0 = torch.randn(numel, device="cuda", generator=gen)
    grads = [torch.randn(numel, device="cuda", generator=gen) for _ in range(5)]
    segs = (_lib.AdamSegment * 3)(_lib.AdamSegment(0, 1000, 1.6e-4, 0.0), _lib.AdamSegment(1003, 7000, 2.5e-3, 0.0),
                                  _lib.AdamSegment(7000, numel, 0.05, 0.0))
    b1, b2, eps, gs = 0.9, 0.999, 1e-15, 0.5
    stream = lambda: torch.cuda.current_stream().cuda_stream

    def state():
        return [p0.clone(), torch.zeros(numel, device="cuda"), torch.zeros(numel, device="cuda")]

    def scalars(step):
        for i, lr in enumerate((1.6e-4 * 0.9 ** step, 2.5e-3, 0.05 / step)):
            segs[i].lr = lr
        out = _lib.AdamScalars()
        assert lib.g4d_adam_scalars(segs, 3, b1, b2, step, gs, C.byref(out)) == 0
        return torch.frombuffer(bytearray(bytes(out)), dtype=torch.float32).cuda()

    host, dev, graphed = state(), state(), state()
    grad = torch.empty(numel, device="cuda")
    block = torch.zeros(C.sizeof(_lib.AdamScalars) // 4, device="cuda")
    ptr = lambda t: t.data_ptr()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        assert lib.g4d_adam_step_device(ws.handle, ptr(graphed[0]), ptr(grad), ptr(graphed[1]), ptr(graphed[2]), numel, segs, 3,
                                        b1, b2, eps, ptr(block), stream()) == 0
    for step in range(1, 6):
        d_scal = scalars(step)
        grad.copy_(grads[step - 1])
        assert lib.g4d_adam_step(ws.handle, ptr(host[0]), ptr(grad), ptr(host[1]), ptr(host[2]), numel, segs, 3, b1, b2, eps, step,
                                 gs, stream()) == 0
        assert lib.g4d_adam_step_device(ws.handle, ptr(dev[0]), ptr(grad), ptr(dev[1]), ptr(dev[2]), numel, segs, 3, b1, b2, eps,
                                        ptr(d_scal), stream()) == 0
        block.copy_(d_scal)
        graph.replay()
        torch.cuda.synchronize()
        for a, b, c in zip(host, dev, graphed):
            assert torch.equal(a, b) and torch.equal(a, c), step
    assert not torch.equal(host[0], p0)
    assert torch.equal(host[0][1000:1003], p0[1000:1003])       # outside every segment: untouched
