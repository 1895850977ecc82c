"""The refusals of the rasterize and fused-render entry points (g4d_api.cu), one row per refusal: a call with exactly one
violated condition returns its error code and message, and launches nothing -- its outputs, gradient sinks and the
contexts' camera-gradient sinks keep what they held, and every context keeps the forward it held.  The capture rows make
the call on a stream that is capturing a CUDA graph, then end the capture and drop the graph.
"""
import ctypes as C
import importlib
import warnings
from types import SimpleNamespace

import pytest
import torch

from util_scene import make_module, synth

_lib = importlib.import_module("4dgaussians_b200._lib")
build = importlib.import_module("4dgaussians_b200.build")
renderer = importlib.import_module("4dgaussians_b200.renderer")
rasterizer = importlib.import_module("4dgaussians_b200.rasterizer")

ARG, STATE = -2, -4
SIZES = ((96, 72), (80, 64))   # (W, H) of cameras 0 and 1


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


@pytest.fixture(scope="module", autouse=True)
def _built():
    build.build()
    _lib.load()


@pytest.fixture(scope="module")
def scene():
    """3000 Gaussians under small128 (tensor cores, SH head) and two cameras at one time"""
    n = 3000
    sc = synth.make_scene(n, seed=11, scale_mean=0.05)
    pc = synth.SyntheticGaussianModel(sc, make_module("small128", seed=2, aabb=sc["aabb"]), sh_degree=3)
    keep = []
    cams = (_lib.Camera * 2)()
    for i, (W, H) in enumerate(SIZES):
        rs, t = renderer.settings_from_camera(synth.make_camera(20.0 + 40.0 * i, W, H, radius=2.4, time=0.4), pc, _Pipe,
                                              torch.zeros(3, device="cuda"))
        cams[i] = rasterizer.camera_from_settings(rs, time=t, keep=keep)
    # the post-activation inputs of the rasterizer entry points: means3D, shs, opacities, scales, rotations
    raster = [pc._xyz.detach(), torch.cat([pc._features_dc, pc._features_rest], 1).detach().contiguous(),
              torch.sigmoid(pc._opacity).detach(), torch.exp(pc._scaling).detach(),
              torch.nn.functional.normalize(pc._rotation, dim=-1).detach()]
    g = _lib.Gaussians(n, *(t.data_ptr() for t in (pc._xyz, pc._scaling, pc._rotation, pc._opacity, pc._features_dc,
                                                   pc._features_rest)))
    return SimpleNamespace(n=n, pc=pc, keep=keep, cams=cams, prm=pc._deformation.c_params(keep), raster=raster, g=g)


def _p(t):
    return t.data_ptr() if isinstance(t, torch.Tensor) else t


def _ptrs(xs):
    return (C.c_void_p * len(xs))(*[_p(x) for x in xs])


class _Rig:
    """A private workspace with three contexts and the arguments of every entry point, which a row changes before its
    call.  ctx[2] never runs a forward."""

    def __init__(self, s):
        n = s.n
        self.n = n
        self.ws = _lib.Workspace(0)
        self.own = [_lib.Context(self.ws) for _ in range(3)]
        self.ctx = list(self.own)
        self.extra = []            # contexts, workspaces and tensors a row makes
        self.k = 1
        self.cams = (_lib.Camera * 2)(*s.cams)
        self.prm = _lib.DeformParams.from_buffer_copy(s.prm)
        self.g = _lib.Gaussians.from_buffer_copy(s.g)
        self.outs = [[torch.empty(3, H, W, device="cuda"), torch.empty(1, H, W, device="cuda"),
                      torch.empty(n, device="cuda", dtype=torch.int32)] for W, H in SIZES]
        self.out_arrays = True
        self.pgrad_list = s.pc._deformation.alloc_grads()
        self.pgrads = s.pc._deformation.c_grads(self.pgrad_list)
        # xyz, scaling, rotation, opacity, features_dc, features_rest, means2D of camera 0, means2D of camera 1
        self.gbuf = [torch.empty(n, w, device="cuda") for w in (3, 3, 4, 1, 3, 45, 3, 3)]
        self.gg = _lib.GaussianGrads(*(t.data_ptr() for t in self.gbuf[:7]))
        self.gg_cams = _lib.GaussianGrads(*(t.data_ptr() for t in self.gbuf[:6]), None)
        self.g_means2D = self.gbuf[6:]
        self.dl = [torch.linspace(-1, 1, o[0].numel(), device="cuda") for o in self.outs]
        self.raster = list(s.raster)
        # the rasterize backward's sinks: means3D, means2D, shs, opacities, scales, rotations
        self.rgrads = [torch.empty(n, w, device="cuda") for w in (3, 3, 48, 1, 3, 4)]
        self.sinks = torch.empty(2, 35, device="cuda")      # camera gradients of ctx[0], ctx[1]
        self.watched = [x for o in self.outs for x in o] + self.gbuf + self.rgrads + self.pgrad_list + [self.sinks]

    def close(self):
        torch.cuda.synchronize()
        self.ws.freeze(False)
        for c in self.own + [x for x in self.extra if isinstance(x, _lib.Context)]:
            c.__del__()

    # -- the entry points on the rig's arguments ----------------------------------------------------------------------
    @staticmethod
    def stream():
        return torch.cuda.current_stream().cuda_stream

    @staticmethod
    def handle(c):
        return c.handle if c is not None else None

    def rasterize_forward(self):
        return _lib.load().g4d_rasterize_forward(self.handle(self.ctx[0]), C.byref(self.cams[0]), self.n,
                                                 *_ptrs(self.raster + self.outs[0]), self.stream())

    def rasterize_backward(self):
        return _lib.load().g4d_rasterize_backward(self.handle(self.ctx[0]), C.byref(self.cams[0]), self.n,
                                                  *_ptrs(self.raster + [self.dl[0]] + self.rgrads), self.stream())

    def render_forward(self):
        return _lib.load().g4d_render_forward(self.handle(self.ctx[0]), C.byref(self.cams[0]), self.prm, C.byref(self.g),
                                              *_ptrs(self.outs[0]), self.stream())

    def render_backward(self):
        return _lib.load().g4d_render_backward(self.handle(self.ctx[0]), C.byref(self.cams[0]), self.prm, self.pgrads,
                                               C.byref(self.g), _p(self.dl[0]), C.byref(self.gg), self.stream())

    def forward_cameras(self):
        k = self.k
        ctxs = None if self.ctx is None else _ptrs([self.handle(c) for c in self.ctx[:k]])
        outs = [_ptrs([o[j] for o in self.outs[:k]]) for j in range(3)]
        if not self.out_arrays:
            outs[0] = None
        return _lib.load().g4d_render_forward_cameras(ctxs, k, self.cams, self.prm, C.byref(self.g), *outs, self.stream())

    def backward_cameras(self):
        k = self.k
        dl = None if self.dl is None else _ptrs(self.dl[:k])
        return _lib.load().g4d_render_backward_cameras(_ptrs([self.handle(c) for c in self.ctx[:k]]), k, self.cams, self.prm,
                                                       self.pgrads, C.byref(self.g), dl, C.byref(self.gg_cams),
                                                       _ptrs(self.g_means2D[:k]), self.stream())

    # -- state --------------------------------------------------------------------------------------------------------
    def prep(self, kind):
        """the forward a row's call finds: 'raster' or 'fused' on ctx[0], 'group' on ctx[0] and ctx[1]; '-nograd': with
        camera 0 marked G4D_CAM_NO_GRAD"""
        base, _, nograd = kind.partition("-")
        if nograd:
            self.cams[0].debug |= _lib.CAM_NO_GRAD
        self.k = 2 if base == "group" else 1
        rc = {"raster": self.rasterize_forward, "fused": self.render_forward, "group": self.forward_cameras}[base]()
        assert rc == 0, _lib.load().g4d_last_error()
        self.cams[0].debug &= ~_lib.CAM_NO_GRAD
        self.held = self.ctx[:self.k]

    def poison(self, sinks):
        """NaN (radii: -7) into every output and gradient sink, the camera-gradient sinks set on ctx[0] and ctx[1] when
        `sinks`; and the statistics of the forwards the contexts hold"""
        torch.cuda.synchronize()
        for t in self.watched:
            t.fill_(-7 if t.dtype == torch.int32 else float("nan"))
        if sinks:
            for i in range(2):
                self.ctx[i].set_camera_grad(self.sinks[i].data_ptr())
        torch.cuda.synchronize()
        self.stats = [self.stats_of(c) for c in self.held]

    @staticmethod
    def stats_of(c):
        st = c.stats()
        return st.num_rendered, st.num_visible, st.instance_capacity, st.tiles_x, st.tiles_y

    def assert_untouched(self):
        torch.cuda.synchronize()
        for t in self.watched:
            assert bool((t == -7).all()) if t.dtype == torch.int32 else bool(torch.isnan(t).all())
        assert [self.stats_of(c) for c in self.held] == self.stats


# -- the one change of a row ---------------------------------------------------------------------------------------------
def _set(path, value):
    """set rig.<path> to value (dotted; a number indexes)"""
    *head, last = path.split(".")

    def change(r):
        obj = r
        for p in head:
            obj = obj[int(p)] if p.isdigit() else getattr(obj, p)
        if last.isdigit():
            obj[int(last)] = value
        else:
            setattr(obj, last, value)
    return change


def _all(*changes):
    def change(r):
        for f in changes:
            f(r)
    return change


def _sh(m, degree, cams=(0, 1)):
    """the cameras `cams` render with M = m SH coefficients at SH degree `degree`"""
    return _all(*(_all(_set("cams.%d.sh_coeffs" % i, m), _set("cams.%d.sh_degree" % i, degree)) for i in cams))


def _no_sh_head(r):
    r.prm.head_mask &= ~_lib.HEAD_SHS


def _misaligned_plane_sink(r):
    r.pgrads = _lib.DeformGrads.from_buffer_copy(r.pgrads)
    r.pgrads.planes[0][0] += 4


def _other_workspace(r):
    ws = _lib.Workspace(0)
    c = _lib.Context(ws)
    r.extra += [c, ws]
    r.ctx[1] = c


def _time_source(r):
    t = torch.full((1,), 0.4, device="cuda")
    r.extra.append(t)
    r.ctx[1].set_time_source(t.data_ptr())


def _same_context(r):
    r.ctx[1] = r.ctx[0]


def _exact(r):
    r.ws.set_option(_lib.OPT_SYNC_MODE, 1)


def _debug(i):
    return lambda r: setattr(r.cams[i], "debug", r.cams[i].debug | _lib.CAM_DEBUG)


def _timing(r):
    r.ws.set_option(_lib.OPT_STAGE_TIMING, 1)


def _unlearnt(r):
    """the call's last context has run no forward"""
    r.ctx[r.k - 1] = r.ctx[2]


def _camera_sink(r):
    for i in range(2):
        r.ctx[i].set_camera_grad(r.sinks[i].data_ptr())


_PREP = {"rasterize_forward": "raster", "rasterize_backward": "raster", "render_forward": "fused",
         "render_backward": "fused", "forward_cameras": "group", "backward_cameras": "group"}

# (entry point, change, code, message[, the forward the call finds when it is not the entry point's own])
ROWS = [
    ("rasterize_forward", _set("ctx.0", None), ARG, "context is NULL"),
    ("rasterize_forward", _set("cams.0.image_height", 0), ARG, "image size out of range"),
    ("rasterize_forward", _set("outs.0.0", None), ARG, "bad n / output pointers"),
    ("rasterize_forward", _set("raster.0", None), ARG, "Please provide means3D"),
    ("rasterize_forward", _set("n", 1 << 31), ARG, "n too large"),
    ("rasterize_backward", _set("ctx.0", None), ARG, "context is NULL"),
    ("rasterize_backward", None, STATE, "g4d_rasterize_backward needs the matching g4d_rasterize_forward", "fused"),
    ("rasterize_backward", _set("n", 2999), STATE, "g4d_rasterize_backward needs the matching g4d_rasterize_forward"),
    ("rasterize_backward", _set("cams.0.tanfovx", 0.0), ARG, "tanfov must be positive"),
    ("rasterize_backward", _set("cams.0.image_width", 80), STATE, "camera differs from the forward's"),
    ("rasterize_backward", _sh(4, 1, (0,)), STATE, "sh_coeffs differs from the forward's"),
    ("rasterize_backward", _set("dl.0", None), ARG, "NULL gradient pointer"),
    ("rasterize_backward", _set("rgrads.1", None), ARG, "NULL gradient pointer"),
    ("render_forward", _set("ctx.0", None), ARG, "context is NULL"),
    ("render_forward", _set("cams.0.tanfovy", -1.0), ARG, "tanfov must be positive"),
    ("render_forward", _set("prm.levels", 0), ARG, "levels must be in 1..4"),
    ("render_forward", _sh(9, 2, (0,)), ARG, "the SHS head deforms 16 SH coefficients"),
    ("render_forward", _set("outs.0.0", None), ARG, "bad gaussians / outputs"),
    ("render_forward", _set("g.xyz", None), ARG, "NULL gaussian tensor"),
    ("render_backward", _set("ctx.0", None), ARG, "context is NULL"),
    ("render_backward", None, STATE, "g4d_render_backward needs the matching g4d_render_forward", "raster"),
    ("render_backward", _set("g.n", 2999), STATE, "g4d_render_backward needs the matching g4d_render_forward"),
    ("render_backward", None, STATE, "use g4d_render_backward_cameras", "group"),
    ("render_backward", None, STATE, "g4d_render_backward after a G4D_CAM_NO_GRAD forward", "fused-nograd"),
    ("render_backward", _set("prm", None), STATE, "deform params differ from the forward's"),
    ("render_backward", _set("cams.0.image_height", 20000), ARG, "image size out of range"),
    ("render_backward", _set("prm.channels", 6), ARG, "channels must be a multiple of 4"),
    ("render_backward", _set("pgrads", None), ARG, "pgrads is NULL"),
    ("render_backward", _misaligned_plane_sink, ARG, "spatial-plane gradient sinks must be 16-byte aligned"),
    ("render_backward", _set("cams.0.image_width", 80), STATE, "camera differs from the forward's"),
    ("render_backward", _all(_sh(4, 1, (0,)), _no_sh_head), STATE, "sh_coeffs differs from the forward's"),
    ("render_backward", _set("dl.0", None), ARG, "NULL gradient pointer"),
    ("render_backward", _set("gg.means2D", None), ARG, "NULL gradient pointer"),
    ("render_backward", _set("gg.opacity", None), ARG, "NULL gradient pointer"),
    ("render_backward", _set("gg.features_rest", None), ARG, "features_rest gradient sink is NULL"),
    ("forward_cameras", _set("k", 0), ARG, "the number of cameras must be in 1..G4D_MAX_CAMERAS"),
    ("forward_cameras", _set("k", 33), ARG, "the number of cameras must be in 1..G4D_MAX_CAMERAS"),
    ("forward_cameras", _set("cams", None), ARG, "cameras are NULL"),
    ("forward_cameras", _set("cams.1.image_width", -1), ARG, "image size out of range"),
    ("forward_cameras", _sh(9, 2, (1,)), ARG, "the cameras of one call must share sh_coeffs"),
    ("forward_cameras", _set("cams.1.time", 0.5), ARG, "the cameras of one call must share their time bit for bit"),
    ("forward_cameras", _set("ctx", None), ARG, "contexts are NULL"),
    ("forward_cameras", _set("ctx.1", None), ARG, "context is NULL"),
    ("forward_cameras", _other_workspace, ARG, "the contexts of one call must belong to one workspace"),
    ("forward_cameras", _time_source, ARG, "the contexts of one call must share their time source"),
    ("forward_cameras", _same_context, ARG, "the contexts of one call must be pairwise distinct"),
    ("forward_cameras", _set("out_arrays", False), ARG, "output arrays are NULL"),
    ("forward_cameras", _set("prm.net_width", 96), ARG, "net_width must be 64 or 128"),
    ("forward_cameras", _sh(9, 2), ARG, "the SHS head deforms 16 SH coefficients"),
    ("forward_cameras", _set("outs.1.1", None), ARG, "bad gaussians / outputs"),
    ("forward_cameras", _set("g.opacity", None), ARG, "NULL gaussian tensor"),
    ("backward_cameras", _set("k", 0), ARG, "the number of cameras must be in 1..G4D_MAX_CAMERAS"),
    ("backward_cameras", _set("cams.1.time", 0.5), ARG, "the cameras of one call must share their time bit for bit"),
    ("backward_cameras", _same_context, ARG, "the contexts of one call must be pairwise distinct"),
    ("backward_cameras", _other_workspace, ARG, "the contexts of one call must belong to one workspace"),
    ("backward_cameras", _time_source, ARG, "the contexts of one call must share their time source"),
    ("backward_cameras", _set("dl", None), ARG, "NULL argument"),
    ("backward_cameras", _set("gg_cams.means2D", 256), ARG, "gg->means2D must be NULL"),
    ("backward_cameras", None, STATE, "g4d_render_backward_cameras needs the matching g4d_render_forward_cameras", "fused"),
    ("backward_cameras", _set("k", 1), STATE, "g4d_render_backward_cameras needs the matching g4d_render_forward_cameras"),
    ("backward_cameras", _set("g.n", 2999), STATE, "g4d_render_backward_cameras needs the matching g4d_render_forward_cameras"),
    ("backward_cameras", _set("cams.1.image_height", 60), STATE, "camera differs from the forward's"),
    ("backward_cameras", _all(_sh(4, 1), _no_sh_head), STATE, "sh_coeffs differs from the forward's"),
    ("backward_cameras", None, STATE, "g4d_render_backward_cameras after a G4D_CAM_NO_GRAD forward", "group-nograd"),
    ("backward_cameras", _set("prm", None), STATE, "deform params differ from the forward's"),
    ("backward_cameras", _set("prm.levels", 5), ARG, "levels must be in 1..4"),
    ("backward_cameras", _set("pgrads", None), ARG, "pgrads is NULL"),
    ("backward_cameras", _misaligned_plane_sink, ARG, "spatial-plane gradient sinks must be 16-byte aligned"),
    ("backward_cameras", _set("gg_cams.xyz", None), ARG, "NULL gradient pointer"),
    ("backward_cameras", _set("gg_cams.features_rest", None), ARG, "features_rest gradient sink is NULL"),
]

# the same on a stream that is capturing: (entry point, change, message); every one is G4D_ERR_STATE.  The workspace is in
# no-sync mode, and the contexts learnt their capacity, unless the change says otherwise.
CAPTURE_ROWS = []
for _entry, _last in (("rasterize_forward", 0), ("render_forward", 0), ("forward_cameras", 1)):
    CAPTURE_ROWS += [(_entry, _exact, "cannot capture a forward in exact sync mode"),
                     (_entry, _unlearnt, "has not learnt its instance capacity"),
                     (_entry, _debug(_last), "cannot capture with G4D_CAM_DEBUG"),
                     (_entry, _timing, "cannot capture with G4D_OPT_STAGE_TIMING")]
for _entry, _last in (("rasterize_backward", 0), ("render_backward", 0), ("backward_cameras", 1)):
    CAPTURE_ROWS += [(_entry, _camera_sink, "cannot capture a backward on a context with a camera gradient set"),
                     (_entry, _debug(_last), "cannot capture with G4D_CAM_DEBUG"),
                     (_entry, _timing, "cannot capture with G4D_OPT_STAGE_TIMING")]


def _table():
    rows = [pytest.param(entry, change, code, msg, rest[0] if rest else _PREP[entry], False, id="%s-%d" % (entry, i))
            for i, (entry, change, code, msg, *rest) in enumerate(ROWS)]
    rows += [pytest.param(entry, change, STATE, msg, _PREP[entry], True, id="%s-capture-%d" % (entry, i))
             for i, (entry, change, msg) in enumerate(CAPTURE_ROWS)]
    return rows


@pytest.fixture
def rig(scene):
    r = _Rig(scene)
    yield r
    r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("entry,change,code,msg,prep,capture", _table())
def test_refusal(rig, entry, change, code, msg, prep, capture):
    with torch.no_grad():
        rig.prep(prep)
        rig.k = 2 if entry.endswith("_cameras") else 1
        rig.poison(sinks=not capture)
        if capture:
            rig.ws.set_option(_lib.OPT_SYNC_MODE, 0)
        if change is not None:
            change(rig)
        call = getattr(rig, entry)
        if capture:
            graph, rc = torch.cuda.CUDAGraph(), []
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")      # (torch may warn that the graph is empty)
                with torch.cuda.graph(graph):
                    rc.append(call())
            del graph
            rc = rc[0]
        else:
            rc = call()
        err = _lib.load().g4d_last_error().decode()
        assert rc == code and msg in err, (rc, err)
        rig.assert_untouched()
