"""The forward a context holds (ForwardRecord, g4d_api.cu): a forward entry point clears the record of every context it
writes before its first launch and writes it only once the whole call has succeeded, so no read or backward can act on
what an earlier or a failed forward left in a context's buffers.
"""
import ctypes as C
import importlib

import pytest
import torch

from util_scene import make_module, synth

_lib = importlib.import_module("4dgaussians_b200._lib")
build = importlib.import_module("4dgaussians_b200.build")
renderer = importlib.import_module("4dgaussians_b200.renderer")
rasterizer = importlib.import_module("4dgaussians_b200.rasterizer")


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


@pytest.fixture(scope="module", autouse=True)
def _built():
    build.build()
    _lib.load()


@pytest.fixture
def private():
    """a private workspace and two contexts on it; the contexts are destroyed first, also when the test fails (its traceback
    would otherwise leave their order to the garbage collector)"""
    ws = _lib.Workspace(0)
    ctxs = [_lib.Context(ws), _lib.Context(ws)]
    yield ws, ctxs
    torch.cuda.synchronize()
    ws.freeze(False)
    for c in ctxs:
        c.__del__()


def _stream():
    return torch.cuda.current_stream().cuda_stream


class _Scene:
    """n Gaussians under small128 (tensor cores: a grad-enabled forward keeps its features), the C structs of its grad-enabled
    forwards through the cameras `sizes` ((W, H) each, one time) and their outputs"""

    def __init__(self, n, sizes, seed=11):
        scene = synth.make_scene(n, seed=seed, scale_mean=0.05)
        self.pc = synth.SyntheticGaussianModel(scene, make_module("small128", seed=2, aabb=scene["aabb"]), sh_degree=3)
        self.n = n
        self.keep = []
        bg = torch.zeros(3, device="cuda")
        self.cams = (_lib.Camera * len(sizes))()
        self.outs = []
        for i, (W, H) in enumerate(sizes):
            rs, t = renderer.settings_from_camera(synth.make_camera(20.0 + 40.0 * i, W, H, radius=2.4, time=0.4), self.pc, _Pipe, bg)
            self.cams[i] = rasterizer.camera_from_settings(rs, time=t, keep=self.keep)
            self.outs.append((torch.empty(3, H, W, device="cuda"), torch.empty(1, H, W, device="cuda"),
                              torch.empty(n, device="cuda", dtype=torch.int32)))
        self.prm = self.pc._deformation.c_params(self.keep)
        pc = self.pc
        self.g = _lib.Gaussians(n, *(t.data_ptr() for t in (pc._xyz, pc._scaling, pc._rotation, pc._opacity, pc._features_dc,
                                                             pc._features_rest)))

    def forward(self, ctx, i=0):
        return _lib.load().g4d_render_forward(ctx.handle, C.byref(self.cams[i]), C.byref(self.prm), C.byref(self.g),
                                              *(t.data_ptr() for t in self.outs[i]), _stream())

    def forward_cameras(self, ctxs):
        k = len(ctxs)
        ptrs = lambda xs: (C.c_void_p * k)(*xs)
        return _lib.load().g4d_render_forward_cameras(ptrs([c.handle for c in ctxs]), k, self.cams, C.byref(self.prm),
                                                      C.byref(self.g), *(ptrs([o[j].data_ptr() for o in self.outs[:k]])
                                                                         for j in range(3)), _stream())

    def backward(self, ctx):
        """g4d_render_backward on ctx with camera 0"""
        self.pgrads = self.pc._deformation.alloc_grads()
        self.gbuf = [torch.zeros(self.n, w, device="cuda") for w in (3, 3, 4, 1, 3, 45, 3)]
        gg = _lib.GaussianGrads(*(t.data_ptr() for t in self.gbuf))
        self.dl = torch.linspace(-1, 1, self.outs[0][0].numel(), device="cuda")
        return _lib.load().g4d_render_backward(ctx.handle, C.byref(self.cams[0]), C.byref(self.prm),
                                               C.byref(self.pc._deformation.c_grads(self.pgrads)), C.byref(self.g),
                                               self.dl.data_ptr(), C.byref(gg), _stream())


@pytest.mark.gpu
def test_other_cameras_of_a_group_hold_no_features(private):
    """Cameras 1..k-1 of g4d_render_forward_cameras keep no features of their own: reading them is refused, whatever a
    larger earlier forward left in the context's feature buffer."""
    _, (a, b) = private
    with torch.no_grad():
        earlier = _Scene(2000, [(96, 72)], seed=5)
        assert earlier.forward(b) == 0, _lib.load().g4d_last_error()
        assert b.read("features").size == 2000 * earlier.prm.levels * earlier.prm.channels
        group = _Scene(1000, [(96, 72), (80, 64)])
        assert group.forward_cameras([a, b]) == 0, _lib.load().g4d_last_error()
        with pytest.raises(_lib.G4DError, match=r"code -4"):
            b.read("features")
        assert a.read("features").size == 1000 * group.prm.levels * group.prm.channels


@pytest.mark.gpu
def test_failed_group_leaves_no_forward_on_camera_0(private):
    """A group call refused at camera 1 (its image buffer would have to grow on a frozen workspace) leaves camera 0 without
    a forward, although camera 0's own forward ran to its end: a backward on it is refused."""
    W, H = 96, 72
    ws, (a, b) = private
    with torch.no_grad():
        s = _Scene(1500, [(W, H), (W, H)])
        small = _Scene(1500, [(W // 2 - 8, H // 2 - 6)])     # the same N, under half the pixels of camera 1
        assert s.forward(a) == 0 and s.backward(a) == 0, _lib.load().g4d_last_error()
        assert small.forward(b) == 0, _lib.load().g4d_last_error()
        torch.cuda.synchronize()
        ws.freeze(True)
        assert s.forward_cameras([a, b]) == -4
        assert b"would have to grow" in _lib.load().g4d_last_error()
        assert s.backward(a) == -4
        assert b"g4d_render_backward needs the matching g4d_render_forward" in _lib.load().g4d_last_error()
