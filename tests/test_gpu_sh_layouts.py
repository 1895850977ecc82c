"""The fused SH layout of the render entry points: features_dc holds all 16 coefficients [N,16,3] and features_rest is NULL.

render() always passes the split layout (features_dc [N,1,3] + features_rest [N,15,3]); this file calls the C-ABI directly
with both layouts on the same scene.  The layout only changes where the coefficients are read from and where their
gradient is written to, so every image, radius and context buffer must be bit-identical, and the fused features_dc gradient
must equal the split dc and rest gradients concatenated: bit for bit whenever the split call repeats bit for bit (the
blend backward adds with atomics, whose order may vary from run to run), otherwise within test_gpu_multicam.py's 2e-5 x max.
"""
import ctypes as C
import importlib

import numpy as np
import pytest
import torch

from util_scene import make_module, synth

_lib = importlib.import_module("4dgaussians_b200._lib")
renderer = importlib.import_module("4dgaussians_b200.renderer")
rasterizer = importlib.import_module("4dgaussians_b200.rasterizer")

SUM_TOL = 2e-5
# every g4d_context_read buffer but bin_phases (clock readings)
BUFFERS = [b for b in _lib.BUF if b != "bin_phases"]


class _Pipe:
    debug = False


# small64: FFMA network without the SHS head; small128: SHS head, on the tensor cores (tc 2) and on the FFMA kernels (tc 0)
CASES = {"ffma": dict(net="small64", tc=2, n=900, wh=(96, 64), theta=20.0, radius=4.0, t=0.3, deg=3),
         "tc": dict(net="small128", tc=2, n=1100, wh=(80, 112), theta=-50.0, radius=2.0, t=0.8, deg=3),
         "ffma_sh": dict(net="small128", tc=0, n=1100, wh=(80, 112), theta=-50.0, radius=2.0, t=0.8, deg=2)}


def _run(c, stage, k, fused):
    """forward + backward of k cameras (g4d_render_forward / _backward when k == 1, the _cameras entry points otherwise)"""
    lib = _lib.load()
    ws = _lib.Workspace(0)
    ws.set_option(_lib.OPT_TENSOR_CORES, c["tc"])
    scene = synth.make_scene(c["n"], seed=11, scale_mean=0.06)
    mod = make_module(c["net"], seed=2, aabb=scene["aabb"]) if stage == "fine" else None
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=c["deg"], requires_grad=False)
    n = c["n"]
    W, H = c["wh"]
    views = [synth.make_camera(c["theta"] + 55.0 * i, W + 13 * i, H, radius=c["radius"], time=c["t"]) for i in range(k)]
    bg = torch.tensor([0.2, 0.1, 0.0], device="cuda")
    keep = []
    cams = (_lib.Camera * k)()
    for i, v in enumerate(views):
        rs, t = renderer.settings_from_camera(v, pc, _Pipe, bg)
        cams[i] = rasterizer.camera_from_settings(rs, time=t, keep=keep)
    prm = mod.c_params(keep, fresh=True) if mod is not None else None
    x, s, r, o = (p.detach().float().contiguous() for p in (pc._xyz, pc._scaling, pc._rotation, pc._opacity))
    if fused:
        dc, rest = torch.cat([pc._features_dc, pc._features_rest], dim=1).detach().float().contiguous(), None
    else:
        dc, rest = pc._features_dc.detach().float().contiguous(), pc._features_rest.detach().float().contiguous()
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
                reads.append((b, None))           # not kept by this forward (e.g. deformed_shs without the SHS head)
    # backward of sum_i <w_i, image_i>
    gen = torch.Generator().manual_seed(5)
    dL = [torch.rand(cl.shape, generator=gen).cuda() for cl in colors]
    pgrads = mod.alloc_grads() if mod is not None else []
    cg = C.byref(mod.c_grads(pgrads)) if mod is not None else None
    gx, gs, gm2 = torch.empty(n, 3, device="cuda"), torch.empty(n, 3, device="cuda"), [torch.empty(n, 3, device="cuda") for _ in range(k)]
    gr, go = torch.empty(n, 4, device="cuda"), torch.empty(n, 1, device="cuda")
    gdc = torch.empty(n, 16 if fused else 1, 3, device="cuda")
    grest = None if fused else torch.empty(n, 15, 3, device="cuda")
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
    grads = [gx, gs, gr, go, sh] + gm2 + list(pgrads)
    return colors + depths + radii, reads, [t.clone() for t in grads]


@pytest.mark.gpu
@pytest.mark.parametrize("case,stage,k", [("ffma", "fine", 1), ("tc", "fine", 1), ("ffma_sh", "fine", 1), ("ffma", "coarse", 1),
                                          ("tc", "fine", 2), ("ffma_sh", "fine", 2), ("tc", "coarse", 2)])
def test_fused_layout_equals_split_layout(case, stage, k):
    c = CASES[case]
    outs, reads, grads = _run(c, stage, k, fused=True)
    outs1, reads1, grads1 = _run(c, stage, k, fused=False)
    _, _, grads2 = _run(c, stage, k, fused=False)
    for a, b in zip(outs, outs1):
        assert torch.equal(a, b)
    for (name, a), (_, b) in zip(reads, reads1):
        assert (a is None) == (b is None), name
        if a is not None:
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), name
    assert any(name == "deformed_shs" and a is not None for name, a in reads) == (stage == "fine" and c["net"] == "small128")
    repeatable = all(torch.equal(a, b) for a, b in zip(grads1, grads2))
    assert len(grads) == len(grads1)
    for i, (a, b) in enumerate(zip(grads, grads1)):
        if repeatable:
            assert torch.equal(a, b), i
        else:
            assert float((a - b).abs().max()) <= SUM_TOL * max(1e-3, float(b.abs().max())), i
