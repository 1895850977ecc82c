"""The spatial walk order of the HexPlane gather (G4D_OPT_GATHER_ORDER, DESIGN.md §4.1).

The order is a permutation of the Gaussians that the workspace builds when the xyz pointer or N changes and keeps
otherwise.  It can never change a result: every Gaussian's features come from its own taps and land in its own row.  So every
output of the spatial order is compared bit for bit with index order (G4D_OPT_GATHER_ORDER = 0).  Gradients are compared bit
for bit whenever index order itself repeats bit for bit; the atomics of the backward kernels may add in another order from
one run to the next.
"""
import ctypes as C
import importlib

import numpy as np
import pytest
import torch

from util_scene import g4d, make_module, synth

_lib = importlib.import_module("4dgaussians_b200._lib")

SUM_TOL = 2e-5   # fp32 atomics in another order (test_gpu_multicam.py)


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


@pytest.fixture
def ws():
    w = _lib.Workspace.get(0)
    yield w
    w.set_option(_lib.OPT_GATHER_ORDER, 1)


def _model(n, seed=3, net="dynerf", grad=False, scale=0.02):
    scene = synth.make_scene(n, seed=seed, scale_mean=scale)
    mod = make_module(net, seed=seed, aabb=scene["aabb"])
    return scene, mod, synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=grad)


def _read_order(ctx):
    """the workspace's walk order (G4D_BUF_GATHER_ORDER), read through a context of that workspace"""
    lib = _lib.load()
    nb = lib.g4d_context_read(ctx.handle, _lib.BUF_GATHER_ORDER, None, 0)
    _lib.check(min(int(nb), 0), "g4d_context_read")
    out = np.zeros(max(int(nb) // 4, 1), dtype=np.uint32)
    _lib.check(min(int(lib.g4d_context_read(ctx.handle, _lib.BUF_GATHER_ORDER, out.ctypes.data_as(C.c_void_p), nb)), 0),
               "g4d_context_read")
    return out[:int(nb) // 4]


def _assert_permutation(order, n):
    assert order.shape == (n,)
    assert np.array_equal(np.sort(order), np.arange(n, dtype=np.uint32))


def _render(pc, cam, ws, order, grad=False):
    ws.set_option(_lib.OPT_GATHER_ORDER, order)
    bg = torch.zeros(3, device="cuda")
    with torch.set_grad_enabled(grad):
        out = g4d.render(cam, pc, _Pipe, bg)
    torch.cuda.synchronize()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 63, 64, 65, 4097, 300_000])
def test_order_is_a_permutation(ws, n):
    """Deform-only forward over points inside the aabb, exactly on its faces, outside it, infinite and NaN."""
    scene, mod, pc = _model(max(n, 64))
    keep = _render(pc, synth.make_camera(30.0, 64, 48, radius=4.0, time=0.3), ws, 1, grad=True)   # a context to read through
    ctx = keep["render"].grad_fn.lease.ctx
    hi, lo = scene["aabb"][0], scene["aabb"][1]
    nan, inf = float("nan"), float("inf")
    special = torch.stack([torch.tensor([nan, 0.0, 0.0]), hi, lo, torch.tensor([hi[0], lo[1], hi[2]]), hi + 1.0, lo - 1.0,
                           torch.full((3,), nan), torch.full((3,), inf), torch.full((3,), -inf), torch.tensor([0.0, inf, nan]),
                           hi * 1e30, torch.tensor([lo[0], 0.0, nan])])
    xyz = scene["xyz"][:n].clone()
    k = min(n, special.shape[0])
    xyz[:k] = special[:k]
    shs = torch.cat([scene["features_dc"], scene["features_rest"]], dim=1)[:n]
    ws.set_option(_lib.OPT_GATHER_ORDER, 1)
    with torch.no_grad():
        mod(xyz.cuda().contiguous(), scene["scaling"][:n].cuda().contiguous(), scene["rotation"][:n].cuda().contiguous(),
            scene["opacity"][:n].cuda().contiguous(), shs.cuda().contiguous(), torch.tensor(0.4))
    torch.cuda.synchronize()
    _assert_permutation(_read_order(ctx), n)


def _outputs(out, ctx, features=True):
    bufs = ("features", "deformed", "deformed_shs", "sorted_ids") if features else ("deformed", "sorted_ids")
    return [out["render"].detach(), out["depth"].detach(), out["radii"]] + [torch.from_numpy(ctx.read(b).copy()) for b in bufs]


def _same_bits_in_either_order(ws, workload):
    w = synth.WORKLOADS[workload]
    _, _, pc = _model(w["n"], seed=0, net=w["net"], grad=True, scale=w["scale_mean"])
    cams = synth.orbit_cameras(2, w["width"], w["height"], radius=w["radius"], focal=w["focal"])
    for cam in cams:
        cam.time = 0.35
    tc = workload == "C3"
    res = {}
    for order in (1, 0, 1):
        out = _render(pc, cams[0], ws, order, grad=True)
        res.setdefault(order, []).append(_outputs(out, out["render"].grad_fn.lease.ctx, features=tc))
        del out
    assert len(res[1][0]) == len(res[0][0]) == (7 if tc else 5)
    for got in (res[1][0], res[1][1]):
        for i, (a, b) in enumerate(zip(got, res[0][0])):
            assert torch.equal(a, b), (workload, i)
    assert int((res[0][0][2] > 0).sum()) > 1000
    # render_cameras, k = 2: deformed once, both cameras from the same features
    multi = {}
    for order in (1, 0):
        ws.set_option(_lib.OPT_GATHER_ORDER, order)
        with torch.no_grad():
            outs = g4d.render_cameras(cams, pc, _Pipe, torch.zeros(3, device="cuda"))
        multi[order] = [(o["render"].clone(), o["depth"].clone(), o["radii"].clone()) for o in outs]
    for a, b in zip(multi[1], multi[0]):
        assert all(torch.equal(x, y) for x, y in zip(a, b)), workload


@pytest.mark.gpu
def test_full_size_C3_same_bits_in_either_order(ws):
    """C3 (the tensor-core network), then an FFMA arm at C1 size (dnerf net, net_width 64), which keeps no features."""
    _same_bits_in_either_order(ws, "C3")
    _same_bits_in_either_order(ws, "C1")


@pytest.mark.gpu
def test_stale_order_and_growth(ws):
    scene, mod, pc = _model(20_000, seed=4)
    cam = synth.make_camera(40.0, 160, 120, radius=3.0, time=0.6)
    _render(pc, cam, ws, 1, grad=True)
    ctx_of = lambda o: o["render"].grad_fn.lease.ctx
    first = _render(pc, cam, ws, 1, grad=True)
    built = _read_order(ctx_of(first)).copy()
    _assert_permutation(built, 20_000)
    # xyz moved in place (a training step): the order is kept, the results are still those of index order
    with torch.no_grad():
        pc._xyz.add_(0.05 * torch.randn(pc._xyz.shape, generator=torch.Generator().manual_seed(9)).cuda())
    moved = _render(pc, cam, ws, 1, grad=True)
    assert np.array_equal(_read_order(ctx_of(moved)), built)
    ref = _render(pc, cam, ws, 0, grad=True)
    for a, b in zip(_outputs(moved, ctx_of(moved)), _outputs(ref, ctx_of(ref))):
        assert torch.equal(a, b)
    # more Gaussians (densification appends): a new order for the new N
    extra = synth.make_scene(3_001, seed=5, scale_mean=0.02)
    grown = {k: torch.cat([pc_t.detach().cpu(), extra[k]]) for k, pc_t in
             (("xyz", pc._xyz), ("scaling", pc._scaling), ("rotation", pc._rotation), ("opacity", pc._opacity),
              ("features_dc", pc._features_dc), ("features_rest", pc._features_rest))}
    pc2 = synth.SyntheticGaussianModel(grown, mod, sh_degree=3, requires_grad=True)
    big = _render(pc2, cam, ws, 1, grad=True)
    _assert_permutation(_read_order(ctx_of(big)), 23_001)
    ref2 = _render(pc2, cam, ws, 0, grad=True)
    for a, b in zip(_outputs(big, ctx_of(big)), _outputs(ref2, ctx_of(ref2))):
        assert torch.equal(a, b)


def _compare_grads(spatial, index, index_again):
    repeatable = all(torch.equal(a, b) for a, b in zip(index, index_again))
    for a, b in zip(spatial, index):
        if repeatable:
            assert torch.equal(a, b)
        else:
            assert float((a - b).abs().max()) <= SUM_TOL * max(1e-3, float(b.abs().max()))


@pytest.mark.gpu
def test_render_backward_same_gradients(ws):
    cam = synth.make_camera(100.0, 203, 152, radius=2.2, time=0.5)
    wgt = torch.rand(3, cam.image_height, cam.image_width, generator=torch.Generator().manual_seed(3)).cuda()
    runs = {}
    for order in (1, 0, 0):
        _, mod, pc = _model(2500, seed=6, grad=True, scale=0.04)
        out = _render(pc, cam, ws, order, grad=True)
        (out["render"] * wgt).sum().backward()
        runs.setdefault(order, []).append([p.grad.clone() for p in pc.gaussian_parameters()] +
                                          [p.grad.clone() for p in mod.flat_parameters() if p.grad is not None])
    _compare_grads(runs[1][0], runs[0][0], runs[0][1])


@pytest.mark.gpu
def test_deform_only_backward_same_gradients(ws):
    """g4d_deform_backward gathers the features again, in the workspace's order."""
    scene = synth.make_scene(5000, seed=8)
    runs = {}
    for order in (1, 0, 0):
        ws.set_option(_lib.OPT_GATHER_ORDER, order)
        mod = make_module("dynerf", seed=8, aabb=scene["aabb"])
        leaves = [scene[k].cuda().requires_grad_(True) for k in ("xyz", "scaling", "rotation", "opacity")]
        shs = torch.cat([scene["features_dc"], scene["features_rest"]], dim=1).cuda().requires_grad_(True)
        outs = mod(*leaves, shs, torch.tensor(0.7))
        fwd = [o.detach().clone() for o in outs]
        sum((o * (1.0 + 0.1 * i)).sum() for i, o in enumerate(outs)).backward()
        torch.cuda.synchronize()
        runs.setdefault(order, []).append((fwd, [t.grad.clone() for t in leaves + [shs]] +
                                           [p.grad.clone() for p in mod.flat_parameters() if p.grad is not None]))
    for a, b in zip(runs[1][0][0], runs[0][0][0]):
        assert torch.equal(a, b)
    _compare_grads(runs[1][0][1], runs[0][0][1], runs[0][1][1])
