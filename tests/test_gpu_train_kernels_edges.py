"""The training-step kernels on their edges, each against a plain high-precision reference: L1 (g4d_loss.cu) at every tail,
storage offset, dtype and layout; SSIM at clipped windows, tile seams, many channels and near-flat images, per pixel; the
plane regulariser per texel at 4 levels, time resolution 3 and odd channel counts; the flat Adam of g4d_optim.cu element by
element through the C-ABI and through FlatState; the kNN of g4d_knn.cu bit for bit on degenerate and far-off-origin clouds.
The cases live in util_train_kernels.py; test_train_kernels_edge_cases.py checks on the CPU that each reaches its condition."""
import ctypes as C
import importlib

import numpy as np
import pytest
import torch

import util_train_kernels as ut
from oracle import knn_ref
from oracle import loss_ref as lr
from util_scene import g4d

pytestmark = pytest.mark.gpu
losses = importlib.import_module("4dgaussians_b200.losses")
knn = importlib.import_module("4dgaussians_b200.simple_knn")
td = importlib.import_module("4dgaussians_b200.train_dp")
_lib = importlib.import_module("4dgaussians_b200._lib")
G4D_ERR_ARG = -2


def _abi():
    return _lib.load(), _lib.Workspace.get(torch.cuda.current_device()).handle, int(torch.cuda.current_stream().cuda_stream)


# ---- L1 ------------------------------------------------------------------------------------------------------------------------
def _l1_check(out_leaf, out, gt_leaf, gt, up=0.37):
    """losses.l1_loss(out, gt) with gradients to both sides: value within 1e-6 of the fp64 mean; every gradient element equal to
    sign(out - gt) * (fp32(1/n) * fp32(up)) formed in fp32 (cast to the input dtype), bit for bit, and within 1 ulp of fp64."""
    n = out.numel()
    v = losses.l1_loss(out, gt)
    (v * up).backward()
    a64, b64 = out.detach().double().cpu(), gt.detach().double().cpu()
    ref = float((a64 - b64).abs().mean())
    assert abs(float(v.detach()) - ref) <= 1e-6 * abs(ref) + 1e-30, (n, float(v.detach()), ref)
    s32 = np.float32(np.float32(1.0 / n) * np.float32(up))
    sign = torch.sign(a64 - b64).float()
    want = (sign * float(s32)).to(out.dtype)
    for leaf, view, w, side in ((out_leaf, out, want, 1.0), (gt_leaf, gt, -want, -1.0)):
        got = leaf.grad
        if view is not leaf:                       # the gradient reaches the base tensor through the view, zeros elsewhere
            mask = torch.zeros_like(leaf, dtype=torch.bool)
            mask.view(-1)[(view.data_ptr() - leaf.data_ptr()) // leaf.element_size():][:n] = True
            assert view.is_contiguous() and not bool(got[~mask].any())
            got = got.view(-1)[mask.view(-1)]
        got = got.detach().cpu().reshape(-1)
        assert torch.equal(got, w.reshape(-1)), (n, int((got != w.reshape(-1)).sum()))
        if out.dtype == torch.float32:
            # one rounding from the fp64 product of the two fp32 factors the kernel receives; two (1/n, then the product)
            # from the exact fp32(up) / n
            up32 = float(np.float32(up))
            for exact, ulps in ((float(np.float32(1.0 / n)) * up32, 1), (up32 / n, 2)):
                e = (sign.double() * side * exact).reshape(-1).numpy()
                assert (np.abs(got.double().numpy() - e) <= ulps * ut.ulp32(e)).all(), (n, ulps)


def _leaf(t):
    return t.detach().clone().requires_grad_(True)


@pytest.mark.parametrize("n", ut.L1_NUMELS)
def test_l1_every_tail(n):
    a, b = ut.pair((n,), n, "cuda")
    a, b = _leaf(a), _leaf(b)
    _l1_check(a, a, b, b)


def test_l1_full_size_batch():
    a, b = ut.pair(ut.L1_BATCH, 5, "cuda")
    a, b = _leaf(a), _leaf(b)
    _l1_check(a, a, b, b, up=0.25)


@pytest.mark.parametrize("case", range(18))
def test_l1_misaligned_views(case):
    """batch[i] of an odd-H*W batch and flat[k:] views start 4, 8 or 12 bytes off a 16-byte boundary: the scalar-load kernels"""
    cases = ut.offset_views("cuda")
    name, out, gt = cases[case]
    ob, gb = out._base if out._base is not None else out, gt._base if gt._base is not None else gt
    ob, gb = ob.detach().clone().requires_grad_(True), gb.detach().clone().requires_grad_(True)
    # the same views of the leaves (clone keeps the storage offsets modulo 16: fresh allocations are 512-byte aligned)
    o = ob.view(-1)[out.storage_offset():out.storage_offset() + out.numel()].view(out.shape)
    g = gb.view(-1)[gt.storage_offset():gt.storage_offset() + gt.numel()].view(gt.shape)
    side = name.rsplit(":", 1)[1]
    assert (ut.misalignment(o) != 0) == (side in ("out", "both")) and (ut.misalignment(g) != 0) == (side in ("gt", "both"))
    _l1_check(ob, o, gb, g)


def test_l1_misaligned_gradient_sink_through_the_abi():
    lib, ws, st = _abi()
    for n in (1, 5, 1023, 4096):
        a, b = ut.pair((n,), n + 1, "cuda")
        buf = torch.full((n + 8,), 7.0, device="cuda")
        for k in (1, 2, 3):
            buf.fill_(7.0)
            grad = buf[k:k + n]
            assert ut.misalignment(grad) == 4 * k
            _lib.check(lib.g4d_l1_loss_backward(ws, a.data_ptr(), b.data_ptr(), n, 1.0 / n, None, grad.data_ptr(), st), "l1 bwd")
            torch.cuda.synchronize()
            want = torch.sign(a.double() - b.double()).float() * float(np.float32(1.0 / n))
            assert torch.equal(grad, want) and bool((buf[:k] == 7).all()) and bool((buf[k + n:] == 7).all())


def test_l1_non_contiguous_rgba_ground_truth():
    out, _ = ut.pair((2, 3) + ut.ODD_HW, 21, "cuda")
    rgba, _ = ut.pair((2, 4) + ut.ODD_HW, 22, "cuda")
    o, g = _leaf(out), _leaf(rgba)
    gt = g[:, :3]
    assert not gt.is_contiguous()
    v = losses.l1_loss(o, gt)
    (v * 0.37).backward()
    ref = float((o.detach().double() - gt.detach().double()).abs().mean())
    assert abs(float(v) - ref) <= 1e-6 * ref
    want = torch.sign(o.detach().double() - gt.detach().double()).float() * float(np.float32(np.float32(1.0 / o.numel()) * np.float32(0.37)))
    assert torch.equal(o.grad, want) and torch.equal(g.grad[:, :3], -want) and not bool(g.grad[:, 3].any())
    # one image, as train.py:201 passes it: gt[:3] of a [4,H,W] frame
    o1, g1 = _leaf(out[0]), _leaf(rgba[0])
    _l1_check(o1, o1, g1, g1[:3])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_l1_half_inputs(dtype):
    for shape in ((1025,), (3,) + ut.ODD_HW):
        a, b = ut.pair(shape, 31, "cuda", dtype)
        a, b = _leaf(a), _leaf(b)
        _l1_check(a, a, b, b)
        assert a.grad.dtype == dtype and b.grad.dtype == dtype


# ---- SSIM ----------------------------------------------------------------------------------------------------------------------
def _ssim_check(shape, kind, seed, record_property, up=0.37):
    x, y = ut.ssim_images(shape, kind, seed)
    a = x.float().cuda().requires_grad_(True)
    v = losses.ssim(a, y.float().cuda())
    (v * up).backward()
    got = a.grad.double().cpu().numpy()
    v64, g64 = ut.ssim_ref(x, y, torch.float64, up)
    v32, g32 = ut.ssim_ref(x, y, torch.float32, up)
    if kind == "same":                    # the map is 1 everywhere and the fp64 gradient 0 to rounding
        assert abs(float(v) - 1.0) <= 1e-6
        bound = 1e-4 * up / x.numel()     # 1e-4 of one pixel's share of the mean
        record_property("ssim_same_grad_over_bound", float(np.abs(got).max() / bound))
        assert np.abs(got).max() <= bound
        return
    dv = abs(float(v) - v64)
    assert dv <= max(ut.SSIM_K * abs(v32 - v64), 2e-6 * abs(v64)), (float(v), v64, v32)
    e_k, e_32 = ut.pixel_err(got, g64), ut.pixel_err(g32, g64)
    record_property("ssim_pixel_err", (e_k, e_32))
    # floor on the fp32 distance: below 1e-5 both sides are a few roundings of the pixel's own value
    assert e_k <= ut.SSIM_K * max(e_32, 1e-5), (shape, kind, e_k, e_32)


@pytest.mark.parametrize("i", range(len(ut.SSIM_HW)))
def test_ssim_windows_and_seams(i, record_property):
    h, w = ut.SSIM_HW[i]
    _ssim_check(ut.ssim_shape(i, h, w), "rand", i, record_property)


@pytest.mark.parametrize("kind", ["same", "const", "bright"])
@pytest.mark.parametrize("shape", [(3, 32, 33), (4, 3, 17, 12)])
def test_ssim_special_images(shape, kind, record_property):
    _ssim_check(shape, kind, 7 if len(shape) == 3 else 8, record_property)


def test_ssim_many_channels(record_property):
    _ssim_check(ut.SSIM_MANY, "rand", 3, record_property)


# ---- plane regulariser -------------------------------------------------------------------------------------------------------
def _reg_module(args, seed):
    torch.manual_seed(seed)
    mod = g4d.deform_network(args).cuda()
    planes = ut.reg_planes(args, seed)
    with torch.no_grad():
        for lvl_m, lvl_r in zip(mod.deformation_net.grid.grids, planes):
            for p, q in zip(lvl_m, lvl_r):
                p.copy_(q)
    return mod, planes


def _reg_errs(mod, g64, g32, scale=1.0, grads=None):
    worst = 0.0
    gm = grads or [p.grad for lvl in mod.deformation_net.grid.grids for p in lvl]
    i = 0
    for l64, l32 in zip(g64, g32):
        for r64, r32 in zip(l64, l32):
            got = gm[i].detach().double().cpu().numpy()
            i += 1
            e_k, e_32 = ut.texel_err(got, r64 * scale), ut.texel_err(r32 * scale, r64 * scale)
            assert e_k <= ut.REG_K * e_32 + ut.REG_ABS, (i - 1, e_k, e_32)
            worst = max(worst, e_k)
    return worst


@pytest.mark.parametrize("name", list(ut.REG_CONFIGS))
def test_plane_regulation_per_texel(name, record_property):
    args = ut.reg_args(**ut.REG_CONFIGS[name])
    worst = 0.0
    for j, w in enumerate(ut.REG_WEIGHTS):
        mod, planes = _reg_module(args, 3)
        v64, g64 = ut.reg_ref(planes, w, torch.float64, 1.7)
        _, g32 = ut.reg_ref(planes, w, torch.float32, 1.7)
        # compute_regulation: autograd node, upstream 1.7
        loss = losses.compute_regulation(mod, *w)
        (loss * 1.7).backward()
        assert abs(float(loss) * 1.7 - v64 * 1.7) <= 2e-6 * abs(v64 * 1.7) + 1e-12, (w, float(loss), v64)
        worst = max(worst, _reg_errs(mod, g64, g32))
        # accumulate_regulation: twice into zeroed .grad (exactly 2x one call), value into loss_accum
        for p in mod.deformation_net.grid.parameters():
            p.grad = torch.zeros_like(p)
        acc = torch.zeros((), device="cuda")
        losses.accumulate_regulation(mod, *w, loss_accum=acc)
        losses.accumulate_regulation(mod, *w, loss_accum=acc)
        assert abs(float(acc) - 2 * v64) <= 2e-6 * abs(2 * v64) + 1e-12
        worst = max(worst, _reg_errs(mod, g64, g32, scale=2.0 / 1.7))
        # the C-ABI's device upstream scalar
        lib, ws, st = _abi()
        keep = []
        prm = mod.c_params(keep)
        grads = mod.alloc_plane_grads()
        cg = _lib.DeformGrads()
        for k, gk in enumerate(grads):
            cg.planes[k // 6][k % 6] = gk.data_ptr()
        up = torch.tensor(0.3, device="cuda")
        acc.zero_()
        _lib.check(lib.g4d_plane_regulation(ws, C.byref(prm), C.byref(cg), float(w[2]), float(w[0]), float(w[1]), up.data_ptr(),
                                            acc.data_ptr(), st), "g4d_plane_regulation")
        torch.cuda.synchronize()
        assert abs(float(acc) - v64) <= 2e-6 * abs(v64) + 1e-12
        worst = max(worst, _reg_errs(mod, g64, g32, scale=0.3 / 1.7, grads=grads))
    record_property("reg_texel_err", worst)


def test_plane_regulation_refuses_channels_off_a_multiple_of_four():
    mod, _ = _reg_module(ut.reg_args(channels=6), 1)
    with pytest.raises(RuntimeError, match="multiple of 4"):
        losses.compute_regulation(mod, 1e-3, 1e-4, 2e-4)


# ---- flat Adam -----------------------------------------------------------------------------------------------------------------
def _adam_call(bufs, numel, segs, step, gs, shift=0):
    lib, ws, st = _abi()
    arr = (_lib.AdamSegment * max(1, len(segs)))()
    for i, (b, e, lr_) in enumerate(segs):
        arr[i].begin, arr[i].end, arr[i].lr = b, e, lr_
    p, g, m, v = (t.data_ptr() + shift for t in bufs)
    return lib.g4d_adam_step(ws, p, g, m, v, numel, arr, len(segs), ut.ADAM_BETAS[0], ut.ADAM_BETAS[1], ut.ADAM_EPS, step, gs, st)


def _adam_run(numel, segs, steps, gs, seed, warm):
    rng = np.random.default_rng(seed)
    lrs = [float(10.0 ** -rng.uniform(1, 4)) for _ in segs]
    sl = [(b, e, lr_) for (b, e), lr_ in zip(segs, lrs)]
    live = ut.adam_live(numel, segs)
    lr_elem = np.zeros(numel)
    for b, e, lr_ in sl:
        lr_elem[b:e] = np.float32(lr_)
    p = rng.standard_normal(numel).astype(np.float32)
    m = (rng.standard_normal(numel) * 1e-2).astype(np.float32) if warm else np.zeros(numel, np.float32)
    v = (np.abs(rng.standard_normal(numel)) * 1e-3).astype(np.float32) if warm else np.zeros(numel, np.float32)
    bufs = [torch.from_numpy(x.copy()).cuda() for x in (p, np.zeros(numel, np.float32), m, v)]
    for j, step in enumerate(steps):
        g = ut.adam_grads(numel, seed * 100 + j)
        bufs[1].copy_(torch.from_numpy(g))
        prev = [t.cpu().numpy().copy() for t in (bufs[0], bufs[2], bufs[3])]
        _lib.check(_adam_call(bufs, numel, sl, step, gs), "g4d_adam_step")
        torch.cuda.synchronize()
        p1, m1, v1 = (t.cpu().numpy() for t in (bufs[0], bufs[2], bufs[3]))
        for new, old in ((p1, prev[0]), (m1, prev[1]), (v1, prev[2])):        # gaps: bitwise untouched
            assert np.array_equal(new[~live].view(np.uint32), old[~live].view(np.uint32)), step
        em, ev, tm, tv, param = ut.adam_expect(prev[0], g, prev[1], prev[2], lr_elem, step, gs)
        assert (np.abs(m1 - em) <= tm)[live].all(), (step, float(np.max(np.abs(m1 - em) / np.maximum(tm, 1e-300) * live)))
        assert (np.abs(v1 - ev) <= tv)[live].all(), (step, float(np.max(np.abs(v1 - ev) / np.maximum(tv, 1e-300) * live)))
        ep, tp = param(m1, v1)
        assert (np.abs(p1 - ep) <= tp)[live].all(), (step, float(np.max(np.abs(p1 - ep) / tp * live)))
        assert (p1[live] != prev[0][live]).any()


@pytest.mark.parametrize("name", list(ut.ADAM_LAYOUTS))
def test_flat_adam_element_by_element(name):
    numel, segs = ut.ADAM_LAYOUTS[name]
    _adam_run(numel, segs, [1, 2, 3, 4], 1.0 / 3.0, 1, warm=False)
    _adam_run(numel, segs, [100000, 100001], 0.25, 2, warm=True)
    _adam_run(numel, segs, [7], 1.0, 3, warm=True)


def test_flat_adam_refuses_bad_calls_without_a_launch():
    numel = 64
    bufs = [torch.randn(numel + 4, device="cuda") for _ in range(4)]
    before = [t.clone() for t in bufs]
    ok = [(0, 8, 1e-3), (8, 40, 1e-2)]
    assert _adam_call(bufs, numel - 2, ok, 1, 1.0) == G4D_ERR_ARG                                 # numel & 3
    assert _adam_call(bufs, numel, [(i * 3, i * 3 + 2, 1e-3) for i in range(17)], 1, 1.0) == G4D_ERR_ARG   # 17 segments
    assert _adam_call(bufs, numel, [(8, 40, 1e-2), (0, 8, 1e-3)], 1, 1.0) == G4D_ERR_ARG        # unsorted
    assert _adam_call(bufs, numel, [(0, 10, 1e-3), (8, 40, 1e-2)], 1, 1.0) == G4D_ERR_ARG       # overlapping
    for shift in (4, 8, 12):                                                                    # misaligned pointers
        assert _adam_call(bufs, numel, ok, 1, 1.0, shift=shift) == G4D_ERR_ARG
    torch.cuda.synchronize()
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(bufs, before))
    assert _adam_call(bufs, numel, ok, 1, 1.0) == 0                                              # the same call, aligned
    torch.cuda.synchronize()
    assert not torch.equal(bufs[0], before[0])


def _flat_states(seed):
    torch.manual_seed(seed)
    shapes = {"a": [(1001, 3)], "b": [(77,), (5, 3)], "c": [(6, 4, 3, 2)], "d": [(33, 33)], "e": [(3,), (130,)]}
    ps = {k: [torch.nn.Parameter(torch.randn(s, device="cuda")) for s in v] for k, v in shapes.items()}
    qs = {k: [torch.nn.Parameter(p.detach().clone()) for p in v] for k, v in ps.items()}
    dev = torch.device("cuda", 0)
    return td.FlatState(list(ps.items()), dev), td.FlatState(list(qs.items()), dev)


def _state_bits(st):
    return [t.detach().clone().view(torch.int32) for t in (st.param, st.exp_avg, st.exp_avg_sq)]


LRS = {"a": 1.6e-4, "b": 2.5e-3, "c": 5e-2, "d": 1e-3, "e": 1e-2}


def test_flat_state_only_leaves_other_groups_bitwise():
    st, _ = _flat_states(0)
    st.grad.normal_()
    st.adam_step(LRS, grad_scale=0.5)
    st.grad.normal_()
    before = _state_bits(st)
    st.adam_step(LRS, grad_scale=0.5, only=("a", "c", "e"))
    after = _state_bits(st)
    changed = torch.zeros(st.numel, dtype=torch.bool, device="cuda")
    for name in ("a", "c", "e"):
        b, e = st.segments[name]
        changed[b:e] = True
    for x, y in zip(before, after):
        assert torch.equal(x[~changed], y[~changed])
        assert bool((x[changed] != y[changed]).any())


def test_flat_state_four_slice_pipeline_is_bit_identical_to_one_call():
    whole, piped = _flat_states(1)
    k = 4
    chunk = (whole.numel // k + 3) // 4 * 4                       # DPTrainer._launch_allreduce's slices
    spans = [(b, min(whole.numel, b + chunk)) for b in range(0, whole.numel, chunk)]
    assert len(spans) == k and any(whole.segments["a"][0] < b < whole.segments["a"][1] for b, _ in spans[1:])
    g = torch.Generator(device="cuda").manual_seed(5)
    for it in range(4):
        gr = torch.randn(whole.numel, device="cuda", generator=g) * 10.0 ** (it - 2)
        whole.grad.copy_(gr); piped.grad.copy_(gr)
        whole.adam_step(LRS, grad_scale=0.5)
        for i, span in enumerate(spans):
            piped.adam_step(LRS, grad_scale=0.5, span=span, count_step=(i == 0))
        assert whole.step_count == piped.step_count == it + 1
        for x, y in zip(_state_bits(whole), _state_bits(piped)):
            assert torch.equal(x, y), it


# ---- kNN -----------------------------------------------------------------------------------------------------------------------
def _knn_exact(pts):
    got = knn.distCUDA2(torch.from_numpy(pts).cuda()).cpu().numpy()
    want = knn_ref.dist2_knn3_bruteforce(pts)
    bad = int((got != want).sum())
    assert got.shape == want.shape and bad == 0, (bad, len(pts))
    return got


@pytest.mark.parametrize("kind", ut.KNN_KINDS)
def test_knn_degenerate_clouds_bit_exact(kind, record_property):
    pts = ut.knn_cloud(kind)
    got = _knn_exact(pts)
    if kind == "identical":
        assert (got == 0).all()
    if kind == "cluster + outliers":
        x = torch.from_numpy(pts).cuda()
        knn.distCUDA2(x)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record(); knn.distCUDA2(x); t1.record(); torch.cuda.synchronize()
        record_property("knn_cluster_outliers_ms", t0.elapsed_time(t1))


@pytest.mark.parametrize("centre,n", ut.KNN_OFFSETS)
def test_knn_dense_cloud_far_from_the_origin_bit_exact(centre, n):
    _knn_exact(ut.knn_offset_cloud(centre, n))
