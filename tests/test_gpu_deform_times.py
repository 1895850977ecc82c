"""GPU: deform_network with one time per Gaussian (times_sel rows that differ) -- the per-row HexPlane gather and scatter
(g4d_deform_forward_times / _backward_times) against the fp64 oracle, forward and backward including dL/dt; the per-row path at
equal times against the one-time path, bit for bit, on both engines and both gather orders; a trajectory batch over T frames
against T one-time calls; the Python surface of times_sel and the C-ABI's refusals and FP16x2 range flag.

Rows near a ReLU kink or a texel line (the time axis included) are masked from the gradient comparisons, as in
test_gpu_deep_network."""
import ctypes as C
import importlib

import numpy as np
import pytest
import torch

from oracle import deform_ref as dr
from oracle.make_golden_deform import synth_inputs
from util_deep_network import deform_forward, fp64_leaves, oracle_from_module
from util_scene import g4d, make_module, rel_err

pytestmark = pytest.mark.gpu
_lib = importlib.import_module("4dgaussians_b200._lib")
deformation = importlib.import_module("4dgaussians_b200.deformation")

FWD_TOL = 2e-5        # the forward parity tolerance of both engines (test_gpu_parity, test_gpu_deep_network)
GRAD_TOL = 2e-3
WEIGHT_TOL = 3 * GRAD_TOL   # MLP weights through the BF16x2 wgrad of the tensor-core backward
ATOMIC_TOL = 1e-5     # weight and plane gradients summed by atomics in another order
NAMES = ("pts", "scales", "rot", "opacity", "shs")
AABB = torch.tensor([[1.31, 1.27, 1.3], [-1.29, -1.3, -1.22]])


class _Opts:
    """the shared workspace with G4D_OPT_TENSOR_CORES / G4D_OPT_GATHER_ORDER set, restored to their defaults on exit"""

    def __init__(self, tc=2, order=1):
        self.tc, self.order = tc, order

    def __enter__(self):
        self.ws = _lib.Workspace.get(torch.cuda.current_device())
        self.ws.set_option(_lib.OPT_TENSOR_CORES, self.tc)
        self.ws.set_option(_lib.OPT_GATHER_ORDER, self.order)
        return self.ws

    def __exit__(self, *a):
        torch.cuda.synchronize()
        self.ws.set_option(_lib.OPT_TENSOR_CORES, 2)
        self.ws.set_option(_lib.OPT_GATHER_ORDER, 1)


def _module(net, seed=3):
    return make_module(net, seed=seed, aabb=AABB)


def _edge_times(T):
    """rows at 0 and +-1, on time-grid lines, and outside [-1, 1]"""
    lines = [2.0 * k / (T - 1) - 1.0 for k in range(T)]
    return torch.tensor([0.0, 1.0, -1.0, 1.5, -1.5, 7.0, -3.25] + lines, dtype=torch.float32)


def _times(n, T, seed):
    g = torch.Generator().manual_seed(500 + seed)
    t = torch.rand(n, generator=g) * 2.4 - 1.2
    e = _edge_times(T)
    t[:min(n, e.numel())] = e[:min(n, e.numel())]
    return t


def _kink_rows(cfg, prm, trunk, xyz, tt, delta_act=2e-6, delta_grid=2e-4):
    """[N] bool: util_scene.kink_rows / util_deep_network.kink_rows with one time per row -- a HexPlane coordinate (time
    included) within delta_grid texels of a grid line, or a ReLU pre-activation within delta_act of 0, in fp64 on the oracle"""
    with torch.no_grad():
        x64 = xyz.detach().double().cpu()
        t64 = tt.detach().double().cpu().reshape(-1)
        planes = [[p.detach().double() for p in lvl] for lvl in prm.planes]
        aabb = prm.aabb.detach().double()
        q = torch.cat([dr.normalize(x64, aabb), t64.reshape(-1, 1)], dim=-1)
        mask = torch.zeros(x64.shape[0], dtype=torch.bool)
        for lvl in planes:
            for k, (c0, c1) in enumerate(dr.PLANE_AXES):
                _, _, H, W = lvl[k].shape
                for coord, size in ((q[:, c0], W), (q[:, c1], H)):
                    g = (coord + 1.0) / 2.0 * (size - 1)
                    mask |= ((g - torch.round(g)).abs() < delta_grid) & (g > -delta_grid) & (g < size - 1 + delta_grid)
        hidden = dr.hexplane_features(planes, x64, aabb, t64) @ prm.w0.detach().double().t() + prm.b0.detach().double()
        mask |= (hidden.abs() < delta_act).any(dim=1)
        for w, b in trunk:
            hidden = torch.relu(hidden) @ w.detach().double().t() + b.detach().double()
            mask |= (hidden.abs() < delta_act).any(dim=1)
        a = torch.relu(hidden)
        for name in cfg.active_heads():
            w1, b1, _, _ = prm.heads[name]
            mask |= ((a @ w1.detach().double().t() + b1.detach().double()).abs() < delta_act).any(dim=1)
    return mask


def _run(mod, ins, times, probes=None):
    """module forward at times_sel = times (and the backward of <outs, probes>): (outs, input grads, times grad, param grads)"""
    mod.zero_grad(set_to_none=True)
    dev_in = [x.cuda().clone().requires_grad_(probes is not None) for x in ins]
    with torch.set_grad_enabled(probes is not None):
        outs = mod(*dev_in, times)
        if probes is not None:
            torch.autograd.backward(list(outs), [p.cuda().float() for p in probes])
    gi = [x.grad.clone() if x.grad is not None else None for x in dev_in] if probes is not None else None
    gt = times.grad.clone() if torch.is_tensor(times) and times.grad is not None else None
    gp = {k: p.grad.clone() for k, p in mod.named_parameters() if p.grad is not None}
    return [o.detach().clone() for o in outs], gi, gt, gp


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# (net, G4D_OPT_TENSOR_CORES): FFMA at W = 64; the FP16x2 tensor-core forward and its FFMA fallback at W = 128; a depth-3
# trunk; C/4 = 1; C/4 = 3 with L = 3; F = 128
CONFIGS = [("small64", 2), ("small128", 2), ("small128", 0), ("c32w128sh", 2), ("c32w128sh", 0), ("deep128", 2),
           ("c4w64", 2), ("c12w128", 2), ("f128w64", 2)]


@pytest.mark.parametrize("net,tc", CONFIGS)
def test_per_row_forward_and_backward_vs_fp64_oracle(net, tc):
    n = 777
    mod = _module(net)
    cfg, prm, trunk = oracle_from_module(mod)
    ins, probes = synth_inputs(n, 7)
    T = int(mod.args.kplanes_config["resolution"][3])
    tt = _times(n, T, 7)
    kink = _kink_rows(cfg, prm, trunk, ins[0], tt)
    assert float(kink.float().mean()) <= 0.1
    for p in probes:
        p[kink] = 0
    times = tt.cuda().reshape(n, 1).requires_grad_(True)
    with _Opts(tc):
        outs, gi, gt, gp = _run(mod, ins, times, probes)
    p64, tr64 = fp64_leaves(prm, trunk)
    x64 = [v.double().requires_grad_(True) for v in ins]
    t64 = tt.double().requires_grad_(True)
    want = deform_forward(cfg, p64, tr64, *x64, t64)
    torch.autograd.backward(list(want), [p.double() for p in probes])
    for o, w, nm in zip(outs, want, NAMES):
        err = float((o.cpu().double() - w.detach()).abs().max())
        assert err <= FWD_TOL, (net, tc, nm, err)
    for a, b, nm in zip(gi, x64, NAMES):
        if b.grad is not None and a is not None:
            assert rel_err(a.cpu().numpy(), b.grad.numpy()) <= GRAD_TOL, (nm, rel_err(a.cpu().numpy(), b.grad.numpy()))
    g_t = gt.cpu().reshape(-1)
    ok = ~kink
    assert rel_err(g_t[ok].numpy(), t64.grad[ok].numpy()) <= GRAD_TOL, rel_err(g_t[ok].numpy(), t64.grad[ok].numpy())
    clamped = tt.abs() >= 1.0                       # the time coordinate sits on or past the border: ATen's gradient is 0
    assert bool((g_t[clamped] == 0).all()), g_t[clamped]
    net_ = mod.deformation_net
    for l, lvl in enumerate(net_.grid.grids):
        for k, p in enumerate(lvl):
            e = rel_err(p.grad.cpu().numpy(), p64.planes[l][k].grad.numpy())
            assert e <= GRAD_TOL, ("plane", l, k, e)
    pairs = [(net_.feature_out[0].weight, p64.w0), (net_.feature_out[0].bias, p64.b0)]
    for lin, (w, b) in zip(mod.trunk_layers(), tr64):
        pairs += [(lin.weight, w), (lin.bias, b)]
    heads = dict(zip(("pos", "scales", "rotations", "opacity", "shs"), deformation._HEADS))
    for h in cfg.active_heads():
        seq = getattr(net_, heads[h])
        pairs += list(zip((seq[1].weight, seq[1].bias, seq[3].weight, seq[3].bias), p64.heads[h]))
    for p, r in pairs:
        e = rel_err(p.grad.cpu().numpy(), r.grad.numpy())
        assert e <= WEIGHT_TOL, (tuple(p.shape), e)


def _assert_weights_close(gp, want):
    assert sorted(gp) == sorted(want)
    for k in gp:
        scale = max(1e-30, float(want[k].abs().max()))
        assert float((gp[k] - want[k]).abs().max()) <= ATOMIC_TOL * scale, (k, float((gp[k] - want[k]).abs().max()) / scale)


@pytest.mark.parametrize("order", [1, 0])
@pytest.mark.parametrize("net,tc", [("small64", 2), ("small128", 2), ("small128", 0), ("c32w128sh", 2), ("deep128", 2),
                                    ("c12w128", 0)])
def test_uniform_rows_equal_the_one_time_path_bit_for_bit(net, tc, order):
    n, t = 1001, 0.3715
    mod = _module(net)
    ins, probes = synth_inputs(n, 8)
    with _Opts(tc, order):
        ref = _run(mod, ins, torch.full((n, 1), t, device="cuda"), probes)            # uniform, no grad: one-time path
        times = torch.full((n, 1), t, device="cuda", requires_grad=True)               # requires grad: the per-row path
        got = _run(mod, ins, times, probes)
    for a, b, nm in zip(got[0], ref[0], NAMES):
        assert _bits_equal(a, b), nm
    for a, b, nm in zip(got[1], ref[1], NAMES):
        assert (a is None) == (b is None) and (a is None or _bits_equal(a, b)), nm
    assert got[2] is not None and got[2].shape == (n, 1) and ref[2] is None
    _assert_weights_close(got[3], ref[3])


@pytest.mark.parametrize("net,tc", [("small64", 2), ("small128", 2), ("small128", 0), ("c32w128sh", 2)])
def test_trajectory_batch_equals_one_call_per_frame(net, tc):
    n, frames = 301, torch.tensor([-0.9, -0.2, 0.35, 0.8, 1.0])
    T = frames.numel()
    mod = _module(net)
    ins, probes = synth_inputs(n, 9)
    with _Opts(tc):
        per_frame = [_run(mod, ins, torch.full((n, 1), float(t), device="cuda"), probes) for t in frames]
        want_w = {k: sum(r[3][k] for r in per_frame) for k in per_frame[0][3]}
        big_in = [x.repeat((T,) + (1,) * (x.dim() - 1)) for x in ins]
        big_pr = [p.repeat((T,) + (1,) * (p.dim() - 1)) for p in probes]
        times = frames.repeat_interleave(n).cuda()
        got = _run(mod, big_in, times, big_pr)
    for i, nm in enumerate(NAMES):
        assert _bits_equal(got[0][i], torch.cat([r[0][i] for r in per_frame])), nm
        if got[1][i] is not None:
            assert _bits_equal(got[1][i], torch.cat([r[1][i] for r in per_frame])), nm
    _assert_weights_close(got[3], want_w)


def test_times_sel_layouts_dtypes_and_devices_give_the_same_bits():
    n = 513
    mod = _module("small128")
    ins, _ = synth_inputs(n, 10)
    tt = (torch.arange(n) % 3 - 1).float()          # -1, 0, 1: exact in every dtype below
    ref = _run(mod, ins, tt.cuda().reshape(n, 1))[0]
    for times in (tt.cuda(), tt.double().cuda().reshape(n, 1), tt.long().cuda(), tt.reshape(n, 1), tt.double(), tt.long()):
        got = _run(mod, ins, times)[0]
        for a, b, nm in zip(got, ref, NAMES):
            assert _bits_equal(a, b), (times.dtype, times.device, tuple(times.shape), nm)


def test_uniform_times_that_require_grad_get_dl_dt_in_their_own_shape_dtype_and_device():
    n = 200
    mod = _module("small64")
    ins, probes = synth_inputs(n, 11)
    ref = _run(mod, ins, 0.25, probes)
    for times in (torch.full((n,), 0.25, dtype=torch.float64, requires_grad=True),
                  torch.full((n, 1), 0.25, device="cuda", requires_grad=True)):
        got = _run(mod, ins, times, probes)
        for a, b, nm in zip(got[0], ref[0], NAMES):
            assert _bits_equal(a, b), nm
        assert got[2] is not None and got[2].shape == times.shape and got[2].dtype == times.dtype
        assert got[2].device == times.device and bool(torch.isfinite(got[2]).all())


def test_a_wrong_element_count_is_refused_before_any_launch(monkeypatch):
    n = 64
    mod = _module("small64")
    x = torch.zeros(n, 3, device="cuda")

    def no_launch():
        raise AssertionError("the library was called")
    monkeypatch.setattr(_lib, "load", no_launch)
    for times in (torch.linspace(0, 1, n + 1, device="cuda"), torch.linspace(0, 1, n - 1),
                  torch.full((n + 3,), 0.5, requires_grad=True)):
        with pytest.raises(ValueError, match="times_sel"):
            mod(x, None, None, None, None, times)


def _oracle_dt(mod, ins, probes, tt):
    """fp64 oracle of <outs, probes>, the probes of rows near a kink zeroed (in place): (dL/dt, dL/d(xyz), kink mask)"""
    cfg, prm, trunk = oracle_from_module(mod)
    kink = _kink_rows(cfg, prm, trunk, ins[0], tt)
    for p in probes:
        p[kink] = 0
    p64, tr64 = fp64_leaves(prm, trunk)
    t64 = tt.double().requires_grad_(True)
    x64 = ins[0].double().requires_grad_(True)
    want = deform_forward(cfg, p64, tr64, x64, *[v.double() for v in ins[1:]], t64)
    live = [(o, p.double()) for o, p in zip(want, probes) if o.requires_grad]   # (inactive heads pass inputs through)
    torch.autograd.backward([o for o, _ in live], [p for _, p in live])
    return t64.grad, x64.grad, kink


@pytest.mark.parametrize("n", [0, 1, 63, 65, 191, 193])
def test_row_counts_off_every_tile(n):
    """per-row calls at N off every tile size (FFMA 128 / 64 / 32, tensor-core 128 / 192, gather and scatter blocks): the first
    and the last rows -- those past the last full tile -- against the one-time path at each row's time, outputs and input
    gradients bit for bit; dL/dt against the fp64 oracle, and on those rows bit for bit equal to the same rows at other positions
    of the tiles (a call over the rows twice).  N = 1 is a one-element times_sel, the one-time path itself."""
    mod = _module("small128")
    ins, probes = synth_inputs(n, 12)
    tt = _times(n, 8, 12) if n else torch.zeros(0)
    want_dt, _, kink = _oracle_dt(mod, ins, probes, tt) if n > 1 else (None, None, None)
    rows = sorted({i for i in (0, 1, n - 2, n - 1) if 0 <= i < n})
    for tc in (2, 0):
        with _Opts(tc):
            times = tt.cuda().reshape(n, 1).requires_grad_(True)
            got = _run(mod, ins, times, probes)
            for o, x in zip(got[0], ins):
                assert o.shape == x.shape
            for i in rows:
                ref = _run(mod, [x[i:i + 1] for x in ins], float(tt[i]), [p[i:i + 1] for p in probes])
                for a, b, nm in zip(got[0], ref[0], NAMES):
                    assert _bits_equal(a[i:i + 1], b), (n, tc, i, nm)
                for a, b, nm in zip(got[1], ref[1], NAMES):
                    assert (a is None) == (b is None) and (a is None or _bits_equal(a[i:i + 1], b)), (n, tc, i, nm)
            if n == 1:
                assert got[2] is None
                continue
            assert got[2] is not None and got[2].shape == (n, 1)
            if n == 0:
                continue
            g_t = got[2].reshape(-1)
            ok = ~kink
            assert rel_err(g_t.cpu()[ok].numpy(), want_dt[ok].numpy()) <= GRAD_TOL, (n, tc)
            twice = torch.cat([tt, tt]).cuda().requires_grad_(True)
            g2 = _run(mod, [torch.cat([x, x]) for x in ins], twice, [torch.cat([p, p]) for p in probes])[2]
            for i in rows:                  # row i sits at i and at n + i: two positions in every tile size
                assert _bits_equal(g_t[i:i + 1], g2[i:i + 1]) and _bits_equal(g_t[i:i + 1], g2[n + i:n + i + 1]), (n, tc, i)


@pytest.mark.parametrize("tc", [2, 0])
def test_dl_dt_is_exactly_zero_on_and_past_the_time_border(tc):
    """gmul_t = 0 where the time coordinate is clamped, the border itself included (ATen's clip_coordinates_set_grad): rows at
    exactly +-1 and past it get dL/dt = 0 with every probe live; rows just inside get a gradient"""
    n = 400
    mod = _module("small128")
    ins, probes = synth_inputs(n, 14)
    border = torch.tensor([1.0, -1.0, 1.5, -7.0])
    inside = torch.tensor([0.999, -0.999])
    tt = torch.cat([border.repeat(n // 8), inside.repeat(n // 4)])
    with _Opts(tc):
        times = tt.cuda().reshape(n, 1).requires_grad_(True)
        g_t = _run(mod, ins, times, probes)[2].cpu().reshape(-1)
    on = tt.abs() >= 1.0
    assert int(on.sum()) == n // 2 and bool((g_t[on] == 0).all()), g_t[on][g_t[on] != 0]
    assert float((g_t[~on] != 0).float().mean()) > 0.9


@pytest.mark.parametrize("net,tc", [("small128", 2), ("small128", 0), ("small64", 2)])
def test_second_backward_through_a_retained_graph_runs_at_the_per_row_times(net, tc):
    """two torch.autograd.grad calls through one per-row forward (retain_graph=True): both against the fp64 oracle (dL/dt and
    d(xyz)).  On the FFMA engine, which derives its ReLU signs in every backward, the two are equal: the per-row gradients bit
    for bit, the weight and plane gradients within the atomics' reordering.  (The tensor-core backward reads the signs the
    forward saved once, and recomputes them in a second backward, as on the one-time path.)"""
    n = 700
    mod = _module(net)
    ins, probes = synth_inputs(n, 15)
    tt = _times(n, int(mod.args.kplanes_config["resolution"][3]), 15)
    want_dt, want_dx, kink = _oracle_dt(mod, ins, probes, tt)
    with _Opts(tc):
        x = ins[0].cuda().clone().requires_grad_(True)
        times = tt.cuda().reshape(n, 1).requires_grad_(True)
        outs = mod(x, *[v.cuda() for v in ins[1:]], times)
        live = [(o, p.cuda().float()) for o, p in zip(outs, probes) if o.requires_grad]   # (inactive heads pass inputs through)
        outs, cot = [o for o, _ in live], [c for _, c in live]
        leaves = [x, times] + [p for p in mod.parameters() if p.requires_grad]
        first = torch.autograd.grad(outs, leaves, cot, retain_graph=True, allow_unused=True)
        second = torch.autograd.grad(outs, leaves, cot, allow_unused=True)
    ok = ~kink
    for g in (first, second):
        assert rel_err(g[1].cpu().reshape(-1)[ok].numpy(), want_dt[ok].numpy()) <= GRAD_TOL
        assert rel_err(g[0].cpu().numpy(), want_dx.numpy()) <= GRAD_TOL
    if tc == 0 or net == "small64":
        assert _bits_equal(first[0], second[0]) and _bits_equal(first[1], second[1])
        for a, b in zip(first[2:], second[2:]):
            assert (a is None) == (b is None)
            if a is not None:
                assert float((a - b).abs().max()) <= ATOMIC_TOL * max(1e-30, float(a.abs().max()))


def test_times_changed_in_place_before_the_backward_are_refused():
    n = 300
    mod = _module("small64")
    ins, probes = synth_inputs(n, 16)
    times = _times(n, 7, 16).cuda().reshape(n, 1).requires_grad_(True)
    t = times.detach()          # the caller's storage, as the per-row path reads it
    x = ins[0].cuda().clone().requires_grad_(True)
    outs = mod(x, *[v.cuda() for v in ins[1:]], times)
    t.add_(0.25)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        torch.autograd.backward(outs[0], probes[0].cuda().float())


def _abi_rc(fn_name, use_null):
    lib = _lib.load()
    mod = _module("small64")
    keep = []
    prm = mod.c_params(keep)
    n = 64
    x = torch.zeros(n, 3, device="cuda")
    tt = torch.zeros(n, device="cuda")
    out = torch.full((n, 3), 7.0, device="cuda")
    ws = _lib.Workspace.get(torch.cuda.current_device())
    st = _lib.stream_of(x.device)
    d_times = None if use_null else tt.data_ptr()
    if fn_name == "forward":
        rc = lib.g4d_deform_forward_times(ws.handle, C.byref(prm), n, x.data_ptr(), None, None, None, None, d_times,
                                          out.data_ptr(), None, None, None, None, None, st)
    else:
        grads = mod.alloc_grads()
        cg = mod.c_grads(grads)
        g_t = torch.full((n,), 7.0, device="cuda")
        go = torch.ones(n, 3, device="cuda")
        rc = lib.g4d_deform_backward_times(ws.handle, C.byref(prm), C.byref(cg), n, x.data_ptr(), d_times, go.data_ptr(),
                                           None, None, None, None, out.data_ptr(), None, None, None, None, g_t.data_ptr(),
                                           None, st)
        out = torch.cat([out.reshape(-1), g_t])
    torch.cuda.synchronize()
    return rc, lib.g4d_last_error().decode(), bool((out == 7.0).all())


def test_c_abi_refuses_null_times_before_any_launch():
    for which in ("forward", "backward"):
        ok = _abi_rc(which, False)
        assert ok[0] == 0, ok
        rc, msg, untouched = _abi_rc(which, True)
        assert rc == -2 and "d_times" in msg and untouched, (which, rc, msg)


def test_per_row_forward_that_leaves_the_fp16x2_range_is_flagged_on_the_next_call():
    n = 256
    mod = _module("small128")
    with torch.no_grad():
        mod.deformation_net.feature_out[0].weight[5].zero_()          # a1[5] = b0[5] exactly: past 65504 / 8
        mod.deformation_net.feature_out[0].bias[5] = 8188.0
    mod.invalidate_cache()
    ins, _ = synth_inputs(n, 13)
    ins = [x.cuda() for x in ins]
    times = _times(n, 8, 13).cuda()
    with _Opts(2), torch.no_grad():
        mod(*ins, times)
        torch.cuda.synchronize()
        with pytest.raises(_lib.G4DError, match="f16 operand range"):
            mod(*ins, times)
