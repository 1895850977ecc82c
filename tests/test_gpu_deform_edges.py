"""GPU: the deformation network's kernels on the edge scenes of util_deform_edges -- the HexPlane gather and scatter at faces,
outside the AABB and at NaN / inf, the time-row collapse and distribution at the ends of the time axis, plane values that are
zero, negative or span 1e-6 .. 1e2, one texel hit by 65536 Gaussians, the FP16x2 operand range on both sides of its limits,
tile tails of every engine, partial upstream gradients, and gradient sinks the scatter cannot take.

Engines: forward FFMA (G4D_OPT_TENSOR_CORES = 0) at net_width 64 and 128 and FP16x2 (2); backward FFMA and BF16x2
(the tensor-core backward, after the tensor-core forward).  The scenes' cells are exact in fp32 and fp64, so only rows near a
ReLU kink are masked (util_deep_network.kink_rows with the texel-line test off)."""
import ctypes as C
import importlib

import numpy as np
import pytest
import torch

import util_deform_edges as ue
from util_deep_network import deform_forward, fp64_leaves, kink_rows, oracle_from_module
from util_scene import g4d, row_err, synth

pytestmark = pytest.mark.gpu
_lib = importlib.import_module("4dgaussians_b200._lib")
dp = importlib.import_module("4dgaussians_b200.dp")
losses = importlib.import_module("4dgaussians_b200.losses")

FWD_TOL = 2e-5
GRAD_TOL = 2e-3
WEIGHT_TOL = 3 * GRAD_TOL          # weights through the BF16x2 wgrad (test_tensor_core_paths_corner_cases_vs_oracle)
NAMES = ("pts", "scales", "rot", "opacity", "shs")
F16_LIMIT = "f16 operand range"

# (net, tensor-core mode): the three (C, L) the tensor-core kernels take at W = 128 with every head, the FFMA kernels at W = 64,
# a half-tile FFMA configuration (L = 3, C = 20, all heads) and a D = 2 trunk
TC_NETS = [ue.Net("small128", ue.RES[0]), ue.Net("small128", ue.RES[1], (1, 2, 4)), ue.Net("c32w128sh", ue.RES[2])]
FFMA_NETS = [ue.Net("small64", ue.RES[1]), ue.Net("c20w128sh", ue.RES[0], (1, 2, 4)), ue.Net("deep64", ue.RES[2], depth=2)]
ENGINES = [(n, 0) for n in TC_NETS + FFMA_NETS] + [(n, 2) for n in TC_NETS]
SEEN = {}                          # worst row error per case group (printed with -s; DESIGN.md §4.4 quotes one run)


def _note(group, e):
    SEEN[group] = max(SEEN.get(group, 0.0), float(e))
    print("\n[deform-edges] %-12s worst %.3g" % (group, SEEN[group]))


class _Mode:
    def __init__(self, tc):
        self.tc = tc

    def __enter__(self):
        self.ws = _lib.Workspace.get(torch.cuda.current_device())
        self.ws.set_option(_lib.OPT_TENSOR_CORES, self.tc)
        return self.ws

    def __exit__(self, *a):
        torch.cuda.synchronize()
        self.ws.set_option(_lib.OPT_TENSOR_CORES, 2)


def _run(mod, ins, probes, t, tc, backward=True):
    """module forward (and backward of <outs, probes>) at time t on engine tc: (outs, input grads, {param: grad})"""
    n = ins[0].shape[0]
    mod.zero_grad(set_to_none=True)
    with _Mode(tc):
        dev_in = [x.cuda().clone().requires_grad_(backward) for x in ins]
        with torch.set_grad_enabled(backward):
            outs = mod(*dev_in, torch.tensor(float(t)).repeat(n, 1).cuda())
        if backward:
            torch.autograd.backward(list(outs), [p.cuda() for p in probes])
    outs = [o.detach().cpu() for o in outs]
    gi = [x.grad.cpu() if backward else None for x in dev_in]
    gp = {k: p.grad.cpu() for k, p in mod.named_parameters() if p.grad is not None}
    return outs, gi, gp


def _oracle(mod, ins, probes, t, backward=True):
    cfg, prm, trunk = oracle_from_module(mod)
    p64, tr64 = fp64_leaves(prm, trunk)
    x = [v.double().requires_grad_(backward) for v in ins]
    outs = deform_forward(cfg, p64, tr64, *x, float(t))
    if backward:
        torch.autograd.backward(list(outs), [p.double() for p in probes])
    return cfg, prm, trunk, p64, tr64, [o.detach() for o in outs], [v.grad for v in x]


def _mask_kinks(mod, ins, probes, t):
    """zero the upstream gradient of rows with a ReLU pre-activation within rounding of 0 (no texel-line masking)"""
    cfg, prm, trunk = oracle_from_module(mod)
    xyz = ins[0].clone()
    xyz[~torch.isfinite(xyz)] = 0.0
    kink = kink_rows(cfg, prm, trunk, xyz, t, delta_grid=-1.0)
    assert float(kink.float().mean()) <= 0.1
    probes = [p.clone() for p in probes]
    for p in probes:
        p[kink] = 0
    return probes


def _fwd_err(got, ref):
    """per row: max |got - ref| / max(1, max |ref|) -- the existing absolute 2e-5 at unit scale, relative beyond"""
    g, r = got.double().reshape(got.shape[0], -1), ref.double().reshape(ref.shape[0], -1)
    return float(((g - r).abs().max(dim=1).values / r.abs().max(dim=1).values.clamp_min(1.0)).max())


def _param_pairs(mod, p64, tr64):
    """[(name, kernel gradient, fp64 oracle gradient)] of every parameter with a gradient"""
    net = mod.deformation_net
    out = []
    for l, lvl in enumerate(net.grid.grids):
        for k, p in enumerate(lvl):
            out.append(("plane%d.%d" % (l, k), p, p64.planes[l][k]))
    out += [("w0", net.feature_out[0].weight, p64.w0), ("b0", net.feature_out[0].bias, p64.b0)]
    for lin, (w, b) in zip(mod.trunk_layers(), tr64):
        out += [("wt", lin.weight, w), ("bt", lin.bias, b)]
    heads = dict(zip(("pos", "scales", "rotations", "opacity", "shs"),
                     ("pos_deform", "scales_deform", "rotations_deform", "opacity_deform", "shs_deform")))
    for h, key in heads.items():
        seq = getattr(net, key)
        out += [(h + n, q, r) for n, q, r in zip(("w1", "b1", "w2", "b2"), (seq[1].weight, seq[1].bias, seq[3].weight,
                                                                          seq[3].bias), p64.heads[h])]
    return out


def _magnitudes(mod, ins, probes, t):
    """the fp64 network with every weight, bias, plane, input and probe replaced by its absolute value: per row, a bound on
    the magnitude of every term the outputs and input gradients sum (ReLU passes non-negative values unchanged)"""
    cfg, prm, trunk = oracle_from_module(mod)
    p64, tr64 = fp64_leaves(prm, trunk)
    with torch.no_grad():
        for q in p64.leaves() + [x for wb in tr64 for x in wb]:
            q.abs_()
    x = [v.double().requires_grad_(True) if i == 0 else v.double().abs().requires_grad_(True) for i, v in enumerate(ins)]
    outs = deform_forward(cfg, p64, tr64, *x, float(t))
    torch.autograd.backward(list(outs), [p.double().abs() for p in probes])
    return [o.detach() for o in outs], [v.grad.abs() for v in x]


def _scaled_err(got, ref, mag):
    """per row: max |got - ref| / max(max |ref|, max mag, 1e-30)"""
    g, r, m = (np.asarray(v, np.float64).reshape(v.shape[0], -1) for v in (got, ref, mag))
    scale = np.maximum(np.maximum(np.abs(r).max(axis=1), np.abs(m).max(axis=1)), 1e-30)
    return float((np.abs(g - r).max(axis=1) / scale).max())


def _check_vs_oracle(mod, ins, probes, t, tc, group, backward=True, conditioned=False):
    """forward and backward against fp64, per Gaussian.  conditioned: errors relative to _magnitudes (planes whose values
    span 1e-6 .. 1e2 make sums whose terms cancel by many orders of magnitude; fp32 is then exact to its rounding of the
    terms, not of the result)"""
    if backward:
        probes = _mask_kinks(mod, ins, probes, t)
    outs, gi, _ = _run(mod, ins, probes, t, tc, backward)
    _, _, _, p64, tr64, want, wgi = _oracle(mod, ins, probes, t, backward)
    mag = _magnitudes(mod, ins, probes, t) if conditioned else None
    for i, (o, w, nm) in enumerate(zip(outs, want, NAMES)):
        e = _scaled_err(o, w, mag[0][i]) if conditioned else _fwd_err(o, w)
        assert e <= FWD_TOL, (group, nm, e)
        _note(group + "/fwd", e)
    if not backward:
        return outs, gi
    for i, (a, b, nm) in enumerate(zip(gi, wgi, ("xyz",) + NAMES[1:])):
        if conditioned:
            e, worst = _scaled_err(a, b, mag[1][i]), [None, None]
        else:
            e, worst = row_err(a.numpy(), b.numpy())
        assert e <= GRAD_TOL, (group, nm, e, worst[:2])
        _note(group + "/grad", e)
    for nm, p, r in _param_pairs(mod, p64, tr64):
        if r.grad is None or float(r.grad.abs().max()) == 0.0:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, nm
            continue
        a, b = p.grad.cpu().double().numpy(), r.grad.numpy()
        e = float(np.abs(a - b).max() / np.abs(b).max())
        assert e <= (GRAD_TOL if nm.startswith("plane") else WEIGHT_TOL), (group, nm, e)
    return outs, gi


# --------------------------------------------------------------------------------------------------- faces and planes
@pytest.mark.parametrize("net,tc", ENGINES, ids=lambda v: v.name if isinstance(v, ue.Net) else str(v))
@pytest.mark.parametrize("kind", ["default", "zero", "negative", "wide"])
def test_faces_and_plane_values_vs_oracle(net, tc, kind):
    """faces, one ulp inside them, outside, edges, corners, the last texel, res = 2 axes: forward and backward per Gaussian
    against fp64.  A face row takes no coordinate gradient from the planes: d(xyz) there is the residual's alone, bit for
    bit.  (wide planes leave the FP16x2 range: they run on the FFMA forward.)"""
    if kind == "wide" and tc == 2:
        pytest.skip("features up to 1e12 are outside the FP16x2 operand range by design")
    mod = ue.make_edge_module(net, seed=3)
    if kind != "default":
        ue.set_planes(mod, kind, seed=4)
    sc = ue.face_scene()
    ins, probes = ue.inputs(sc.xyz, seed=7)
    probes = _mask_kinks(mod, ins, probes, 0.25)
    _, gi = _check_vs_oracle(mod, ins, probes, 0.25, tc, "faces" if kind == "default" else "planes-" + kind,
                             conditioned=kind == "wide")
    for row, a, claim in sc.claims:
        if claim != ue.INSIDE:
            assert gi[0][row, a] == probes[0][row, a], (row, a, claim)


@pytest.mark.parametrize("tc", [0, 2])
def test_corner_gradients_land_on_border_texels_only(tc):
    net = ue.Net("small128", ue.RES[0])
    mod = ue.make_edge_module(net, seed=3)
    corners = np.array([[1.0 if (s >> a) & 1 else -1.0 for a in range(3)] for s in range(8)], np.float32)
    ins, probes = ue.inputs(corners, seed=2)
    _run(mod, ins, probes, 0.25, tc)
    for l, lvl in enumerate(mod.deformation_net.grid.grids):
        for k, p in enumerate(lvl):
            if k in (2, 4, 5):
                continue                       # time planes: t = 0.25 is interior
            g = p.grad.abs().sum(dim=(0, 1)).cpu()         # [H, W]
            inner = g.clone()
            inner[[0, -1], :] = 0
            inner[:, [0, -1]] = 0
            assert float(g.max()) > 0 and float(inner.max()) == 0.0, (l, k)
            if g.shape[0] > 2 and g.shape[1] > 2:
                assert float(g[1:-1].max()) == 0.0 and float(g[:, 1:-1].max()) == 0.0, (l, k)


# --------------------------------------------------------------------------------------------------- NaN and inf
@pytest.mark.parametrize("net,tc", ENGINES, ids=lambda v: v.name if isinstance(v, ue.Net) else str(v))
def test_nan_and_inf_coordinates_behave_as_their_faces(net, tc):
    """kernel-defined behaviour: make_tap's fmaxf drops a NaN, so a NaN coordinate samples the xyz_max face, +inf too and -inf
    the xyz_min face.  Every output but the deformed position (NaN + delta) and every per-Gaussian input gradient equals the
    twin row's bit for bit, and every gradient is finite."""
    mod = ue.make_edge_module(net, seed=5)
    sc = ue.nonfinite_scene()
    ins, probes = ue.inputs(sc.xyz, seed=9)
    for i, j in sc.twins:
        for v in ins[1:] + probes:
            v[i] = v[j]
    outs, gi, gp = _run(mod, ins, probes, 0.25, tc)
    for (i, j), (row, a, claim) in zip(sc.twins, [c for c in sc.claims if c[2] in (ue.NAN, ue.POS_INF, ue.NEG_INF)]):
        assert row == i
        for o, nm in zip(outs, NAMES):
            if nm == "pts":
                other = [b for b in range(3) if b != a]
                assert torch.equal(o[i, other], o[j, other]) and not torch.isfinite(o[i, a]), (i, nm)
            else:
                assert torch.equal(o[i], o[j]), (i, nm, claim)
        for g in gi:
            assert torch.equal(g[i], g[j]), (i, claim)
    assert all(bool(torch.isfinite(g).all()) for g in gi)
    assert all(bool(torch.isfinite(g).all()) for g in gp.values())


# --------------------------------------------------------------------------------------------------- time
@pytest.mark.parametrize("net,tc", [(ue.Net("small128", r), tc) for r in ue.RES for tc in (0, 2)] +
                         [(ue.Net("small64", ue.RES[1]), 0)], ids=lambda v: v.name if isinstance(v, ue.Net) else str(v))
def test_time_ends_and_lines(net, tc):
    """t at 0 (the centre row, a texel line for odd T), 1 (the last row, i0 == i1), beyond both ends, and on a line away from
    the centre with its neighbours: forward, input and parameter gradients against fp64, and the time planes' gradients
    (the collapse and the distribution of the time rows) row by row.  At t >= 1 and t <= -1 every time-plane gradient lies
    on the one clamped row."""
    mod = ue.make_edge_module(net, seed=6)
    T = net.res[3]
    sc = ue.tile_scene(300, seed=4)
    for t in ue.TIME_ENDS + ue.TIME_LINE:
        ins, probes = ue.inputs(sc.xyz, seed=11)
        probes = _mask_kinks(mod, ins, probes, t)
        _check_vs_oracle(mod, ins, probes, t, tc, "time")
        _, _, _, p64, _, _, _ = _oracle(mod, ins, probes, t)
        for l, lvl in enumerate(mod.deformation_net.grid.grids):
            for k in (2, 4, 5):
                got = lvl[k].grad.cpu().double()[0].permute(1, 0, 2).numpy()       # [T, C, W]: one row per time texel
                ref = p64.planes[l][k].grad[0].permute(1, 0, 2).numpy()
                e, worst = row_err(got, ref)
                assert e <= GRAD_TOL, (t, l, k, e, worst[:1])
                _note("time-rows", e)
                if t >= 1.0 or t <= -1.0:
                    row = T - 1 if t >= 1.0 else 0
                    assert np.abs(np.delete(got, row, axis=0)).max() == 0.0 and np.abs(got[row]).max() > 0, (t, l, k)


# --------------------------------------------------------------------------------------------------- hot texel
def _plane_grads(mod):
    return [p.grad.cpu().double().numpy() for lvl in mod.deformation_net.grid.grids for p in lvl]


def test_hot_texel_vs_fp64():
    """65536 Gaussians at one point, each with its own inputs and upstream gradients (FFMA engine): every plane gradient is
    one fp32 sum of 65536 red.global.add contributions; it must match the fp64 sum to n 2^-24 relative, the worst case of fp32
    accumulation"""
    mod = ue.make_edge_module(ue.Net("small128", ue.RES[0]), seed=8)
    sc = ue.hot_scene()
    n = sc.xyz.shape[0]
    ins, probes = ue.inputs(sc.xyz, seed=13)
    _run(mod, ins, probes, 0.25, 0)
    _, _, _, p64, _, _, _ = _oracle(mod, ins, probes, 0.25)
    ref = [p.grad.numpy() for lvl in p64.planes for p in lvl]
    worst = max(float(np.abs(a - b).max() / np.abs(b).max()) for a, b in zip(_plane_grads(mod), ref))
    assert worst <= n * 2.0 ** -24, worst
    _note("hot-texel-fp64", worst)


@pytest.mark.parametrize("tc", [0, 2])
def test_hot_texel_accumulation(tc):
    """65536 copies of ONE Gaussian (same inputs, same upstream gradient): every copy adds the same contribution c to a texel,
    so the engine's own c is its plane gradient at n = 1 (checked against fp64 there, which covers the BF16x2 dgrad's error),
    and at n = 65536 the red.global.add sum must equal n c to n 2^-24 relative (no cancellation: every term is c), plus one
    rounding of the time-row distribution's weight"""
    mod = ue.make_edge_module(ue.Net("small128", ue.RES[0]), seed=8)
    sc = ue.hot_scene()
    n = sc.xyz.shape[0]
    ins1, probes1 = ue.inputs(sc.xyz[:1], seed=13)
    _run(mod, ins1, probes1, 0.25, tc)
    g1 = _plane_grads(mod)
    _, _, _, p64, _, _, _ = _oracle(mod, ins1, probes1, 0.25)
    for a, b in zip(g1, [p.grad.numpy() for lvl in p64.planes for p in lvl]):
        assert float(np.abs(a - b).max() / np.abs(b).max()) <= GRAD_TOL
    rep = lambda ts: [t.expand((n,) + tuple(t.shape[1:])).contiguous() for t in ts]
    _run(mod, rep(ins1), rep(probes1), 0.25, tc)
    worst = 0.0
    for gn, c in zip(_plane_grads(mod), g1):
        want = n * c                                        # exact: n is a power of two
        assert np.all(np.abs(gn - want) <= (n * 2.0 ** -24 + 2.0 ** -23) * np.abs(want)), float(np.abs(gn - want).max())
        nz = want != 0
        assert np.array_equal(gn != 0, nz)
        worst = max(worst, float((np.abs(gn - want)[nz] / np.abs(want)[nz]).max()))
    _note("hot-texel-tc%d" % tc, worst)


# --------------------------------------------------------------------------------------------------- FP16x2 range
def _fp16_case(edit):
    """(module, inputs) of small128 on the edge AABB with edit(mod) applied"""
    mod = ue.make_edge_module(ue.Net("small128", ue.RES[0]), seed=9)
    edit(mod)
    mod.invalidate_cache()
    ins, _ = ue.inputs(ue.tile_scene(200, seed=8).xyz, seed=3)
    return mod, [x.cuda() for x in ins]


def _b0_edit(v):
    def f(mod):
        with torch.no_grad():
            mod.deformation_net.feature_out[0].weight[5].zero_()          # a1[5] = b0[5] exactly
            mod.deformation_net.feature_out[0].bias[5] = v
    return f


def _sh_b1_edit(v):
    def f(mod):
        with torch.no_grad():
            mod.deformation_net.shs_deform[1].weight[7].zero_()          # a2[7] of the SH head = b1[7] exactly
            mod.deformation_net.shs_deform[1].bias[7] = v
    return f


def _w1_edit(v):
    def f(mod):
        with torch.no_grad():
            mod.deformation_net.pos_deform[1].weight[0, 0] = v
    return f


def _feature_edit(v):
    return lambda mod: ue.set_uniform_planes(mod, v)


BELOW = float(np.nextafter(np.float32(8188.0), np.float32(0)))
FP16_CASES = {                     # name: (edit, flagged)
    "feature_1023.5": (_feature_edit(1023.5), True), "feature_1023.4": (_feature_edit(1023.4), False),
    "a1_8188": (_b0_edit(8188.0), True), "a1_below": (_b0_edit(BELOW), False),
    "a2_8188": (_sh_b1_edit(8188.0), True), "a2_below": (_sh_b1_edit(BELOW), False),
    "w1_255.875": (_w1_edit(255.875), True), "w1_255.8": (_w1_edit(255.8), False),
}


@pytest.mark.parametrize("name", sorted(FP16_CASES))
def test_fp16x2_range_on_both_sides_of_each_limit(name):
    """s |x| >= 65504 raises the flag (features s = 2^6, activations 2^3, weights 2^8): the NEXT call reports it.  Just below
    the limit the FP16x2 forward matches the FFMA forward to 5e-6 and no flag is raised."""
    edit, flagged = FP16_CASES[name]
    mod, ins = _fp16_case(edit)
    n = ins[0].shape[0]
    t = torch.tensor(0.25).repeat(n, 1).cuda()
    ws = _lib.Workspace.get(0)
    try:
        with torch.no_grad():
            ws.set_option(_lib.OPT_TENSOR_CORES, 0)
            ref = [o.clone() for o in mod(*ins, t)]
            ws.set_option(_lib.OPT_TENSOR_CORES, 2)
            got = [o.clone() for o in mod(*ins, t)]
            torch.cuda.synchronize()
            if flagged:
                with pytest.raises(_lib.G4DError, match=F16_LIMIT):
                    mod(*ins, t)
            else:
                mod(*ins, t)                    # no flag from the first call
                torch.cuda.synchronize()
                for x, y, nm in zip(got, ref, NAMES):
                    e = float((x - y).abs().max() / max(1.0, float(y.abs().max())))
                    assert e <= 5e-6, (name, nm, e)
                    _note("fp16-range", e)
    finally:
        ws.set_option(_lib.OPT_TENSOR_CORES, 2)


def test_fp16x2_tiny_features_within_the_absolute_floor():
    """features in [1e-9, 1.8e-9], where the FP16x2 split's absolute floor 2^-25 / 2^6 ~ 4.7e-10 is a large part of each
    feature.  The network makes every feature visible: all biases 0, every weight positive (no cancellation, no ReLU kink),
    W0 ~ 225 so the activations stay far above their own floor 2^-25 / 2^3, and zero residual inputs, so each output is the
    network's delta alone (~0.1).  The FP16x2 forward must match the FFMA forward to the error bound propagated from
    max(2^-22 |x|, 2^-25 / s) of every split operand (features, activations, weights) through |W0|, |W1|, |W2|, plus both
    engines' fp32 accumulation; and that bound must be tighter than what dropping the features would cost."""
    from oracle import deform_ref as dr
    u = 2.0 ** -24

    def edit(mod):
        g = torch.Generator().manual_seed(1)
        rnd = lambda t, lo, hi: t.copy_((lo + (hi - lo) * torch.rand(t.shape, generator=g)).to(t.device))
        net = mod.deformation_net
        with torch.no_grad():
            for lvl in net.grid.grids:
                for p in lvl:
                    rnd(p, 10.0 ** -1.5, 1.1 * 10.0 ** -1.5)
            rnd(net.feature_out[0].weight, 200.0, 250.0)
            net.feature_out[0].bias.zero_()
            for key in ("pos_deform", "scales_deform", "rotations_deform", "opacity_deform", "shs_deform"):
                seq = getattr(net, key)
                rnd(seq[1].weight, 0.5, 1.0); seq[1].bias.zero_()
                rnd(seq[3].weight, 0.5, 1.0); seq[3].bias.zero_()
    mod, ins = _fp16_case(edit)
    ins = [x.cpu() for x in ins]
    for x in ins[1:]:
        x.zero_()
    n = ins[0].shape[0]
    got, _, _ = _run(mod, ins, None, 0.25, 2, backward=False)
    ffma, _, _ = _run(mod, ins, None, 0.25, 0, backward=False)
    with _Mode(2):
        with torch.no_grad():
            mod(*[x.cuda() for x in ins], torch.tensor(0.25).repeat(n, 1).cuda())   # raises if a call set the range flag

    cfg, prm, _ = oracle_from_module(mod)
    p64 = prm.to(torch.float64)
    with torch.no_grad():
        f = dr.hexplane_features(p64.planes, ins[0].double(), p64.aabb, torch.full((n,), 0.25, dtype=torch.float64))
    assert float(f.min()) >= 2.0 * 2.0 ** -25 / 64 and float(f.max()) <= 2e-9
    split = lambda x, s: torch.maximum(2.0 ** -22 * x.abs(), torch.full_like(x, 2.0 ** -25 / s))
    W0 = p64.w0.detach()
    F, Wd = W0.shape[1], W0.shape[0]
    m1 = f @ W0.t()
    e1 = split(f, 64) @ W0.t() + f @ split(W0, 256).t() + 2 * (F + 4) * u * m1
    e1 = e1 + split(m1 + e1, 8)
    heads = ("pos", "scales", "rotations", "opacity", "shs")
    for i, h in enumerate(heads):
        W1, _, W2, _ = (t.detach() for t in p64.heads[h])
        m2 = m1 @ W1.t()
        e2 = e1 @ W1.t() + (m1 + e1) @ split(W1, 256).t() + 2 * (Wd + 4) * u * m2
        e2 = e2 + split(m2 + e2, 8)
        m3 = m2 @ W2.t()
        e3 = e2 @ W2.t() + (m2 + e2) @ split(W2, 256).t() + 2 * (Wd + 4) * u * m3
        a, b = got[i].double().reshape(n, -1), ffma[i].double().reshape(n, -1)
        if h == "pos":
            x = ins[0].double()
            e3 = e3 + 2.0 ** -23 * (x + m3).abs()         # each engine rounds xyz + delta once
            assert torch.all((b - x - m3).abs() <= (F + 2 * Wd + 3) * u * m3 + u * (x + m3).abs()), h
        else:
            assert torch.all((b - m3).abs() <= (F + 2 * Wd + 3) * u * m3), h        # FFMA: fp32 sums of positive terms
        assert torch.all(e3 < 0.75 * m3), h                 # non-vacuous: outputs without the features break the bound
        assert torch.all((a - b).abs() <= e3), (h, float(((a - b).abs() / e3).max()))
        _note("fp16-tiny", float(((a - b).abs() / m3).max()))


# --------------------------------------------------------------------------------------------------- tiles
# (net, engine, tile sizes in Gaussians): the tensor-core forward (FP16x2: 128 per CTA pass as two warpgroups of 64) and the
# BF16x2 backward (128) at W = 128; the FFMA kernels at W = 64 (128 per tile) and in half tiles (C = 20, L = 3, every head,
# D = 2: 32 per tile)
TILE_CASES = [(ue.Net("small128", ue.RES[0]), 2, (64, 128)),
              (ue.Net("small64", ue.RES[1]), 0, (128,)), (ue.Net("c20w128sh", ue.RES[0], (1, 2, 4), depth=2), 0, (32,))]


@pytest.mark.parametrize("net,tc,tiles", TILE_CASES, ids=lambda v: v.name if isinstance(v, ue.Net) else str(v))
def test_tile_tails_match_ffma_and_oracle(net, tc, tiles):
    """n in {1, 63 .. 129} and k S T + {-1, 0, 1} (S SMs, T the engine's tiles, k = 1, 2: the persistent grid's last CTA takes
    one tile more, or one fewer): forward and backward against fp64 per Gaussian, and the tensor-core engines against the
    FFMA engine"""
    mod = ue.make_edge_module(net, seed=10)
    for n in ue.tile_sizes(torch.cuda.get_device_properties(0).multi_processor_count, tiles):
        ins, probes = ue.inputs(ue.tile_scene(n, seed=n).xyz, seed=n)
        probes = _mask_kinks(mod, ins, probes, 0.25)
        outs, gi = _check_vs_oracle(mod, ins, probes, 0.25, tc, "tiles")
        if tc == 0:
            continue
        o_ff, gi_ff, _ = _run(mod, ins, probes, 0.25, 0)
        for a, b, nm in zip(outs, o_ff, NAMES):
            assert float((a - b).abs().max()) <= 5e-6, (n, nm)
        for a, b in zip(gi, gi_ff):
            e, _ = row_err(a.numpy(), b.numpy())
            assert e <= GRAD_TOL, (n, e)


# --------------------------------------------------------------------------------------------------- partial gradients
def _direct(mod, x, others, t, go, gi_mask, tc, sink_offset=0):
    """g4d_deform_forward + g4d_deform_backward through the C-ABI with the upstream gradients go (None = NULL) and input
    gradient sinks where gi_mask is True (else NULL).  Returns (rc, input grads, {plane/weight sinks}) ."""
    lib = _lib.load()
    n = x.shape[0]
    keep = []
    prm = mod.c_params(keep, fresh=True)
    outs = [torch.empty_like(v) for v in [x] + others]
    bits = torch.empty(_lib.relu_bits_words(n), device="cuda", dtype=torch.int32)
    ptr = lambda v: v.data_ptr() if v is not None else None
    grads = mod.alloc_grads()
    if sink_offset:
        buf = torch.zeros(sum(g.numel() for g in grads) + 4, device="cuda")
        off, moved = sink_offset, []
        for g in grads:
            if g.dim() == 4:
                b_, c, h, w = g.shape
                moved.append(buf[off:off + g.numel()].view(b_, h, w, c).permute(0, 3, 1, 2))
            else:
                moved.append(buf[off:off + g.numel()].view(g.shape))
            off += g.numel()
        grads = moved
    cg = mod.c_grads(grads)
    gi = [torch.zeros_like(v) if m else None for v, m in zip([x] + others, gi_mask)]
    with _Mode(tc):
        ws = _lib.workspace_of(x.device)
        _lib.check(lib.g4d_deform_forward(ws.handle, C.byref(prm), n, ptr(x), *[ptr(v) for v in others], float(t),
                                          *[ptr(v) for v in outs], ptr(bits), _lib.stream_of(x.device)), "forward")
        rc = lib.g4d_deform_backward(ws.handle, C.byref(prm), C.byref(cg), n, ptr(x), float(t), *[ptr(v) for v in go],
                                     *[ptr(v) for v in gi], ptr(bits), _lib.stream_of(x.device))
    return rc, gi, grads


@pytest.mark.parametrize("tc", [0, 2])
def test_partial_upstream_gradients_equal_explicit_zeros(tc):
    """a loss over one output passes NULL for the other upstream gradients: the per-Gaussian input gradients equal those of
    explicit zero cotangents bit for bit, plane and weight gradients (float atomics in varying order) to 1e-6 of their max.
    NULL input-gradient sinks leave the other gradients unchanged to the same bounds."""
    net = ue.Net("small128", ue.RES[0])
    mod = ue.make_edge_module(net, seed=12)
    sc = ue.face_scene()
    ins, probes = ue.inputs(sc.xyz, seed=17)
    x, *others = [v.cuda().contiguous() for v in ins]
    pr = [p.cuda().contiguous() for p in probes]

    def close(a, b):
        for p, q in zip(a, b):
            m = float(q.abs().max())
            assert float((p - q).abs().max()) <= 1e-6 * max(m, 1e-30), (tuple(p.shape), m)

    full = _direct(mod, x, others, 0.25, pr, [True] * 5, tc)
    assert full[0] == 0
    for h in range(5):
        null = _direct(mod, x, others, 0.25, [p if i == h else None for i, p in enumerate(pr)], [True] * 5, tc)
        zero = _direct(mod, x, others, 0.25, [p if i == h else torch.zeros_like(p) for i, p in enumerate(pr)], [True] * 5, tc)
        assert null[0] == 0 and zero[0] == 0
        for a, b in zip(null[1], zero[1]):
            assert torch.equal(a, b), h
        close(null[2], zero[2])
    for drop in range(1, 5):           # xyz's sink is required; any other may be NULL
        mask = [i != drop for i in range(5)]
        part = _direct(mod, x, others, 0.25, pr, mask, tc)
        assert part[0] == 0
        for i in range(5):
            if mask[i]:
                assert torch.equal(part[1][i], full[1][i]), (drop, i)
        close(part[2], full[2])


# --------------------------------------------------------------------------------------------------- sinks and planes the kernels cannot take
def test_misaligned_plane_gradient_sink_is_refused_before_any_launch():
    """the scatter adds float4s: a plane-gradient sink one float off 16-byte alignment returns G4D_ERR_ARG and no sink is
    written"""
    mod = ue.make_edge_module(ue.Net("small128", ue.RES[0]), seed=1)
    ins, probes = ue.inputs(ue.face_scene().xyz, seed=1)
    x, *others = [v.cuda().contiguous() for v in ins]
    rc, gi, grads = _direct(mod, x, others, 0.25, [p.cuda() for p in probes], [True] * 5, 0, sink_offset=1)
    torch.cuda.synchronize()
    assert rc == -2, rc
    assert "16-byte" in _lib.load().g4d_last_error().decode()
    assert all(float(g.abs().max()) == 0.0 for g in grads)
    assert all(float(g.abs().max()) == 0.0 for g in gi if g is not None)


def test_misaligned_or_oversized_planes_are_refused_before_any_launch():
    lib = _lib.load()
    mod = ue.make_edge_module(ue.Net("small128", ue.RES[0]), seed=1)
    n = 64
    x = torch.zeros(n, 3, device="cuda")
    out = torch.full((n, 3), 7.0, device="cuda")
    ws = _lib.Workspace.get(0)

    def rc_of(edit):
        keep = []
        prm = mod.c_params(keep)
        edit(prm)
        rc = lib.g4d_deform_forward(ws.handle, C.byref(prm), n, x.data_ptr(), None, None, None, None, 0.0, out.data_ptr(), None,
                                    None, None, None, None, _lib.stream_of(x.device))
        torch.cuda.synchronize()
        return rc, lib.g4d_last_error().decode()

    def misalign(p):
        p.planes[1][3] = p.planes[1][3] + 4

    def oversize(p):
        p.res[0][0] = p.res[0][1] = 11586              # 11586^2 * 16 >= 2^31 floats in plane (x, y)
    for edit, what in ((misalign, "16-byte"), (oversize, "2^31")):
        rc, msg = rc_of(edit)
        assert rc == -2 and what in msg, (rc, msg)
    assert bool((out == 7.0).all())


@pytest.mark.parametrize("n", [2501, 2502, 2503])
def test_fused_grad_accumulation_with_unaligned_bucket_views(n):
    """FlatGradBucket(gaussian_parameters() + flat_parameters()) at n = 1, 2, 3 (mod 4): the plane .grad views are not 16-byte
    aligned, grad_sinks() hands the kernels staging buffers, and two views' gradients plus the plane regulariser's (added
    straight into the unaligned views) equal the unfused path's"""
    res = []
    for fused in (False, True):
        scene = synth.make_scene(n, seed=11, scale_mean=0.08)
        torch.manual_seed(1236)
        mod = g4d.deform_network(synth.hidden_args("small128"))
        synth.perturb_deformation(mod, 2)
        mod.deformation_net.set_aabb(scene["aabb"][0].tolist(), scene["aabb"][1].tolist())
        mod = mod.cuda()
        pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
        bucket = dp.FlatGradBucket(pc.gaussian_parameters() + list(mod.flat_parameters()))
        mod.fused_grad_accumulation = fused
        bucket.zero_()
        if fused:
            planes = [p.grad for lvl in mod.deformation_net.grid.grids for p in lvl]
            assert any(g.data_ptr() % 16 for g in planes) and mod.grad_sinks() is None
        for th in (20.0, 45.0):
            cam = synth.make_camera(th, 96, 64, radius=4.0, time=0.3)

            class P:
                convert_SHs_python = False; compute_cov3D_python = False; debug = False
            out = g4d.render(cam, pc, P, torch.tensor([1.0, 1.0, 1.0], device="cuda"))
            (out["render"] * 0.5).abs().mean().backward()
        losses.accumulate_regulation(mod, 1e-3, 1e-4, 2e-4)     # scalar adds: takes the unaligned views as they are
        res.append(bucket.flat.clone())
    a, b = res
    assert float(b.abs().max()) > 0
    assert float((a - b).abs().max()) <= 1e-5 * float(b.abs().max())
