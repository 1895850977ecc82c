"""Deformation networks with trunk layers (defor_depth 2..8) on the CPU: the fp64 restatement against the reference's own
module, state_dict and checkpoint round trips, the parameter plumbing of the C-ABI and the refusals."""
import importlib
import os
import subprocess
import types

import pytest
import torch

from oracle import deform_ref as dr
from oracle import ref_loader
from oracle.make_golden_deform import synth_inputs
from util_deep_network import deform_forward, random_trunk, reference_module, trunk_to_state_dict

g4d = importlib.import_module("4dgaussians_b200")
synth = importlib.import_module("4dgaussians_b200.synth")
ck = importlib.import_module("4dgaussians_b200.checkpoint")
td = importlib.import_module("4dgaussians_b200.train_dp")
g4d_lib = importlib.import_module("4dgaussians_b200._lib")

AABB = torch.tensor([[1.31, 1.27, 1.3], [-1.29, -1.3, -1.22]])
needs_reference = pytest.mark.skipif(not ref_loader.reference_available(), reason="reference module not available")


def _deep_args(net, depth):
    a = synth.hidden_args(net)
    a.defor_depth = depth
    return a


@needs_reference
@pytest.mark.parametrize("depth", [2, 3, 8])
@pytest.mark.parametrize("name", ["dnerf", "dynerf"])
def test_restatement_matches_reference_module_fp64(name, depth):
    """forward outputs and autograd gradients of every parameter, trunk included, against the reference's deform_network"""
    cfg = dr.CONFIGS[name]
    prm = dr.random_params(cfg, seed=11, aabb=AABB, dtype=torch.float64)
    trunk = random_trunk(cfg.net_width, depth, seed=5, dtype=torch.float64)
    net = reference_module(cfg, depth).double()
    sd = net.state_dict()
    mine = dict(dr.params_to_state_dict(prm), **trunk_to_state_dict(trunk))
    assert set(k for k in sd if k.startswith("deformation_net.feature_out.")) == \
        set(k for k in mine if k.startswith("deformation_net.feature_out."))
    sd.update(mine)
    net.load_state_dict(sd)
    (xyz, sc, rot, op, shs), probes = synth_inputs(129, 7, dtype=torch.float64)
    xyz_r = xyz.clone().requires_grad_(True)
    t = 0.73
    ref = net(xyz_r, sc, rot, op, shs, torch.tensor(t, dtype=torch.float64).repeat(129, 1))
    leaves = [p.clone().requires_grad_(True) for p in prm.leaves()]
    lw = iter(leaves)
    p2 = dr.DeformParams(aabb=prm.aabb, planes=[[next(lw) for _ in range(6)] for _ in range(cfg.levels)], w0=next(lw), b0=next(lw),
                         heads={k: tuple(next(lw) for _ in range(4)) for k in dr.HEAD_NAMES})
    tr2 = [(w.clone().requires_grad_(True), b.clone().requires_grad_(True)) for w, b in trunk]
    xyz_m = xyz.clone().requires_grad_(True)
    got = deform_forward(cfg, p2, tr2, xyz_m, sc, rot, op, shs, t)
    for o, r in zip(got, ref):
        assert (o - r).abs().max().item() <= 1e-12
    sum(((r * p).sum() for r, p in zip(ref, probes))).backward()
    sum(((o * p).sum() for o, p in zip(got, probes))).backward()
    named = dict(net.named_parameters())
    pre = "deformation_net."
    pairs = [(xyz_r.grad, xyz_m.grad)]
    pairs += [(named[f"{pre}feature_out.0.weight"].grad, p2.w0.grad), (named[f"{pre}feature_out.0.bias"].grad, p2.b0.grad)]
    for j, (w, b) in enumerate(tr2, start=1):
        pairs += [(named[f"{pre}feature_out.{2 * j}.weight"].grad, w.grad), (named[f"{pre}feature_out.{2 * j}.bias"].grad, b.grad)]
    for l in range(cfg.levels):
        for k in range(6):
            pairs.append((named[f"{pre}grid.grids.{l}.{k}"].grad, p2.planes[l][k].grad))
    for name_h, key in dr._HEAD_KEY.items():
        if name_h not in cfg.active_heads():
            continue
        for i, idx in enumerate(("1.weight", "1.bias", "3.weight", "3.bias")):
            pairs.append((named[f"{pre}{key}.{idx}"].grad, p2.heads[name_h][i].grad))
    for r, m in pairs:
        assert r is not None and m is not None
        assert (r - m).abs().max().item() <= 1e-10 * max(1.0, r.abs().max().item())
    assert all(w.grad.abs().max() > 0 for w, _ in tr2)


@needs_reference
def test_state_dict_round_trip_with_reference_at_depth_3():
    cfg = dr.CONFIGS["dynerf"]
    mine = g4d.deform_network(_deep_args("dynerf", 3))
    synth.perturb_deformation(mine, 2)
    theirs = reference_module(cfg, 3)
    a, b = mine.state_dict(), theirs.state_dict()
    assert list(a.keys()) == list(b.keys()) and all(a[k].shape == b[k].shape for k in a)
    assert "deformation_net.feature_out.4.weight" in a and "deformation_net.feature_out.6.weight" not in a
    theirs.load_state_dict({k: v.contiguous() for k, v in a.items()})
    for k, v in theirs.state_dict().items():
        assert torch.equal(v, a[k]), k
    gen = torch.Generator().manual_seed(9)
    rnd = {k: torch.rand(v.shape, generator=gen) for k, v in b.items()}
    theirs.load_state_dict(rnd)
    mine.load_state_dict(theirs.state_dict())
    for k, v in mine.state_dict().items():
        assert torch.equal(v, rnd[k]), k


def test_checkpoint_round_trip_at_depth_3(tmp_path):
    mod = g4d.deform_network(_deep_args("deep128", 3))
    synth.perturb_deformation(mod, 4)
    scene = synth.make_scene(37, seed=2)
    pc = types.SimpleNamespace(_xyz=scene["xyz"], _features_dc=scene["features_dc"], _features_rest=scene["features_rest"],
                               _opacity=scene["opacity"], _scaling=scene["scaling"], _rotation=scene["rotation"], _deformation=mod)
    ck.save_iteration(str(tmp_path), 7, pc)
    other = g4d.deform_network(_deep_args("deep128", 3))
    g, table, _ = ck.load_iteration(str(tmp_path), 7, other, device="cpu")
    assert torch.equal(g["xyz"], scene["xyz"]) and table.shape == (37,)
    sa, sb = mod.state_dict(), other.state_dict()
    assert list(sa) == list(sb) and "deformation_net.feature_out.4.bias" in sb
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k


@pytest.mark.parametrize("depth", [0, 1, 2, 8])
def test_feature_out_layout_and_flat_parameters(depth):
    mod = g4d.deform_network(_deep_args("small64", depth))
    net = mod.deformation_net
    fo = list(net.feature_out)
    ntrunk = max(depth, 1) - 1
    assert len(fo) == 1 + 2 * ntrunk
    assert all(isinstance(m, torch.nn.ReLU) for m in fo[1::2]) and all(isinstance(m, torch.nn.Linear) for m in fo[0::2])
    flat = mod.flat_parameters()
    n_planes = len(net.grid.grids) * 6
    assert len(flat) == n_planes + 2 + 4 * 5 + 2 * ntrunk
    for j, lin in enumerate(mod.trunk_layers()):
        assert flat[n_planes + 22 + 2 * j] is lin.weight and flat[n_planes + 23 + 2 * j] is lin.bias
    mlp = {id(p) for p in mod.get_mlp_parameters()}
    assert all(id(lin.weight) in mlp and id(lin.bias) in mlp for lin in mod.trunk_layers())
    grads = mod.alloc_grads()
    assert [g.shape for g in grads] == [p.shape for p in flat]


def test_trunk_lands_in_the_mlp_learning_rate_segment():
    torch.manual_seed(3)
    scene = synth.make_scene(200, seed=1, scale_mean=0.05)
    mod = g4d.deform_network(synth.hidden_args("deep128"))
    tr = td.DPTrainer(td.GaussianSet(scene, mod, device="cpu"), td.default_opt(), cameras_extent=2.0)
    b, e = tr.state.segments["deformation"]
    for lin in mod.trunk_layers():
        for p in (lin.weight, lin.bias):
            off, n = tr.state.slices(p)
            assert b <= off and off + n <= e


def test_refusals_in_python():
    with pytest.raises(NotImplementedError, match="defor_depth"):
        g4d.deform_network(_deep_args("small64", 9))
    a = synth.hidden_args("small128")
    a.net_width = 256
    with pytest.raises(NotImplementedError, match="net_width must be 64 or 128"):
        g4d.deform_network(a)


def test_params_struct_tail_matches_the_header(tmp_path):
    """offsets of the trunk tail of G4DDeformParams / G4DDeformGrads in C and in the ctypes mirrors"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    prog = tmp_path / "off.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "g4d.h"\nint main(){printf("%d %zu %zu %zu %zu %zu\\n", '
                    'G4D_MAX_DEPTH, offsetof(G4DDeformParams, depth), offsetof(G4DDeformParams, wt), offsetof(G4DDeformParams, bt),'
                    ' offsetof(G4DDeformGrads, wt), offsetof(G4DDeformGrads, bt));return 0;}')
    exe = tmp_path / "off"
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(prog), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    P, G = g4d_lib.DeformParams, g4d_lib.DeformGrads
    assert got == [g4d_lib.MAX_DEPTH, P.depth.offset, P.wt.offset, P.bt.offset, G.wt.offset, G.bt.offset]
    zero = P()
    assert zero.depth == 0 and all(not zero.wt[j] for j in range(g4d_lib.MAX_DEPTH - 1))


def test_gradient_sinks_carry_the_trunk():
    mod = g4d.deform_network(_deep_args("small64", 4))
    grads = mod.alloc_grads()
    cg = mod._build_c_grads(grads)
    n = len(mod.deformation_net.grid.grids) * 6 + 22
    for j in range(3):
        assert cg.wt[j] == grads[n + 2 * j].data_ptr() and cg.bt[j] == grads[n + 2 * j + 1].data_ptr()
    assert not cg.wt[3] and not cg.bt[3]
