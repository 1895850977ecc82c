"""GPU: the FP16x2 tensor-core forward (deform_tc_kernel) with three consumer warpgroups per CTA (192 Gaussians per W1 image
load) and with two (F = 48 / 64 with the SH head, whose shared memory does not fit a third stage slab).

The count is chosen from the network alone; G4D_OPT_TC_DEBUG reports it per CTA (g4d_debug_tc_cycles [2], averaged over the
SMs).  Tile tails of both counts, forward (no-grad and grad-enabled) against fp64 and against the FFMA engine, input gradients
against the FFMA engine; fused renders at the C3 and C2 shapes against the FFMA engine."""
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

FWD_TOL = 2e-5
GRAD_TOL = 2e-3
NAMES = ("pts", "scales", "rot", "opacity", "shs")


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _expected_counter(nwg, n):
    """g4d_debug_tc_cycles [2]: nwg in each CTA of the persistent grid (min(tiles, SMs) CTAs), averaged over the SMs"""
    s = _sm_count()
    return nwg * min(-(-n // (64 * nwg)), s) / s


class _Engine:
    """G4D_OPT_TENSOR_CORES = tc on the shared workspace, with the per-CTA counters on"""
    def __init__(self, tc):
        self.tc = tc

    def __enter__(self):
        self.ws = _lib.Workspace.get(torch.cuda.current_device())
        self.ws.set_option(_lib.OPT_TENSOR_CORES, self.tc)
        self.ws.set_option(_lib.OPT_TC_DEBUG, 1)
        return self

    def warpgroups(self):
        out = (C.c_double * 12)()
        _lib.check(_lib.load().g4d_debug_tc_cycles(self.ws.handle, out), "g4d_debug_tc_cycles")
        return out[2]

    def __exit__(self, *a):
        torch.cuda.synchronize()
        self.ws.set_option(_lib.OPT_TC_DEBUG, 0)
        self.ws.set_option(_lib.OPT_TENSOR_CORES, 2)


def _fwd_err(got, ref):
    """per row: max |got - ref| / max(1, max |ref|)"""
    g, r = got.double().reshape(got.shape[0], -1), ref.double().reshape(ref.shape[0], -1)
    return float(((g - r).abs().max(dim=1).values / r.abs().max(dim=1).values.clamp_min(1.0)).max())


def _deform(mod, ins, probes, t, eng, backward):
    """module forward on the engine's settings (grad-enabled with a backward of <outs, probes>, or no-grad)"""
    n = ins[0].shape[0]
    dev_in = [x.cuda().clone().requires_grad_(backward) for x in ins]
    with torch.set_grad_enabled(backward):
        outs = mod(*dev_in, torch.tensor(float(t)).repeat(n, 1).cuda())
    counter = eng.warpgroups() if eng.tc else None
    if backward:
        torch.autograd.backward(list(outs), [p.cuda() for p in probes])
    return [o.detach().cpu() for o in outs], [x.grad.cpu() if backward else None for x in dev_in], counter


# (net, warpgroups the launch must choose): F = 32 with the SH head (the C3 shape), and F = 48 with it (two warpgroups)
TAIL_CASES = [(ue.Net("small128", ue.RES[0]), 3), (ue.Net("small128", ue.RES[1], (1, 2, 4)), 2)]


@pytest.mark.parametrize("net,nwg", TAIL_CASES, ids=lambda v: v.name if isinstance(v, ue.Net) else str(v))
def test_tile_tails_of_each_warpgroup_count(net, nwg):
    """n at every warpgroup boundary of a 192-Gaussian tile (191 .. 257) and k S T + {-1, 0, 1} (S SMs, T = 64 nwg, k = 1, 2:
    the persistent grid's last CTA takes one tile more, or one fewer): the no-grad and the grad-enabled forward agree bit for
    bit, match fp64 and the FFMA engine, and the input gradients match the FFMA engine's"""
    t = 0.25
    mod = ue.make_edge_module(net, seed=11)
    cfg, prm, trunk = oracle_from_module(mod)
    p64, tr64 = fp64_leaves(prm, trunk)
    for n in sorted(set(ue.tile_sizes(_sm_count(), (64 * nwg,)) + [191, 192, 193, 255, 256, 257])):
        ins, probes = ue.inputs(ue.tile_scene(n, seed=n).xyz, seed=n)
        kink = kink_rows(cfg, prm, trunk, ins[0].clone(), t, delta_grid=-1.0)
        for p in probes:
            p[kink] = 0
        with _Engine(2) as eng:
            nograd, _, c0 = _deform(mod, ins, probes, t, eng, backward=False)
            outs, gi, c1 = _deform(mod, ins, probes, t, eng, backward=True)
        assert c0 == c1 == pytest.approx(_expected_counter(nwg, n)), (n, c0, c1)
        with _Engine(0) as eng:
            o_ff, gi_ff, _ = _deform(mod, ins, probes, t, eng, backward=True)
        with torch.no_grad():
            want = deform_forward(cfg, p64, tr64, *[v.double() for v in ins], float(t))
        for a, b, f, w, nm in zip(nograd, outs, o_ff, want, NAMES):
            assert torch.equal(a, b), (n, nm)
            assert _fwd_err(b, w) <= FWD_TOL, (n, nm, _fwd_err(b, w))
            assert float((b - f).abs().max()) <= 5e-6, (n, nm)
        for a, b in zip(gi, gi_ff):
            e, _ = row_err(a.numpy(), b.numpy())
            assert e <= GRAD_TOL, (n, e)


class Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


def _workload_net(workload, sh_head):
    a = synth.hidden_args(synth.WORKLOADS[workload]["net"])
    a.no_dshs = not sh_head
    return a


# (workload, SH head, warpgroups): C3 (dynerf: F = 32 with the SH head), C2 (hypernerf: F = 48 without it), and the C2
# network with the SH head (F = 48: two warpgroups)
RENDER_CASES = [("C3", True, 3), ("C2", False, 3), ("C2", True, 2)]


@pytest.mark.parametrize("workload,sh_head,nwg", RENDER_CASES)
def test_fused_render_chooses_warpgroups_and_matches_ffma(workload, sh_head, nwg):
    """a fused no-grad render() of the workload's scene and camera: the launch runs nwg warpgroups per CTA, and the image and
    radii agree with the FFMA engine's (pixels off by more than 1e-4 are rare: a visibility or alpha threshold the two
    roundings of the network decide differently)"""
    w = synth.WORKLOADS[workload]
    scene = synth.make_scene(w["n"], seed=0, scale_mean=w["scale_mean"])
    torch.manual_seed(1234)
    mod = g4d.deform_network(_workload_net(workload, sh_head))
    synth.perturb_deformation(mod, 0)
    mod.deformation_net.set_aabb(scene["aabb"][0].tolist(), scene["aabb"][1].tolist())
    mod = mod.cuda()
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3)
    bg = torch.tensor([float(x) for x in w["bg"]], device="cuda")
    cam = synth.orbit_cameras(1, w["width"], w["height"], radius=w["radius"], focal=w["focal"], timestamps=300)[0]
    res = {}
    for tc in (2, 0):
        with _Engine(tc) as eng, torch.no_grad():
            out = g4d.render(cam, pc, Pipe, bg)
            res[tc] = (out["render"].cpu(), out["radii"].cpu())
            if tc:
                assert eng.warpgroups() == pytest.approx(_expected_counter(nwg, w["n"]))
    img, ref = res[2][0], res[0][0]
    err = (img - ref).abs().amax(dim=0)
    assert int((res[2][1] != res[0][1]).sum()) <= 1e-4 * w["n"] + 2
    assert int((err > 1e-4).sum()) <= 1e-4 * err.numel() + 2, int((err > 1e-4).sum())
    assert float(err.max()) <= 6e-3, float(err.max())
