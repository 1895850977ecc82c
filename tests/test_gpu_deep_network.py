"""Deformation networks with trunk layers (defor_depth D >= 2) on the GPU: the FFMA forward and backward against the fp64
oracle, an exactness case against the network without trunk, the fused render / multi-camera / CUDA-graph paths, one training
step, and the C-ABI's refusals.

Tolerances are DESIGN.md §2.2's for the FFMA network: forward 2e-5 absolute on the pre-activation outputs; gradients 2e-3 of the
tensor's max, with the upstream gradient of the Gaussians at a kink of the network (found in fp64 on the oracle, now including
the trunk's pre-activations) zeroed on both sides; network weights and biases 2e-4 of the tensor's max.
"""
import ctypes as C
import importlib

import pytest
import torch

from util_deep_network import deform_forward, fp64_leaves, kink_rows, oracle_from_module
from util_scene import g4d, rel_err, synth

pytestmark = pytest.mark.gpu
_lib = importlib.import_module("4dgaussians_b200._lib")
graphs = importlib.import_module("4dgaussians_b200.graphs")
td = importlib.import_module("4dgaussians_b200.train_dp")

FWD_TOL = 2e-5
GRAD_TOL = 2e-3
WEIGHT_TOL = 2e-4
ATOMIC_TOL = 1e-4      # the same per-CTA partials summed by fp32 atomics in another order
NAMES = ("xyz", "scales", "rot", "opacity", "shs")


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


def _deep_module(net, depth, seed=3, aabb=None):
    """make_module at another defor_depth: same seed discipline, so D = 0 / 1 are the shipped networks"""
    args = synth.hidden_args(net)
    args.defor_depth = depth
    torch.manual_seed(1234 + seed)
    m = g4d.deform_network(args)
    synth.perturb_deformation(m, seed)
    if aabb is not None:
        m.deformation_net.set_aabb(aabb[0].tolist(), aabb[1].tolist())
    return m.cuda()


def _inputs(n, seed):
    from oracle.make_golden_deform import synth_inputs
    (xyz, sc, rot, op, shs), probes = synth_inputs(n, seed)
    return [t.cuda() for t in (xyz, sc, rot, op, shs)], probes


class _Ffma:
    """the shared workspace with tensor cores off (the D <= 1 reference engine of the exactness case)"""

    def __enter__(self):
        self.ws = _lib.Workspace.get(torch.cuda.current_device())
        self.ws.set_option(_lib.OPT_TENSOR_CORES, 0)

    def __exit__(self, *a):
        torch.cuda.synchronize()
        self.ws.set_option(_lib.OPT_TENSOR_CORES, 2)


# deep64: the dnerf heads (pos, scales, rotations) at W = 64; deep128: all five dynerf heads at W = 128.  c32w128sh (L = 2,
# C = 32, all heads: the tensor cores' configuration at D <= 1) and c20w128sh (L = 3, C = 20, all heads) need more shared memory
# than a tile of 64 Gaussians leaves once the trunk biases are added: the FFMA forward runs them in tiles of 32.  N is not a
# multiple of any tile (128 / 64 / 32 Gaussians).
@pytest.mark.parametrize("depth", [0, 2, 3, 8])
@pytest.mark.parametrize("net,n", [("deep64", 1001), ("deep128", 777), ("c32w128sh", 333), ("c20w128sh", 301)])
def test_deform_forward_and_backward_vs_oracle(net, n, depth):
    t = 0.61
    mod = _deep_module(net, depth)
    cfg, prm, trunk = oracle_from_module(mod)
    assert len(trunk) == max(depth, 1) - 1
    ins, probes = _inputs(n, 6)
    kink = kink_rows(cfg, prm, trunk, ins[0], t)
    # the statement must not be vacuous; a deeper trunk has more pre-activations that can sit near 0 (5.3 % of the rows at
    # D = 8, W = 128: 8 x 128 + 5 x 128 ReLUs per Gaussian)
    assert float(kink.float().mean()) <= 0.1
    for p in probes:
        p[kink] = 0
    dev_in = [x.clone().requires_grad_(True) for x in ins]
    outs = mod(*dev_in, torch.tensor(t).repeat(n, 1).cuda())
    sum((o * p.cuda()).sum() for o, p in zip(outs, probes)).backward()
    p64, tr64 = fp64_leaves(prm, trunk)
    cpu_in = [x.cpu().double().requires_grad_(True) for x in ins]
    want = deform_forward(cfg, p64, tr64, *cpu_in, t)
    sum((o * p.double()).sum() for o, p in zip(want, probes)).backward()
    for o, w, nm in zip(outs, want, NAMES):
        assert o.shape == w.shape, nm
        err = float((o.detach().cpu().double() - w.detach()).abs().max())
        assert err <= FWD_TOL, (nm, err)
    for a, b, nm in zip(dev_in, cpu_in, NAMES):
        if b.grad is not None:
            e = rel_err(a.grad.cpu().numpy(), b.grad.numpy())
            assert e <= GRAD_TOL, (nm, e)
    net_ = mod.deformation_net
    pairs = [(net_.feature_out[0].weight, p64.w0), (net_.feature_out[0].bias, p64.b0)]
    for lin, (w, b) in zip(mod.trunk_layers(), tr64):
        pairs += [(lin.weight, w), (lin.bias, b)]
    heads = dict(zip(("pos", "scales", "rotations", "opacity", "shs"), ("pos_deform", "scales_deform", "rotations_deform",
                                                                       "opacity_deform", "shs_deform")))
    for h in cfg.active_heads():
        seq = getattr(net_, heads[h])
        pairs += list(zip((seq[1].weight, seq[1].bias, seq[3].weight, seq[3].bias), p64.heads[h]))
    for l, lvl in enumerate(net_.grid.grids):
        for k, p in enumerate(lvl):
            e = rel_err(p.grad.cpu().numpy(), p64.planes[l][k].grad.numpy())
            assert e <= GRAD_TOL, ("plane", l, k, e)
    for p, r in pairs:
        e = rel_err(p.grad.cpu().numpy(), r.grad.numpy())
        assert e <= WEIGHT_TOL, (tuple(p.shape), e)


@pytest.mark.parametrize("net", ["deep64", "deep128"])
def test_identity_trunk_layer_is_bit_exact(net):
    """D = 2 with W_1 = I, b_1 = 0: relu(I relu(h_0)) = relu(h_0), so outputs and every shared gradient equal the D = 1
    network's on the FFMA engine: the outputs and the per-Gaussian input gradients bit for bit.  The weight and plane gradients
    add per-CTA partials with fp32 atomics, in an order that is not fixed from one launch to the next (not even between two
    runs of one network): those agree up to that reordering, 1e-4 of the tensor's max (1.7e-5 measured on an H100 for the
    opacity head's b2, a sum with cancellation).  dW_1 = dz_1^T a_0 against fp64, db_1 = db_0 of the D = 1 run."""
    n, t = 3001, 0.37
    m1 = _deep_module(net, 1)
    m2 = _deep_module(net, 2)
    sd = m2.state_dict()
    sd.update(m1.state_dict())
    w = m1.deformation_net.W
    sd["deformation_net.feature_out.2.weight"] = torch.eye(w, device="cuda")
    sd["deformation_net.feature_out.2.bias"] = torch.zeros(w, device="cuda")
    m2.load_state_dict(sd)
    ins, probes = _inputs(n, 8)
    cfg, prm, _ = oracle_from_module(m1)
    kink = kink_rows(cfg, prm, [], ins[0], t)     # (for the fp64 check of dW_1 only)
    for p in probes:
        p[kink] = 0
    res = []
    with _Ffma():
        for m in (m1, m2):
            dev_in = [x.clone().requires_grad_(True) for x in ins]
            outs = m(*dev_in, torch.tensor(t).repeat(n, 1).cuda())
            sum((o * p.cuda()).sum() for o, p in zip(outs, probes)).backward()
            res.append(([o.detach().clone() for o in outs], [x.grad for x in dev_in]))
    (o1, g1), (o2, g2) = res
    for a, b, nm in zip(o1, o2, NAMES):
        assert torch.equal(a, b), nm
    for a, b, nm in zip(g1, g2, NAMES):
        assert (a is None) == (b is None) and (a is None or torch.equal(a, b)), nm
    named1 = dict(m1.named_parameters())
    for k, p in m2.named_parameters():
        if k in named1 and p.grad is not None:
            assert float((p.grad - named1[k].grad).abs().max()) <= ATOMIC_TOL * float(named1[k].grad.abs().max()), k
    lin = m2.trunk_layers()[0]
    b0 = m1.deformation_net.feature_out[0].bias.grad
    assert float((lin.bias.grad - b0).abs().max()) <= ATOMIC_TOL * float(b0.abs().max())
    # dz_1 = dL/dh_0 of the D = 1 network, in fp64: dW_1 = dz_1^T a_0
    from oracle import deform_ref as dr
    p64, _ = fp64_leaves(prm, [])
    with torch.no_grad():
        feat = dr.hexplane_features(p64.planes, ins[0].cpu().double(), p64.aabb, torch.full((n,), t, dtype=torch.float64))
    hidden = (feat @ p64.w0.t() + p64.b0).detach().requires_grad_(True)
    heads = ("pos", "scales", "rotations", "opacity", "shs")
    sum((dr.mlp_head(hidden, p64.heads[h]).reshape(n, -1) * pr.double().reshape(n, -1)).sum()
        for h, pr in zip(heads, probes) if h in cfg.active_heads()).backward()
    want = hidden.grad.t() @ torch.relu(hidden.detach())
    e = rel_err(lin.weight.grad.cpu().numpy(), want.numpy())
    assert e <= WEIGHT_TOL, e


def _render_setup(net, depth, n=1500, t=0.45, grad=True, seed=11):
    scene = synth.make_scene(n, seed=seed, scale_mean=0.05)
    mod = _deep_module(net, depth, seed=2, aabb=scene["aabb"])
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=grad)
    return scene, mod, pc


def _settings(cam, bg):
    import math
    return g4d.GaussianRasterizationSettings(
        image_height=cam.image_height, image_width=cam.image_width, tanfovx=math.tan(cam.FoVx * 0.5),
        tanfovy=math.tan(cam.FoVy * 0.5), bg=torch.tensor(bg, dtype=torch.float32, device="cuda"), scale_modifier=1.0,
        viewmatrix=cam.world_view_transform.cuda(), projmatrix=cam.full_proj_transform.cuda(), sh_degree=3,
        campos=cam.camera_center.cuda(), prefiltered=False, debug=False)


@pytest.mark.parametrize("net", ["deep64", "deep128"])
def test_fused_render_vs_oracle_deformation_and_dropin_rasterizer(net):
    """render() at D = 3 against the reference-style composition: the fp64 oracle deformation, activations, then the drop-in
    GaussianRasterizer; the backward chains the rasterizer's gradients back through the oracle in fp64"""
    t, bg = 0.45, (0.0, 0.0, 0.0)
    scene, mod, pc = _render_setup(net, 3)
    cam = synth.make_camera(40.0, 120, 96, radius=2.6, time=t)
    out = g4d.render(cam, pc, _Pipe(), torch.tensor(bg, device="cuda"), stage="fine")
    gen = torch.Generator().manual_seed(1)
    dL = torch.randn(out["render"].shape, generator=gen).cuda()
    (out["render"] * dL).sum().backward()
    cfg, prm, trunk = oracle_from_module(mod)
    p64, tr64 = fp64_leaves(prm, trunk)
    leaves = {k: v.detach().cpu().double().requires_grad_(True) for k, v in scene.items() if k != "aabb"}
    shs = torch.cat([leaves["features_dc"], leaves["features_rest"]], dim=1)
    deformed = deform_forward(cfg, p64, tr64, leaves["xyz"], leaves["scaling"], leaves["rotation"], leaves["opacity"], shs, t)
    dev = [d.detach().float().cuda().requires_grad_(True) for d in deformed]
    m3, sc, rot, op, sh = dev
    rast = g4d.GaussianRasterizer(_settings(cam, bg))
    img, radii, _ = rast(means3D=m3, means2D=torch.zeros_like(m3), shs=sh, colors_precomp=None, opacities=torch.sigmoid(op),
                         scales=torch.exp(sc), rotations=torch.nn.functional.normalize(rot), cov3D_precomp=None)
    err = (out["render"].detach() - img.detach()).abs()
    assert float((err > 1e-4).float().mean()) <= 1e-3 and float(err.max()) <= 1e-2, float(err.max())
    assert float((out["radii"] != radii).float().mean()) <= 2e-3
    (img * dL).sum().backward()
    torch.autograd.backward(deformed, [d.grad.cpu().double() for d in dev])
    pairs = [(pc._xyz, leaves["xyz"]), (pc._scaling, leaves["scaling"]), (pc._rotation, leaves["rotation"]),
             (pc._opacity, leaves["opacity"]), (pc._features_dc, leaves["features_dc"]), (pc._features_rest, leaves["features_rest"])]
    for p, r in pairs:
        e = rel_err(p.grad.cpu().numpy(), r.grad.numpy())
        assert e <= 3 * GRAD_TOL, (tuple(p.shape), e)
    net_ = mod.deformation_net
    wpairs = [(net_.feature_out[0].weight, p64.w0)] + [(lin.weight, w) for lin, (w, _) in zip(mod.trunk_layers(), tr64)]
    for p, r in wpairs:
        e = rel_err(p.grad.cpu().numpy(), r.grad.numpy())
        assert e <= 3 * GRAD_TOL, (tuple(p.shape), e)


def test_render_cameras_equal_separate_renders_at_depth_3():
    t = 0.6
    scene, mod, pc = _render_setup("deep128", 3)
    bg = torch.zeros(3, device="cuda")
    cams = [synth.make_camera(30.0, 120, 90, radius=2.4, time=t), synth.make_camera(85.0, 120, 90, radius=2.6, time=t),
            synth.make_camera(-50.0, 157, 79, radius=2.4, time=t)]
    outs = g4d.render_cameras(cams, pc, _Pipe, bg)
    gen = torch.Generator().manual_seed(4)
    ws = [torch.rand(3, c.image_height, c.image_width, generator=gen).cuda() for c in cams]
    sum((o["render"] * w).sum() for o, w in zip(outs, ws)).backward()
    ga = [p.grad.clone() for p in pc.gaussian_parameters()] + [p.grad.clone() for p in mod.flat_parameters()]
    for p in pc.gaussian_parameters() + list(mod.flat_parameters()):
        p.grad = None
    singles = []
    for cam, w in zip(cams, ws):
        o = g4d.render(cam, pc, _Pipe, bg)
        (o["render"] * w).sum().backward()
        singles.append(o)
    gb = [p.grad.clone() for p in pc.gaussian_parameters()] + [p.grad.clone() for p in mod.flat_parameters()]
    for o, s in zip(outs, singles):
        assert torch.equal(o["render"].detach(), s["render"].detach()) and torch.equal(o["radii"], s["radii"])
    assert len(ga) == len(gb)
    for a, b in zip(ga, gb):
        assert float((a - b).abs().max()) <= 1e-5 * max(1e-3, float(b.abs().max()))


def test_graphed_render_replays_equal_eager_renders_at_depth_3():
    scene, mod, pc = _render_setup("deep64", 3, grad=False)
    bg = torch.ones(3, device="cuda")
    cams = synth.orbit_cameras(5, 96, 72, radius=4.0)
    for i, cam in enumerate(cams):
        cam.time = (i + 1) / 6.0
    ws = _lib.Workspace.get(torch.cuda.current_device())
    with torch.no_grad():
        ws.set_option(_lib.OPT_SYNC_MODE, 0)
        try:
            gr = graphs.GraphedRender(pc, _Pipe, bg, cams[0])
            for cam in cams:
                got = {k: v.clone() for k, v in gr(cam).items()}
                ref = g4d.render(cam, pc, _Pipe, bg)
                for key in ("render", "depth", "radii", "visibility_filter"):
                    assert torch.equal(got[key], ref[key]), key
            gr.check()
        finally:
            torch.cuda.synchronize()
            ws.set_option(_lib.OPT_SYNC_MODE, 1)


def test_training_step_and_densify_at_depth_3():
    scene = synth.make_scene(1500, seed=5, scale_mean=0.05)
    mod = _deep_module("deep128", 3, seed=2, aabb=scene["aabb"])
    opt = td.default_opt()
    opt.densify_from_iter, opt.pruning_from_iter, opt.min_gaussians_for_prune = 1, 1, 100
    opt.densification_interval = opt.pruning_interval = 2
    opt.densify_grad_threshold_fine_init = opt.densify_grad_threshold_after = 5e-6
    tr = td.DPTrainer(td.GaussianSet(scene, mod), opt, cameras_extent=2.6)
    W, H = 96, 80
    cams = [synth.make_camera(th, W, H, radius=4.0, time=t) for th, t in ((0.0, 0.1), (60.0, 0.5))]
    gts = [torch.full((3, H, W), 0.25, device="cuda") for _ in cams]
    bg = torch.zeros(3, device="cuda")
    b, e = tr.state.segments["deformation"]
    tr.step(cams, gts, bg, _Pipe)
    torch.cuda.synchronize()
    for lin in mod.trunk_layers():
        off, cnt = tr.state.slices(lin.weight)
        assert b <= off and off + cnt <= e
        assert float(tr.state.grad[off:off + cnt].abs().max()) > 0       # the trunk's gradient landed in the MLP segment
    before = [lin.weight.detach().clone() for lin in mod.trunk_layers()]
    n0 = tr.g._xyz.shape[0]
    for _ in range(3):
        tr.step(cams, gts, bg, _Pipe)
    torch.cuda.synchronize()
    assert tr.rebuilds > 1 and tr.g._xyz.shape[0] != n0
    assert all(not torch.equal(a, lin.weight) for a, lin in zip(before, mod.trunk_layers()))
    assert bool(torch.isfinite(tr.state.param).all())


def _forward_rc(mod, edit):
    lib = _lib.load()
    keep = []
    prm = mod.c_params(keep)
    edit(prm)
    n = 64
    x = torch.zeros(n, 3, device="cuda")
    out = torch.full((n, 3), 7.0, device="cuda")
    ws = _lib.Workspace.get(torch.cuda.current_device())
    rc = lib.g4d_deform_forward(ws.handle, C.byref(prm), n, x.data_ptr(), None, None, None, None, 0.0, out.data_ptr(), None,
                                None, None, None, None, _lib.stream_of(x.device))
    torch.cuda.synchronize()
    return rc, lib.g4d_last_error().decode(), bool((out == 7.0).all())


def test_c_abi_refuses_bad_trunks_before_any_launch():
    mod = _deep_module("deep64", 3)
    ok = _forward_rc(mod, lambda p: None)
    assert ok[0] == 0 and not ok[2]

    def depth9(p):
        p.depth = 9

    def null_trunk(p):
        p.wt[1] = None

    def width256(p):
        p.net_width = 256
    for edit, what in ((depth9, "depth"), (null_trunk, "NULL"), (width256, "net_width")):
        rc, msg, untouched = _forward_rc(mod, edit)
        assert rc == -2 and what in msg and untouched, (rc, msg)
