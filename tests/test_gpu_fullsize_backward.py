"""Full-size fused training backward (render() forward + backward) against a decomposed fp64 oracle, Gaussian by Gaussian.

Same proof structure as the forward in test_gpu_fullsize.py: compare on IDENTICAL post-deformation inputs, then chain.
  (1) GPU forward in training mode; before the backward releases the context, read the deformed [N,11] (and deformed SH)
      tensors the fused kernel projected from, plus n_contrib, radii and clamped;
  (2) the raster oracle on exactly those tensors: index data bit-exact (colours to fp32 rounding);
  (3) flip pixels -- n_contrib differs, or a channel differs by more than 1e-4 -- are bounded (the forward's 2e-5 H W + 2);
      so are threshold pixels, where an instance before the pixel's stop sits within rounding of alpha = 1/255, alpha = 0.99,
      T = 1e-4 or power = 0 (util_scene.threshold_pixels, the forward's explained-flip predicate).  A threshold flip of an
      instance that is not the pixel's last contributor, behind a small T, moves the image by less than 1e-4 yet gives that
      Gaussian a gradient term on one side only.  The upstream gradient is zeroed at both kinds of pixel on BOTH sides (every
      backward term of a pixel, background included, is proportional to that pixel's upstream gradient);
  (4) the raster oracle's backward with that upstream gives the post-activation cotangents, chained back through the
      deformation in fp64 (util_scene.oracle_chain_backward); means2D comes straight from the raster oracle.
Gaussians where fp32 may legitimately take the other branch are silenced BEFORE the GPU forward, by rules fixed in advance
and evaluated in fp64: a kink of the network (util_scene.kink_rows) or an SH colour channel within 1e-5 of the clamp for a
camera of the arm (util_scene.colour_kink_rows).  Their opacity logit is set to -40, so their alpha stays below 1/255 at
every pixel on both sides; their gradients, and those of Gaussians no camera sees, must then be exactly zero.

Every other row is compared per row (util_scene.row_err): |got - ref| / max(|ref row|, FLOOR max|ref|) <= ROW_TOL.  Network
weights and biases are compared as whole tensors.  Measured statistics go to parity_fullsize_backward.json, in the directory
where test_gpu_fullsize.py writes its own (quoted in DESIGN.md §2.3).
"""
import json
import os
import time

import numpy as np
import pytest
import torch

from oracle import deform_ref as dr
from oracle import raster_ref as rr
from test_gpu_fullsize import STATS as FWD_STATS, _assert_index_data_bit_exact
from util_scene import (SCENE_LEAVES, cam_tuple, colour_kink_rows, deformed_fp64, g4d, kink_rows, make_module,
                        oracle_chain_backward, oracle_params_from_module, raster_oracle_inputs, rel_err, row_err, row_errors,
                        synth, threshold_pixels)

pytestmark = pytest.mark.gpu
IMG_TOL = 1e-4
ROW_TOL = 2e-3
FLOOR = 1e-4
PLANE_FLOOR = 1e-2              # plane texels: a texel's gradient sums many Gaussians' terms that cancel (fp32 rounding)
MLP_TOL = {"ffma": 2e-4, "bf16x2": 5e-4}
FLIP_FRAC = 2e-5
THRESHOLD_FRAC = 0.03            # pixels with an instance on a compositing threshold (1.3-1.4 % at C1 and C3)
KINK_FRAC = 0.05
SILENCED_LOGIT = -40.0
T = 0.4
THETAS = (30.0, 120.0)          # camera 0 is the one of test_full_size_fused_forward_vs_oracle
STATS = os.path.join(os.path.dirname(FWD_STATS), "parity_fullsize_backward.json")

ARMS = [
    dict(id="C1", wl="C1", mlp="ffma"),                                   # dnerf: FFMA backward, width 64, C = 32
    dict(id="C1_modifier0.7", wl="C1", mlp="ffma", modifier=0.7),
    dict(id="C2", wl="C2", mlp="bf16x2"),                                 # hypernerf: three levels, tensor-core backward
    dict(id="C3", wl="C3", mlp="bf16x2"),                                 # dynerf: five heads incl. SHS
    dict(id="C3_ffma", wl="C3", mlp="ffma", tensor_cores=0),
    dict(id="C3_two_cameras", wl="C3", mlp="bf16x2", cameras=2),          # render_cameras, one summed backward
]


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


def _record(key, val):
    try:
        os.makedirs(os.path.dirname(STATS), exist_ok=True)
        cur = json.load(open(STATS)) if os.path.isfile(STATS) else {}
        cur[key] = val
        json.dump(cur, open(STATS, "w"), indent=1, sort_keys=True)
    except Exception:
        pass


@pytest.fixture(scope="module")
def workload():
    """Per BASELINE config: scene (silenced rows already at logit -40), module, oracle parameters, cameras, silenced set."""
    cache = {}

    def get(wl):
        if wl not in cache:
            w = synth.WORKLOADS[wl]
            scene = synth.make_scene(w["n"], seed=0, scale_mean=w["scale_mean"])
            mod = make_module(w["net"], seed=0, aabb=scene["aabb"])
            cfg, prm = oracle_params_from_module(mod)
            for p in prm.leaves():
                p.requires_grad_(False)
            cams = [synth.make_camera(th, w["width"], w["height"], radius=w["radius"], focal=w["focal"], time=T) for th in THETAS]
            t = float(np.float32(T))
            net_k = kink_rows(cfg, prm, scene["xyz"], t)
            pts, shs = deformed_fp64(cfg, prm, scene, t)
            col_k = colour_kink_rows(pts, shs, cams, sh_degree=3)
            silenced = (net_k | col_k).numpy()
            scene = dict(scene)
            scene["opacity"] = scene["opacity"].clone()
            scene["opacity"][torch.from_numpy(silenced)] = SILENCED_LOGIT
            cache[wl] = dict(w=w, scene=scene, mod=mod, cfg=cfg, prm=prm, cams=cams, t=t, silenced=silenced,
                             n_net_kinks=int(net_k.sum()), n_colour_kinks=int(col_k.sum()))
        return cache[wl]
    return get


def _stats(got, ref, floor=FLOOR):
    e = row_errors(got, ref, floor)
    emax, worst = row_err(got, ref, floor)
    return {"p50": float(np.quantile(e, 0.5)), "p99.99": float(np.quantile(e, 0.9999)), "max": emax,
            "worst": [(i, [float(x) for x in g[:6]], [float(x) for x in r[:6]]) for i, g, r in worst]}


def _plane_rows(a):
    """[1,C,H,W] -> [texels, C]"""
    a = np.asarray(a)
    return a[0].transpose(1, 2, 0).reshape(-1, a.shape[1])


@pytest.mark.parametrize("arm", ARMS, ids=[a["id"] for a in ARMS])
def test_fused_backward_vs_fp64_oracle(arm, workload):
    t0 = time.time()
    W = workload(arm["wl"])
    w, scene, mod, cfg, prm, t = W["w"], W["scene"], W["mod"], W["cfg"], W["prm"], W["t"]
    n = scene["xyz"].shape[0]
    silenced = W["silenced"]
    assert silenced.sum() <= KINK_FRAC * n, int(silenced.sum())
    cams = W["cams"][:arm.get("cameras", 1)]
    modifier = arm.get("modifier", 1.0)
    has_sh = not mod.args.no_dshs
    H, Wd = w["height"], w["width"]
    gen = torch.Generator().manual_seed(sum(map(ord, arm["id"])))
    dLs = [torch.randn(3, H, Wd, generator=gen) for _ in cams]
    mod.zero_grad(set_to_none=True)
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
    bg = torch.tensor(w["bg"], dtype=torch.float32, device="cuda")
    ws = g4d._lib.Workspace.get(0)
    stats = {"n": n, "silenced_network_kinks": W["n_net_kinks"], "silenced_colour_kinks": W["n_colour_kinks"],
             "silenced": int(silenced.sum()), "flip_pixels": [], "threshold_pixels": [], "R": []}
    cots, m2_ref = [], []
    try:
        ws.set_option(g4d._lib.OPT_TENSOR_CORES, arm.get("tensor_cores", 2))
        # ---- (1) GPU forward in training mode; read what the backward will use before it releases the contexts
        if len(cams) == 1:
            outs = [g4d.render(cams[0], pc, _Pipe, bg, scaling_modifier=modifier)]
            ctxs = [outs[0]["render"].grad_fn.lease.ctx]
        else:
            outs = g4d.render_cameras(cams, pc, _Pipe, bg, scaling_modifier=modifier)
            ctxs = [lease.ctx for lease in outs[0]["render"].grad_fn.leases]
        torch.cuda.synchronize()
        dfm = ctxs[0].read("deformed")
        shs_gpu = ctxs[0].read("deformed_shs") if has_sh else \
            torch.cat([scene["features_dc"], scene["features_rest"]], dim=1).numpy()
        ins = raster_oracle_inputs(dfm, shs_gpu)
        fwds = []
        for i, (cam, ctx, o, dL) in enumerate(zip(cams, ctxs, outs, dLs)):
            rc, _ = cam_tuple(cam, w["bg"], sh_degree=3, scale_modifier=modifier)
            # ---- (2) the raster oracle on the GPU's own deformed tensors: identical index data
            fwd = rr.rasterize_forward(rc, *ins)
            stats["R"].append(int(_assert_index_data_bit_exact(ctx, o["radii"].cpu().numpy(), fwd, colour_exact=False)))
            # ---- (3) flip pixels and threshold pixels: bounded, and silenced on both sides
            err = np.abs(o["render"].detach().cpu().numpy() - fwd["color"]).max(axis=0)
            flip = (ctx.read("n_contrib").reshape(H, Wd) != fwd["n_contrib"]) | (err > IMG_TOL)
            near = threshold_pixels(fwd, Wd, H)
            stats["flip_pixels"].append(int(flip.sum()))
            stats["threshold_pixels"].append(int(near.sum()))
            assert flip.sum() <= FLIP_FRAC * H * Wd + 2, (i, int(flip.sum()))
            assert near.sum() <= THRESHOLD_FRAC * H * Wd, (i, int(near.sum()))
            dL[:, torch.from_numpy(flip | near)] = 0.0
            fwds.append((rc, fwd))
        sum((o["render"] * dL.cuda()).sum() for o, dL in zip(outs, dLs)).backward()
        torch.cuda.synchronize()
    finally:
        ws.set_option(g4d._lib.OPT_TENSOR_CORES, 2)
    # ---- (4) oracle backward per camera, cotangents summed, one fp64 chain
    for (rc, fwd), dL in zip(fwds, dLs):
        g = rr.rasterize_backward(rc, *ins, fwd, dL.numpy())
        cots.append(g)
        m2_ref.append(g["means2D"])
    cot = {nm: sum(g[nm].astype(np.float64) for g in cots) for nm in ("means3D", "scales", "rots", "opacities", "shs")}
    ref, p64 = oracle_chain_backward(cfg, prm, scene, t, cot)
    got = {k: getattr(pc, "_" + k).grad.cpu().numpy().reshape(ref[k].shape) for k in SCENE_LEAVES}

    # exact zeros: silenced rows and rows no camera sees
    unseen = np.logical_and.reduce([o["radii"].cpu().numpy() == 0 for o in outs])
    stats["unseen"] = int(unseen.sum())
    failures = []
    for k in SCENE_LEAVES:
        for nm, rows in (("silenced", silenced), ("unseen", unseen)):
            nz = int((got[k][rows].reshape(int(rows.sum()), -1) != 0).any(axis=1).sum())
            if nz:
                failures.append(("%s rows with a nonzero gradient" % nm, k, nz))
    # per-row comparisons
    rows = {}
    for k in SCENE_LEAVES:
        rows[k] = _stats(got[k], ref[k])
    for i, (o, m2) in enumerate(zip(outs, m2_ref)):
        rows["viewspace_points_%d" % i] = _stats(o["viewspace_points"].grad.cpu().numpy(), m2)
    gp = {k: p.grad for k, p in mod.named_parameters()}
    mlp = {}
    for key, p in dr.params_to_state_dict(p64).items():
        if key not in gp:
            continue
        if p.grad is None:                                        # an inactive head: no gradient on the GPU either
            if gp[key] is not None and float(gp[key].abs().max()) != 0.0:
                failures.append(("inactive head has a gradient", key))
            continue
        g_ = gp[key].cpu().numpy()
        if key.startswith("deformation_net.grid.grids."):
            rows[key] = _stats(_plane_rows(g_), _plane_rows(p.grad.numpy()), PLANE_FLOOR)
        else:
            mlp[key] = rel_err(g_, p.grad.numpy())
    stats["rows"] = rows
    stats["mlp_rel_err_max"] = max(mlp.values())
    stats["mlp_rel_err"] = mlp
    stats["wall_s"] = time.time() - t0
    _record(arm["id"], stats)
    for k, s in rows.items():
        if s["max"] > ROW_TOL:
            failures.append(("row", k, s["max"], s["worst"][:2]))
    for k, e in mlp.items():
        if e > MLP_TOL[arm["mlp"]]:
            failures.append(("mlp", k, e))
    assert not failures, failures
