"""Deformation networks with trunk layers (defor_depth D >= 2) on the CPU side of the tests: an independent restatement of the
reference's trunk (scene/deformation.py:55-60: ``feature_out = Linear(F, W), [ReLU, Linear(W, W)] * (D - 1)``) on top of the
oracle's HexPlane field and heads, the reference's own module built at any depth, and the conversions between them.

The trunk: h_0 = W_0 feat + b_0, h_j = W_j relu(h_{j-1}) + b_j for j = 1 .. D-1; every head starts with its own ReLU of
h_{D-1}.  The trunk layers are the state_dict entries ``deformation_net.feature_out.{2j}.{weight,bias}``.
"""
from __future__ import annotations

import contextlib
import io
from typing import List, Tuple

import torch

from oracle import deform_ref as dr
from oracle import ref_loader

PRE = "deformation_net.feature_out."


def trunk_from_state_dict(sd, depth: int) -> List[Tuple[torch.Tensor, torch.Tensor]]:
    """[(W_j [W,W], b_j [W])] for j = 1 .. depth-1"""
    return [(sd[f"{PRE}{2 * j}.weight"], sd[f"{PRE}{2 * j}.bias"]) for j in range(1, depth)]


def trunk_to_state_dict(trunk) -> dict:
    out = {}
    for j, (w, b) in enumerate(trunk, start=1):
        out[f"{PRE}{2 * j}.weight"], out[f"{PRE}{2 * j}.bias"] = w, b
    return out


def random_trunk(width: int, depth: int, seed: int, dtype=torch.float32):
    """xavier-uniform weights and default-Linear-like biases, as oracle.deform_ref.random_params draws them"""
    g = torch.Generator().manual_seed(seed)
    bound = (6.0 / (2 * width)) ** 0.5
    out = []
    for _ in range(1, depth):
        w = (torch.rand(width, width, generator=g, dtype=torch.float64) * 2 - 1) * bound
        b = (torch.rand(width, generator=g, dtype=torch.float64) * 2 - 1) / width ** 0.5
        out.append((w.to(dtype), b.to(dtype)))
    return out


def deform_forward(cfg: dr.DeformConfig, prm: dr.DeformParams, trunk, xyz, scales, rotations, opacity, shs, t):
    """deform_network.forward (deformation.py:185-212 -> :97-148) with the trunk; the 5-tuple of pre-activation tensors"""
    n = xyz.shape[0]
    tt = torch.as_tensor(t, dtype=xyz.dtype).reshape(-1)
    if tt.numel() == 1:
        tt = tt.expand(n)
    feat = dr.hexplane_features(prm.planes, xyz, prm.aabb, tt)
    hidden = feat @ prm.w0.t() + prm.b0
    for w, b in trunk:
        hidden = torch.relu(hidden) @ w.t() + b
    pts = xyz if cfg.no_dx else xyz + dr.mlp_head(hidden, prm.heads["pos"])
    sc = scales if cfg.no_ds else scales + dr.mlp_head(hidden, prm.heads["scales"])
    rot = rotations if cfg.no_dr else rotations + dr.mlp_head(hidden, prm.heads["rotations"])
    op = opacity if cfg.no_do else opacity + dr.mlp_head(hidden, prm.heads["opacity"])
    sh = shs if cfg.no_dshs else shs + dr.mlp_head(hidden, prm.heads["shs"]).reshape(n, 16, 3)
    return pts, sc, rot, op, sh


def oracle_from_module(module):
    """(DeformConfig, DeformParams, trunk) as CPU fp32 leaves with requires_grad, mirroring a g4d deform_network"""
    a = module.args
    kc = a.kplanes_config
    cfg = dr.DeformConfig(channels=kc["output_coordinate_dim"], resolution=tuple(kc["resolution"]), multires=tuple(a.multires),
                          net_width=a.net_width, no_dx=a.no_dx, no_ds=a.no_ds, no_dr=a.no_dr, no_do=a.no_do, no_dshs=a.no_dshs)
    sd = {k: v.detach().cpu().contiguous().clone() for k, v in module.state_dict().items()}
    prm = dr.params_from_state_dict(sd, cfg.levels)
    trunk = trunk_from_state_dict(sd, module.deformation_net.D)
    for t in prm.leaves() + [x for wb in trunk for x in wb]:
        t.requires_grad_(True)
    return cfg, prm, trunk


def reference_module(cfg: dr.DeformConfig, depth: int):
    """the reference's own scene.deformation.deform_network at defor_depth = depth (CPU, fp32)"""
    if not ref_loader.reference_available():
        raise RuntimeError("reference tree not present at %s" % ref_loader.REF_ROOT)
    ref_loader._install_shims()
    from scene.deformation import deform_network  # type: ignore
    args = ref_loader.hidden_args(cfg)
    args.defor_depth = depth
    with contextlib.redirect_stdout(io.StringIO()):
        return deform_network(args)


def kink_rows(cfg, prm, trunk, xyz, t, delta_act=2e-6, delta_grid=2e-4):
    """[N] bool: util_scene.kink_rows extended to the trunk -- a HexPlane coordinate within delta_grid texels of a grid line, or
    a ReLU pre-activation within delta_act of 0 anywhere in the network (h_0 .. h_{D-1} and every active head's hidden layer,
    fed by relu(h_{D-1})), in fp64 on the oracle"""
    from util_scene import kink_rows as grid_and_first_layer_kinks
    mask = grid_and_first_layer_kinks(cfg, prm, xyz, t, delta_act, delta_grid)
    with torch.no_grad():
        x64 = xyz.detach().double().cpu()
        n = x64.shape[0]
        planes = [[p.detach().double() for p in lvl] for lvl in prm.planes]
        tt = torch.full((n,), float(t), dtype=torch.float64)
        feat = dr.hexplane_features(planes, x64, prm.aabb.detach().double(), tt)
        hidden = feat @ prm.w0.detach().double().t() + prm.b0.detach().double()
        for w, b in trunk:
            hidden = torch.relu(hidden) @ w.detach().double().t() + b.detach().double()
            mask |= (hidden.abs() < delta_act).any(dim=1)
        a = torch.relu(hidden)
        for name in cfg.active_heads():
            w1, b1, _, _ = prm.heads[name]
            mask |= ((a @ w1.detach().double().t() + b1.detach().double()).abs() < delta_act).any(dim=1)
    return mask


def fp64_leaves(prm, trunk):
    """fp64 copies of (prm, trunk) as fresh leaves that collect gradients"""
    p = prm.to(torch.float64)
    for q in p.leaves():
        q.detach_().requires_grad_(True)
    tr = [(w.detach().double().requires_grad_(True), b.detach().double().requires_grad_(True)) for w, b in trunk]
    return p, tr
