"""Data-parallel training harness around the render path (SURVEY.md 8f N1).

Mirrors the shape of the reference's fine-stage loop -- /root/reference/train.py:108-296 (``scene_reconstruction``) with the
optimizer / densification bookkeeping of /root/reference/scene/gaussian_model.py:165-212, 316-413, 415-523 -- but GPU-first:

  * scene replicated, views sharded round-robin over ranks (one process per GPU); every rank renders its B views
    (fused forward + backward), the image loss and the HexPlane regularisers are the fused kernels of ``losses.py``;
  * ALL parameters and ALL gradients live in two flat fp32 buffers (``FlatState``): ``.data`` / ``.grad`` of every
    nn.Parameter are views, so the step's communication is ONE ``all_reduce`` over the gradient buffer and the optimizer
    step is ONE launch (``g4d_adam_step``: 8 learning-rate segments = the reference's 8 param groups, 1 / world folded in);
  * densification statistics (sum of ||grad means2D||, visible counts, max radii) are all-reduced, the split noise comes
    from a generator seeded by (seed, iteration): densify / prune decisions are IDENTICAL on every rank, so the replicas
    stay bit-identical without ever broadcasting parameters;
  * growing / shrinking N rebuilds the flat buffers once (every ``densification_interval`` = 100 steps), carrying the Adam
    moments of surviving Gaussians exactly like ``cat_tensors_to_optimizer`` / ``_prune_optimizer``.
The reference's learning-rate schedules (``get_expon_lr_func``, utils/general_utils.py:60-93) are restated in ``expon_lr``.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from argparse import Namespace
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn as nn

from . import _lib, losses
from .renderer import render

GAUSSIAN_GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")


def default_opt() -> Namespace:
    """OptimizationParams defaults (arguments/__init__.py:108-150) that the harness reads."""
    return Namespace(position_lr_init=0.00016, position_lr_final=0.0000016, position_lr_delay_mult=0.01,
                     position_lr_max_steps=20_000, deformation_lr_init=0.00016, deformation_lr_final=0.000016,
                     deformation_lr_delay_mult=0.01, grid_lr_init=0.0016, grid_lr_final=0.00016, feature_lr=0.0025,
                     opacity_lr=0.05, scaling_lr=0.005, rotation_lr=0.001, percent_dense=0.01, lambda_dssim=0.0,
                     densification_interval=100, opacity_reset_interval=3000, densify_from_iter=500, densify_until_iter=15_000,
                     densify_grad_threshold_fine_init=0.0002, densify_grad_threshold_after=0.0002,
                     opacity_threshold_fine_init=0.005, opacity_threshold_fine_after=0.005, pruning_from_iter=500,
                     pruning_interval=100, batch_size=2, time_smoothness_weight=0.001, l1_time_planes=0.0001,
                     plane_tv_weight=0.0002, max_gaussians=360_000, min_gaussians_for_prune=200_000)


def expon_lr(step, lr_init, lr_final, lr_delay_steps=0, lr_delay_mult=1.0, max_steps=1000000):
    """utils/general_utils.py:60-93 get_expon_lr_func (log-linear interpolation with an optional delayed warm-up)"""
    if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
        return 0.0
    if lr_delay_steps > 0:
        delay_rate = lr_delay_mult + (1 - lr_delay_mult) * math.sin(0.5 * math.pi * min(max(step / lr_delay_steps, 0.0), 1.0))
    else:
        delay_rate = 1.0
    t = min(max(step / max_steps, 0.0), 1.0)
    return delay_rate * math.exp(math.log(lr_init) * (1 - t) + math.log(lr_final) * t)


def inverse_sigmoid(x):
    return torch.log(x / (1 - x))


def build_rotation(r: torch.Tensor) -> torch.Tensor:
    """utils/general_utils.py:84-106"""
    q = r / r.norm(dim=1, keepdim=True)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], dim=1)
    return R.view(-1, 3, 3)


class FlatState:
    """Flat parameter / gradient / Adam-moment buffers; ``.data`` and ``.grad`` of every parameter are views.

    groups: ordered list of (name, [parameters]); the order fixes the layout and the Adam segments."""

    def __init__(self, groups: Sequence, device):
        self.groups = [(n, list(ps)) for n, ps in groups]
        self.device = device
        # every tensor starts on a 16-byte boundary: the kernels read rotations / SH rows / planes with 128-bit loads
        self.numel = sum((p.numel() + 3) // 4 * 4 for _, ps in self.groups for p in ps)
        self.param = torch.zeros(self.numel, device=device)
        self.grad = torch.zeros(self.numel, device=device)
        self.exp_avg = torch.zeros(self.numel, device=device)
        self.exp_avg_sq = torch.zeros(self.numel, device=device)
        self.segments: Dict[str, tuple] = {}
        self._views = []
        off = 0
        for name, ps in self.groups:
            begin = off
            for p in ps:
                n = p.numel()
                cl = p.dim() == 4 and p.is_contiguous(memory_format=torch.channels_last) and not p.is_contiguous()

                def view(buf, p=p, off=off, n=n, cl=cl):
                    seg = buf[off:off + n]
                    if cl:
                        b, c, h, w = p.shape
                        return seg.view(b, h, w, c).permute(0, 3, 1, 2)
                    return seg.view(p.shape)
                pv = view(self.param)
                pv.copy_(p.data)
                p.data = pv
                gv = view(self.grad)
                p.grad = gv
                self._views.append((p, pv, gv, off, n))
                off += (n + 3) // 4 * 4
            self.segments[name] = (begin, off)
        self.step_count = 0

    def slices(self, param: torch.Tensor):
        for p, _, _, off, n in self._views:
            if p is param:
                return off, n
        raise KeyError("parameter is not part of this FlatState")

    def moments(self, param):
        off, n = self.slices(param)
        return self.exp_avg[off:off + n].view(param.shape), self.exp_avg_sq[off:off + n].view(param.shape)

    def attached(self) -> bool:
        return all(p.grad is not None and p.grad.data_ptr() == gv.data_ptr() and p.data.data_ptr() == pv.data_ptr()
                   for p, pv, gv, _, _ in self._views)

    def zero_grad(self):
        self.grad.zero_()

    def adam_step(self, lrs: Dict[str, float], grad_scale: float = 1.0, betas=(0.9, 0.999), eps=1e-15, only=None,
                  span=None, count_step: bool = True):
        """``only``: restrict the update to these groups (the rest is left untouched, moments included).
        ``span`` = (begin, end), multiples of 4: update only that slice of the flat buffers (chunked all-reduce pipeline)."""
        if not self.attached():
            raise RuntimeError("FlatState: a parameter's .data / .grad is no longer a view of the flat buffers (zero_grad("
                               "set_to_none=True) or a parameter swap); use zero_grad() of this object and rebuild after densify")
        if count_step:
            self.step_count += 1
        b0, e0 = (0, self.numel) if span is None else span
        clipped = []
        for n, _ in self.groups:
            if only is not None and n not in only:
                continue
            sb, se = max(self.segments[n][0], b0), min(self.segments[n][1], e0)
            if se > sb:
                clipped.append((sb - b0, se - b0, float(lrs[n])))
        if not clipped:
            return
        segs = (_lib.AdamSegment * len(clipped))()
        for i, (sb, se, lr) in enumerate(clipped):
            segs[i].begin, segs[i].end, segs[i].lr = sb, se, lr
        dev = self.device
        off = 4 * b0
        with torch.cuda.device(dev):
            ws = _lib.Workspace.get(dev.index if dev.index is not None else torch.cuda.current_device())
            _lib.check(_lib.load().g4d_adam_step(ws.handle, self.param.data_ptr() + off, self.grad.data_ptr() + off,
                                                 self.exp_avg.data_ptr() + off, self.exp_avg_sq.data_ptr() + off, e0 - b0, segs,
                                                 len(clipped), betas[0], betas[1], eps, self.step_count, float(grad_scale),
                                                 int(torch.cuda.current_stream(dev).cuda_stream)), "g4d_adam_step")


class GaussianSet:
    """The GaussianModel tensors render() reads + the densification bookkeeping (scene/gaussian_model.py:46-131, 165-170)."""

    def __init__(self, tensors: Dict[str, torch.Tensor], deformation, device="cuda", sh_degree: int = 3):
        mk = lambda t: nn.Parameter(t.detach().to(device).float().contiguous(), requires_grad=True)
        self._xyz, self._features_dc, self._features_rest = mk(tensors["xyz"]), mk(tensors["features_dc"]), mk(tensors["features_rest"])
        self._opacity, self._scaling, self._rotation = mk(tensors["opacity"]), mk(tensors["scaling"]), mk(tensors["rotation"])
        self._deformation = deformation
        self.active_sh_degree, self.max_sh_degree = sh_degree, 3
        self.scaling_activation, self.opacity_activation = torch.exp, torch.sigmoid
        self.rotation_activation = torch.nn.functional.normalize
        self.reset_stats()

    def reset_stats(self):
        n, dev = self._xyz.shape[0], self._xyz.device
        self.xyz_gradient_accum = torch.zeros(n, 1, device=dev)
        self.denom = torch.zeros(n, 1, device=dev)
        self.max_radii2D = torch.zeros(n, device=dev)
        self._deformation_table = torch.ones(n, dtype=torch.bool, device=dev)
        self._deformation_accum = torch.zeros(n, 3, device=dev)

    @property
    def get_xyz(self):
        return self._xyz

    @property
    def get_features(self):
        return torch.cat((self._features_dc, self._features_rest), dim=1)

    @property
    def get_scaling(self):
        return torch.exp(self._scaling)

    @property
    def get_opacity(self):
        return torch.sigmoid(self._opacity)

    def named(self):
        return {"xyz": self._xyz, "f_dc": self._features_dc, "f_rest": self._features_rest, "opacity": self._opacity,
                "scaling": self._scaling, "rotation": self._rotation}

    def assign(self, d):
        self._xyz, self._features_dc, self._features_rest = d["xyz"], d["f_dc"], d["f_rest"]
        self._opacity, self._scaling, self._rotation = d["opacity"], d["scaling"], d["rotation"]


class DPTrainer:
    def __init__(self, gaussians: GaussianSet, opt: Optional[Namespace] = None, dist=None, world_size: int = 1, rank: int = 0,
                 spatial_lr_scale: float = 1.0, cameras_extent: float = 1.0, seed: int = 0):
        self.g, self.opt = gaussians, opt or default_opt()
        self.dist, self.world, self.rank = dist, world_size, rank
        self.spatial_lr_scale, self.extent, self.seed = spatial_lr_scale, cameras_extent, seed
        self.iteration = 0
        self.rebuilds = 0
        self.loss_accum = torch.zeros((), device=gaussians._xyz.device)
        self._rebuilt_this_step = False
        self._build_state(None)

    # ---- flat buffers -------------------------------------------------------------------------------------------
    def _build_state(self, carried: Optional[Dict[str, tuple]]):
        g, mod = self.g, self.g._deformation
        groups = [(n, [p]) for n, p in g.named().items()]
        flat = mod.flat_parameters()
        n_planes = len(mod.deformation_net.grid.grids) * 6
        groups += [("grid", flat[:n_planes]), ("deformation", flat[n_planes:])]
        old = getattr(self, "state", None)
        self.state = FlatState(groups, g._xyz.device)
        if old is not None:
            self.state.step_count = old.step_count
            for name in ("grid", "deformation"):      # network moments (and this step's gradients) carry over unchanged
                b0, e0 = old.segments[name]; b1, e1 = self.state.segments[name]
                self.state.exp_avg[b1:e1].copy_(old.exp_avg[b0:e0]); self.state.exp_avg_sq[b1:e1].copy_(old.exp_avg_sq[b0:e0])
                self.state.grad[b1:e1].copy_(old.grad[b0:e0])
        if carried is not None:
            for name, p in g.named().items():
                m, v = self.state.moments(p)
                m.copy_(carried[name][0]); v.copy_(carried[name][1])
        mod.fused_grad_accumulation = True            # network gradients accumulate straight into the flat buffer
        mod._sink_cache = None
        self.rebuilds += 1

    def learning_rates(self, iteration: int) -> Dict[str, float]:
        o, s = self.opt, self.spatial_lr_scale
        return {"xyz": expon_lr(iteration, o.position_lr_init * s, o.position_lr_final * s, 0, o.position_lr_delay_mult, o.position_lr_max_steps),
                "deformation": expon_lr(iteration, o.deformation_lr_init * s, o.deformation_lr_final * s, 0, o.deformation_lr_delay_mult, o.position_lr_max_steps),
                "grid": expon_lr(iteration, o.grid_lr_init * s, o.grid_lr_final * s, 0, o.deformation_lr_delay_mult, o.position_lr_max_steps),
                "f_dc": o.feature_lr, "f_rest": o.feature_lr / 20.0, "opacity": o.opacity_lr, "scaling": o.scaling_lr,
                "rotation": o.rotation_lr}

    # ---- one optimisation step (train.py:180-226, 259-292) ----------------------------------------------------------
    def step(self, cameras: Sequence, gt_images: Sequence[torch.Tensor], background: torch.Tensor, pipe, stage: str = "fine"):
        """cameras / gt_images: this rank's B views of the global batch.  Returns the (device) loss of this rank's views."""
        g, o = self.g, self.opt
        self.iteration += 1
        it = self.iteration
        B = len(cameras)
        self.state.zero_grad()
        self.loss_accum.zero_()
        dev = g._xyz.device
        radii_max = torch.zeros(g._xyz.shape[0], device=dev)
        vis_any = torch.zeros(g._xyz.shape[0], dtype=torch.bool, device=dev)
        m2d_grad = torch.zeros(g._xyz.shape[0], 3, device=dev)
        for cam, gt in zip(cameras, gt_images):
            out = render(cam, g, pipe, background, stage=stage)
            loss = losses.l1_loss(out["render"], gt[:3]) / B                       # mean over the concatenated batch (train.py:201)
            if o.lambda_dssim != 0:
                loss = loss + o.lambda_dssim * (1.0 - losses.ssim(out["render"], gt[:3])) / B
            loss.backward()
            self.loss_accum += loss.detach()
            radii_max = torch.maximum(radii_max, out["radii"].float())
            vis_any |= out["visibility_filter"]
            m2d_grad += out["viewspace_points"].grad
        if stage == "fine" and o.time_smoothness_weight != 0:
            # view-independent: computed identically on every rank, scaled so that the 1 / world of the reduction restores it
            w = float(self.world)
            losses.accumulate_regulation(g._deformation, o.time_smoothness_weight * w, o.l1_time_planes * w, o.plane_tv_weight * w,
                                         loss_accum=None)
        # ---- the step's ONE exchange: the flat gradient buffer, reduced in `comm_chunks` back-to-back slices so that Adam on
        #      slice i overlaps the reduction of slice i + 1 (the collective runs on the backend's own stream)
        works = None
        if self.dist is not None and self.world > 1:
            works = self._launch_allreduce()
        if it < o.densify_until_iter:
            # train.py:252-255 / gaussian_model.py:636-638 without the boolean-mask indexing (each `x[mask]` is a nonzero() ->
            # one host synchronisation per statement): the same values, masked arithmetically (radii and the statistics
            # are >= 0; an invisible Gaussian's screen-space gradient is exactly zero)
            vis_f = vis_any.unsqueeze(-1).to(g.denom.dtype)
            torch.maximum(g.max_radii2D, radii_max * vis_f.squeeze(-1), out=g.max_radii2D)
            g.xyz_gradient_accum.add_(torch.norm(m2d_grad[:, :2], dim=-1, keepdim=True) * vis_f)
            g.denom.add_(vis_f)
            if it % o.densification_interval == 0 or it % o.pruning_interval == 0:
                if works is not None:                  # a rebuild copies the reduced network gradients: finish the exchange first
                    for _, _, w in works:
                        self._wait(w)
                self._densify_and_prune(it, stage)
            if it % o.opacity_reset_interval == 0:
                self.reset_opacity()
        # after a densify / prune the per-Gaussian tensors are new Parameters without gradients: like the reference's
        # optimizer.step() (which skips grad-less parameters, train.py:290), this step only updates the network
        only = ("grid", "deformation") if self._rebuilt_this_step else None
        lrs = self.learning_rates(it)
        if works is None or self._rebuilt_this_step:
            if works is not None:
                for _, _, w in works:
                    self._wait(w)
            self.state.adam_step(lrs, grad_scale=1.0 / self.world, only=only)
        else:
            for i, (b, e, w) in enumerate(works):
                self._wait(w)                              # the current stream waits for slice i only
                self.state.adam_step(lrs, grad_scale=1.0 / self.world, span=(b, e), count_step=(i == 0))
        self._rebuilt_this_step = False
        return self.loss_accum

    comm_chunks = 4

    def _host_staged_collectives(self) -> bool:
        """gloo stages CUDA tensors through pinned host memory on its own streams (the CPU-side test configuration): it is
        handed finished buffers and its results are awaited on the host.  NCCL (the production path) is stream-ordered and
        needs no host synchronisation."""
        return self.state.device.type == "cuda" and self.dist.get_backend() != "nccl"

    def _sync_device(self):
        torch.cuda.synchronize(self.state.device)

    def _wait(self, work):
        work.wait()
        if self._host_staged_collectives():
            self._sync_device()

    def _launch_allreduce(self):
        st = self.state
        if self._host_staged_collectives():
            self._sync_device()
        k = max(1, int(self.comm_chunks))
        step = (st.numel // k + 3) // 4 * 4
        works, b = [], 0
        while b < st.numel:
            e = min(st.numel, b + step)
            works.append((b, e, self.dist.all_reduce(st.grad[b:e], op=self.dist.ReduceOp.SUM, async_op=True)))
            b = e
        return works

    def _global_stats(self):
        """(sum of ||grad means2D||, visible count, max radii) over ALL ranks.  The per-rank accumulators stay local (they
        keep accumulating until a densify / prune resets them), the reduced copies drive the decisions."""
        g = self.g
        if self.dist is None or self.world <= 1:
            return g.xyz_gradient_accum, g.denom, g.max_radii2D
        packed = torch.cat([g.xyz_gradient_accum.reshape(-1), g.denom.reshape(-1)])
        self.dist.all_reduce(packed, op=self.dist.ReduceOp.SUM)
        n = g.xyz_gradient_accum.numel()
        radii = g.max_radii2D.clone()
        self.dist.all_reduce(radii, op=self.dist.ReduceOp.MAX)
        return packed[:n].view_as(g.xyz_gradient_accum), packed[n:].view_as(g.denom), radii

    # ---- densification (gaussian_model.py:415-506; schedule train.py:259-285) -------------------------------------------
    def _thresholds(self, it):
        o = self.opt
        op_t = o.opacity_threshold_fine_init - it * (o.opacity_threshold_fine_init - o.opacity_threshold_fine_after) / o.densify_until_iter
        gr_t = o.densify_grad_threshold_fine_init - it * (o.densify_grad_threshold_fine_init - o.densify_grad_threshold_after) / o.densify_until_iter
        return op_t, gr_t

    @torch.no_grad()
    def _densify_and_prune(self, it, stage):
        g, o = self.g, self.opt
        n = g._xyz.shape[0]
        op_t, gr_t = self._thresholds(it)
        size_threshold = 20 if it > o.opacity_reset_interval else None
        changed = False
        accum, denom, radii = self._global_stats()
        if it > o.densify_from_iter and it % o.densification_interval == 0 and n < o.max_gaussians:
            changed |= self.densify(gr_t, it, accum, denom)
        if it > o.pruning_from_iter and it % o.pruning_interval == 0 and g._xyz.shape[0] > o.min_gaussians_for_prune:
            mask = (g.get_opacity < op_t).squeeze(-1)
            if size_threshold:
                if radii.shape[0] != mask.shape[0]:          # a densify just happened: its postfix reset the radii (as upstream)
                    radii = g.max_radii2D
                mask |= radii > size_threshold
                mask |= g.get_scaling.max(dim=1).values > 0.1 * self.extent
            changed |= self.prune_points(mask)
        return changed

    @torch.no_grad()
    def densify(self, grad_threshold: float, iteration: int, accum: Optional[torch.Tensor] = None,
                denom: Optional[torch.Tensor] = None) -> bool:
        g = self.g
        grads = (g.xyz_gradient_accum if accum is None else accum) / (g.denom if denom is None else denom)
        grads[grads.isnan()] = 0.0
        small = g.get_scaling.max(dim=1).values <= self.opt.percent_dense * self.extent
        clone = (torch.norm(grads, dim=-1) >= grad_threshold) & small
        split = (grads.squeeze(-1) >= grad_threshold) & ~small
        if not bool(clone.any()) and not bool(split.any()):
            return False
        named = g.named()
        N = 2
        # the split noise must be identical on every rank: generator seeded by (seed, iteration), drawn on the device
        gen = torch.Generator(device=g._xyz.device).manual_seed((self.seed * 1_000_003 + iteration) & 0x7FFFFFFF)
        stds = g.get_scaling[split].repeat(N, 1)
        samples = torch.randn(stds.shape, generator=gen, device=stds.device) * stds
        rots = build_rotation(g._rotation[split]).repeat(N, 1, 1)
        new = {
            "xyz": torch.cat([g._xyz[clone], torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + g._xyz[split].repeat(N, 1)]),
            "f_dc": torch.cat([g._features_dc[clone], g._features_dc[split].repeat(N, 1, 1)]),
            "f_rest": torch.cat([g._features_rest[clone], g._features_rest[split].repeat(N, 1, 1)]),
            "opacity": torch.cat([g._opacity[clone], g._opacity[split].repeat(N, 1)]),
            "scaling": torch.cat([g._scaling[clone], torch.log(g.get_scaling[split].repeat(N, 1) / (0.8 * N))]),
            "rotation": torch.cat([g._rotation[clone], g._rotation[split].repeat(N, 1)]),
        }
        keep = ~split                                   # the split parents are removed (prune_filter, gaussian_model.py:448-449)
        self._replace({k: torch.cat([named[k].data[keep], new[k]]) for k in named},
                      {k: tuple(torch.cat([m[keep], torch.zeros_like(new[k])]) for m in self.state.moments(named[k])) for k in named})
        return True

    @torch.no_grad()
    def prune_points(self, mask: torch.Tensor) -> bool:
        if not bool(mask.any()):
            return False
        named = self.g.named()
        keep = ~mask
        self._replace({k: named[k].data[keep] for k in named},
                      {k: tuple(m[keep] for m in self.state.moments(named[k])) for k in named})
        return True

    @torch.no_grad()
    def reset_opacity(self):
        """gaussian_model.py:270-273: opacities clamped to 0.01, their Adam moments zeroed"""
        g = self.g
        g._opacity.data.copy_(inverse_sigmoid(torch.minimum(g.get_opacity, torch.ones_like(g._opacity) * 0.01)))
        m, v = self.state.moments(g._opacity)
        m.zero_(); v.zero_()

    def _replace(self, tensors: Dict[str, torch.Tensor], moments: Dict[str, tuple]):
        g = self.g
        tensors = {k: v.clone() for k, v in tensors.items()}
        moments = {k: tuple(x.clone() for x in v) for k, v in moments.items()}
        g.assign({k: nn.Parameter(v.contiguous(), requires_grad=True) for k, v in tensors.items()})
        g.reset_stats()                                 # densification_postfix / prune_points reset the statistics
        self._build_state(moments)
        self._rebuilt_this_step = True
