"""Drop-in for ``scene.deformation.deform_network`` (/root/reference/scene/deformation.py:161-216) backed by
the sm_90a kernels of libg4d.so.

Contract kept (SURVEY.md §8b, App. B.4):
  * ctor reads the same ``args`` fields; ``forward(point, scales, rotations, opacity, shs, times_sel)`` -> 5-tuple;
  * ``state_dict()`` keys / shapes identical to the reference (planes ``[1,C,H,W]``, all five heads and the dead
    ``timenet`` always present), so reference checkpoints load and ours load in the reference;
  * ``get_mlp_parameters()`` / ``get_grid_parameters()`` split by ``"grid" in name``;
    ``deformation_net.set_aabb`` / ``get_aabb`` / ``deformation_net.grid.grids`` as used by
    scene/__init__.py:83 and scene/gaussian_model.py:539-564;
  * parameters are ordinary leaf ``nn.Parameter`` objects that an optimizer updates in place.

Kernel-native storage: every plane Parameter is a ``[1,C,H,W]`` tensor in ``torch.channels_last`` memory, i.e.
physically ``[H][W][C]`` -- the kernels read it (and scatter gradients into a same-layout tensor) directly, no
per-step transposes; shape-wise it is indistinguishable from the reference's tensor.
"""
from __future__ import annotations

import ctypes as C
import itertools
from typing import List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.init as init

from . import _lib

_VERSION_COUNTER = itertools.count(1)   # process-global: a fresh module can never reuse a (version, pointer) pair

_HEADS = ("pos_deform", "scales_deform", "rotations_deform", "opacity_deform", "shs_deform")
_HEAD_OUT = (3, 3, 4, 1, 48)


class HexPlaneField(nn.Module):
    """Parameter container mirroring scene/hexplane.py:109-183 (no compute here; the kernels sample the planes)."""

    def __init__(self, bounds, planeconfig, multires):
        super().__init__()
        aabb = torch.tensor([[bounds, bounds, bounds], [-bounds, -bounds, -bounds]], dtype=torch.float32)
        self.aabb = nn.Parameter(aabb, requires_grad=False)
        self.grid_config = [planeconfig]
        self.multiscale_res_multipliers = list(multires)
        self.concat_features = True
        self.grids = nn.ModuleList()
        self.feat_dim = 0
        cdim = planeconfig["output_coordinate_dim"]
        for res in self.multiscale_res_multipliers:
            reso = [r * res for r in planeconfig["resolution"][:3]] + list(planeconfig["resolution"][3:])
            gp = nn.ParameterList()
            for comb in itertools.combinations(range(planeconfig["input_coordinate_dim"]), planeconfig["grid_dimensions"]):
                t = torch.empty([1, cdim] + [reso[cc] for cc in comb[::-1]]).contiguous(memory_format=torch.channels_last)
                if 3 in comb:
                    init.ones_(t)           # time planes start at 1 (hexplane.py:64-65)
                else:
                    init.uniform_(t, a=0.1, b=0.5)
                gp.append(nn.Parameter(t))
            self.feat_dim += cdim
            self.grids.append(gp)

    @property
    def get_aabb(self):
        return self.aabb[0], self.aabb[1]

    def set_aabb(self, xyz_max, xyz_min):
        aabb = torch.tensor([list(xyz_max), list(xyz_min)], dtype=torch.float32)
        self.aabb = nn.Parameter(aabb.to(self.aabb.device), requires_grad=False)


class Deformation(nn.Module):
    """Mirrors scene/deformation.py:16-160 for the live configuration (no_grid / grid_pe / empty_voxel /
    static_mlp / apply_rotation are dead options in every shipped config and are rejected).  ``feature_out`` is built as
    the reference builds it: ``Linear(F, W)`` followed by ``[ReLU, Linear(W, W)] * (D - 1)`` (D = 0 and 1 are the same
    network), so state_dict keys and shapes match for every depth the kernels take."""

    def __init__(self, D=8, W=256, args=None):
        super().__init__()
        self.D, self.W, self.args = D, W, args
        if getattr(args, "no_grid", False) or getattr(args, "grid_pe", 0) or getattr(args, "empty_voxel", False) or \
                getattr(args, "static_mlp", False) or getattr(args, "apply_rotation", False):
            raise NotImplementedError("no_grid / grid_pe / empty_voxel / static_mlp / apply_rotation are dead options "
                                      "in the reference configs and are not provided by the g4d path")
        if not 0 <= D <= _lib.MAX_DEPTH:
            raise NotImplementedError("defor_depth must be in 0..%d (the trunk layers the g4d kernels take), got %d"
                                      % (_lib.MAX_DEPTH, D))
        if W not in (64, 128):
            raise NotImplementedError("net_width must be 64 or 128, got %d: one fp32 W x W weight image of a wider network "
                                      "does not fit in an SM's shared memory (the FFMA network kernels stage one whole)" % W)
        self.grid = HexPlaneField(args.bounds, args.kplanes_config, args.multires)
        trunk = [nn.Linear(self.grid.feat_dim, W)]
        for _ in range(D - 1):
            trunk += [nn.ReLU(), nn.Linear(W, W)]
        self.feature_out = nn.Sequential(*trunk)
        for name, k in zip(_HEADS, _HEAD_OUT):
            setattr(self, name, nn.Sequential(nn.ReLU(), nn.Linear(W, W), nn.ReLU(), nn.Linear(W, k)))
        self.ratio = 0

    @property
    def get_aabb(self):
        return self.grid.get_aabb

    def set_aabb(self, xyz_max, xyz_min):
        self.grid.set_aabb(xyz_max, xyz_min)

    @property
    def get_empty_ratio(self):
        return self.ratio

    def get_mlp_parameters(self):
        return [p for n, p in self.named_parameters() if "grid" not in n]

    def get_grid_parameters(self):
        return [p for n, p in self.named_parameters() if "grid" in n]


def _initialize_weights(m):
    if isinstance(m, nn.Linear):
        init.xavier_uniform_(m.weight, gain=1)   # deformation.py:218-224 (bias keeps the default init)


class deform_network(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.args = args
        times_ch = 2 * args.timebase_pe + 1
        self.timenet = nn.Sequential(nn.Linear(times_ch, args.timenet_width), nn.ReLU(),
                                     nn.Linear(args.timenet_width, args.timenet_output))   # dead in the reference too
        self.deformation_net = Deformation(W=args.net_width, D=args.defor_depth, args=args)
        self.register_buffer('time_poc', torch.FloatTensor([(2 ** i) for i in range(args.timebase_pe)]))
        self.register_buffer('pos_poc', torch.FloatTensor([(2 ** i) for i in range(args.posebase_pe)]))
        self.register_buffer('rotation_scaling_poc', torch.FloatTensor([(2 ** i) for i in range(args.scale_rotation_pe)]))
        self.register_buffer('opacity_poc', torch.FloatTensor([(2 ** i) for i in range(args.opacity_pe)]))
        self.apply(_initialize_weights)
        self._version_seen = None
        self._param_version = 0
        self._dirty = False
        self._flat_cache = None          # the Parameter objects in C-ABI order (nn.Module container indexing is slow: ~90 calls per render)
        self._cparams_cache = None       # (key, struct, keep): the ctypes struct is rebuilt only when a pointer / the head mask changes

    # ---- reference surface -------------------------------------------------------------------------
    @property
    def get_aabb(self):
        return self.deformation_net.get_aabb

    @property
    def get_empty_ratio(self):
        return self.deformation_net.get_empty_ratio

    def get_mlp_parameters(self):
        return self.deformation_net.get_mlp_parameters() + list(self.timenet.parameters())

    def get_grid_parameters(self):
        return self.deformation_net.get_grid_parameters()

    def forward(self, point, scales=None, rotations=None, opacity=None, shs=None, times_sel=None):
        return self.forward_dynamic(point, scales, rotations, opacity, shs, times_sel)

    def forward_dynamic(self, point, scales=None, rotations=None, opacity=None, shs=None, times_sel=None):
        t, times = classify_times(times_sel, point.shape[0])
        flat = self.flat_parameters()
        outs = _DeformFunction.apply(self, t, times, torch.is_grad_enabled(), point, scales, rotations, opacity, shs, *flat)
        pts, sc, rot, op, sh = outs
        a = self.args
        # inactive heads hand the input tensor back, exactly like the reference (deformation.py:106-145)
        return (point if a.no_dx else pts, scales if a.no_ds else sc, rotations if a.no_dr else rot,
                opacity if a.no_do else op, shs if a.no_dshs else sh)

    # ---- plumbing for the C-ABI ---------------------------------------------------------------------
    def head_mask(self) -> int:
        a = self.args
        return ((0 if a.no_dx else _lib.HEAD_POS) | (0 if a.no_ds else _lib.HEAD_SCALES) | (0 if a.no_dr else _lib.HEAD_ROT)
                | (0 if a.no_do else _lib.HEAD_OPACITY) | (0 if a.no_dshs else _lib.HEAD_SHS))

    def trunk_layers(self) -> List[nn.Linear]:
        """feature_out.{2j} for j = 1 .. D-1: the trunk layers behind feature_out.0"""
        return list(self.deformation_net.feature_out)[2::2]

    def flat_parameters(self) -> List[torch.Tensor]:
        """planes (level-major), w0, b0, then (w1, b1, w2, b2) per head, then (w, b) per trunk layer -- the order
        _DeformFunction uses.
        The list of Parameter OBJECTS is cached (they survive .to() / load_state_dict / optimizer steps, which all write in
        place); ``invalidate_cache()`` drops it after module surgery."""
        if self._flat_cache is None:
            net = self.deformation_net
            out = [p for lvl in net.grid.grids for p in lvl]
            out += [net.feature_out[0].weight, net.feature_out[0].bias]
            for name in _HEADS:
                seq = getattr(net, name)
                out += [seq[1].weight, seq[1].bias, seq[3].weight, seq[3].bias]
            for lin in self.trunk_layers():
                out += [lin.weight, lin.bias]
            self._flat_cache = out
        return list(self._flat_cache)

    def _apply(self, fn, *a, **k):       # .cuda() / .float() / .to(): pointers change, and so may the Parameter objects
        self._flat_cache = None
        self._cparams_cache = None
        return super()._apply(fn, *a, **k)

    def _ensure_layout(self):
        for lvl in self.deformation_net.grid.grids:
            for p in lvl:
                if not p.is_contiguous(memory_format=torch.channels_last) or p.dtype != torch.float32:
                    p.data = p.data.float().contiguous(memory_format=torch.channels_last)
        for p in self.flat_parameters()[len(self.deformation_net.grid.grids) * 6:]:
            if not p.is_contiguous() or p.dtype != torch.float32:
                p.data = p.data.float().contiguous()

    def param_version(self, fresh: bool = False) -> int:
        """Key of the library's packed weight images (transposes / FP16 / BF16 operand images of the MLP weights).

        It changes whenever a parameter tensor was replaced or modified through an op that bumps ``Tensor._version``
        (``load_state_dict``, ``copy_``, foreach / plain optimizers), whenever the head mask changes, after
        ``invalidate_cache()``, and -- ``fresh=True`` -- on EVERY forward that a backward can follow: fused optimizers
        (``torch.optim.Adam(fused=True)``) and writes through ``param.data`` update the weights WITHOUT bumping
        ``_version``, so in training the images are simply rebuilt per forward (three tiny kernels over ~100k floats)."""
        sig = (self.head_mask(),) + tuple((p.data_ptr(), p._version) for p in self.flat_parameters())
        # a training forward is normally followed by an optimizer step the version counters may not show: the first
        # no_grad forward after it refreshes once more (self._dirty)
        if fresh or self._dirty or sig != self._version_seen:
            self._version_seen = sig
            self._param_version = next(_VERSION_COUNTER)
        self._dirty = fresh
        return self._param_version

    def invalidate_cache(self):
        """Call after changing weights in a way autograd's version counters cannot see (``p.data.copy_``, a custom fused
        optimizer) while rendering under ``torch.no_grad()``; training forwards refresh the images on their own."""
        self._version_seen = None
        self._flat_cache = None
        self._cparams_cache = None

    def c_params(self, keep: list, fresh: bool = False) -> _lib.DeformParams:
        self._ensure_layout()
        net = self.deformation_net
        key = (self.head_mask(), net.grid.aabb.data_ptr()) + tuple(p.data_ptr() for p in self.flat_parameters())
        if self._cparams_cache is not None and self._cparams_cache[0] == key:
            _, prm0, keep0 = self._cparams_cache
            prm = _lib.DeformParams.from_buffer_copy(prm0)       # callers keep their struct (its version) for the backward
            keep.extend(keep0)
            prm.version = self.param_version(fresh)
            return prm
        keep_local = []
        prm = self._build_c_params(keep_local)
        self._cparams_cache = (key, _lib.DeformParams.from_buffer_copy(prm), keep_local)
        keep.extend(keep_local)
        prm.version = self.param_version(fresh)
        return prm

    def _build_c_params(self, keep: list) -> _lib.DeformParams:
        net = self.deformation_net
        kc = net.grid.grid_config[0]
        prm = _lib.DeformParams()
        prm.levels = len(net.grid.grids)
        prm.channels = int(kc["output_coordinate_dim"])
        prm.net_width = int(net.W)
        prm.head_mask = self.head_mask()
        base = list(kc["resolution"])
        for l, m in enumerate(net.grid.multiscale_res_multipliers):
            for a in range(3):
                prm.res[l][a] = int(base[a] * m)
            prm.res[l][3] = int(base[3])
            for k in range(6):
                p = net.grid.grids[l][k]
                if not p.is_cuda:
                    raise RuntimeError("deform_network parameters must live on a CUDA device (no CPU fallback)")
                prm.planes[l][k] = p.data_ptr()
        aabb = _lib.cuda_f32(net.grid.aabb, "aabb")
        keep.append(aabb)
        prm.aabb = aabb.data_ptr()
        prm.w0 = net.feature_out[0].weight.data_ptr()
        prm.b0 = net.feature_out[0].bias.data_ptr()
        for h, name in enumerate(_HEADS):
            seq = getattr(net, name)
            prm.w1[h], prm.b1[h] = seq[1].weight.data_ptr(), seq[1].bias.data_ptr()
            prm.w2[h], prm.b2[h] = seq[3].weight.data_ptr(), seq[3].bias.data_ptr()
        prm.depth = int(net.D)
        for j, lin in enumerate(self.trunk_layers()):
            prm.wt[j], prm.bt[j] = lin.weight.data_ptr(), lin.bias.data_ptr()
        return prm

    def alloc_grads(self) -> List[torch.Tensor]:
        """Zeroed gradient sinks for flat_parameters(): ONE allocation + ONE memset, handed out as views with the
        parameters' own memory layout (channel-last for the planes) -- instead of 33 zeros_like launches."""
        flat = self.flat_parameters()
        total = sum(p.numel() for p in flat)
        buf = torch.zeros(total, device=flat[0].device, dtype=torch.float32)
        out, off = [], 0
        for p in flat:
            n = p.numel()
            seg = buf[off:off + n]
            if p.dim() == 4 and not p.is_contiguous():      # channels_last plane [1,C,H,W]
                b, c, h, w = p.shape
                out.append(seg.view(b, h, w, c).permute(0, 3, 1, 2))
            else:
                out.append(seg.view(p.shape))
            off += n
        return out

    def alloc_plane_grads(self) -> List[torch.Tensor]:
        """zeroed channel-last gradient sinks for the planes only (one allocation), level-major"""
        planes = [p for lvl in self.deformation_net.grid.grids for p in lvl]
        buf = torch.zeros(sum(p.numel() for p in planes), device=planes[0].device, dtype=torch.float32)
        out, off = [], 0
        for p in planes:
            b, c, h, w = p.shape
            out.append(buf[off:off + p.numel()].view(b, h, w, c).permute(0, 3, 1, 2))
            off += p.numel()
        return out

    # Opt-in (default off, autograd semantics untouched): when True and every parameter already owns a `.grad` with the
    # parameter's own memory layout (e.g. views of a dp.FlatGradBucket), the backward kernels -- which ACCUMULATE with
    # atomics anyway -- add straight into those tensors and autograd receives None for the parameters: no per-view
    # zero-filled staging buffer and no 47 AccumulateGrad `add_` launches per view.
    fused_grad_accumulation = False

    def grad_sinks(self) -> Optional[List[torch.Tensor]]:
        """the parameters' own .grad tensors when fused accumulation is possible, else None.  The plane scatter adds float4s,
        so a spatial plane's .grad that is not 16-byte aligned (a view into a FlatGradBucket behind a parameter of 4k+1
        floats, say) takes the staging path."""
        if not self.fused_grad_accumulation:
            return None
        flat = self.flat_parameters()
        cache = getattr(self, "_sink_cache", None)
        if cache is not None and len(cache[0]) == len(flat) and all(p.grad is g for p, g in zip(flat, cache[0])):
            return cache[0]                       # same .grad objects as last time: already validated
        out = []
        nplanes = len(self.deformation_net.grid.grids) * 6
        for i, p in enumerate(flat):
            g = p.grad
            if g is None or g.dtype != torch.float32 or g.shape != p.shape or g.stride() != p.stride() or g.device != p.device:
                return None
            if i < nplanes and i % 6 in (0, 1, 3) and g.data_ptr() % 16:
                return None
            out.append(g)
        self._sink_cache = [out, None]
        return out

    def c_grad_sinks(self) -> Tuple[_lib.DeformGrads, List[Optional[torch.Tensor]]]:
        """(C-ABI gradient sinks of flat_parameters(), the gradients autograd receives for them): the parameters' own
        .grad and Nones when fused accumulation is possible (``grad_sinks``), else ``alloc_grads()`` and those tensors."""
        sinks = self.grad_sinks()
        if sinks is not None:
            return self.c_grads(sinks), [None] * len(sinks)
        grads = self.alloc_grads()
        return self.c_grads(grads), grads

    def c_grads(self, grads: List[torch.Tensor]) -> _lib.DeformGrads:
        cache = getattr(self, "_sink_cache", None)
        if cache is not None and grads is cache[0] and cache[1] is not None:
            return cache[1]
        g = self._build_c_grads(grads)
        if cache is not None and grads is cache[0]:
            cache[1] = g
        return g

    def c_plane_grads(self, grads: List[torch.Tensor]) -> _lib.DeformGrads:
        """C-ABI sinks for the planes only: grads[:6 * levels], level-major; the MLP sinks stay NULL."""
        g = _lib.DeformGrads()
        for i in range(len(self.deformation_net.grid.grids) * 6):
            g.planes[i // 6][i % 6] = grads[i].data_ptr()
        return g

    def _build_c_grads(self, grads: List[torch.Tensor]) -> _lib.DeformGrads:
        g = self.c_plane_grads(grads)
        i = len(self.deformation_net.grid.grids) * 6
        g.w0, g.b0 = grads[i].data_ptr(), grads[i + 1].data_ptr()
        i += 2
        for h in range(5):
            g.w1[h], g.b1[h], g.w2[h], g.b2[h] = (grads[i + j].data_ptr() for j in range(4))
            i += 4
        for j in range(len(self.trunk_layers())):
            g.wt[j], g.bt[j] = grads[i].data_ptr(), grads[i + 1].data_ptr()
            i += 2
        return g


def scalar_time(times_sel) -> float:
    """The time of row 0 of ``times_sel``: the one timestamp of a camera.  The renderer builds an [N,1] tensor whose rows are
    identical (gaussian_renderer/__init__.py:52); python floats, 0-d tensors and the int 0 all occur (SURVEY.md §8b 'Input
    quirks').  ``deform_network.forward`` takes rows that differ too (``classify_times``)."""
    if times_sel is None:
        raise RuntimeError("times_sel is required (forward_static is a dead path in the reference)")
    if torch.is_tensor(times_sel):
        if times_sel.numel() == 0:
            return 0.0
        return float(times_sel.reshape(-1)[0].item())
    return float(times_sel)


def classify_times(times_sel, n: int):
    """(t, None): every one of the n rows at the time t -- a Python number, a one-element tensor, or a tensor whose elements
    are all equal and that does not require grad (one host sync, as ``scalar_time``'s).  Such a tensor takes this path
    whatever its element count, an empty one included (t = 0), exactly as before per-row times existed, so no caller of the
    one-time path sees a new error.  (None, times_sel): one time per row -- any other tensor with n elements ([n] or [n, 1],
    any real dtype and device), which receives dL/dt when it requires grad.  Any other tensor -- elements that differ, or
    that require grad, in a count that is neither 1 nor n -- raises ValueError."""
    if not torch.is_tensor(times_sel) or times_sel.numel() == 1:
        return scalar_time(times_sel), None
    if not times_sel.requires_grad:
        if times_sel.numel() == 0:
            return scalar_time(times_sel), None
        lo, hi = torch.aminmax(times_sel.detach().reshape(-1))
        lo, hi = torch.stack([lo, hi]).tolist()
        if lo == hi:
            return float(lo), None
    if times_sel.numel() != n:
        raise ValueError("times_sel must hold one time or one per row: %d elements for %d rows" % (times_sel.numel(), n))
    return None, times_sel


class _DeformFunction(torch.autograd.Function):
    """t: the time of every row, or times (a tensor of N elements, t None): one time per row"""

    @staticmethod
    def forward(ctx, module: deform_network, t: Optional[float], times, grad_mode: bool, xyz, scales, rotations, opacity, shs,
                *params):
        lib = _lib.load()
        dev = xyz.device
        n = xyz.shape[0]
        x, s, r, o, sh = (_lib.cuda_f32(v, nm) for v, nm in ((xyz, "point"), (scales, "scales"), (rotations, "rotations"),
                                                             (opacity, "opacity"), (shs, "shs")))
        keep = []
        needs_bwd = grad_mode and any(ctx.needs_input_grad)      # (grad mode is always off INSIDE Function.forward)
        prm = module.c_params(keep, fresh=needs_bwd)
        hm = prm.head_mask
        if sh is not None and (hm & _lib.HEAD_SHS):     # the SH head deforms exactly 16 coefficients per Gaussian
            _lib.check_sh_degree(_lib.sh_coeffs(sh, n, "shs"), 0, hm)
        ox = torch.empty_like(x)
        os_ = torch.empty_like(s) if s is not None else None
        orr = torch.empty_like(r) if r is not None else None
        oo = torch.empty_like(o) if o is not None else None
        osh = torch.empty_like(sh) if (sh is not None and (hm & _lib.HEAD_SHS)) else None
        ptr = lambda v: v.data_ptr() if v is not None else None
        # what autograd would save for the ReLU backward: one sign bit per hidden unit (only when a backward can follow)
        relu_bits = torch.empty(_lib.relu_bits_words(n), device=dev, dtype=torch.int32) if needs_bwd else None
        # per-row times as a contiguous fp32 device copy (N = 0: nothing to sample, the one-time call does it)
        tt = times.detach().reshape(-1).to(device=dev, dtype=torch.float32).contiguous() if times is not None and n else None
        with torch.cuda.device(dev):
            ws = _lib.workspace_of(dev)
            if tt is None:
                _lib.check(lib.g4d_deform_forward(ws.handle, C.byref(prm), n, ptr(x), ptr(s), ptr(r), ptr(o), ptr(sh),
                                                  float(t or 0.0), ptr(ox), ptr(os_), ptr(orr), ptr(oo), ptr(osh), ptr(relu_bits),
                                                  _lib.stream_of(dev)), "g4d_deform_forward")
            else:
                _lib.check(lib.g4d_deform_forward_times(ws.handle, C.byref(prm), n, ptr(x), ptr(s), ptr(r), ptr(o), ptr(sh),
                                                        ptr(tt), ptr(ox), ptr(os_), ptr(orr), ptr(oo), ptr(osh), ptr(relu_bits),
                                                        _lib.stream_of(dev)), "g4d_deform_forward_times")
        ctx.module, ctx.t, ctx.n = module, float(t or 0.0), n
        ctx.per_row = times is not None
        ctx.times_meta = (times.shape, times.dtype, times.device) if times is not None else None
        ctx.relu_bits = relu_bits
        # the times are saved like xyz: every backward of the graph reads them, and autograd's version check refuses a
        # backward after either was changed in place
        ctx.save_for_backward(x, tt)
        ctx.has = (s is not None, r is not None, o is not None, sh is not None)
        outs = (ox, os_ if os_ is not None else x.new_zeros(0), orr if orr is not None else x.new_zeros(0),
                oo if oo is not None else x.new_zeros(0), osh if osh is not None else x.new_zeros(0))
        return outs

    @staticmethod
    def backward(ctx, g_xyz, g_sc, g_rot, g_op, g_sh):
        lib = _lib.load()
        module, t, n = ctx.module, ctx.t, ctx.n
        x, tt = ctx.saved_tensors
        dev = x.device
        keep = []
        prm = module.c_params(keep, fresh=True)      # (keeps the "an optimizer step may follow" mark, see param_version)
        hm = prm.head_mask
        cg, pgrads = module.c_grad_sinks()

        def gin(g, shape_ok):
            if g is None or not shape_ok or g.numel() == 0:
                return None
            return _lib.cuda_f32(g, "grad")
        has_s, has_r, has_o, has_sh = ctx.has
        go_x = gin(g_xyz, True)
        go_s, go_r, go_o = gin(g_sc, has_s), gin(g_rot, has_r), gin(g_op, has_o)
        go_sh = gin(g_sh, has_sh and bool(hm & _lib.HEAD_SHS))
        gi_x = torch.empty(n, 3, device=dev)
        gi_s = torch.empty(n, 3, device=dev) if has_s else None
        gi_r = torch.empty(n, 4, device=dev) if has_r else None
        gi_o = torch.empty(n, 1, device=dev) if has_o else None
        gi_sh = torch.empty(n, 16, 3, device=dev) if (has_sh and (hm & _lib.HEAD_SHS)) else None
        ptr = lambda v: v.data_ptr() if v is not None else None
        per_row = ctx.per_row and n > 0      # (N = 0: the forward made the one-time call, which launches nothing per row)
        g_t = torch.empty(n, device=dev) if ctx.needs_input_grad[2] else None
        with torch.cuda.device(dev):
            ws = _lib.workspace_of(dev)
            if not per_row:
                _lib.check(lib.g4d_deform_backward(ws.handle, C.byref(prm), C.byref(cg), n, ptr(x), float(t), ptr(go_x),
                                                   ptr(go_s), ptr(go_r), ptr(go_o), ptr(go_sh), ptr(gi_x), ptr(gi_s), ptr(gi_r),
                                                   ptr(gi_o), ptr(gi_sh), ptr(ctx.relu_bits), _lib.stream_of(dev)),
                           "g4d_deform_backward")
            else:
                _lib.check(lib.g4d_deform_backward_times(ws.handle, C.byref(prm), C.byref(cg), n, ptr(x), ptr(tt), ptr(go_x),
                                                         ptr(go_s), ptr(go_r), ptr(go_o), ptr(go_sh), ptr(gi_x), ptr(gi_s),
                                                         ptr(gi_r), ptr(gi_o), ptr(gi_sh), ptr(g_t), ptr(ctx.relu_bits),
                                                         _lib.stream_of(dev)), "g4d_deform_backward_times")
        ctx.relu_bits = None      # a second backward through the graph derives the ReLU signs itself, as the C-ABI allows
        if g_t is not None:   # dL/dt in the shape, dtype and device of times_sel
            times = ctx.times_meta
            g_t = g_t.reshape(times[0]).to(device=times[2], dtype=times[1])
        return (None, None, g_t, None, gi_x, gi_s, gi_r, gi_o, gi_sh) + tuple(pgrads)
