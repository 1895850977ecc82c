"""CUDA-graph capture of no-grad rendering: ``render()`` and ``render_cameras()`` recorded once and replayed per call.

A replay re-runs the device work of a render with no host work in between: no C-ABI structs rebuilt, no weight-image
decision, no host synchronisation.  What changes from one call to the next -- the view and projection matrices, the camera
centre and the timestamp -- goes through one pinned staging block into device memory the captured kernels read
(``G4DCamera.d_*`` and ``g4d_context_set_time_source``).  Everything else is fixed by the template the graph was built
from: the model's tensors (their storage; in-place updates are seen), the image size, FoV and SH degree of every view, the
background and the stage.

The graph owns a private workspace and its contexts, frozen after the capture, so that no eager call can move a buffer
the graph points at.  Forwards run in no-sync mode (G4D_OPT_SYNC_MODE = 0): the instance capacity is learnt from the
template views, and a replay whose views need more instances gives incomplete images.  ``check()`` reports that (and the
FP16x2 range flag of the tensor-core network) as ``G4DError``.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import List, Sequence

import torch

from . import _lib
from .deformation import deform_network, scalar_time
from .rasterizer import camera_from_settings
from .renderer import _stage_module, _time_bits, _zero_points, settings_from_camera

_VIEW_FLOATS = 36        # per view in the staging block: view matrix [16], projection matrix [16], camera centre [3], time
ERR_OVERFLOW = -5        # G4D_ERR_OVERFLOW


class ViewBlock:
    """The device block captured kernels read a call's views from -- per view its view matrix [16], projection matrix [16],
    camera centre [3] and time [1], then ``extra`` floats -- and its pinned host twin: ``stage`` writes host values into the
    twin, copies it over in one host-to-device copy, and copies device tensors device to device behind it."""

    def __init__(self, dev: torch.device, k: int, extra: int = 0):
        self.k, self.extra_at = k, k * _VIEW_FLOATS
        self.block = torch.zeros(k * _VIEW_FLOATS + extra, device=dev, dtype=torch.float32)
        self._staging = torch.zeros(k * _VIEW_FLOATS + extra, dtype=torch.float32, pin_memory=True)
        self._staging_np = self._staging.numpy()
        self._staged = torch.cuda.Event()

    def view(self, i: int):
        """view i's (view matrix [4,4], projection matrix [4,4], camera centre [3]): views of the block"""
        o = i * _VIEW_FLOATS
        b = self.block
        return b[o:o + 16].view(4, 4), b[o + 16:o + 32].view(4, 4), b[o + 32:o + 35]

    def time_ptr(self, i: int) -> int:
        return self.block.data_ptr() + 4 * (i * _VIEW_FLOATS + 35)

    def stage(self, views: Sequence, extra: Sequence = ()) -> List[float]:
        """Views and ``extra`` ((offset past the views, tensor or numpy array), ...) into the block; returns the views' times."""
        times = []
        dev_copies = []
        self._staged.synchronize()          # the previous call's copy has read the staging block
        st = self._staging_np
        for i, v in enumerate(views):
            if isinstance(v, dict):
                raise NotImplementedError("PanopticSports cameras are not supported by a CUDA graph")
            times.append(scalar_time(v.time))
            o = i * _VIEW_FLOATS
            for j, (t, w) in enumerate(((v.world_view_transform, 16), (v.full_proj_transform, 16), (v.camera_center, 3))):
                t = t if torch.is_tensor(t) else torch.as_tensor(t, dtype=torch.float32)
                if t.numel() != w:
                    raise RuntimeError("camera matrix has %d elements, expected %d" % (t.numel(), w))
                if t.is_cuda:
                    dev_copies.append((o + 16 * j, w, t))
                else:
                    st[o + 16 * j:o + 16 * j + w] = t.detach().reshape(-1).float().numpy()
            st[o + 35] = times[-1]
        for off, t in extra:
            o = self.extra_at + off
            if torch.is_tensor(t) and t.is_cuda:
                dev_copies.append((o, t.numel(), t))
            else:
                t = t.detach().reshape(-1).float().numpy() if torch.is_tensor(t) else t.reshape(-1)
                st[o:o + t.size] = t
        stream = torch.cuda.current_stream(self.block.device)
        self.block.copy_(self._staging, non_blocking=True)
        self._staged.record(stream)
        for o, w, t in dev_copies:
            self.block[o:o + w].copy_(t.detach().reshape(-1))
        return times


def status_error(s: _lib.GraphStatus):
    """The G4DError a graph status reports (None: nothing to report)."""
    if s.overflows:
        return _lib.G4DError("graphed render failed (code %d): %d replayed view(s) needed up to %d tile instances, more than "
                             "the capacity learnt at capture; their images are incomplete (build the graph with a larger "
                             "min_capacity)" % (ERR_OVERFLOW, s.overflows, s.max_instances))
    if s.f16_range:
        return _lib.G4DError("graphed render failed (code %d): an FP16x2 tensor-core launch met a value outside the f16 "
                             "operand range; its results were saturated (G4D_OPT_TENSOR_CORES = 0, the FFMA kernels, has no range limit)"
                             % ERR_OVERFLOW)
    return None


class GraphWorkspace:
    """The private workspace of a CUDA graph and one context per view.  It runs in no-sync mode (G4D_OPT_SYNC_MODE = 0):
    a context's first forward reads its instance count R back once and keeps R + 50 % (at least ``min_capacity``) as its
    capacity, later forwards -- and every replay -- are bounded by it.  Context i reads its timestamp from the device float
    at time_ptrs[i].  ``capture`` freezes the workspace, so that no call can move a buffer the graph points at."""

    def __init__(self, dev: torch.device, time_ptrs: Sequence[int], min_capacity: int = 0):
        self.ws = _lib.Workspace(dev.index)
        self.ws.set_option(_lib.OPT_SYNC_MODE, 0)
        if min_capacity:
            self.ws.set_option(_lib.OPT_INSTANCE_CAPACITY, int(min_capacity))
        self.ctxs = [_lib.Context(self.ws) for _ in time_ptrs]
        for c, t in zip(self.ctxs, time_ptrs):
            c.set_time_source(t)

    def routed(self):
        """``with gws.routed():`` -- the library calls of the block run on this workspace and its contexts (``_lib.routed``)."""
        return _lib.routed(self.ws, self.ctxs)

    def capture(self, launch) -> torch.cuda.CUDAGraph:
        """Record launch() on a private memory pool, then freeze the workspace."""
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            launch()
        self.ws.freeze(True)
        self.ws.graph_status(sync=True)   # (clear: nothing has been replayed yet)
        return graph

    def check(self, sync: bool = True) -> None:
        err = status_error(self.ws.graph_status(sync))
        if err is not None:
            raise err


class GraphedRender:
    """``render()`` (template: one camera) or ``render_cameras()`` (template: a list of at most 32 cameras at one time)
    under ``torch.no_grad()``, replayed from a CUDA graph.

    ``__call__`` takes a camera (or a list of cameras) with the template's image sizes and FoVs and returns the result
    dict(s) ``render()`` returns.  Their tensors are the graph's static outputs: the next call overwrites them.
    ``min_capacity`` raises the instance capacity learnt from the template views (G4D_OPT_INSTANCE_CAPACITY).
    ``return_alpha``: the result dicts also hold ``alpha``, as ``render(..., return_alpha=True)`` returns it."""

    def __init__(self, pc, pipe, bg_color: torch.Tensor, template, stage: str = "fine", scaling_modifier: float = 1.0,
                 min_capacity: int = 0, return_alpha: bool = False):
        self.multi = isinstance(template, (list, tuple))
        views = list(template) if self.multi else [template]
        if not views or len(views) > _lib.MAX_CAMERAS:
            raise ValueError("a graphed render takes 1..%d views, got %d" % (_lib.MAX_CAMERAS, len(views)))
        module = _stage_module(pc, stage)
        if "coarse" not in stage and not isinstance(module, deform_network):
            raise NotImplementedError("a graphed render needs the g4d deformation network (or the coarse stage)")
        if getattr(pipe, "debug", False):
            raise ValueError("a graphed render cannot run with pipe.debug (it synchronises after every stage)")
        xyz = pc.get_xyz
        dev = xyz.device
        self.pc, self.k, self.n, self.dev = pc, len(views), int(xyz.shape[0]), dev
        self.sh_degree = int(pc.active_sh_degree)
        n, k = self.n, self.k
        lib = _lib.load()
        settings = [settings_from_camera(v, pc, pipe, bg_color, scaling_modifier) for v in views]
        self._shape = [self._view_key(rs) for rs, _ in settings]
        # the model's tensors are read in place: a copy (non-contiguous or non-fp32 storage) would freeze their values
        self._tensors = (pc._xyz, pc._scaling, pc._rotation, pc._opacity, pc._features_dc, pc._features_rest)
        staged = [_lib.cuda_f32(t, name) for t, name in zip(self._tensors, ("xyz", "scaling", "rotation", "opacity",
                                                                            "features_dc", "features_rest"))]
        if any(a.data_ptr() != b.data_ptr() for a, b in zip(staged, self._tensors)):
            raise ValueError("a graphed render reads the model's tensors in place: they must be contiguous fp32 CUDA tensors")
        self._ptrs = tuple(t.data_ptr() for t in self._tensors)
        m = _lib.sh_coeffs(pc._features_rest, n, "features_rest", skip=1)
        _lib.check_sh_degree(m, self.sh_degree, module.head_mask() if module is not None else 0)
        self._bg = _lib.cuda_f32(bg_color, "bg", 3)

        # device block the captured kernels read: k views; every context takes view 0's timestamp
        self._views = ViewBlock(dev, k)
        self._gws = GraphWorkspace(dev, [self._views.time_ptr(0)] * k, min_capacity)
        self.ws, self.ctxs = self._gws.ws, self._gws.ctxs
        self._cams = (_lib.Camera * k)(*[camera_from_settings(rs._replace(bg=self._bg), sh_coeffs=m)
                                          for rs, _ in settings])
        for i, cam in enumerate(self._cams):      # the view matrices and camera centre: read from the staging block's copy
            cam.debug = _lib.CAM_NO_GRAD
            view, proj, campos = self._views.view(i)
            cam.d_viewmatrix, cam.d_projmatrix, cam.d_campos = view.data_ptr(), proj.data_ptr(), campos.data_ptr()
        self._keep: list = []
        # fresh: the capture records the weight repack, so every replay packs the parameters as they are then
        self._prm = module.c_params(self._keep, fresh=True) if module is not None else None
        self._module = module
        self._net_key = self._network_key()
        self._g = _lib.Gaussians(n, *self._ptrs)
        self.colors = [torch.zeros(3, int(rs.image_height), int(rs.image_width), device=dev) for rs, _ in settings]
        self.depths = [torch.zeros(1, int(rs.image_height), int(rs.image_width), device=dev) for rs, _ in settings]
        self.alphas = [torch.zeros(1, int(rs.image_height), int(rs.image_width), device=dev) for rs, _ in settings] \
            if return_alpha else []
        for c, a in zip(self.ctxs, self.alphas):     # the private contexts write their alpha maps into the static outputs
            c.set_alpha_out(a.data_ptr())
        self.radii = [torch.zeros(n, device=dev, dtype=torch.int32) for _ in range(k)]
        self.visible = [torch.zeros(n, device=dev, dtype=torch.bool) for _ in range(k)]
        ptrs = lambda ts: (C.c_void_p * k)(*[t.data_ptr() for t in ts])
        self._out = (ptrs(self.colors), ptrs(self.depths), ptrs(self.radii))
        self._handles = (C.c_void_p * k)(*[c.handle for c in self.ctxs])
        self._lib = lib

        with torch.cuda.device(dev):
            self._stage(views)
            # eager: the first call learns each context's instance capacity (it reads R back once), the second is the
            # no-sync warm-up; the stats read reports an overflow of the warm-up
            self._launch()
            self._launch()
            for c in self.ctxs:
                c.stats()
            self.graph = self._gws.capture(self._launch)

    @staticmethod
    def _view_key(rs):
        return (int(rs.image_height), int(rs.image_width), _time_bits(rs.tanfovx), _time_bits(rs.tanfovy), int(rs.sh_degree))

    def _launch(self):
        """The captured work: one C-ABI render call, then the visibility masks."""
        stream = _lib.stream_of(self.dev)
        prm = C.byref(self._prm) if self._prm is not None else None
        if self.multi:
            _lib.check(self._lib.g4d_render_forward_cameras(self._handles, self.k, self._cams, prm, C.byref(self._g), *self._out,
                                                            stream), "g4d_render_forward_cameras")
        else:
            _lib.check(self._lib.g4d_render_forward(self.ctxs[0].handle, C.byref(self._cams[0]), prm, C.byref(self._g),
                                                    self.colors[0].data_ptr(), self.depths[0].data_ptr(),
                                                    self.radii[0].data_ptr(), stream), "g4d_render_forward")
        for r, v in zip(self.radii, self.visible):
            torch.gt(r, 0, out=v)

    def _stage(self, views: Sequence) -> None:
        times = self._views.stage(views)
        if any(_time_bits(t) != _time_bits(times[0]) for t in times):
            raise ValueError("a graphed render_cameras renders one timestamp: the cameras' times differ (%s)" % sorted(set(times)))

    def _network_key(self):
        """what the captured G4DDeformParams points at: the module, its head mask, aabb and parameter storage"""
        m = self._module
        if m is None:
            return None
        return (id(self.pc._deformation), m.head_mask(), m.deformation_net.grid.aabb.data_ptr()) + \
            tuple(p.data_ptr() for p in m.flat_parameters())

    def _check_template(self, views: List) -> None:
        if len(views) != self.k:
            raise ValueError("the graph was captured for %d views, got %d" % (self.k, len(views)))
        pc = self.pc
        if int(pc.get_xyz.shape[0]) != self.n:
            raise ValueError("the model has %d Gaussians, the graph was captured for %d" % (pc.get_xyz.shape[0], self.n))
        if int(pc.active_sh_degree) != self.sh_degree:
            raise ValueError("the SH degree changed from %d to %d since the capture" % (self.sh_degree, pc.active_sh_degree))
        if tuple(t.data_ptr() for t in (pc._xyz, pc._scaling, pc._rotation, pc._opacity, pc._features_dc,
                                        pc._features_rest)) != self._ptrs:
            raise ValueError("the model's tensors were replaced since the capture: build a new GraphedRender")
        if self._network_key() != self._net_key:
            raise ValueError("the deformation network's parameters were replaced (or its head mask changed) since the capture: "
                             "build a new GraphedRender")
        for i, v in enumerate(views):
            key = (int(v.image_height), int(v.image_width), _time_bits(math.tan(v.FoVx * 0.5)), _time_bits(math.tan(v.FoVy * 0.5)),
                   self.sh_degree)
            if key != self._shape[i]:
                raise ValueError("view %d differs from the template (image size or FoV): %s vs %s" % (i, key[:2], self._shape[i][:2]))

    def __call__(self, cameras):
        if self.multi != isinstance(cameras, (list, tuple)):
            raise ValueError("the graph was captured for %s" % ("render_cameras() of %d cameras, got one camera" % self.k
                                                                if self.multi else "render() of one camera, got a list"))
        views = list(cameras) if self.multi else [cameras]
        self._check_template(views)
        with torch.cuda.device(self.dev):
            self._stage(views)
            self.graph.replay()
        pts = _zero_points(self.pc.get_xyz)
        out = [{"render": c, "viewspace_points": pts, "visibility_filter": v, "radii": r, "depth": d}
               for c, v, r, d in zip(self.colors, self.visible, self.radii, self.depths)]
        for o, a in zip(out, self.alphas):
            o["alpha"] = a
        return out if self.multi else out[0]

    def check(self, sync: bool = True) -> None:
        """Raise G4DError when a replay since the last check overflowed its instance capacity (its images are incomplete) or
        met a value outside the FP16x2 operand range.  sync: wait for the replays first."""
        self._gws.check(sync)
