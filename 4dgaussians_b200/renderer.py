"""Drop-in for ``gaussian_renderer.render`` (/root/reference/gaussian_renderer/__init__.py:18-138).

Same signature, same result dict (``render, viewspace_points, visibility_filter, radii, depth``), same quirks
(``time`` may be a float / 0-d tensor / int; PanopticSports cameras are dicts carrying a prebuilt settings object).
What changes is underneath: when ``pc._deformation`` is the g4d ``deform_network`` the whole of
deform -> activations -> rasterize runs as ONE C-ABI call into hand-written sm_90a kernels
(``g4d_render_forward`` / ``g4d_render_backward``): no [N,F] feature temporaries, no ``time.repeat(N,1)``,
no ``torch.cat`` of the SH features, no per-call ``.cuda()`` copies of the camera matrices.

``render_cameras`` renders one timestamp from several cameras (a camera rig at frame t) in one call: the deformation
network runs once, forward and backward (``g4d_render_forward_cameras`` / ``g4d_render_backward_cameras``).
"""
from __future__ import annotations

import ctypes as C
import math
import struct
from typing import Optional

import torch

from . import _lib
from .deformation import deform_network, scalar_time
from .rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, _ContextLease, _dev_f32, _stream_ptr,
                         camera_from_settings)


def settings_from_camera(viewpoint_camera, pc, pipe, bg_color, scaling_modifier=1.0, cam_type=None):
    """gaussian_renderer/__init__.py:35-56, minus the three per-call .cuda() copies (CPU matrices travel inside the
    C-ABI camera struct as kernel parameters)."""
    if cam_type != "PanopticSports":
        rs = GaussianRasterizationSettings(
            image_height=int(viewpoint_camera.image_height), image_width=int(viewpoint_camera.image_width),
            tanfovx=math.tan(viewpoint_camera.FoVx * 0.5), tanfovy=math.tan(viewpoint_camera.FoVy * 0.5),
            bg=bg_color, scale_modifier=scaling_modifier, viewmatrix=viewpoint_camera.world_view_transform,
            projmatrix=viewpoint_camera.full_proj_transform, sh_degree=pc.active_sh_degree,
            campos=viewpoint_camera.camera_center, prefiltered=False, debug=bool(getattr(pipe, "debug", False)))
        t = scalar_time(viewpoint_camera.time)
    else:
        rs = viewpoint_camera['camera']
        t = scalar_time(viewpoint_camera['time'])
    return rs, t


def _fused_forward(module: Optional[deform_network], rs, t, needs_bwd, xyz, scaling, rotation, opacity, f_dc, f_rest):
    """One g4d_render_forward call.  Shared by the autograd Function and by the no-grad fast path of render()."""
    lib = _lib.load()
    dev = xyz.device
    n = xyz.shape[0]
    x = _dev_f32(xyz, n * 3, "xyz"); s = _dev_f32(scaling, n * 3, "scaling"); r = _dev_f32(rotation, n * 4, "rotation")
    o = _dev_f32(opacity, n, "opacity"); dc = _dev_f32(f_dc, n * 3, "features_dc"); rest = _dev_f32(f_rest, n * 45, "features_rest")
    H, W = int(rs.image_height), int(rs.image_width)
    color = torch.empty(3, H, W, device=dev, dtype=torch.float32)
    depth = torch.empty(1, H, W, device=dev, dtype=torch.float32)
    radii = torch.empty(n, device=dev, dtype=torch.int32)
    keep = []
    cam = camera_from_settings(rs, time=t, keep=keep)
    if not needs_bwd:
        cam.debug |= _lib.CAM_NO_GRAD      # torch.no_grad() rendering: nothing is saved for a backward
    # training forwards rebuild the packed weight images (fused optimizers do not bump Tensor._version)
    prm = module.c_params(keep, fresh=needs_bwd) if module is not None else None
    g = _lib.Gaussians(n, x.data_ptr(), s.data_ptr(), r.data_ptr(), o.data_ptr(), dc.data_ptr(), rest.data_ptr())
    with torch.cuda.device(dev):
        lease = _ContextLease(_lib.Workspace.get(dev.index if dev.index is not None else torch.cuda.current_device()))
        _lib.check(lib.g4d_render_forward(lease.ctx.handle, C.byref(cam), C.byref(prm) if prm is not None else None,
                                          C.byref(g), color.data_ptr(), depth.data_ptr(), radii.data_ptr(),
                                          _stream_ptr(dev)), "g4d_render_forward")
    cstructs = (cam, prm, g, keep, int(prm.version) if prm is not None else None)
    return color, radii, depth, lease, cstructs, (x, s, r, o, dc, rest)


class _FusedRender(torch.autograd.Function):
    """inputs: xyz, scaling, rotation, opacity, features_dc, features_rest, means2D, *deform parameters"""

    @staticmethod
    def forward(ctx, module: Optional[deform_network], rs, t, grad_mode, xyz, scaling, rotation, opacity, f_dc, f_rest, means2D, *params):
        needs_bwd = grad_mode and any(ctx.needs_input_grad)    # (grad mode is always off INSIDE Function.forward)
        color, radii, depth, lease, cstructs, saved = _fused_forward(module, rs, t, needs_bwd, xyz, scaling, rotation, opacity, f_dc, f_rest)
        ctx.module, ctx.rs, ctx.t, ctx.n, ctx.lease = module, rs, t, xyz.shape[0], lease
        # the C-ABI structs (and the tensors whose pointers they carry) are kept for the backward: rebuilding them costs the
        # host ~0.3 ms per view, during which the GPU has nothing queued behind the forward's last kernel
        ctx.cstructs = cstructs
        ctx.save_for_backward(*saved)
        ctx.mark_non_differentiable(radii, depth)
        return color, radii, depth

    @staticmethod
    def backward(ctx, grad_color, _gr, _gd):
        lib = _lib.load()
        x, s, r, o, dc, rest = ctx.saved_tensors
        dev, n, rs, module = x.device, ctx.n, ctx.rs, ctx.module
        gcol = _dev_f32(grad_color, 3 * int(rs.image_height) * int(rs.image_width), "grad_out_color")
        cam, prm, g, keep, version = ctx.cstructs
        if module is not None and version != module._param_version:      # another forward ran since: take the current key
            keep = []
            prm = module.c_params(keep, fresh=True)
        pgrads, cg = [], None
        if module is not None:
            sinks = module.grad_sinks()
            if sinks is not None:          # opt-in fused accumulation: kernels add into the parameters' own .grad
                cg = module.c_grads(sinks)
                pgrads = [None] * len(sinks)
            else:
                pgrads = module.alloc_grads()
                cg = module.c_grads(pgrads)
        npad = (n + 3) // 4 * 4                                           # keeps every segment 16-byte aligned
        flat = torch.empty(npad * 62, device=dev, dtype=torch.float32)    # one allocation for the seven per-Gaussian gradients
        gx, gs, gr, go, gdc, grest, gm2 = (flat[a * npad:a * npad + w * n].view(shape) for a, w, shape in
                                           ((0, 3, (n, 3)), (3, 3, (n, 3)), (6, 4, (n, 4)), (10, 1, (n, 1)), (11, 3, (n, 1, 3)),
                                            (14, 45, (n, 15, 3)), (59, 3, (n, 3))))
        gg = _lib.GaussianGrads(gx.data_ptr(), gs.data_ptr(), gr.data_ptr(), go.data_ptr(), gdc.data_ptr(), grest.data_ptr(),
                                gm2.data_ptr())
        lease = ctx.lease
        if lease is None or lease.ctx is None:
            raise RuntimeError("render backward called twice (context already released)")
        with torch.cuda.device(dev):
            _lib.check(lib.g4d_render_backward(lease.ctx.handle, C.byref(cam), C.byref(prm) if prm is not None else None,
                                               C.byref(cg) if cg is not None else None, C.byref(g), gcol.data_ptr(),
                                               C.byref(gg), _stream_ptr(dev)), "g4d_render_backward")
        lease.release()
        ctx.lease = None
        return (None, None, None, None, gx, gs, gr, go, gdc, grest, gm2) + tuple(pgrads)


_ZERO_POINTS = {}


def _zero_points(xyz: torch.Tensor) -> torch.Tensor:
    """The ``viewspace_points`` of a no-grad render: all zeros, never written by anything (no gradient can flow into it), so
    one read-only tensor per (device, N) is shared between calls instead of filling a new one per view."""
    key = (xyz.device, xyz.shape[0], xyz.dtype)
    z = _ZERO_POINTS.get(key)
    if z is None:
        if len(_ZERO_POINTS) > 8:
            _ZERO_POINTS.clear()
        z = _ZERO_POINTS[key] = torch.zeros_like(xyz)
    return z


def render(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None, stage="fine",
           cam_type=None):
    """Render the scene.  Background tensor (bg_color) must be on GPU (as in the reference)."""
    if override_color is not None or getattr(pipe, "convert_SHs_python", False) or getattr(pipe, "compute_cov3D_python", False):
        raise NotImplementedError("override_color / convert_SHs_python / compute_cov3D_python are dead or broken paths in "
                                  "the reference (gaussian_renderer/__init__.py:74-78,105-116)")
    xyz = pc.get_xyz
    if torch.is_grad_enabled():
        screenspace_points = torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device=xyz.device) + 0
        try:
            screenspace_points.retain_grad()
        except Exception:
            pass
    else:       # nothing will ever flow into it: a cached all-zero tensor instead of a memset (+ add) launch per view
        screenspace_points = _zero_points(xyz)
    rs, t = settings_from_camera(viewpoint_camera, pc, pipe, bg_color, scaling_modifier, cam_type)
    if "coarse" in stage:
        module = None
    elif "fine" in stage:
        module = pc._deformation
    else:
        raise NotImplementedError
    if module is None or isinstance(module, deform_network):
        if not torch.is_grad_enabled():
            # no autograd node to build: skip Function.apply and its per-input bookkeeping (40 inputs with the network's parameters)
            rendered_image, radii, depth, lease, _, _ = _fused_forward(module, rs, t, False, xyz, pc._scaling, pc._rotation, pc._opacity,
                                                                       pc._features_dc, pc._features_rest)
            lease.release()
        else:
            params = tuple(module.flat_parameters()) if module is not None else ()
            rendered_image, radii, depth = _FusedRender.apply(module, rs, t, True, xyz, pc._scaling, pc._rotation, pc._opacity,
                                                              pc._features_dc, pc._features_rest, screenspace_points, *params)
    else:
        # a foreign (e.g. the reference's own PyTorch) deformation module: keep its semantics, still rasterize with g4d
        n = xyz.shape[0]
        time = torch.tensor(t, device=xyz.device, dtype=torch.float32).repeat(n, 1)
        m3, sc, rot, op, shs = module(xyz, pc._scaling, pc._rotation, pc._opacity, pc.get_features, time)
        rasterizer = GaussianRasterizer(raster_settings=rs)
        rendered_image, radii, depth = rasterizer(means3D=m3, means2D=screenspace_points, shs=shs, colors_precomp=None,
                                                  opacities=pc.opacity_activation(op), scales=pc.scaling_activation(sc),
                                                  rotations=pc.rotation_activation(rot), cov3D_precomp=None)
    return {"render": rendered_image, "viewspace_points": screenspace_points, "visibility_filter": radii > 0,
            "radii": radii, "depth": depth}


def _fused_forward_cameras(module: Optional[deform_network], rss, t, needs_bwd, xyz, scaling, rotation, opacity, f_dc, f_rest):
    """One g4d_render_forward_cameras call over the cameras' settings rss (one context lease per camera)."""
    lib = _lib.load()
    dev = xyz.device
    n, k = xyz.shape[0], len(rss)
    x = _dev_f32(xyz, n * 3, "xyz"); s = _dev_f32(scaling, n * 3, "scaling"); r = _dev_f32(rotation, n * 4, "rotation")
    o = _dev_f32(opacity, n, "opacity"); dc = _dev_f32(f_dc, n * 3, "features_dc"); rest = _dev_f32(f_rest, n * 45, "features_rest")
    colors = [torch.empty(3, int(rs.image_height), int(rs.image_width), device=dev, dtype=torch.float32) for rs in rss]
    depths = [torch.empty(1, int(rs.image_height), int(rs.image_width), device=dev, dtype=torch.float32) for rs in rss]
    radii = [torch.empty(n, device=dev, dtype=torch.int32) for _ in rss]
    keep = []
    cams = (_lib.Camera * k)()
    for i, rs in enumerate(rss):
        cams[i] = camera_from_settings(rs, time=t, keep=keep)
        if not needs_bwd:
            cams[i].debug |= _lib.CAM_NO_GRAD
    prm = module.c_params(keep, fresh=needs_bwd) if module is not None else None
    g = _lib.Gaussians(n, x.data_ptr(), s.data_ptr(), r.data_ptr(), o.data_ptr(), dc.data_ptr(), rest.data_ptr())
    ptrs = lambda ts: (C.c_void_p * k)(*[tt.data_ptr() for tt in ts])
    with torch.cuda.device(dev):
        ws = _lib.Workspace.get(dev.index if dev.index is not None else torch.cuda.current_device())
        leases = [_ContextLease(ws) for _ in range(k)]
        handles = (C.c_void_p * k)(*[lease.ctx.handle for lease in leases])
        _lib.check(lib.g4d_render_forward_cameras(handles, k, cams, C.byref(prm) if prm is not None else None, C.byref(g),
                                                  ptrs(colors), ptrs(depths), ptrs(radii), _stream_ptr(dev)),
                   "g4d_render_forward_cameras")
    cstructs = (cams, prm, g, keep, int(prm.version) if prm is not None else None, handles)
    return colors, radii, depths, leases, cstructs, (x, s, r, o, dc, rest)


class _FusedRenderCameras(torch.autograd.Function):
    """inputs: xyz, scaling, rotation, opacity, features_dc, features_rest, k x means2D, *deform parameters;
    outputs: k images, k radii, k depth maps"""

    @staticmethod
    def forward(ctx, module: Optional[deform_network], rss, t, xyz, scaling, rotation, opacity, f_dc, f_rest, *rest):
        k = len(rss)
        needs_bwd = any(ctx.needs_input_grad)
        colors, radii, depths, leases, cstructs, saved = _fused_forward_cameras(module, rss, t, needs_bwd, xyz, scaling, rotation,
                                                                                opacity, f_dc, f_rest)
        ctx.module, ctx.rss, ctx.n, ctx.leases, ctx.cstructs = module, rss, xyz.shape[0], leases, cstructs
        ctx.save_for_backward(*saved)
        ctx.mark_non_differentiable(*radii, *depths)
        ctx.set_materialize_grads(False)         # an image outside the loss arrives as None: its blend backward is skipped
        return tuple(colors) + tuple(radii) + tuple(depths)

    @staticmethod
    def backward(ctx, *grads):
        lib = _lib.load()
        x, s, r, o, dc, rest = ctx.saved_tensors
        dev, n, rss, module = x.device, ctx.n, ctx.rss, ctx.module
        k = len(rss)
        leases = ctx.leases
        if leases is None:
            raise RuntimeError("render_cameras backward called twice (contexts already released)")
        gcols = [None if gc is None else _dev_f32(gc, 3 * int(rs.image_height) * int(rs.image_width), "grad_out_color")
                 for gc, rs in zip(grads[:k], rss)]
        cams, prm, g, keep, version, handles = ctx.cstructs
        if module is not None and version != module._param_version:      # another forward ran since: take the current key
            keep = []
            prm = module.c_params(keep, fresh=True)
        pgrads, cg = [], None
        if module is not None:
            sinks = module.grad_sinks()
            if sinks is not None:
                cg = module.c_grads(sinks)
                pgrads = [None] * len(sinks)
            else:
                pgrads = module.alloc_grads()
                cg = module.c_grads(pgrads)
        npad = (n + 3) // 4 * 4
        flat = torch.empty(npad * (59 + 3 * k), device=dev, dtype=torch.float32)
        gx, gs, gr, go, gdc, grest = (flat[a * npad:a * npad + w * n].view(shape) for a, w, shape in
                                      ((0, 3, (n, 3)), (3, 3, (n, 3)), (6, 4, (n, 4)), (10, 1, (n, 1)), (11, 3, (n, 1, 3)),
                                       (14, 45, (n, 15, 3))))
        gm2 = [flat[(59 + 3 * i) * npad:(59 + 3 * i) * npad + 3 * n].view(n, 3) for i in range(k)]
        gg = _lib.GaussianGrads(gx.data_ptr(), gs.data_ptr(), gr.data_ptr(), go.data_ptr(), gdc.data_ptr(), grest.data_ptr(), None)
        dl = (C.c_void_p * k)(*[None if gc is None else gc.data_ptr() for gc in gcols])
        m2 = (C.c_void_p * k)(*[t.data_ptr() for t in gm2])
        with torch.cuda.device(dev):
            _lib.check(lib.g4d_render_backward_cameras(handles, k, cams, C.byref(prm) if prm is not None else None,
                                                       C.byref(cg) if cg is not None else None, C.byref(g), dl, C.byref(gg), m2,
                                                       _stream_ptr(dev)), "g4d_render_backward_cameras")
        for lease in leases:
            lease.release()
        ctx.leases = None
        return (None, None, None, gx, gs, gr, go, gdc, grest) + tuple(gm2) + tuple(pgrads)


def _time_bits(t) -> bytes:
    return struct.pack("<f", float(t))


def render_cameras(viewpoint_cameras, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None, stage="fine",
                   cam_type=None):
    """Render one timestamp from several cameras: one result dict per camera, each with the keys render() returns and its
    own ``viewspace_points``.  The cameras must share their time (as float32, bit for bit; else ValueError) and there may
    be at most G4D_MAX_CAMERAS (32) of them.  With the g4d deformation network the deformation runs once for all cameras,
    forward and backward; a foreign deformation module is run once and its output rasterized per camera."""
    if override_color is not None or getattr(pipe, "convert_SHs_python", False) or getattr(pipe, "compute_cov3D_python", False):
        raise NotImplementedError("override_color / convert_SHs_python / compute_cov3D_python are dead or broken paths in "
                                  "the reference (gaussian_renderer/__init__.py:74-78,105-116)")
    cams = list(viewpoint_cameras)
    if not cams:
        raise ValueError("render_cameras needs at least one camera")
    if len(cams) > _lib.MAX_CAMERAS:
        raise ValueError("render_cameras takes at most %d cameras per call, got %d" % (_lib.MAX_CAMERAS, len(cams)))
    settings = [settings_from_camera(c, pc, pipe, bg_color, scaling_modifier, cam_type) for c in cams]
    rss = [rs for rs, _ in settings]
    t = settings[0][1]
    if any(_time_bits(ti) != _time_bits(t) for _, ti in settings):
        raise ValueError("render_cameras renders one timestamp: the cameras' times differ (%s)" % sorted({float(ti) for _, ti in settings}))
    if "coarse" in stage:
        module = None
    elif "fine" in stage:
        module = pc._deformation
    else:
        raise NotImplementedError
    xyz = pc.get_xyz
    k = len(cams)
    if torch.is_grad_enabled():
        points = [torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device=xyz.device) + 0 for _ in range(k)]
        for p in points:
            p.retain_grad()
    else:
        points = [_zero_points(xyz)] * k
    if module is None or isinstance(module, deform_network):
        if not torch.is_grad_enabled():
            images, radii, depths, leases, _, _ = _fused_forward_cameras(module, rss, t, False, xyz, pc._scaling, pc._rotation,
                                                                         pc._opacity, pc._features_dc, pc._features_rest)
            for lease in leases:
                lease.release()
        else:
            params = tuple(module.flat_parameters()) if module is not None else ()
            outs = _FusedRenderCameras.apply(module, rss, t, xyz, pc._scaling, pc._rotation, pc._opacity, pc._features_dc,
                                             pc._features_rest, *points, *params)
            images, radii, depths = outs[:k], outs[k:2 * k], outs[2 * k:]
    else:
        # a foreign deformation module: deformed once, then rasterized per camera by g4d
        n = xyz.shape[0]
        time = torch.tensor(t, device=xyz.device, dtype=torch.float32).repeat(n, 1)
        m3, sc, rot, op, shs = module(xyz, pc._scaling, pc._rotation, pc._opacity, pc.get_features, time)
        opac, scales, rots = pc.opacity_activation(op), pc.scaling_activation(sc), pc.rotation_activation(rot)
        images, radii, depths = [], [], []
        for rs, p in zip(rss, points):
            img, rad, dep = GaussianRasterizer(raster_settings=rs)(means3D=m3, means2D=p, shs=shs, colors_precomp=None,
                                                                   opacities=opac, scales=scales, rotations=rots,
                                                                   cov3D_precomp=None)
            images.append(img); radii.append(rad); depths.append(dep)
    return [{"render": img, "viewspace_points": p, "visibility_filter": rad > 0, "radii": rad, "depth": dep}
            for img, p, rad, dep in zip(images, points, radii, depths)]
