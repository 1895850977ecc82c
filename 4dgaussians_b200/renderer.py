"""Drop-in for ``gaussian_renderer.render`` (/root/reference/gaussian_renderer/__init__.py:18-138).

Same signature, same result dict (``render, viewspace_points, visibility_filter, radii, depth``), same quirks
(``time`` may be a float / 0-d tensor / int; PanopticSports cameras are dicts carrying a prebuilt settings object).
What changes is underneath: when ``pc._deformation`` is the g4d ``deform_network`` the whole of
deform -> activations -> rasterize runs as ONE C-ABI call into hand-written sm_90a kernels
(``g4d_render_forward`` / ``g4d_render_backward``): no [N,F] feature temporaries, no ``time.repeat(N,1)``,
no ``torch.cat`` of the SH features, no per-call ``.cuda()`` copies of the camera matrices.

``render_cameras`` renders one timestamp from several cameras (a camera rig at frame t) in one call: the deformation
network runs once, forward and backward (``g4d_render_forward_cameras`` / ``g4d_render_backward_cameras``).  ``render``
is its one-camera case, which takes the single-camera entry points.

Both differentiate the camera tensors that require grad (``rasterizer.camera_grad_leaves``) and the camera's time when it
is a tensor that requires grad (``time_grad_leaf``): dL/dt comes from the network's backward, for learning per-camera time
offsets.  The ``depth`` maps they return are differentiable too, for depth supervision.  With ``return_alpha=True`` each
result dict also holds ``alpha``, the accumulated opacity 1 - T of each pixel, differentiable as well, for mask supervision
and compositing.
"""
from __future__ import annotations

import ctypes as C
import math
import struct
from typing import Optional

import torch

from . import _lib
from .deformation import deform_network, scalar_time
from .rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, ViewTerms, _ContextLease, camera_from_settings,
                         per_view)


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


def time_grad_leaf(viewpoint_cameras, cam_type=None):
    """The cameras' time tensor that takes a gradient (grad mode on, ``requires_grad``), or None.  The cameras of one call
    share one deformation and so one dL/dt: when one camera's time takes a gradient, every camera must hold that same
    tensor object (ValueError otherwise, before anything runs)."""
    if not torch.is_grad_enabled():
        return None
    times = [c['time'] if cam_type == "PanopticSports" else c.time for c in viewpoint_cameras]
    leaves = [t for t in times if torch.is_tensor(t) and t.requires_grad]
    if not leaves:
        return None
    if any(t is not leaves[0] for t in times):
        raise ValueError("render_cameras deforms once for all cameras, so it has one time gradient: a camera's time requires "
                         "grad, and then every camera must hold that same time tensor.  Call render() per camera to learn "
                         "a time per camera")
    if leaves[0].numel() != 1:
        raise ValueError("a camera time that requires grad must have one element, got shape %s" % (tuple(leaves[0].shape),))
    return leaves[0]


def _fused_forward(module: Optional[deform_network], terms: ViewTerms, t, needs_bwd, xyz, scaling, rotation, opacity, f_dc,
                   f_rest):
    """One fused render call over the views of ``terms``, one context lease per camera: g4d_render_forward for one camera,
    g4d_render_forward_cameras for several.  Shared by the autograd Function and by the no-grad fast path."""
    lib = _lib.load()
    dev = xyz.device
    n, k = xyz.shape[0], terms.k
    x, s = _lib.cuda_f32(xyz, "xyz", n * 3), _lib.cuda_f32(scaling, "scaling", n * 3)
    r, o = _lib.cuda_f32(rotation, "rotation", n * 4), _lib.cuda_f32(opacity, "opacity", n)
    m = _lib.sh_coeffs(f_rest, n, "features_rest", skip=1)
    _lib.check_sh_degree(m, int(terms.rss[0].sh_degree), module.head_mask() if module is not None else 0)
    dc, rest = _lib.cuda_f32(f_dc, "features_dc", n * 3), _lib.cuda_f32(f_rest, "features_rest", n * 3 * (m - 1))
    colors, radii, depths, alphas = terms.outputs(dev, n)
    keep = []
    cams = [camera_from_settings(rs, time=t, keep=keep, sh_coeffs=m) for rs in terms.rss]
    if not needs_bwd:
        for cam in cams:
            cam.debug |= _lib.CAM_NO_GRAD      # torch.no_grad() rendering: nothing is saved for a backward
    # training forwards rebuild the packed weight images (fused optimizers do not bump Tensor._version)
    prm = module.c_params(keep, fresh=needs_bwd) if module is not None else None
    # at M = 1 rest is empty and its data_ptr() may be 0: the library then takes the fused layout [N,M,3] in dc, which at
    # M = 1 is the same tensor as the split dc [N,1,3] (include/g4d.h, G4DGaussians)
    g = _lib.Gaussians(n, x.data_ptr(), s.data_ptr(), r.data_ptr(), o.data_ptr(), dc.data_ptr(), rest.data_ptr())
    with torch.cuda.device(dev):
        ws = _lib.workspace_of(dev)
        leases = [_ContextLease(ws) for _ in cams]
        pm = C.byref(prm) if prm is not None else None
        with terms.forward([lease.ctx for lease in leases], alphas):
            if k == 1:
                cams, handles = cams[0], None       # one camera: the Camera itself, several: a Camera array
                _lib.check(lib.g4d_render_forward(leases[0].ctx.handle, C.byref(cams), pm, C.byref(g), colors[0].data_ptr(),
                                                  depths[0].data_ptr(), radii[0].data_ptr(), _lib.stream_of(dev)),
                           "g4d_render_forward")
            else:
                cams, handles = (_lib.Camera * k)(*cams), (C.c_void_p * k)(*[lease.ctx.handle for lease in leases])
                _lib.check(lib.g4d_render_forward_cameras(handles, k, cams, pm, C.byref(g), _pointers(colors), _pointers(depths),
                                                          _pointers(radii), _lib.stream_of(dev)), "g4d_render_forward_cameras")
    cstructs = (cams, prm, g, keep, int(prm.version) if prm is not None else None, handles)
    return colors, radii, depths, alphas, leases, cstructs, (x, s, r, o, dc, rest)


def _pointers(tensors):
    return (C.c_void_p * len(tensors))(*[None if t is None else t.data_ptr() for t in tensors])


class _FusedRender(torch.autograd.Function):
    """inputs: xyz, scaling, rotation, opacity, features_dc, features_rest, k x means2D, *deform parameters, then
    ``terms.leaves`` (the camera and time tensors that take a gradient); outputs (``per_view``): k images, k radii, k depth
    maps, and with ``terms.alpha`` k alpha maps"""

    @staticmethod
    def forward(ctx, module: Optional[deform_network], terms, t, xyz, scaling, rotation, opacity, f_dc, f_rest, *rest):
        colors, radii, depths, alphas, leases, cstructs, saved = _fused_forward(module, terms, t, any(ctx.needs_input_grad),
                                                                                xyz, scaling, rotation, opacity, f_dc, f_rest)
        ctx.module, ctx.terms, ctx.n, ctx.leases = module, terms, xyz.shape[0], leases
        ctx.lease = leases[0]        # camera 0's context: what a render() caller reads the forward's buffers through
        # the C-ABI structs (and the tensors whose pointers they carry) are kept for the backward: rebuilding them costs the
        # host ~0.3 ms per view, during which the GPU has nothing queued behind the forward's last kernel
        ctx.cstructs = cstructs
        ctx.save_for_backward(*saved)
        ctx.mark_non_differentiable(*radii)
        # an image, depth or alpha map outside the loss arrives as None: a camera with none of them in the loss has its blend
        # backward skipped
        ctx.set_materialize_grads(False)
        return tuple(colors) + tuple(radii) + tuple(depths) + tuple(alphas)

    @staticmethod
    def backward(ctx, *grads):
        lib = _lib.load()
        x, s, r, o, dc, rest = ctx.saved_tensors
        dev, n, terms, module = x.device, ctx.n, ctx.terms, ctx.module
        k = terms.k
        leases = ctx.leases
        if leases is None:
            raise RuntimeError("render backward called twice (context already released)" if k == 1 else
                               "render_cameras backward called twice (contexts already released)")
        gcols, gdeps, galphas = terms.gradients(grads, dev)
        cams, prm, g, keep, version, handles = ctx.cstructs
        if module is not None and version != module._param_version:      # another forward ran since: take the current key
            keep = []
            prm = module.c_params(keep, fresh=True)
        cg, pgrads = module.c_grad_sinks() if module is not None else (None, [])
        # one allocation for the per-Gaussian gradients, every segment 16-byte aligned: xyz, scaling, rotation, opacity,
        # features_dc, features_rest (M - 1 coefficients), then means2D of each camera: 11 + 3M + 3k floats per Gaussian
        npad = (n + 3) // 4 * 4
        m = cams.sh_coeffs if k == 1 else cams[0].sh_coeffs
        end = 11 + 3 * m
        flat = torch.empty(npad * (end + 3 * k), device=dev, dtype=torch.float32)
        gx, gs, gr, go, gdc, grest = (flat[a * npad:a * npad + w * n].view(shape) for a, w, shape in
                                      ((0, 3, (n, 3)), (3, 3, (n, 3)), (6, 4, (n, 4)), (10, 1, (n, 1)), (11, 3, (n, 1, 3)),
                                       (14, 3 * (m - 1), (n, m - 1, 3))))
        gm2 = [flat[(end + 3 * i) * npad:(end + 3 * i) * npad + 3 * n].view(n, 3) for i in range(k)]
        gg = _lib.GaussianGrads(gx.data_ptr(), gs.data_ptr(), gr.data_ptr(), go.data_ptr(), gdc.data_ptr(), grest.data_ptr(),
                                gm2[0].data_ptr() if k == 1 else None)
        with torch.cuda.device(dev), terms.backward([lease.ctx for lease in leases], dev, gdeps, galphas):
            if k == 1:
                _lib.check(lib.g4d_render_backward(leases[0].ctx.handle, C.byref(cams), C.byref(prm) if prm is not None else None,
                                                   C.byref(cg) if cg is not None else None, C.byref(g), gcols[0].data_ptr(),
                                                   C.byref(gg), _lib.stream_of(dev)), "g4d_render_backward")
            else:
                _lib.check(lib.g4d_render_backward_cameras(handles, k, cams, C.byref(prm) if prm is not None else None,
                                                           C.byref(cg) if cg is not None else None, C.byref(g), _pointers(gcols),
                                                           C.byref(gg), _pointers(gm2), _lib.stream_of(dev)),
                           "g4d_render_backward_cameras")
        for lease in leases:
            lease.release()
        ctx.leases = ctx.lease = None
        return (None, None, None, gx, gs, gr, go, gdc, grest) + tuple(gm2) + tuple(pgrads) + terms.leaf_grads()


def _time_bits(t) -> bytes:
    return struct.pack("<f", float(t))


def _stage_module(pc, stage):
    """The deformation module a stage renders with: none in the coarse stage, the model's in the fine stage."""
    if "coarse" in stage:
        return None
    if "fine" in stage:
        return pc._deformation
    raise NotImplementedError


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


def _render(viewpoint_cameras, pc, pipe, bg_color, scaling_modifier, override_color, stage, cam_type, return_alpha):
    """The body of render() and render_cameras(): one result dict per camera."""
    if override_color is not None or getattr(pipe, "convert_SHs_python", False) or getattr(pipe, "compute_cov3D_python", False):
        raise NotImplementedError("override_color / convert_SHs_python / compute_cov3D_python are dead or broken paths in "
                                  "the reference (gaussian_renderer/__init__.py:74-78,105-116)")
    cams = list(viewpoint_cameras)
    if not cams:
        raise ValueError("render_cameras needs at least one camera")
    if len(cams) > _lib.MAX_CAMERAS:
        raise ValueError("render_cameras takes at most %d cameras per call, got %d" % (_lib.MAX_CAMERAS, len(cams)))
    time_leaf = time_grad_leaf(cams, cam_type)
    settings = [settings_from_camera(c, pc, pipe, bg_color, scaling_modifier, cam_type) for c in cams]
    rss = [rs for rs, _ in settings]
    t = settings[0][1]
    if len(cams) > 1 and len({_time_bits(ti) for _, ti in settings}) > 1:
        raise ValueError("render_cameras renders one timestamp: the cameras' times differ (%s)"
                         % sorted({float(ti) for _, ti in settings}))
    module = _stage_module(pc, stage)
    xyz = pc.get_xyz
    k = len(cams)
    if torch.is_grad_enabled():
        points = [torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device=xyz.device) + 0 for _ in range(k)]
        for p in points:
            p.retain_grad()
    else:       # nothing will ever flow into them: a cached all-zero tensor instead of a memset (+ add) launch per view
        points = [_zero_points(xyz)] * k
    if module is None or isinstance(module, deform_network):
        terms = ViewTerms(rss, return_alpha, time_leaf)
        if not torch.is_grad_enabled():
            # no autograd node to build: skip Function.apply and its per-input bookkeeping (40 inputs with the network's parameters)
            images, radii, depths, alphas, leases, _, _ = _fused_forward(module, terms, t, False, xyz, pc._scaling, pc._rotation,
                                                                         pc._opacity, pc._features_dc, pc._features_rest)
            for lease in leases:
                lease.release()
        else:
            params = tuple(module.flat_parameters()) if module is not None else ()
            outs = _FusedRender.apply(module, terms, t, xyz, pc._scaling, pc._rotation, pc._opacity, pc._features_dc,
                                      pc._features_rest, *points, *params, *terms.leaves)
            images, radii, depths, alphas = per_view(outs, k)
    else:
        # a foreign (e.g. the reference's own PyTorch) deformation module: keep its semantics, deform once, then rasterize
        # every camera with g4d
        n = xyz.shape[0]
        if time_leaf is None:
            time = torch.tensor(t, device=xyz.device, dtype=torch.float32).repeat(n, 1)
        else:       # kept in the graph: the module's own autograd gives dL/dt
            time = time_leaf.to(device=xyz.device, dtype=torch.float32).reshape(1, 1).repeat(n, 1)
        m3, sc, rot, op, shs = module(xyz, pc._scaling, pc._rotation, pc._opacity, pc.get_features, time)
        opac, scales, rots = pc.opacity_activation(op), pc.scaling_activation(sc), pc.rotation_activation(rot)
        images, radii, depths, alphas = [], [], [], []
        for rs, p in zip(rss, points):
            r = GaussianRasterizer(raster_settings=rs, differentiable_depth=True, return_alpha=return_alpha)(
                means3D=m3, means2D=p, shs=shs, colors_precomp=None, opacities=opac, scales=scales, rotations=rots,
                cov3D_precomp=None)
            images.append(r[0]); radii.append(r[1]); depths.append(r[2]); alphas.extend(r[3:])
    outs = [{"render": img, "viewspace_points": p, "visibility_filter": rad > 0, "radii": rad, "depth": dep}
            for img, p, rad, dep in zip(images, points, radii, depths)]
    for out, alp in zip(outs, alphas):
        out["alpha"] = alp
    return outs


def render(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None, stage="fine",
           cam_type=None, return_alpha=False):
    """Render the scene.  Background tensor (bg_color) must be on GPU (as in the reference).  return_alpha: the result
    dict also holds ``alpha`` [1,H,W], the accumulated opacity 1 - T of each pixel (render = C_fg + (1 - alpha) * bg up to
    fp32 rounding), which takes a gradient in grad mode."""
    return _render((viewpoint_camera,), pc, pipe, bg_color, scaling_modifier, override_color, stage, cam_type,
                   return_alpha)[0]


def render_cameras(viewpoint_cameras, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None, stage="fine",
                   cam_type=None, return_alpha=False):
    """Render one timestamp from several cameras: one result dict per camera, each with the keys render() returns and its
    own ``viewspace_points``.  The cameras must share their time (as float32, bit for bit; else ValueError) and there may
    be at most G4D_MAX_CAMERAS (32) of them.  With the g4d deformation network the deformation runs once for all cameras,
    forward and backward; a foreign deformation module is run once and its output rasterized per camera.  A time that
    requires grad must be one tensor that every camera holds (ValueError otherwise): the group's one dL/dt goes to it.
    return_alpha: as for render(), per camera."""
    return _render(viewpoint_cameras, pc, pipe, bg_color, scaling_modifier, override_color, stage, cam_type, return_alpha)
