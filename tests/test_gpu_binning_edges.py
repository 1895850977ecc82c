"""Tile binning (g4d_bin.cu) on the branches random scenes never take, against the oracle's key sort bit for bit.

Random scenes all sort 24-27 key bits in 3 radix passes, spread hundreds of visible Gaussians over every chunk, keep their
sub-segments near 4 entries and fit one band.  Each case here builds a scene that forces one other branch, asserts that it
got there (kbits, nvis, the chunk cut, the sub-segment length, the band crossings) and then asserts that radii, depth
bits, rects, tile counts, screen records, colours, sorted keys / ids and tile ranges equal the oracle's and the image is
within 1e-4 except at explained threshold flips.  util_binning.py builds the scenes; test_binning_edge_scenes.py checks on
the oracle alone that they are what is asserted here.
"""
import math

import numpy as np
import pytest
import torch

from oracle import raster_ref as rr
import util_binning as ub
from util_scene import (_assert_index_data_bit_exact, _assert_pixel_outliers_are_threshold_flips, cam_tuple, g4d, make_module,
                        raster_oracle_inputs, synth)

pytestmark = pytest.mark.gpu


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _settings(cam, bg):
    return g4d.GaussianRasterizationSettings(
        image_height=cam.image_height, image_width=cam.image_width, tanfovx=math.tan(cam.FoVx * 0.5),
        tanfovy=math.tan(cam.FoVy * 0.5), bg=torch.tensor(bg, dtype=torch.float32, device="cuda"), scale_modifier=1.0,
        viewmatrix=cam.world_view_transform.cuda(), projmatrix=cam.full_proj_transform.cuda(), sh_degree=3,
        campos=cam.camera_center.cuda(), prefiltered=False, debug=False)


def _kbits(ctx):
    return int(ctx.read("bin_phases")[15])


def _rasterize(cam, ins, bg=(0.1, 0.2, 0.3), sync_mode=1, ref=None, grad=False):
    """drop-in GaussianRasterizer on fp32 numpy inputs; everything checked against the oracle.  sync_mode 0: the capacity-
    bounded device-side binning, on the second forward of a fresh context.  Returns (ctx, ref, colour, inputs on the GPU)."""
    rc, _ = cam_tuple(cam, bg, sh_degree=3)
    ref = rr.rasterize_forward(rc, *ins) if ref is None else ref
    ws = g4d._lib.Workspace.get(0)
    ws._free_contexts.clear()
    try:
        ws.set_option(g4d._lib.OPT_SYNC_MODE, sync_mode)
        for _ in range(2 if sync_mode == 0 else 1):
            color = ctx = None
            # (means3D always requires grad: the context stays leased to the output's grad_fn)
            dev = [torch.from_numpy(a).cuda().requires_grad_(grad or i == 0) for i, a in enumerate(ins)]
            m3, sc, ro, op, sh = dev
            m2 = torch.zeros_like(m3, requires_grad=grad)
            color, radii, _ = g4d.GaussianRasterizer(_settings(cam, bg))(
                means3D=m3, means2D=m2, shs=sh, colors_precomp=None, opacities=op, scales=sc, rotations=ro, cov3D_precomp=None)
            torch.cuda.synchronize()
            ctx = color.grad_fn.lease.ctx
            if sync_mode == 0:
                ctx.stats()
        _assert_index_data_bit_exact(ctx, radii.cpu().numpy(), ref)
        _assert_pixel_outliers_are_threshold_flips(color.detach().cpu().numpy(), ref, cam.image_width)
    finally:
        ws.set_option(g4d._lib.OPT_SYNC_MODE, 1)
        ws.set_option(g4d._lib.OPT_INSTANCE_CAPACITY, 0)
    return ctx, ref, color, dev + [m2]


# ------------------------------------------------------------------------------------------------------------- A
@pytest.mark.parametrize("span", ub.PASS_SPANS)
def test_radix_pass_count(span):
    """visible depth-bit span exactly 0, 2^9 - 1, 2^9, 2^18 - 1, 2^18, 2^27 - 1, 2^27: kbits 1 .. 28, one to four passes"""
    cam, ins = ub.pass_scene(span)
    ctx, ref, _, _ = _rasterize(cam, ins)
    bits = ub.depth_bits(ctx.read("depth"))[ctx.read("tiles_touched") > 0].astype(np.int64)
    assert int(bits.max() - bits.min()) == span                    # on the GPU's own depth bits
    kbits, passes = ub.PASS_KBITS[span]
    assert _kbits(ctx) == kbits and ub.passes_of(kbits) == passes


def test_radix_four_passes_near_cluster_and_far_shell():
    cam, ins = ub.four_pass_scene()
    ctx, _, _, _ = _rasterize(cam, ins, bg=(0.0, 0.0, 0.0))
    assert ub.passes_of(_kbits(ctx)) == 4


# ------------------------------------------------------------------------------------------------------------- B
def _assert_extremes(ref, near, far):
    pr = ref["proj"]
    vis = np.nonzero(pr.tiles_touched > 0)[0]
    b = ub.depth_bits(pr.depth)[vis]
    assert len(vis) == len(pr.depth)                              # every Gaussian visible: the extremes decide the range
    assert vis[np.argmin(b)] == near and (b == b.min()).sum() == 1
    assert vis[np.argmax(b)] == far and (b == b.max()).sum() == 1


@pytest.mark.parametrize("n", ub.EXTREME_NS)
def test_depth_range_extremes_preprocess_kernel(n):
    for near, far in ub.extreme_layouts(n):
        cam, ins = ub.extreme_scene(n, near, far, seed=n)
        ctx, ref, _, _ = _rasterize(cam, ins)
        _assert_extremes(ref, near, far)


FUSED_PATHS = {"ffma": dict(net="small64", tc=0), "fp16x2": dict(net="small128", tc=2),
               "coarse": dict(net="small128", tc=2, stage="coarse"), "cameras3": dict(net="small128", tc=2, cameras=3)}
_MODULES = {}


def _module(net):
    if net not in _MODULES:
        box = torch.tensor([[1.3, 4.0, 1.3], [-1.3, -1.0, -1.3]])
        _MODULES[net] = make_module(net, seed=1, aabb=box)
    return _MODULES[net]


@pytest.mark.parametrize("path", list(FUSED_PATHS))
@pytest.mark.parametrize("n", ub.EXTREME_NS)
def test_depth_range_extremes_fused_paths(path, n):
    """render() fine stage on the FFMA and the tensor-core kernels, the coarse stage, and render_cameras' extra cameras
    (project_cameras_kernel): the oracle runs on the GPU's own deformed tensors"""
    p = FUSED_PATHS[path]
    stage = p.get("stage", "fine")
    mod = _module(p["net"])
    has_sh = stage == "fine" and not mod.args.no_dshs
    ws = g4d._lib.Workspace.get(0)
    bg = torch.tensor([0.2, 0.1, 0.0], device="cuda")
    try:
        ws.set_option(g4d._lib.OPT_TENSOR_CORES, p["tc"])
        for near, far in ub.extreme_layouts(n):
            cam, m3, _ = ub.extreme_points(n, near, far, seed=n)
            scene = synth.make_scene(n, seed=n, scale_mean=0.04)
            scene["xyz"] = torch.from_numpy(m3)
            cam.time = 0.4
            pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
            if p.get("cameras"):
                cams = [cam] + [ub.front_camera(*ub.EXTREME_WH) for _ in (1, 2)]     # every Gaussian visible in each
                for c in cams:
                    c.time = 0.4
                outs = g4d.render_cameras(cams, pc, _Pipe, bg, stage=stage)
                ctxs = [lease.ctx for lease in outs[0]["render"].grad_fn.leases]
            else:
                cams, outs = [cam], [g4d.render(cam, pc, _Pipe, bg, stage=stage)]
                ctxs = [outs[0]["render"].grad_fn.lease.ctx]
            torch.cuda.synchronize()
            shs = ctxs[0].read("deformed_shs") if has_sh else torch.cat([scene["features_dc"], scene["features_rest"]], 1).numpy()
            ins = raster_oracle_inputs(ctxs[0].read("deformed"), shs)
            for c, ctx, o in zip(cams, ctxs, outs):
                rc, _ = cam_tuple(c, (0.2, 0.1, 0.0), sh_degree=3)
                ref = rr.rasterize_forward(rc, *ins)
                _assert_extremes(ref, near, far)
                _assert_index_data_bit_exact(ctx, o["radii"].cpu().numpy(), ref, colour_exact=False)
                _assert_pixel_outliers_are_threshold_flips(o["render"].detach().cpu().numpy(), ref, c.image_width)
            del outs, ctxs
    finally:
        ws.set_option(g4d._lib.OPT_TENSOR_CORES, 2)


# ------------------------------------------------------------------------------------------------------------- C
def _sparse_counts():
    G = _sms()
    return [1, 2, 31, G - 1, G, G + 1, 2 * G + 1]


@pytest.mark.parametrize("which", range(7))
def test_sparse_views(which):
    nvis = _sparse_counts()[which]
    cam, ins = ub.sparse_scene(nvis, 50_000, seed=which)
    ctx, ref, _, _ = _rasterize(cam, ins)
    assert ctx.stats().num_visible == nvis


def test_empty_view_of_many_gaussians():
    """n = 100k, nothing visible: background image exactly, R = 0, every range (0, 0), exactly zero gradients"""
    cam, ins = ub.sparse_scene(0, 100_000, seed=9)
    bg = (0.1, 0.2, 0.3)
    ctx, ref, color, dev = _rasterize(cam, ins, bg=bg, grad=True)
    st = ctx.stats()
    assert st.num_visible == 0 and st.num_rendered == 0 and _kbits(ctx) == 1
    assert not ctx.read("ranges").any()
    want = torch.tensor(bg, device="cuda").reshape(3, 1, 1).expand_as(color)
    assert torch.equal(color.detach(), want)
    color.backward(torch.randn(color.shape, generator=torch.Generator().manual_seed(0)).cuda())
    for t in dev:
        if t.requires_grad:
            assert t.grad is not None and not t.grad.any()


def test_screen_filling_gaussian_opens_several_chunks():
    cam, ins = ub.chunk_cut_scene()
    ctx, ref, _, _ = _rasterize(cam, ins)
    G = _sms()
    perm, starts, w, T = ub.chunk_starts(ref["proj"], G)
    k = int(np.argmax(w))
    assert w[k] > 2 * T and int((starts == k + 1).sum()) >= 2       # the one element ends two or more chunks
    assert ctx.stats().num_visible == len(perm)


# ------------------------------------------------------------------------------------------------------------- D
@pytest.mark.parametrize("L", ub.TIER_LENGTHS)
def test_fix_up_tiers(L):
    """one tile, G L Gaussians: every (tile, chunk) sub-segment of bin_fix holds exactly L entries"""
    G = _sms()
    cam, ins = ub.tier_scene(G, L, seed=L)
    ctx, ref, _, _ = _rasterize(cam, ins)
    assert (ctx.read("tiles_touched") == 1).all()
    assert ctx.read("ranges").tolist() == [[0, G * L]]
    _, starts, _, T = ub.chunk_starts(ref["proj"], G)
    assert T == 5 * L and (np.diff(starts) == L).all()


# ------------------------------------------------------------------------------------------------------------- E / F
_BAND_REFS = {}


def _band_case(W, H, clones):
    key = (W, H, clones)
    if key not in _BAND_REFS:
        cam, ins = ub.band_scene(W, H)
        if clones:
            ins = ub.clone_exactly(ins, 0.3, seed=3)
        rc, _ = cam_tuple(cam, (0.0, 0.0, 0.0), sh_degree=3)
        _BAND_REFS.clear()
        _BAND_REFS[key] = (cam, ins, rr.rasterize_forward(rc, *ins))
    return _BAND_REFS[key]


@pytest.mark.parametrize("sync_mode", [1, 0])
@pytest.mark.parametrize("wh,clones", [((3840, 2160), False), ((5120, 2160), False), ((5120, 2160), True)],
                         ids=["3840x2160", "5120x2160", "5120x2160-clones"])
def test_bands(wh, clones, sync_mode):
    """3840 x 2160 places in two bands, 5120 x 2160 also counts in two; the clone arm puts exact ties across the boundaries"""
    cam, ins, ref = _band_case(*wh, clones)
    cb, pb = ub.band_boundaries(*wh)
    assert pb and (cb or wh == (3840, 2160))
    rect = ref["proj"].rect
    for b in cb + pb:
        s, big, clipped = ub.straddlers(rect, b)
        assert s >= 1000 and big >= 10 and clipped >= 1, (b, s, big, clipped)
    ctx, _, _, _ = _rasterize(cam, ins, bg=(0.0, 0.0, 0.0), sync_mode=sync_mode, ref=ref)
    if clones:
        tied, gap = ub.tie_groups(ref["proj"])
        assert tied >= 30_000 and gap > len(ins[0]) // _sms()


def test_exact_clones_at_scale():
    """densify_and_clone: 30 % of 150k Gaussians appended as exact copies, a tenth of those copied again -- runs of identical
    depth bits whose members lie in different radix slices, ordered by index"""
    cam, ins = ub.tie_scene()
    ctx, ref, _, _ = _rasterize(cam, ins, bg=(0.0, 0.0, 0.0))
    n = len(ins[0])
    tied, gap = ub.tie_groups(ref["proj"])
    assert n >= 195_000 and tied >= 0.3 * ctx.stats().num_visible and gap > n // _sms()
