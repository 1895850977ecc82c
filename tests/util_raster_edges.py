"""Scenes that put Gaussians on the boundaries of the per-Gaussian projection (g4d_math.cuh, geom_finish.cuh) and of the blend
kernels (g4d_raster.cu): clamped opacities, pixels with 255-513 contributors, the 1.3 tanfov guard band, the 0.2 near plane,
rects clamped at every grid side, the SH colour clamp, degenerate covariances and images of 1-33 pixels a side.

Every scene is seen by origin_camera(): a camera at the world origin whose view matrix is a signed permutation, so a
Gaussian's view-space position is its world position permuted and negated, exactly, and a boundary found in fp32 here is the
boundary the kernels and the oracle see.  Each Scene carries rows (named index sets) and claim(rec), which asserts that the
scene reaches its condition on a record of projected data -- the oracle's (test_raster_edge_scenes.py) or the GPU's
(test_gpu_raster_edges.py).  A record is a dict of radii, rect, xy, conic_op, rgb, clamped, n_contrib [H, W], final_T [H, W]
and ranges."""
import dataclasses
import math

import numpy as np
import torch

import util_binning as ub
from util_scene import synth

f32 = np.float32
ALPHA_MAX = f32(0.99)
LONG_OPACITY = 0.011              # about 830 layers before T < 1e-4
LONG_COUNTS = [255, 256, 257, 511, 512, 513]
LONG_SKIP = 1400                  # stops near 833 (later where a network lowers the opacities): > 256 entries to spare
OPAQUE_OPACITIES = [0.995, 0.9999, 1.0]
OPAQUE_LOGITS = {0.995: 6.0, 0.9999: 10.0, 1.0: 20.0}     # fused paths reach opacity through the logit; 20 rounds to 1.0f
SHAPES = [(1, 1), (1, 17), (17, 1), (2, 33), (15, 15), (16, 16), (17, 17), (33, 2)]


@dataclasses.dataclass
class Scene:
    name: str
    group: str
    cam: object
    ins: list                     # post-activation fp32 (means3D, scales, rots, opacities, shs)
    bg: tuple
    deg: int
    rows: dict
    claim: object                 # claim(sc, rec, fused=False): asserts the condition
    fused_claim: bool = True      # the condition survives the network (means exact, other attributes deformed)

    @property
    def W(self):
        return self.cam.image_width

    @property
    def H(self):
        return self.cam.image_height


def origin_camera(W, H):
    """ub.front_camera's orientation (looking down -y) moved to the origin: view (x, y, z) = (-x, -z, -y), exactly"""
    cam = ub.front_camera(W, H)
    wvt = cam.world_view_transform.clone()
    wvt[3, :3] = 0.0
    proj = synth.projection_matrix(0.01, 100.0, cam.FoVx, cam.FoVy).transpose(0, 1)
    full = wvt.unsqueeze(0).bmm(proj.unsqueeze(0)).squeeze(0).contiguous()
    return dataclasses.replace(cam, world_view_transform=wvt, full_proj_transform=full, camera_center=torch.zeros(3))


def tangents(cam):
    """(tanfovx, tanfovy, limx, limy) in fp32, as the oracle and the kernels form them"""
    tx, ty = f32(math.tan(cam.FoVx * 0.5)), f32(math.tan(cam.FoVy * 0.5))
    return tx, ty, f32(1.3) * tx, f32(1.3) * ty


def focal(cam):
    tx, ty, _, _ = tangents(cam)
    return cam.image_width / (2.0 * float(tx)), cam.image_height / (2.0 * float(ty))


def view_of(cam, means):
    """view-space positions in fp32, the operation order of xform4x3"""
    v = cam.world_view_transform.numpy().astype(f32).reshape(16)
    m = np.asarray(means, f32)
    return np.stack([v[r] * m[:, 0] + v[4 + r] * m[:, 1] + v[8 + r] * m[:, 2] + v[12 + r] for r in range(3)], -1)


def world_of(cam, pv):
    """exact inverse of view_of for origin_camera"""
    R, t = ub._view(cam)
    assert not t.any()
    p = (np.asarray(pv, np.float64) @ R.T).astype(f32)
    assert np.array_equal(view_of(cam, p), np.asarray(pv, f32))
    return p


def guard_flags(cam, means):
    """(clampx, clampy) of cov2d_project, evaluated in fp32"""
    pv = view_of(cam, means)
    _, _, limx, limy = tangents(cam)
    with np.errstate(divide="ignore", invalid="ignore"):
        xz, yz = pv[:, 0] / pv[:, 2], pv[:, 1] / pv[:, 2]
    return (xz < -limx) | (xz > limx), (yz < -limy) | (yz > limy)


def pixel_view(cam, px, py, depth):
    """view-space points at pixel (px, py) and view depth `depth` (exact in fp32)"""
    tx, ty, _, _ = tangents(cam)
    W, H = cam.image_width, cam.image_height
    d = np.asarray(depth, np.float64)
    return np.stack([((2 * np.asarray(px, np.float64) + 1) / W - 1) * float(tx) * d,
                     ((2 * np.asarray(py, np.float64) + 1) / H - 1) * float(ty) * d, d], -1).astype(f32)


def gaussians(cam, pv, sigma_px, opac, rng, sh_scale=0.2):
    """Gaussians of about sigma_px pixels at view-space points pv: scales within 20 % of each other and random rotations, so
    that no gradient row is zero by symmetry"""
    pv = np.asarray(pv, f32)
    n = len(pv)
    fx, _ = focal(cam)
    sc = np.repeat((np.broadcast_to(np.asarray(sigma_px, np.float64), (n,)) * np.abs(pv[:, 2]) / fx)[:, None], 3, 1)
    sc = sc * rng.uniform(0.85, 1.0, (n, 3))
    ro = rng.standard_normal((n, 4))
    ro = (ro / np.linalg.norm(ro, axis=1, keepdims=True)).astype(f32)
    op = np.broadcast_to(np.asarray(opac, f32), (n,)).reshape(n, 1).copy()
    sh = (rng.standard_normal((n, 16, 3)) * sh_scale).astype(f32)
    sh[:, 0] = rng.uniform(-1.5, 1.5, (n, 3))
    return [world_of(cam, pv), sc.astype(f32), ro, op, sh]


# ------------------------------------------------------------------------------------------------------------- records
def oracle_record(fwd):
    pr = fwd["proj"]
    return dict(radii=fwd["radii"], rect=pr.rect, xy=pr.xy, conic_op=pr.conic_op, rgb=pr.rgb, clamped=pr.clamped,
                n_contrib=fwd["n_contrib"], final_T=fwd["final_T"], ranges=fwd["bin"].ranges, ids=fwd["bin"].ids)


def gpu_record(ctx, radii, W, H):
    return dict(radii=radii, rect=ctx.read("rect"), xy=ctx.read("xy"), conic_op=ctx.read("conic_opacity"), rgb=ctx.read("rgb"),
                clamped=ctx.read("clamped"), n_contrib=ctx.read("n_contrib").reshape(H, W),
                final_T=ctx.read("final_T").reshape(H, W), ranges=ctx.read("ranges"), ids=ctx.read("sorted_ids"))


def raw_alpha(rec, ids, px, py):
    """o G (before the clamp) of instances ids at pixels (px, py), in fp64: [len(ids), len(px)]"""
    xy = rec["xy"][ids].astype(np.float64); co = rec["conic_op"][ids].astype(np.float64)
    dx = xy[:, 0:1] - np.asarray(px, np.float64)[None]
    dy = xy[:, 1:2] - np.asarray(py, np.float64)[None]
    power = -0.5 * (co[:, 0:1] * dx * dx + co[:, 2:3] * dy * dy) - co[:, 1:2] * dx * dy
    return co[:, 3:4] * np.exp(np.minimum(power, 0.0)), power


def all_clamped_pixels(rec, W, H, margin=1e-4):
    """[H, W] bool: pixels with at least one contributor where every instance up to and including the one that stops the pixel
    (or up to its last contributor when nothing stops it) is either clamped with room to spare (o G >= 0.99 (1 + margin)) or
    far below 1/255.  Their alphas are 0.99f exactly on both sides, so n_contrib and final_T do not depend on exp."""
    nc, out = rec["n_contrib"], np.zeros((H, W), bool)
    gx = (W + 15) // 16
    for y in range(H):
        for x in range(W):
            last = int(nc[y, x])
            if last == 0:
                continue
            lo, hi = (int(v) for v in rec["ranges"][(y // 16) * gx + x // 16])
            ids = rec["ids"][lo:min(hi, lo + last + 1)].astype(np.int64)
            a, power = raw_alpha(rec, ids, [x], [y])
            a, power = a[:, 0], power[:, 0]
            ok = (a >= ALPHA_MAX * (1 + margin)) | (a < (1.0 / 255.0) * (1 - 1e-3)) | (power > 1e-6)
            out[y, x] = ok.all() and (a[:last] >= ALPHA_MAX * (1 + margin)).any()
    return out


def _tile_list_len(rec, tile=0):
    lo, hi = rec["ranges"][tile]
    return int(hi) - int(lo)


# ------------------------------------------------------------------------------------------------------------- opaque
def opaque_scene(opacity, layers, thin=0):
    """`layers` Gaussians of opacity `opacity` stacked on the image centre (sigma 40 px, so o G >= 0.99 on a central disc),
    behind `thin` Gaussians of opacity 0.3; a non-zero background.  Two clamped layers take T to (1 - 0.99f)^2 < 1e-4: the
    pixel stops at the second and shows only the first."""
    rng = np.random.default_rng(int(opacity * 1e4) + 10 * layers + thin)
    W, H = 24, 20
    cam = origin_camera(W, H)
    cx, cy = (W - 1) / 2, (H - 1) / 2
    front = gaussians(cam, pixel_view(cam, [cx] * thin, [cy] * thin, 1.0 + 0.1 * np.arange(thin)), 40.0, 0.3, rng)
    stack = gaussians(cam, pixel_view(cam, [cx] * layers, [cy] * layers, 2.0 + 0.5 * np.arange(layers)), 40.0, opacity, rng)
    ins = ub.concat(front, stack)
    rows = dict(thin=np.arange(thin), opaque=thin + np.arange(layers))

    def claim(sc, rec, fused=False):
        ys, xs = np.mgrid[0:H, 0:W]
        a, _ = raw_alpha(rec, rows["opaque"], xs.reshape(-1), ys.reshape(-1))
        core = (a >= ALPHA_MAX * (1 + 1e-4)).all(axis=0).reshape(H, W)
        assert core.sum() >= 4, int(core.sum())
        nc = rec["n_contrib"][core]
        assert (nc == thin + 1).all(), np.unique(nc)        # thin layers, the first clamped layer, then the stop (or the end)
        if thin == 0:
            assert (rec["final_T"][core] == f32(1.0) - ALPHA_MAX).all()
    return Scene("opaque_o%g_l%d_t%d" % (opacity, layers, thin), "opaque", cam, ins, (0.3, 0.6, 0.9), 3, rows, claim)


# ------------------------------------------------------------------------------------------------------------- long tiles
def long_scene(count):
    """one 16 x 16 tile under `count` Gaussians of opacity 0.011 at distinct depths, each nearly flat over the tile
    (sigma 250 px): every pixel has exactly `count` contributors when count < 830; LONG_SKIP stops every pixel near 833"""
    rng = np.random.default_rng(count)
    cam = origin_camera(16, 16)
    d = (2.0 + 0.0005 * np.arange(count)).astype(f32)
    ins = gaussians(cam, pixel_view(cam, np.full(count, 7.5), np.full(count, 7.5), d), 250.0, LONG_OPACITY, rng)
    rows = dict(all=np.arange(count))

    def claim(sc, rec, fused=False):
        nc = rec["n_contrib"]
        assert _tile_list_len(rec) == count
        if count < 800 and not fused:
            assert (nc == count).all() and (rec["final_T"] > 1e-4).all(), np.unique(nc)
        elif count < 800:     # a fused test silences the Gaussians on a kink of the network, and the network moves opacities
            assert (nc >= 0.9 * count).all() and (rec["final_T"] > 1e-4).all(), np.unique(nc)
        else:
            assert (nc > 800).all() and (nc < count).all(), np.unique(nc)          # every pixel stopped by T < 1e-4
            assert int(nc.max()) + 256 < count                                      # blend backward skips a whole batch
            assert int(nc.max()) + 1 <= 256 * ((count - 1) // 256)                  # blend forward: all done before the last batch
    return Scene("long_%d" % count, "long", cam, ins, (0.1, 0.1, 0.1), 3, rows, claim)


# ------------------------------------------------------------------------------------------------------------- guard band
def guard_scene():
    """view-space x/z and y/z exactly at +-limx / +-limy (not clamped; the comparison is strict) and one float beyond
    (clamped), at depth 2; and large Gaussians whose means lie at 1.6 tanfov beyond the band on each side and at the four
    corners, whose footprints still cover tiles"""
    rng = np.random.default_rng(7)
    W, H = 64, 48
    cam = origin_camera(W, H)
    tx, ty, limx, limy = tangents(cam)
    d = f32(2.0)
    pv = []
    for lim, axis in ((limx, 0), (limy, 1)):
        for v in (lim, -lim, np.nextafter(lim, f32(np.inf)), -np.nextafter(lim, f32(np.inf))):
            p = [f32(0), f32(0), d]
            p[axis] = f32(v * d)                          # v * 2 is exact, and so is (v * 2) / 2
            pv.append(p)
    band = gaussians(cam, np.array(pv, f32), 15.0, 0.7, rng)
    pb = []
    for sx, sy in ((1, 0), (-1, 0), (0, 1), (0, -1), (1, 1), (1, -1), (-1, 1), (-1, -1)):
        pb.append([sx * 1.6 * float(tx) * 2.0, sy * 1.6 * float(ty) * 2.0, 2.0])
    beyond = gaussians(cam, np.array(pb, f32), 30.0, 0.8, rng)
    mid = gaussians(cam, pixel_view(cam, rng.uniform(0, W, 12), rng.uniform(0, H, 12), rng.uniform(1.5, 3.0, 12)), 5.0, 0.5, rng)
    ins = ub.concat(band, beyond, mid)
    rows = dict(exact=np.array([0, 1, 4, 5]), beyond_one_float=np.array([2, 3, 6, 7]), beyond_big=8 + np.arange(8))

    def claim(sc, rec, fused=False):
        cx, cy = guard_flags(cam, sc.ins[0])
        pvv = view_of(cam, sc.ins[0])
        on = np.abs(np.concatenate([pvv[:4, 0] / pvv[:4, 2], pvv[4:8, 1] / pvv[4:8, 2]]))
        assert np.array_equal(on, np.array([limx, limx, np.nextafter(limx, f32(1)), np.nextafter(limx, f32(1)),
                                            limy, limy, np.nextafter(limy, f32(1)), np.nextafter(limy, f32(1))], f32))
        assert not (cx | cy)[rows["exact"]].any()
        assert (cx | cy)[rows["beyond_one_float"]].all()
        bb = rows["beyond_big"]
        assert (cx[bb[[0, 1, 4, 5, 6, 7]]]).all() and (cy[bb[[2, 3, 4, 5, 6, 7]]]).all()
        assert (rec["radii"][:16] > 0).all()
        out = (rec["xy"][bb, 0] < 0) | (rec["xy"][bb, 0] > W) | (rec["xy"][bb, 1] < 0) | (rec["xy"][bb, 1] > H)
        assert out.all()
    return Scene("guard_band", "guard", cam, ins, (0.2, 0.2, 0.2), 3, rows, claim)


# ------------------------------------------------------------------------------------------------------------- near plane
def near_scene():
    """view depth exactly 0.2f (culled: the test is <=), the next float up with a screen-filling footprint (kept, rect clamped
    to the whole grid), depths in (0.2, 0.3), and Gaussians behind the camera and at depth 0"""
    rng = np.random.default_rng(3)
    W, H = 48, 32
    cam = origin_camera(W, H)
    z = f32(0.2)
    at = gaussians(cam, np.array([[0.0, 0.0, z], [0.01, 0.0, z]], f32), 30.0, 0.6, rng)
    up = gaussians(cam, np.array([[0.0, 0.0, np.nextafter(z, f32(1))]], f32), 40.0, 0.5, rng)
    near = gaussians(cam, pixel_view(cam, [5, 40, 20, 30], [5, 8, 25, 16], [0.21, 0.23, 0.25, 0.29]), 4.0, 0.8, rng)
    behind = gaussians(cam, np.array([[0.0, 0.0, -1.0], [0.1, 0.1, -0.1], [0.1, 0.0, 0.0], [0.2, 0.0, -3.0]], f32), 20.0, 0.9,
                       rng)
    behind[1][:] = 0.05
    mid = gaussians(cam, pixel_view(cam, rng.uniform(0, W, 10), rng.uniform(0, H, 10), rng.uniform(1.5, 3.0, 10)), 4.0, 0.5, rng)
    ins = ub.concat(at, up, near, behind, mid)
    rows = dict(at_plane=np.array([0, 1]), above_plane=np.array([2]), near=3 + np.arange(4), behind=7 + np.arange(4))

    def claim(sc, rec, fused=False):
        pvz = view_of(cam, sc.ins[0])[:, 2]
        assert (pvz[rows["at_plane"]] == z).all() and pvz[2] == np.nextafter(z, f32(1))
        assert ((pvz[rows["near"]] > 0.2) & (pvz[rows["near"]] < 0.3)).all() and (pvz[rows["behind"]] <= 0).all()
        assert (rec["radii"][rows["at_plane"]] == 0).all() and (rec["radii"][rows["behind"]] == 0).all()
        assert (rec["radii"][rows["near"]] > 0).all()
        gx, gy = (W + 15) // 16, (H + 15) // 16
        assert rec["radii"][2] > 0 and rec["rect"][2].tolist() == [0, 0, gx, gy]
        r = float(rec["radii"][2])
        assert rec["xy"][2, 0] - r < 0 and rec["xy"][2, 0] + r > W and rec["xy"][2, 1] - r < 0 and rec["xy"][2, 1] + r > H
    return Scene("near_plane", "near", cam, ins, (0.0, 0.3, 0.1), 3, rows, claim)


# ------------------------------------------------------------------------------------------------------------- off-screen
def offscreen_scene():
    """means left of, right of, above and below the image, 30 px out (px -+ rad clamps at that grid edge), and about 1e4 px
    out with footprints (sigma 5000 px; 3 sigma is not an integer, so the radius is not on a rounding edge) that still reach in"""
    rng = np.random.default_rng(5)
    W, H = 48, 40
    cam = origin_camera(W, H)
    cx, cy = (W - 1) / 2, (H - 1) / 2
    px = np.array([-30, W + 30, cx, cx, -1e4, W + 1e4, cx, cx], np.float64)
    py = np.array([cy, cy, -30, H + 30, cy, cy, -1e4, H + 1e4], np.float64)
    edge = gaussians(cam, pixel_view(cam, px[:4], py[:4], np.full(4, 2.0)), 20.0, 0.7, rng)
    far = gaussians(cam, pixel_view(cam, px[4:], py[4:], np.full(4, 2.0)), 5000.37, 0.5, rng)
    mid = gaussians(cam, pixel_view(cam, rng.uniform(0, W, 10), rng.uniform(0, H, 10), rng.uniform(1.5, 3.0, 10)), 4.0, 0.5, rng)
    ins = ub.concat(edge, far, mid)
    rows = dict(edge=np.arange(4), far=4 + np.arange(4))

    def claim(sc, rec, fused=False):
        gx, gy = (W + 15) // 16, (H + 15) // 16
        assert (rec["radii"][:8] > 0).all()
        xy, r, rect = rec["xy"], rec["radii"].astype(np.float64), rec["rect"]
        for k in (0, 4):                                                   # left
            assert xy[k, 0] < 0 and xy[k, 0] - r[k] < 0 and rect[k, 0] == 0
        for k in (1, 5):                                                   # right
            assert xy[k, 0] > W and xy[k, 0] + r[k] + 15 > 16 * gx and rect[k, 2] == gx
        for k in (2, 6):                                                   # above
            assert xy[k, 1] < 0 and rect[k, 1] == 0
        for k in (3, 7):                                                   # below
            assert xy[k, 1] > H and rect[k, 3] == gy
        assert (np.abs(xy[4:8] - np.array([[cx, cy]])).max(axis=1) > 9e3).all()
    return Scene("offscreen", "offscreen", cam, ins, (0.5, 0.4, 0.3), 3, rows, claim)


# ------------------------------------------------------------------------------------------------------------- colour clamp
def colour_scene(deg):
    """per channel, one Gaussian whose SH colour is exactly 0 after the + 0.5 (kept: the gradient flows) and one whose DC
    coefficient is the next float below (clamped: no colour gradient).  Found by walking the DC coefficient float by float
    through the oracle's own evaluation."""
    from oracle import raster_ref as rr
    from util_scene import cam_tuple
    rng = np.random.default_rng(11 + deg)
    W, H = 32, 32
    cam = origin_camera(W, H)
    rc, _ = cam_tuple(cam, (0.0, 0.0, 0.0), sh_degree=deg)
    pts = pixel_view(cam, [6, 16, 26, 6, 16, 26], [8, 8, 8, 24, 24, 24], np.full(6, 2.0))
    base = gaussians(cam, pts, 4.0, 0.8, rng, sh_scale=0.1)
    base[4][:, 0] = rng.uniform(0.5, 1.5, (6, 3))
    from oracle.dense_ref import _sh_color
    span = 512
    steps = np.arange(-span, span + 1)
    for ch in range(3):
        k = ch                                              # Gaussian k: exact zero; k + 3, at the same point: the float below
        for _ in range(20):
            d = base[0][k].astype(np.float64)
            rest = base[4][k:k + 1].astype(np.float64).copy()
            rest[:, 0] = 0.0
            acc_rest = float(_sh_color(deg, torch.from_numpy(rest), torch.from_numpy(d / np.linalg.norm(d))[None])[0, ch])
            guess = f32((-0.5 - acc_rest) / 0.28209479177387814)
            cand = np.unique((guess + steps * np.spacing(guess)).astype(f32))
            sh = np.repeat(base[4][k:k + 1], len(cand), 0)
            sh[:, 0, ch] = cand
            rep = [np.repeat(a[k:k + 1], len(cand), 0) for a in base[:4]]
            pr = rr.preprocess(rc, *rep, sh)
            hit = np.nonzero((pr.rgb[1:, ch] == 0) & (pr.clamped[1:, ch] == 0) & (pr.clamped[:-1, ch] == 1))[0] + 1
            if len(hit) and cand[hit[0] - 1] == np.nextafter(cand[hit[0]], f32(-np.inf)):
                base[4][k, 0, ch] = cand[hit[0]]
                base[4][k + 3] = base[4][k]
                base[4][k + 3, 0, ch] = cand[hit[0] - 1]
                base[0][k + 3] = base[0][k]
                break
            base[4][k, 1:] = (rng.standard_normal((15, 3)) * 0.1).astype(f32)   # the sum skips 0 on this walk: other SH
        else:
            raise AssertionError(("no exact colour zero", deg, ch))
    mid = gaussians(cam, pixel_view(cam, rng.uniform(0, W, 8), rng.uniform(0, H, 8), rng.uniform(1.5, 3.0, 8)), 4.0, 0.5, rng)
    ins = ub.concat(base, mid)
    rows = dict(zero=np.arange(3), below=3 + np.arange(3))

    def claim(sc, rec, fused=False):
        for ch in range(3):
            z, b = rows["zero"][ch], rows["below"][ch]
            assert rec["radii"][z] > 0 and rec["radii"][b] > 0
            assert rec["rgb"][z, ch] == 0 and rec["clamped"][z, ch] == 0
            assert rec["rgb"][b, ch] == 0 and rec["clamped"][b, ch] == 1
            assert sc.ins[4][b, 0, ch] == np.nextafter(sc.ins[4][z, 0, ch], f32(-np.inf))
    return Scene("colour_deg%d" % deg, "colour", cam, ins, (0.1, 0.1, 0.1), deg, rows, claim, fused_claim=False)


# ------------------------------------------------------------------------------------------------------------- covariance
def covariance_scene():
    """needles (two scales of 1e-6), discs (one), Gaussians with every scale 1e-6 (the radius comes from the 0.3 dilation and
    the 0.1 discriminant floor: 3 px), one huge scale, and quaternions of norm 0.5 and 2 and with a negative real part (the
    rasterizer does not normalise them)"""
    rng = np.random.default_rng(13)
    W, H = 48, 32
    cam = origin_camera(W, H)
    n = 14
    ins = gaussians(cam, pixel_view(cam, rng.uniform(4, W - 4, n), rng.uniform(4, H - 4, n), rng.uniform(1.5, 3.0, n)), 5.0, 0.7,
                    rng)
    sc, ro = ins[1], ins[2]
    q = rng.standard_normal((n, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[:, 0] = np.abs(q[:, 0])
    ro[:] = q.astype(f32)
    sc[0:3] = [[0.05, 1e-6, 1e-6], [1e-6, 0.08, 1e-6], [1e-6, 1e-6, 0.06]]          # needles
    sc[3:6] = [[0.05, 0.04, 1e-6], [1e-6, 0.06, 0.03], [0.07, 1e-6, 0.05]]           # discs
    sc[6:8] = 1e-6                                                                   # points
    ro[6] = [1, 0, 0, 0]
    sc[8] = 50.0                                                                     # huge
    ro[9] *= 0.5; ro[10] *= 2.0                                                      # norm 0.5, 2
    ro[11, 0] = -abs(ro[11, 0]); ro[12] = -ro[12]                                    # negative real part
    ins[1], ins[2] = sc.astype(f32), ro.astype(f32)
    rows = dict(needle=np.arange(3), disc=3 + np.arange(3), point=np.array([6, 7]), huge=np.array([8]),
                quat=np.array([9, 10, 11, 12]))

    def claim(sc_, rec, fused=False):
        assert (rec["radii"][:13] > 0).all()
        assert (rec["radii"][rows["point"]] == 3).all(), rec["radii"][rows["point"]]
        gx, gy = (W + 15) // 16, (H + 15) // 16
        assert rec["rect"][8].tolist() == [0, 0, gx, gy]
        if not fused:
            nq = np.linalg.norm(sc_.ins[2][9:13].astype(np.float64), axis=1)
            assert abs(nq[0] - 0.5) < 1e-6 and abs(nq[1] - 2.0) < 1e-6 and (sc_.ins[2][11:13, 0] < 0).all()
    return Scene("covariance", "covariance", cam, ins, (0.2, 0.3, 0.4), 3, rows, claim)


# ------------------------------------------------------------------------------------------------------------- image shapes
def shape_scene(W, H):
    """a W x H image (1 .. 33 px a side): partial tiles and the in0 / in1 lanes of the blend kernels (rows r and r + 2)"""
    rng = np.random.default_rng(100 * W + H)
    cam = origin_camera(W, H)
    n = 24
    ins = gaussians(cam, pixel_view(cam, rng.uniform(-2, W + 2, n), rng.uniform(-2, H + 2, n), rng.uniform(1.5, 3.0, n)),
                    rng.uniform(1.0, 6.0, n), rng.uniform(0.2, 0.9, n).astype(f32), rng)
    rows = dict(all=np.arange(n))

    def claim(sc, rec, fused=False):
        assert rec["n_contrib"].shape == (H, W) and (rec["n_contrib"] > 0).mean() >= 0.5
        assert (rec["radii"] > 0).sum() >= 3
    return Scene("shape_%dx%d" % (W, H), "shape", cam, ins, (0.3, 0.2, 0.1), 3, rows, claim)


def all_scenes():
    out = [opaque_scene(o, l) for o in OPAQUE_OPACITIES for l in (1, 2, 3, 4)]
    out += [opaque_scene(o, 2, thin=3) for o in OPAQUE_OPACITIES]
    out += [long_scene(k) for k in LONG_COUNTS + [LONG_SKIP]]
    out += [guard_scene(), near_scene(), offscreen_scene(), colour_scene(0), colour_scene(3), covariance_scene()]
    out += [shape_scene(W, H) for W, H in SHAPES]
    return out


_CACHE = {}


def scene(name):
    if not _CACHE:
        for s in all_scenes():
            _CACHE[s.name] = s
    return _CACHE[name]


def names():
    """scene names without building them (for parametrize)"""
    out = ["opaque_o%g_l%d_t0" % (o, l) for o in OPAQUE_OPACITIES for l in (1, 2, 3, 4)]
    out += ["opaque_o%g_l2_t3" % o for o in OPAQUE_OPACITIES]
    out += ["long_%d" % k for k in LONG_COUNTS + [LONG_SKIP]]
    out += ["guard_band", "near_plane", "offscreen", "colour_deg0", "colour_deg3", "covariance"]
    out += ["shape_%dx%d" % wh for wh in SHAPES]
    return out
