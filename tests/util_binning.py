"""Scenes that drive the tile binning (g4d_bin.cu) into its rarely taken branches, and a numpy restatement of the quantities
that decide which branch runs: the key width kbits of the radix sort, the chunk cuts of the placement and the band rows of
the counting and placement kernels.  Shared by the GPU test (test_gpu_binning_edges.py) and its CPU companion
(test_binning_edge_scenes.py), which checks on the oracle alone that every scene is what the GPU test says it is."""
import math

import numpy as np

from util_scene import synth

# shared-memory budgets of the two banded binning phases (g4d_bin.cu: kCountSmemBudget for bin_sort's per-tile counts,
# kPlaceSmemBudget for bin_place's per-tile cursors; one 4-byte word per tile of a band)
COUNT_SMEM_BUDGET = 160 * 1024
PLACE_SMEM_BUDGET = 96 * 1024
DIGIT_BITS = 9                      # radix digit of bin_sort's LSD passes
H100_SXM_SMS = 132                  # chunk count G on an H100 SXM; the GPU test reads the device's own SM count


def band_rows(W, H):
    """(count band rows, place band rows) of a W x H frame, as launch_bin_sort / launch_bin_place derive them"""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    return min(gy, COUNT_SMEM_BUDGET // (4 * gx)), min(gy, PLACE_SMEM_BUDGET // (4 * gx))


def band_boundaries(W, H):
    """tile rows at which a new count band / place band starts"""
    gy = (H + 15) // 16
    rc, rp = band_rows(W, H)
    return list(range(rc, gy, rc)), list(range(rp, gy, rp))


def depth_bits(depth):
    return np.ascontiguousarray(depth, np.float32).view(np.uint32)


def kbits_of(pr):
    """key width of bin_sort: significant bits of (max - min) of the visible Gaussians' depth bits (1 when the span is 0)"""
    vis = pr.tiles_touched > 0
    if not vis.any():
        return 1
    b = depth_bits(pr.depth)[vis].astype(np.int64)
    return max(1, int(b.max() - b.min()).bit_length())


def passes_of(kbits):
    return (kbits + DIGIT_BITS - 1) // DIGIT_BITS


def chunk_starts(pr, G):
    """bin_sort phase 2: the depth order of the visible Gaussians (stable by index) cut into G chunks of walk cost
    T = ceil(sum(tiles + 4) / G); element k + 1 opens every chunk j with e0(k) < j T <= e1(k).  Returns (perm, starts[G + 1],
    weights in perm order, T)."""
    vis = np.nonzero(pr.tiles_touched > 0)[0]
    perm = vis[np.argsort(depth_bits(pr.depth)[vis], kind="stable")]
    w = pr.tiles_touched[perm].astype(np.int64) + 4
    e1 = np.cumsum(w)
    total = int(e1[-1]) if len(w) else 0
    T = max(1, -(-total // G))
    starts = np.full(G + 1, len(perm), np.int64)
    starts[0] = 0
    for j in range(1, G):
        k = int(np.searchsorted(e1, j * T, side="left"))
        if k < len(perm):
            starts[j] = k + 1
    return perm, starts, w, T


def straddlers(rect, b):
    """(rects covering tile rows b - 1 and b, those of >= 32 tiles, those of >= 32 tiles with < 32 tiles on one side of b)"""
    minx, miny, maxx, maxy = (rect[:, i].astype(np.int64) for i in range(4))
    w = maxx - minx
    s = (miny < b) & (maxy > b)
    big = s & (w * (maxy - miny) >= 32)
    clipped = big & ((w * (b - miny) < 32) | (w * (maxy - b) < 32))
    return int(s.sum()), int(big.sum()), int(clipped.sum())


# ------------------------------------------------------------------------------------------------------------- placement
def front_camera(W, H):
    """camera at (0, 4, 0) looking down -y: its view matrix is a signed permutation plus a translation, so a Gaussian's view
    depth is 4 - y, one exactly rounded fp32 operation"""
    return synth.make_camera(0.0, W, H, phi_deg=0.0)


def _view(cam):
    M = cam.world_view_transform.double().numpy()
    R, t = M[:3, :3], M[3, :3]
    assert np.array_equal(np.abs(R), np.abs(R).round()) and np.array_equal(np.abs(R).sum(0), np.ones(3)), R
    return R, t


def exact_depth_coordinate(cam, depth):
    """world coordinate along the depth axis whose view depth is exactly `depth` (fp32), and that axis"""
    R, t = _view(cam)
    a = int(np.nonzero(R[:, 2])[0][0])
    s = np.float32(R[a, 2])
    d = np.asarray(depth, np.float32)
    c = ((d.astype(np.float64) - t[2]) * s).astype(np.float32)
    assert np.array_equal(np.float32(s) * c + np.float32(t[2]), d), "depth not exact in fp32"
    return a, c


def world_points(cam, px, py, depth, exact=False):
    """fp32 world positions that project to pixel (px, py) at view depth `depth`.  exact: the depth is reproduced bit for bit"""
    W, H = cam.image_width, cam.image_height
    tx, ty = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    d = np.asarray(depth, np.float64)
    pv = np.stack([((2 * np.asarray(px, np.float64) + 1) / W - 1) * tx * d,
                   ((2 * np.asarray(py, np.float64) + 1) / H - 1) * ty * d, d], axis=-1)
    R, t = _view(cam)
    p = ((pv - t) @ R.T).astype(np.float32)
    if exact:
        a, c = exact_depth_coordinate(cam, np.asarray(depth, np.float32))
        p[:, a] = c
    return p


def gaussians(cam, px, py, depth, r_px, rng, opac=(0.1, 0.6), exact=False):
    """post-activation rasterizer inputs (means3D, scales, rots, opacities, shs) of isotropic Gaussians of about r_px pixels
    (3 sigma) centred on (px, py) at the given view depths"""
    n = len(depth)
    fx = cam.image_width / (2 * math.tan(cam.FoVx * 0.5))
    m3 = world_points(cam, px, py, depth, exact)
    sc = np.repeat((np.asarray(r_px, np.float64) / 3.0 * np.asarray(depth, np.float64) / fx)[:, None], 3, 1).astype(np.float32)
    ro = np.zeros((n, 4), np.float32); ro[:, 0] = 1.0
    op = rng.uniform(opac[0], opac[1], (n, 1)).astype(np.float32)
    sh = (rng.standard_normal((n, 16, 3)) * 0.2).astype(np.float32)
    sh[:, 0] = rng.uniform(-1.5, 1.5, (n, 3))
    return [m3, sc, ro, op, sh]


def concat(*parts):
    return [np.ascontiguousarray(np.concatenate([p[i] for p in parts])) for i in range(5)]


def take(ins, idx):
    return [np.ascontiguousarray(a[idx]) for a in ins]


# ------------------------------------------------------------------------------------------------------------- A. pass counts
PASS_SPANS = [0, 2 ** 9 - 1, 2 ** 9, 2 ** 18 - 1, 2 ** 18, 2 ** 27 - 1, 2 ** 27]
PASS_KBITS = {0: (1, 1), 2 ** 9 - 1: (9, 1), 2 ** 9: (10, 2), 2 ** 18 - 1: (18, 2), 2 ** 18: (19, 3), 2 ** 27 - 1: (27, 3),
              2 ** 27: (28, 4)}                                     # span -> (kbits, radix passes)
PASS_WH = (256, 192)


def pass_scene(span, n_mid=30_000, seed=0):
    """visible depth-bit span exactly `span`: two anchors at the ends (the nearest at n // 3, the farthest at 2 n // 3) and
    n_mid Gaussians strictly between; span 0 is a fronto-parallel sheet of 20k overlapping Gaussians at one depth (tie order
    is compositing order there)"""
    rng = np.random.default_rng(seed)
    cam = front_camera(*PASS_WH)
    W, H = PASS_WH
    if span == 0:
        n = 20_000
        d = np.full(n, 3.0, np.float32)
        return cam, gaussians(cam, rng.uniform(0, W, n), rng.uniform(0, H, n), d, rng.uniform(6, 20, n), rng, exact=True)
    lo = np.float32(4.0) if span < 2 ** 23 else np.float32(0.25)
    lo_b = int(depth_bits(np.array([lo]))[0])
    mid_b = rng.integers(lo_b + 1, lo_b + span, n_mid, endpoint=False) if span > 1 else np.zeros(0, np.int64)
    n = len(mid_b) + 2
    anchors = np.array([n // 3, 2 * n // 3])
    d = np.empty(n, np.float32)
    d[np.setdiff1d(np.arange(n), anchors)] = mid_b.astype(np.uint32).view(np.float32)
    d[anchors] = np.array([lo_b, lo_b + span], np.uint32).view(np.float32)
    ins = gaussians(cam, rng.uniform(0, W, n), rng.uniform(0, H, n), d, rng.uniform(2, 6, n), rng)
    # the anchors' depths exactly; the others round monotonically, so they stay inside [lo, hi]
    a, c = exact_depth_coordinate(cam, d[anchors])
    ins[0][anchors, a] = c
    return cam, ins


def four_pass_scene(seed=1):
    """a near cluster at ~0.3 in front of a background shell at ~2e4, sizes proportional to depth"""
    rng = np.random.default_rng(seed)
    cam = front_camera(*PASS_WH)
    W, H = PASS_WH
    n_near, n_far = 4_000, 30_000
    near = gaussians(cam, rng.uniform(0.35 * W, 0.65 * W, n_near), rng.uniform(0.35 * H, 0.65 * H, n_near),
                     rng.uniform(0.27, 0.34, n_near), rng.uniform(2, 12, n_near), rng)
    far = gaussians(cam, rng.uniform(0, W, n_far), rng.uniform(0, H, n_far), rng.uniform(1.8e4, 2.2e4, n_far),
                    rng.uniform(2, 6, n_far), rng)
    ins = concat(far, near)
    return cam, take(ins, rng.permutation(len(ins[0])))


# ------------------------------------------------------------------------------------------------------------- B. extremes
EXTREME_NS = [1, 31, 33, 63, 65, 127, 129, 4097]
EXTREME_WH = (128, 96)


def extreme_positions(n):
    """index 0, n - 1 and the last lane of the last full warp / 64- and 128-Gaussian tensor-core tile before the partial one"""
    cand = {0, n - 1} | {q * ((n - 1) // q) - 1 for q in (32, 64, 128)}
    return sorted(i for i in cand if 0 <= i < n)


def extreme_layouts(n):
    pos = extreme_positions(n)
    return [(a, b) for a in pos for b in pos if a != b] or [(0, 0)]


def extreme_points(n, near, far, seed):
    """[n, 3] positions in front of front_camera(*EXTREME_WH): the Gaussian at `near` is the unique nearest (depth 1.5), the one
    at `far` the unique farthest (depth 3.6); the others lie at depths in [2.2, 2.9], which no deformation of the test nets
    moves across those two"""
    rng = np.random.default_rng(seed)
    cam = front_camera(*EXTREME_WH)
    W, H = EXTREME_WH
    d = rng.uniform(2.2, 2.9, n)
    d[far] = 3.6
    d[near] = 1.5
    return cam, world_points(cam, rng.uniform(0.1 * W, 0.9 * W, n), rng.uniform(0.1 * H, 0.9 * H, n), d), d


def extreme_scene(n, near, far, seed=0):
    cam, m3, d = extreme_points(n, near, far, seed)
    rng = np.random.default_rng(seed + 1)
    ins = gaussians(cam, *np.zeros((2, n)), d, rng.uniform(3, 10, n), rng)
    ins[0] = m3
    return cam, ins


# ------------------------------------------------------------------------------------------------------------- C. sparse / empty / chunk cut
SPARSE_WH = (320, 240)


def sparse_scene(nvis, n, seed=0):
    """n Gaussians of which exactly nvis are visible; the rest are culled in equal shares: behind the camera, nearer than the
    0.2 near plane, and on screen depth but far off the image"""
    rng = np.random.default_rng(seed)
    cam = front_camera(*SPARSE_WH)
    W, H = SPARSE_WH
    m = n - nvis
    k = np.array_split(np.arange(m), 3)
    d = np.concatenate([rng.uniform(2.0, 4.0, nvis), rng.uniform(-3.0, -0.5, len(k[0])), rng.uniform(0.02, 0.19, len(k[1])),
                        rng.uniform(2.0, 4.0, len(k[2]))])
    px = np.concatenate([rng.uniform(0, W, nvis + len(k[0]) + len(k[1])), rng.uniform(-40 * W, -20 * W, len(k[2]))])
    py = rng.uniform(0, H, n)
    r = np.concatenate([rng.uniform(3, 12, nvis + len(k[0]) + len(k[1])), np.full(len(k[2]), 3.0)])
    ins = gaussians(cam, px, py, np.abs(d), r, rng)
    ins[0] = world_points(cam, px, py, d)          # negative depths: behind the camera
    return cam, take(ins, rng.permutation(n))


def chunk_cut_scene(seed=0):
    """one screen-filling Gaussian (walk cost well above the chunk target: it opens several chunks on its own) among 2000
    small ones"""
    rng = np.random.default_rng(seed)
    cam = front_camera(512, 512)
    n = 2000
    small = gaussians(cam, rng.uniform(0, 512, n), rng.uniform(0, 512, n), rng.uniform(2.0, 4.0, n), rng.uniform(2, 8, n), rng)
    big = gaussians(cam, np.array([256.0]), np.array([256.0]), np.array([3.0]), np.array([1200.0]), rng, opac=(0.3, 0.3))
    return cam, concat(take(small, np.arange(n // 2)), big, take(small, np.arange(n // 2, n)))


# ------------------------------------------------------------------------------------------------------------- D. fix-up tiers
TIER_LENGTHS = [1, 4, 5, 8, 9, 12, 13, 16, 17, 24, 25, 32, 33, 64, 65, 128, 129, 256, 257, 600]


def tier_scene(G, L, seed=0):
    """n = G L Gaussians at distinct depths on a one-tile (16 x 16) image: every weight is 5, T = 5 L, so every chunk -- and
    with it every (tile, chunk) sub-segment of the fix-up -- holds exactly L entries"""
    rng = np.random.default_rng(seed)
    cam = front_camera(16, 16)
    n = G * L
    base = int(depth_bits(np.array([2.0]))[0])
    d = (base + 7 * rng.permutation(n).astype(np.uint32)).view(np.float32)    # distinct, in random index order
    return cam, gaussians(cam, rng.uniform(6, 10, n), rng.uniform(6, 10, n), d, rng.uniform(2, 5, n), rng, opac=(0.05, 0.3),
                          exact=True)


# ------------------------------------------------------------------------------------------------------------- E. bands
BAND_FRAMES = [(3840, 2160), (5120, 2160)]


def band_scene(W, H, n_total=150_000, seed=0):
    """~n_total Gaussians on a W x H frame; around every count-band and place-band boundary row a strip of medium Gaussians
    that straddle it and some large ones (>= 32 tiles), part of which keep fewer than 32 tiles on one side"""
    rng = np.random.default_rng(seed)
    cam = front_camera(W, H)
    cb, pb = band_boundaries(W, H)
    bounds = sorted(set(cb) | set(pb))
    parts = []
    for b in bounds:
        m = 3000
        parts.append(gaussians(cam, rng.uniform(0, W, m), 16 * b + rng.uniform(-20, 20, m), rng.uniform(2.0, 10.0, m),
                               rng.uniform(12, 40, m), rng, opac=(0.05, 0.4)))
        m = 80
        parts.append(gaussians(cam, rng.uniform(0, W, m), 16 * b + rng.uniform(-40, 40, m), rng.uniform(2.0, 10.0, m),
                               rng.uniform(60, 130, m), rng, opac=(0.05, 0.3)))
    m = n_total - sum(len(p[0]) for p in parts)
    parts.append(gaussians(cam, rng.uniform(0, W, m), rng.uniform(0, H, m), rng.uniform(2.0, 10.0, m), rng.uniform(3, 14, m),
                           rng, opac=(0.05, 0.5)))
    ins = concat(*parts)
    return cam, take(ins, rng.permutation(len(ins[0])))


# ------------------------------------------------------------------------------------------------------------- F. ties
def clone_exactly(ins, frac, seed):
    """densify_and_clone: exact copies of a random `frac` of the Gaussians appended; then a tenth of those copies cloned again"""
    rng = np.random.default_rng(seed)
    n = len(ins[0])
    a = rng.choice(n, int(frac * n), replace=False)
    ins = concat(ins, take(ins, a))
    b = rng.choice(np.arange(n, len(ins[0])), len(a) // 10, replace=False)
    return concat(ins, take(ins, b))


def tie_scene(n_base=150_000, seed=0):
    """~200k Gaussians of a C3-sized view, 30 % of them cloned exactly and appended, some clones cloned again"""
    from util_scene import raster_inputs
    w = synth.WORKLOADS["C3"]
    cam = synth.make_camera(-40.0, w["width"], w["height"], radius=w["radius"], focal=w["focal"])
    ins = [t.float().numpy() for t in raster_inputs(n_base, 5, scale_mean=w["scale_mean"])]
    return cam, clone_exactly(ins, 0.3, seed)


def tie_groups(pr):
    """(visible Gaussians that share their depth bits with another visible one, largest index distance inside such a group)"""
    vis = np.nonzero(pr.tiles_touched > 0)[0]
    b = depth_bits(pr.depth)[vis]
    o = np.argsort(b, kind="stable")
    bs, vs = b[o], vis[o]
    same = np.r_[False, bs[1:] == bs[:-1]]
    tied = same | np.r_[same[1:], False]
    gap = int((vs[1:] - vs[:-1])[same[1:]].max()) if same.any() else 0
    return int(tied.sum()), gap
