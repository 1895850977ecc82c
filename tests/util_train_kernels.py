"""Cases shared by test_gpu_train_kernels_edges.py (the kernels of g4d_loss.cu, g4d_optim.cu and g4d_knn.cu on their edges)
and its CPU companion test_train_kernels_edge_cases.py, which checks that every case reaches the condition it is named for.
Everything here is plain torch / numpy and runs without a GPU."""
from __future__ import annotations

import copy

import numpy as np
import torch

from oracle import loss_ref as lr
from util_scene import row_errors, synth

# ---- L1 --------------------------------------------------------------------------------------------------------------------
L1_NUMELS = (1, 2, 3, 4, 5, 7, 1023, 1025)            # n & 3 takes every value; 1025 = 256 float4s + a block-0 tail
L1_BATCH = (4, 3, 1014, 1352)                          # the train.py batch at the C3 image size
ODD_HW = (5, 7)                                        # 3 * 5 * 7 = 105 floats per image: batch[i] sits i * 105 floats in


def pair(shape, seed, device="cpu", dtype=torch.float32):
    """(out, gt) in [0, 1] with exact ties on every 7th element (sign(0) = 0 in the L1 gradient)."""
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(shape, generator=g)
    b = (a + 0.2 * torch.randn(shape, generator=g)).clamp(0, 1)
    b.view(-1)[::7] = a.view(-1)[::7]
    return a.to(device=device, dtype=dtype), b.to(device=device, dtype=dtype)


def offset_views(device="cpu"):
    """[(name, out, gt)]: contiguous fp32 views whose storage offset is 1, 2 or 3 floats off a 16-byte boundary on out, on
    gt, or on both -- reached as batch[i] of a [4,3,5,7] batch (105 floats per image) and as flat[k:].view(...)."""
    cases = []
    ob, gb = pair((4, 3) + ODD_HW, 11, device)
    oa, ga = pair((3,) + ODD_HW, 12, device)
    for i in (1, 2, 3):
        cases += [("batch[%d]:out" % i, ob[i], ga), ("batch[%d]:gt" % i, oa, gb[i]), ("batch[%d]:both" % i, ob[i], gb[i])]
    fo, fg = pair((1 + 4 * 1023 + 3,), 13, device)
    for k in (1, 2, 3):
        n = 1023 - k                                    # odd and even lengths, tails of every size
        cases += [("flat[%d:]:out" % k, fo[k:k + n].view(n), fg[:n]), ("flat[%d:]:gt" % k, fo[:n], fg[k:k + n].view(n)),
                  ("flat[%d:]:both" % k, fo[k:k + n].view(n), fg[4 - k:4 - k + n].view(n))]
    return cases


def misalignment(t: torch.Tensor) -> int:
    return t.data_ptr() % 16


# ---- SSIM ------------------------------------------------------------------------------------------------------------------
SSIM_TILE, SSIM_R = 16, 5                               # ssim_*_kernel: 16 x 16 outputs per CTA, 5-pixel halo
SSIM_SIDES = (1, 2, 5, 6, 10, 11, 12, 15, 16, 17, 31, 32, 33)
# (H, W) crossed sparsely: every side appears as H and as W, plus 1 x N and N x 1
SSIM_HW = ((1, 1), (1, 2), (2, 5), (5, 6), (6, 10), (10, 11), (11, 12), (12, 15), (15, 16), (16, 17), (17, 31), (31, 32),
           (32, 33), (33, 1), (2, 1), (6, 5), (11, 33), (33, 17), (16, 16), (32, 32), (12, 31), (15, 2), (10, 32), (17, 6),
           (5, 12), (31, 10), (1, 77), (77, 1))
SSIM_FLOOR = 1e-3        # per-pixel gradient error floor, as a fraction of the largest |gradient| (util_scene.row_errors)
SSIM_K = 8.0             # the kernel may be at most SSIM_K x as far from fp64 as loss_ref.ssim run in fp32
SSIM_FP32_BOUND = 0.25   # ... and that fp32 distance stays below this on every case (checked on the CPU)


def ssim_claims(H, W):
    """What an H x W image exercises in the tiled kernels."""
    return {"window_clipped_both_sides_x": W <= 2 * SSIM_R - 1, "window_clipped_both_sides_y": H <= 2 * SSIM_R - 1,
            "smaller_than_window": H < 2 * SSIM_R + 1 or W < 2 * SSIM_R + 1,
            "seams_x": (W - 1) // SSIM_TILE, "seams_y": (H - 1) // SSIM_TILE,
            "partial_tile_x": W % SSIM_TILE != 0, "partial_tile_y": H % SSIM_TILE != 0}


def ssim_shape(i, H, W):
    """channel layout of the i-th (H, W) case: [1,H,W], [3,H,W] or the [4,3,H,W] batch train.py builds with torch.cat"""
    return ((1, H, W), (3, H, W), (4, 3, H, W))[i % 3]


SSIM_MANY = (1000, 3, 10, 11)                           # 3000 channels: gridDim.z far past one wave


def ssim_images(shape, kind, seed):
    """fp32-representable fp64 (x, y) pairs: 'rand', 'same' (y = x), 'const' (two flat images), 'bright' (0.95 +- 1e-3)."""
    g = torch.Generator().manual_seed(seed)
    r = lambda: torch.rand(shape, generator=g, dtype=torch.float64)
    if kind == "rand":
        x = r(); y = (x + 0.2 * torch.randn(shape, generator=g, dtype=torch.float64)).clamp(0, 1)
    elif kind == "same":
        x = r(); y = x.clone()
    elif kind == "const":
        x = torch.full(shape, 0.3, dtype=torch.float64); y = torch.full(shape, 0.7, dtype=torch.float64)
    elif kind == "bright":
        x = 0.95 + 1e-3 * (2 * r() - 1); y = 0.95 + 1e-3 * (2 * r() - 1)
    else:
        raise ValueError(kind)
    return x.float().double(), y.float().double()


def ssim_ref(x, y, dtype, up):
    """loss_ref.ssim in `dtype` on the CPU: (value, d(up * ssim)/dx as fp64 ndarray)."""
    a = x.to(dtype).clone().requires_grad_(True)
    v = lr.ssim(a, y.to(dtype))
    (v * up).backward()
    return float(v.detach()), a.grad.double().numpy()


def pixel_err(got, ref, floor=SSIM_FLOOR):
    """largest per-pixel error (every element is its own row of util_scene.row_errors)"""
    return float(row_errors(np.asarray(got).reshape(-1, 1), np.asarray(ref).reshape(-1, 1), floor).max(initial=0.0))


# ---- plane regulariser -----------------------------------------------------------------------------------------------------
REG_FLOOR = 1e-2         # per-texel floor (a texel = its C channels), DESIGN.md 2.2's plane-texel floor
REG_K = 8.0              # kernel distance to fp64 <= REG_K x (loss_ref.compute_regulation in fp32's distance) + REG_ABS
# the kernel forms each texel's gradient from the 5-tap stencil of second differences, autograd chains them: where the
# stencil cancels the two fp32 orders differ by a few tens of ulp of the texel (2.8e-6 seen at C = 4 on an H100)
REG_ABS = 1e-5
REG_FP32_BOUND = 1e-3


def reg_args(levels=2, channels=16, time_res=8, base="small128"):
    """synth.hidden_args(base) with the number of levels, the channel count and the time resolution replaced."""
    a = copy.deepcopy(synth.hidden_args(base))
    a.multires = [1, 2, 4, 8][:levels]
    a.kplanes_config["output_coordinate_dim"] = channels
    a.kplanes_config["resolution"] = list(a.kplanes_config["resolution"][:3]) + [time_res]
    return a


REG_CONFIGS = {"4 levels (24 planes)": dict(levels=4), "time res 3": dict(time_res=3), "C = 4": dict(channels=4),
               "C = 12": dict(channels=12), "C = 20, 4 levels, time res 3": dict(channels=20, levels=4, time_res=3)}
REG_WEIGHTS = ((0.0, 1e-4, 2e-4), (1e-3, 0.0, 2e-4), (1e-3, 1e-4, 0.0), (1e-3, 1e-4, 2e-4))   # (time_smooth, l1_time, plane_tv)


def reg_planes(args, seed):
    """the module's planes, made like deform_network's (time planes at 1, the others in U(0.1, 0.5)) and then perturbed,
    so that |1 - p| has both signs and exact zeros: [[1,C,H,W] fp32 x 6] per level, CPU."""
    g = torch.Generator().manual_seed(seed)
    C = args.kplanes_config["output_coordinate_dim"]
    res0 = args.kplanes_config["resolution"]
    out = []
    for m in args.multires:
        res = [r * m for r in res0[:3]] + [res0[3]]
        lvl = []
        for c0, c1 in ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)):
            shape = (1, C, res[c1], res[c0])
            if c1 == 3:
                t = 1.0 + 0.05 * torch.randn(shape, generator=g)
                t.view(-1)[::5] = 1.0
            else:
                t = 0.1 + 0.4 * torch.rand(shape, generator=g)
            lvl.append(t.float())
        out.append(lvl)
    return out


def reg_ref(planes, w, dtype, up):
    """loss_ref.compute_regulation in `dtype`: (value, per-plane d(up * value)/dp as fp64 ndarrays [1,C,H,W])."""
    g = [[p.to(dtype).clone().requires_grad_(True) for p in lvl] for lvl in planes]
    v = lr.compute_regulation(g, *w)
    (v * up).backward()
    return float(v.detach()), [[p.grad.double().numpy() for p in lvl] for lvl in g]


def texel_err(got, ref, floor=REG_FLOOR):
    """largest per-texel error of a [1,C,H,W] plane gradient (a row = the C channels of one texel)"""
    t = lambda a: np.moveaxis(np.asarray(a, np.float64)[0], 0, -1).reshape(-1, np.shape(a)[1])
    return float(row_errors(t(got), t(ref), floor).max(initial=0.0))


# ---- flat Adam -------------------------------------------------------------------------------------------------------------
# (numel, [(begin, end), ...]); learning rates are drawn per segment
ADAM_LAYOUTS = {
    "straddle": (40, [(1, 6), (6, 11), (13, 30), (31, 33)]),               # begins and ends inside float4s, back to back
    "zero-length": (32, [(0, 4), (5, 5), (7, 7), (9, 21), (21, 21), (30, 32)]),
    "gaps": (48, [(2, 5), (9, 14), (22, 23), (30, 38), (45, 47)]),
    "sixteen": (160, [(i * 10 + (i % 3), i * 10 + 7 + (i % 4)) for i in range(16)]),
}
ADAM_BETAS = (0.9, 0.999)
ADAM_EPS = 1e-15


def adam_live(numel, segs):
    m = np.zeros(numel, bool)
    for b, e in segs:
        m[b:e] = True
    return m


def adam_claims(numel, segs):
    """does the layout straddle a float4 (a segment edge strictly inside one) and does it leave gaps?"""
    edges = [x for b, e in segs for x in (b, e) if 0 < x < numel]
    return {"straddles": any(x % 4 for x in edges), "gaps": not adam_live(numel, segs).all(),
            "zero_length": any(b == e for b, e in segs), "count": len(segs)}


def adam_grads(numel, seed):
    """gradients of mixed magnitudes: exact zeros, 1e-20 (v underflows into fp32 subnormals), 1e4 and O(1)"""
    g = np.random.default_rng(seed)
    x = g.standard_normal(numel).astype(np.float32)
    kind = np.arange(numel) % 5
    x[kind == 1] = 0.0
    x[kind == 2] = np.float32(1e-20) * np.sign(x[kind == 2])
    x[kind == 3] = np.float32(1e4) * np.sign(x[kind == 3])
    return x


def ulp32(x):
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)


def adam_expect(p, g, m, v, lrs_per_elem, step, grad_scale, b1=ADAM_BETAS[0], b2=ADAM_BETAS[1], eps=ADAM_EPS):
    """fp64 restatement of torch.optim.Adam's update (no weight decay) from the previous fp32 state.  b1, b2, eps are taken
    as the fp32 values the C-ABI receives.  Returns (m', v', tol_m, tol_v) and a function of the new (m', v') giving
    (p', tol_p): the parameter is restated from the kernel's own new moments, so its tolerance is the final few roundings."""
    f = lambda s: float(np.float32(s))
    b1, b2, eps = f(b1), f(b2), f(eps)
    p, g, m, v = (np.asarray(a, np.float64) for a in (p, g, m, v))
    gr = g * f(grad_scale)
    w = 1.0 - b1
    m1 = m + (gr - m) * w
    v1 = v * b2 + (1.0 - b2) * gr * gr
    tol_m = 4 * ulp32(np.abs(m) + np.abs(gr) * w + np.abs(m1))
    tol_v = 4 * ulp32(v1)
    bc1, bc2 = 1.0 - b1 ** step, 1.0 - b2 ** step

    def param(mk, vk):
        upd = lrs_per_elem * (np.asarray(mk, np.float64) / bc1) / (np.sqrt(np.asarray(vk, np.float64)) / np.sqrt(bc2) + eps)
        p1 = p - upd
        return p1, 8 * ulp32(upd) + 0.5 * ulp32(p1)
    return m1, v1, tol_m, tol_v, param


# ---- kNN -------------------------------------------------------------------------------------------------------------------
def knn_cloud(kind, seed=0):
    g = np.random.default_rng(seed)
    if kind == "identical":
        return np.tile(np.float32([0.25, -1.5, 3.0]), (64, 1))
    if kind == "two stacks":
        return np.concatenate([np.tile(np.float32([0.0, 0.0, 0.0]), (40, 1)), np.tile(np.float32([1.0, 2.0, -0.5]), (25, 1))])
    if kind == "collinear":
        p = np.zeros((3000, 3), np.float32); p[:, 0] = g.random(3000, dtype=np.float32) * 7; p[:, 1] = 0.5; p[:, 2] = -2.0
        return p
    if kind == "cluster + outliers":
        p = (g.standard_normal((8000, 3)) * 0.01).astype(np.float32)
        return np.concatenate([p, np.float32([[1e3, 0, 0], [0, -1e3, 0], [0, 0, 1e3]])])
    if kind == "signed zeros":
        p = g.integers(0, 4, (600, 3)).astype(np.float32)
        p[(p == 0) & (g.random((600, 3)) < 0.5)] = np.float32(-0.0)
        return p
    raise ValueError(kind)


KNN_KINDS = ("identical", "two stacks", "collinear", "cluster + outliers", "signed zeros")
KNN_OFFSETS = ((1e3, 5000), (1e3, 20000), (1e4, 5000), (1e4, 20000))   # (centre, points)
KNN_SPACING_ULP = 300


def knn_offset_cloud(centre, n, seed=0):
    """n points on the fp32 lattice around `centre`: integer multiples of ulp(centre), about KNN_SPACING_ULP ulp apart."""
    g = np.random.default_rng(seed)
    u = float(np.spacing(np.float32(centre)))
    side = int(round(KNN_SPACING_ULP * n ** (1.0 / 3.0)))
    k = g.integers(-side // 2, side // 2, (n, 3))
    return (np.float64(centre) + k * u).astype(np.float32)


def knn_grid(xyz):
    """the grid knn_setup_kernel builds, in fp32: (bmin, cs, dim) per axis"""
    p = np.asarray(xyz, np.float32)
    bmin = p.min(axis=0)
    ext = np.maximum(p.max(axis=0) - bmin, np.float32(0))
    longest = max(float(ext.max()), 1e-30)
    target = np.cbrt(np.float32(max(len(p) / 4.0, 1.0)))
    dim = np.clip(np.ceil(target * ext / np.float32(longest)), 1, 128).astype(np.int64)
    cs = np.where(ext > 0, ext / dim.astype(np.float32), np.float32(1)).astype(np.float32)
    return bmin, cs, dim


def knn_face_rounding(xyz):
    """per axis, max over the cell faces k of |fl(bmin + fl(k * cs)) - (bmin + k * cs)| / cs: how far the face position the
    search's stopping rule uses lies from the exact one, in cell sizes"""
    bmin, cs, dim = knn_grid(xyz)
    out = []
    for a in range(3):
        k = np.arange(int(dim[a]) + 1)
        face32 = (np.float32(bmin[a]) + (k.astype(np.float32) * np.float32(cs[a])).astype(np.float32)).astype(np.float32)
        exact = np.float64(bmin[a]) + k * np.float64(cs[a])
        out.append(float(np.abs(face32.astype(np.float64) - exact).max() / float(cs[a])))
    return out
