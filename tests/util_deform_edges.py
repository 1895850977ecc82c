"""Deformation-network scenes that sit exactly on the edges of the HexPlane field and of the network's kernels.

Every scene uses the AABB [[1, 1, 1], [-1, -1, -1]] (xyz_max | xyz_min): scale = 2 / (xyz_min - xyz_max) = -1, so the
normalised coordinate (hexplane.cuh AabbNorm, oracle.deform_ref.normalize) is exactly -x in fp32 and in fp64 for the dyadic
coordinates used here, and the texel coordinate ((u + 1) / 2) * (size - 1) lands exactly on a texel line in fp32 only where it
does in fp64.  So fp32 and fp64 take every cell decision (floor, border clamp, the coordinate-gradient multiplier) identically,
and no row needs masking near a texel line.
Interior texel lines are only reached on levels whose size - 1 is a power of two (the level-0 sizes 3 and 5 below).

Each scene records, per row and axis, the condition it claims (FACE_MAX ... NEG_INF); tests/test_deform_edge_cases.py checks
the claims with an fp32 restatement of AabbNorm / make_tap.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from util_scene import g4d, synth

F32 = np.float32
AABB = np.array([[1.0, 1.0, 1.0], [-1.0, -1.0, -1.0]], dtype=np.float32)

# claims about one coordinate of one row (per spatial axis, at every level unless stated)
FACE_MAX = "face_max"          # u = -1 exactly: texel coordinate 0, coordinate gradient 0 (the xyz_max face)
FACE_MIN = "face_min"          # u = +1 exactly: texel coordinate size - 1, coordinate gradient 0 (the xyz_min face)
INSIDE = "inside"              # 0 < texel coordinate < size - 1 at every level (one ulp inside a face, or interior)
OUT_MAX = "out_max"            # u < -1: clamped to texel 0
OUT_MIN = "out_min"            # u > +1: clamped to size - 1
NAN = "nan"                    # a NaN coordinate: the kernels clamp it to texel 0 (fmaxf drops the NaN)
POS_INF = "pos_inf"            # x = +inf: u = -inf, clamped like FACE_MAX
NEG_INF = "neg_inf"            # x = -inf: u = +inf, clamped like FACE_MIN

INTERIOR = (F32(0.375), F32(-0.125), F32(0.8125))   # coordinates of the axes not under test (no texel line at any level)
JUST_IN_MAX = F32(1.0 - 2.0 ** -24)                 # u = -1 + 2^-24 (exact: x - 1 = -2^-24)
JUST_IN_MIN = F32(-1.0 + 2.0 ** -23)                # u = 1 - 2^-23 (-1 + 2^-24 would round x - 1 to -2, onto the face)
OUT_NEAR_MAX = F32(1.0 + 2.0 ** -23)
OUT_NEAR_MIN = F32(-1.0 - 2.0 ** -22)


# --------------------------------------------------------------------------------------------------- fp32 restatement
def norm32(x) -> np.ndarray:
    """hexplane.cuh AabbNorm at this AABB: __fadd_rn(__fmul_rn(x - amax, scale), -1) in fp32"""
    x = np.asarray(x, dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        return ((x - F32(1.0)) * F32(-1.0)) + F32(-1.0)


def tap32(u, size: int):
    """hexplane.cuh make_tap in fp32: (x before the clamp, i0, i1, w0, w1, gmul) as arrays"""
    u = np.asarray(u, dtype=np.float32)
    hi = F32(size - 1)
    with np.errstate(invalid="ignore", over="ignore"):
        x = ((u + F32(1.0)) / F32(2.0)) * hi
        gmul = np.where((x > 0) & (x < hi), F32(0.5) * hi, F32(0.0)).astype(np.float32)
        xc = np.fmin(np.fmax(x, F32(0.0)), hi)                     # fmaxf / fminf: a NaN operand yields the other
        x0 = np.floor(xc)
        i0 = x0.astype(np.int64)
        i1 = np.minimum(i0 + 1, size - 1)
        w0 = (x0 + F32(1.0)) - xc
        w1 = xc - x0
    return x, i0, i1, w0, w1, gmul


def u64(x) -> np.ndarray:
    """oracle.deform_ref.normalize at this AABB in fp64"""
    return (np.asarray(x, dtype=np.float64) - 1.0) * (2.0 / (-1.0 - 1.0)) - 1.0


# --------------------------------------------------------------------------------------------------- configurations
@dataclass
class Net:
    """a deformation network on the edge AABB: a shipped synth config with its plane resolutions replaced"""
    base: str                       # synth.hidden_args name (channels, width, heads)
    res: Tuple[int, int, int, int]  # base resolution x, y, z, t (level l multiplies x, y, z by multires[l])
    multires: Tuple[int, ...] = (1, 2)
    depth: int = 1

    @property
    def name(self) -> str:
        return "%s_r%s_m%s_d%d" % (self.base, "x".join(map(str, self.res)), "".join(map(str, self.multires)), self.depth)

    def args(self):
        a = synth.hidden_args(self.base)
        a.kplanes_config = dict(a.kplanes_config, resolution=list(self.res))
        a.multires = list(self.multires)
        a.defor_depth = self.depth
        return a

    def level_sizes(self) -> List[Tuple[int, int, int, int]]:
        return [tuple(r * m for r in self.res[:3]) + (self.res[3],) for m in self.multires]


def make_edge_module(net: Net, seed: int = 0, device="cuda"):
    torch.manual_seed(1234 + seed)
    m = g4d.deform_network(net.args())
    synth.perturb_deformation(m, seed)
    m.deformation_net.set_aabb(AABB[0].tolist(), AABB[1].tolist())
    return m.to(device)


# res = 2 on each spatial axis in turn (level 0), mixed with sizes 3 and 5 (dyadic lines on level 0) and their doubles /
# quadruples (no dyadic line); every plane non-square, so an H / W swap changes the result.  T: 2, 5 and 9.
RES = ((2, 3, 5, 5), (5, 2, 3, 9), (3, 5, 2, 2))


# --------------------------------------------------------------------------------------------------- scenes
@dataclass
class Scene:
    name: str
    xyz: np.ndarray                                   # [n, 3] float32
    claims: List[Tuple[int, int, str]] = field(default_factory=list)   # (row, axis, claim)
    twins: List[Tuple[int, int]] = field(default_factory=list)         # (NaN / inf row, the finite row it must equal)


def _row(claims, rows, a, v, claim, other=INTERIOR):
    p = list(other)
    p[a] = v
    rows.append(p)
    claims.append((len(rows) - 1, a, claim))
    return len(rows) - 1


def face_scene() -> Scene:
    """faces, one ulp inside them, outside by a little and by 1e30, edges and corners, the last interior texel, and dyadic
    interior points (some on the level-0 texel lines)"""
    rows, claims = [], []
    for a in range(3):
        for v, c in ((F32(1.0), FACE_MAX), (F32(-1.0), FACE_MIN), (JUST_IN_MAX, INSIDE), (JUST_IN_MIN, INSIDE),
                     (OUT_NEAR_MAX, OUT_MAX), (OUT_NEAR_MIN, OUT_MIN), (F32(1e30), OUT_MAX), (F32(-1e30), OUT_MIN)):
            _row(claims, rows, a, v, c)
    for a in range(3):                       # edges: two axes on faces
        b = (a + 1) % 3
        for sa in (1.0, -1.0):
            for sb in (1.0, -1.0):
                p = list(INTERIOR); p[a] = F32(sa); p[b] = F32(sb)
                rows.append(p)
                claims += [(len(rows) - 1, a, FACE_MAX if sa > 0 else FACE_MIN), (len(rows) - 1, b, FACE_MAX if sb > 0 else FACE_MIN)]
    for s in range(8):                       # corners
        p = [F32(1.0 if (s >> a) & 1 else -1.0) for a in range(3)]
        rows.append(p)
        claims += [(len(rows) - 1, a, FACE_MAX if p[a] > 0 else FACE_MIN) for a in range(3)]
    for a in range(3):                       # last interior texel on level 0 (size 3: x = 1 <=> u = 0; size 5: x = 3 <=> u = 0.5)
        for v in (F32(0.0), F32(-0.5)):
            _row(claims, rows, a, v, None)
    g = np.random.default_rng(5)             # dyadic interior points (multiples of 1/64 in (-1, 1))
    for _ in range(64):
        rows.append([F32(k / 64.0) for k in g.integers(-63, 64, size=3)])
    return Scene("faces", np.array(rows, dtype=np.float32), [c for c in claims if c[2] is not None])


def nonfinite_scene() -> Scene:
    """NaN and +-inf coordinates, each followed by the finite row it must equal: NaN and +inf behave as the xyz_max face,
    -inf as the xyz_min face"""
    rows, claims, twins = [], [], []
    for a in range(3):
        for v, c, twin in ((F32("nan"), NAN, F32(1.0)), (F32("inf"), POS_INF, F32(1.0)), (F32("-inf"), NEG_INF, F32(-1.0))):
            i = _row(claims, rows, a, v, c)
            j = _row(claims, rows, a, twin, FACE_MAX if twin > 0 else FACE_MIN)
            twins.append((i, j))
    return Scene("nonfinite", np.array(rows, dtype=np.float32), claims, twins)


def hot_scene(n: int = 65536) -> Scene:
    """n Gaussians at one dyadic point: every one adds into the same texels (red.global.add.v4 contention)"""
    return Scene("hot", np.tile(np.array([[0.25, -0.375, 0.5]], dtype=np.float32), (n, 1)))


def tile_scene(n: int, seed: int = 3) -> Scene:
    """n dyadic interior points (multiples of 1/64), for the tile-tail sizes"""
    g = np.random.default_rng(seed)
    return Scene("tiles%d" % n, (g.integers(-63, 64, size=(n, 3)) / 64.0).astype(np.float32))


def tile_sizes(sm_count: int, tiles: Sequence[int] = (64, 128)) -> List[int]:
    """1 and 63 ... 129 (the FP16x2 kernel's two warpgroups of 64), and k * S * T + {-1, 0, 1} for every tile size T and
    k = 1, 2, S = the SM count: the persistent grid's last CTA takes one tile more, or one fewer"""
    out = [1, 63, 64, 65, 127, 128, 129]
    for t in tiles:
        for k in (1, 2):
            out += [k * sm_count * t - 1, k * sm_count * t, k * sm_count * t + 1]
    return sorted(set(out))


# time values: the centre row (t = 0 is a texel line when T is odd), the last row (t = 1: i0 == i1), clamped beyond both
# ends, and a texel line away from the centre with its fp32 neighbours one ulp of (t + 1) either side
TIME_ENDS = (0.0, 1.0, -1.0, -0.5, 1.5)
TIME_LINE = (0.5, 0.5 - 2.0 ** -23, 0.5 + 2.0 ** -23)   # on a line for T - 1 = 4 and 8; exact in fp32 for every T


# --------------------------------------------------------------------------------------------------- plane edits
def set_planes(mod, kind: str, seed: int = 0):
    """overwrite the planes in place.  zero: level 0 plane (x, z) is exactly 0 over its x < 0 half (texels 0 .. W/2 - 1 of
    u = -x), the others keep their values; negative: every second plane negated; wide: |values| log-uniform in
    [1e-6, 1e2] with random signs on the spatial planes (the time planes stay near 1)"""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for l, lvl in enumerate(mod.deformation_net.grid.grids):
            for k, p in enumerate(lvl):
                if kind == "zero" and l == 0 and k == 1:
                    w = p.shape[3]
                    p[..., : (w + 1) // 2] = 0.0
                elif kind == "negative" and k % 2 == 1:
                    p.neg_()
                elif kind == "wide" and k in (0, 1, 3):
                    mag = torch.pow(10.0, torch.rand(p.shape, generator=g, dtype=torch.float64) * 8.0 - 6.0)
                    sign = torch.where(torch.rand(p.shape, generator=g) < 0.5, -1.0, 1.0).double()
                    p.copy_((mag * sign).float().to(p.device))
    mod.invalidate_cache()


def set_uniform_planes(mod, target: float, channel: int = 0):
    """every plane 1, except channel `channel` of level 0's first plane = target: feature[channel] = target exactly"""
    with torch.no_grad():
        for l, lvl in enumerate(mod.deformation_net.grid.grids):
            for k, p in enumerate(lvl):
                p.fill_(1.0)
                if l == 0 and k == 0:
                    p[:, channel] = target
    mod.invalidate_cache()


def inputs(xyz: np.ndarray, seed: int):
    """(xyz, scales, rotations, opacity, shs) and probes (upstream gradients) for the rows of xyz, CPU fp32"""
    n = xyz.shape[0]
    g = torch.Generator().manual_seed(seed)
    ins = [torch.from_numpy(np.ascontiguousarray(xyz)), 0.1 * torch.randn(n, 3, generator=g) - 3.0,
           torch.nn.functional.normalize(torch.randn(n, 4, generator=g), dim=1), torch.randn(n, 1, generator=g),
           0.3 * torch.randn(n, 16, 3, generator=g)]
    probes = [torch.randn(tuple(x.shape), generator=g) for x in ins]
    return ins, probes
