"""A backward taps the texel cells its forward sampled.

The HexPlane coordinate of a Gaussian is p = (x - xyz_max) * scale - 1 (normalize_aabb).  Evaluated as a multiply and a
subtract it can round one ulp away from the same expression contracted to one fused multiply-add; when a texel line of a
plane lies between the two values, floor() picks neighbouring cells.  The forward gather and the backward scatter must
agree, so the scene below holds Gaussians exactly there: the gradient w.r.t. xyz at such a point must be the one of its
neighbouring floats on the forward's side of the line, not the one of the other side (where the slope of the bilinear
sample changes).
"""
from fractions import Fraction

import numpy as np
import pytest
import torch

from util_scene import g4d, make_module

NET = "small128"                 # C = 16, L = 2: both the FFMA and the tensor-core network take it
AABB = np.array([[1.31, 1.27, 1.3], [-1.29, -1.3, -1.22]], dtype=np.float32)   # [xyz_max | xyz_min]
T = 0.43
OTHER = (np.float32(0.1234), np.float32(-0.2345), np.float32(0.3071))          # coordinates of the axes not under test


def _level_sizes():
    from oracle import deform_ref as dr
    cfg = dr.DeformConfig(channels=16, resolution=(9, 12, 10, 8), multires=(1, 2), net_width=128)
    return [[r * m for r in cfg.resolution[:3]] for m in cfg.multires]


def _round_f32(q: Fraction) -> np.float32:
    """q rounded to the nearest float32, ties to even"""
    c = np.float32(float(q))
    best = None
    for v in (np.nextafter(c, np.float32(-np.inf)), c, np.nextafter(c, np.float32(np.inf))):
        d = abs(Fraction(float(v)) - q)
        even = (int(np.array(v).view(np.int32)) & 1) == 0
        if best is None or d < best[0] or (d == best[0] and even and not best[2]):
            best = (d, v, even)
    return best[1]


def _coords(a, x):
    """(plain, contracted) normalised coordinate of world coordinate x (float32) on axis a"""
    amax, amin = AABB[0, a], AABB[1, a]
    scale = np.float32(2.0) / np.float32(amin - amax)
    sub = np.float32(x - amax)
    plain = np.float32(np.float32(sub * scale) - np.float32(1.0))
    fused = _round_f32(Fraction(float(sub)) * Fraction(float(scale)) - 1)
    return plain, fused


def _cell(u, size):
    """make_tap's floor() (grid_sample unnormalise, align_corners=True, border clamp)"""
    hi = np.float32(size - 1)
    x = np.float32(np.float32(np.float32(u + np.float32(1.0)) / np.float32(2.0)) * hi)
    return int(np.floor(min(max(x, np.float32(0.0)), hi)))


def _cells(a, x):
    plain, fused = _coords(a, x)
    return [(_cell(plain, s[a]), _cell(fused, s[a])) for s in _level_sizes()]


def find_crossings(limit=6):
    """Points whose plain and contracted coordinates fall in different texel cells, with the nearest floats on either side
    of the line whose two roundings agree: [(axis, x, forward-side neighbour, other-side neighbour)]"""
    out = []
    for a in range(3):
        amax, amin = AABB[0, a], AABB[1, a]
        for sizes in _level_sizes():
            hi = sizes[a] - 1
            for k in range(1, hi):
                x0 = np.float32(amax + (2.0 * k / hi) * (float(amin) - float(amax)) / 2.0)
                bits = int(np.array(x0).view(np.int32))
                for d in range(-48, 49):
                    x = np.array(bits + d, dtype=np.int32).view(np.float32)[()]
                    cs = _cells(a, x)
                    if all(p == f for p, f in cs):
                        continue
                    sides = {}
                    for direction in (np.float32(np.inf), np.float32(-np.inf)):
                        y = x
                        for _ in range(64):
                            y = np.nextafter(y, direction)
                            cy = _cells(a, y)
                            if all(p == f for p, f in cy):
                                sides[[p for p, f in cy] == [p for p, f in cs]] = y
                                break
                    if True in sides and False in sides:
                        out.append((a, x, sides[True], sides[False]))
                        break          # one point per line
                if len(out) >= limit:
                    return out
    return out


def _scene(crossings):
    rows = []
    for a, x, same, other in crossings:
        for v in (x, same, other):
            p = list(OTHER)
            p[a] = v
            rows.append(p)
    return np.array(rows, dtype=np.float32)


def test_scene_reaches_the_condition():
    """CPU: the roundings differ in the cell at each point found, and both neighbours round the same either way."""
    cr = find_crossings()
    assert len(cr) >= 3
    for a, x, same, other in cr:
        cs = _cells(a, x)
        assert any(p != f for p, f in cs)
        assert [p for p, _ in _cells(a, same)] == [p for p, _ in cs]       # the forward's side: the plain rounding's cells
        assert [p for p, _ in _cells(a, other)] == [f for _, f in cs]      # the other side: the contracted rounding's cells
        assert abs(int(np.array(same).view(np.int32)) - int(np.array(x).view(np.int32))) <= 64


@pytest.mark.gpu
@pytest.mark.parametrize("tensor_cores", [0, 2])
def test_backward_takes_the_forwards_cell(tensor_cores):
    cr = find_crossings()
    xyz = torch.from_numpy(_scene(cr))
    n = xyz.shape[0]
    gen = torch.Generator().manual_seed(11)
    # the three rows of a point share every other input and the upstream gradient: only x differs
    rep = lambda t: t.repeat_interleave(3, dim=0)
    m = len(cr)
    ins = [xyz] + [rep(t) for t in (0.1 * torch.randn(m, 3, generator=gen) - 3.0,
                                    torch.nn.functional.normalize(torch.randn(m, 4, generator=gen), dim=1),
                                    torch.randn(m, 1, generator=gen), 0.3 * torch.randn(m, 16, 3, generator=gen))]
    probes = [rep(torch.randn((m,) + tuple(o.shape[1:]), generator=gen)) for o in ins]
    mod = make_module(NET, seed=7, aabb=torch.from_numpy(AABB))
    ws = g4d._lib.Workspace.get(0)
    try:
        ws.set_option(g4d._lib.OPT_TENSOR_CORES, tensor_cores)
        dev_in = [x.cuda().contiguous().requires_grad_(True) for x in ins]
        outs = mod(*dev_in, torch.tensor(T).repeat(n, 1).cuda())
        sum((o * p.cuda()).sum() for o, p in zip(outs, probes)).backward()
        g = dev_in[0].grad.cpu().numpy()
    finally:
        ws.set_option(g4d._lib.OPT_TENSOR_CORES, 2)
    checked = 0
    for i, (a, _, _, _) in enumerate(cr):
        at, same, other = g[3 * i, a], g[3 * i + 1, a], g[3 * i + 2, a]
        jump = abs(same - other)
        if jump <= 1e-3 * np.abs(g[:, a]).max():
            continue             # the two cells happen to have nearly the same slope here: nothing to tell apart
        assert abs(at - same) <= 0.01 * jump, (i, a, at, same, other)
        checked += 1
    assert checked >= 2, checked
