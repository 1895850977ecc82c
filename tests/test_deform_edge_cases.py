"""CPU: the deformation edge scenes (util_deform_edges) reach the conditions they claim, in the fp32 arithmetic of hexplane.cuh,
with fp32 and fp64 taking the same cell decision on every row; and the fp64 oracle (oracle.deform_ref) equals F.grid_sample
(fp64, padding_mode='border', align_corners=True) on every scene, forward and backward per row."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import util_deform_edges as ue
from oracle import deform_ref as dr

MULTIRES = ((1, 2), (1, 2, 4))


def _sizes(res, multires):
    return [tuple(r * m for r in res[:3]) + (res[3],) for m in multires]


def _claim_holds(claim, u32, x, size):
    hi = float(size - 1)
    if claim == ue.FACE_MAX:
        return u32 == -1.0 and x == 0.0
    if claim == ue.FACE_MIN:
        return u32 == 1.0 and x == hi
    if claim == ue.INSIDE:
        return 0.0 < x < hi
    if claim in (ue.OUT_MAX, ue.POS_INF):
        return u32 < -1.0 and x < 0.0 and (claim != ue.POS_INF or np.isneginf(u32))
    if claim in (ue.OUT_MIN, ue.NEG_INF):
        return u32 > 1.0 and x > hi and (claim != ue.NEG_INF or np.isposinf(u32))
    if claim == ue.NAN:
        return bool(np.isnan(u32))
    raise AssertionError(claim)


@pytest.mark.parametrize("res", ue.RES)
@pytest.mark.parametrize("multires", MULTIRES)
def test_scenes_reach_their_conditions(res, multires):
    sizes = _sizes(res, multires)
    for sc in (ue.face_scene(), ue.nonfinite_scene()):
        u32 = ue.norm32(sc.xyz)
        for row, a, claim in sc.claims:
            for lv in sizes:
                x, i0, i1, w0, w1, gmul = ue.tap32(u32[row, a], lv[a])
                assert _claim_holds(claim, float(u32[row, a]), float(x), lv[a]), (sc.name, row, a, claim, lv)
                if claim in (ue.FACE_MAX, ue.FACE_MIN, ue.OUT_MAX, ue.OUT_MIN, ue.NAN, ue.POS_INF, ue.NEG_INF):
                    assert gmul == 0.0
                else:
                    assert gmul > 0.0
        # NaN / inf rows tap exactly what their finite twins tap
        for i, j in sc.twins:
            for lv in sizes:
                for a in range(3):
                    ti, tj = ue.tap32(u32[i, a], lv[a]), ue.tap32(u32[j, a], lv[a])
                    assert all(np.array_equal(p, q) for p, q in zip(ti[1:], tj[1:]))
    # the last interior texel of level 0 on every axis whose size is at least 3
    xs = ue.norm32(ue.face_scene().xyz)
    for a in range(3):
        if sizes[0][a] >= 3:
            assert any(float(ue.tap32(u, sizes[0][a])[0]) == sizes[0][a] - 2 for u in xs[:, a]), a
    # interior texel lines are reached, on level 0 only
    hit = [any(0 < float(ue.tap32(u, lv[a])[0]) < lv[a] - 1 and float(ue.tap32(u, lv[a])[0]).is_integer()
               for a in range(3) for u in xs[:, a]) for lv in sizes]
    assert hit[0] and not any(hit[1:]), hit


@pytest.mark.parametrize("res", ue.RES)
def test_fp32_and_fp64_take_the_same_cell_on_every_row(res):
    """the normalised coordinate is exact in fp32; floor() and the border test of make_tap decide as in fp64"""
    sizes = _sizes(res, (1, 2, 4))
    xyz = np.concatenate([ue.face_scene().xyz, ue.nonfinite_scene().xyz, ue.tile_scene(500).xyz])
    fin = np.isfinite(xyz)
    u32, u = ue.norm32(xyz), ue.u64(xyz)
    assert np.array_equal(u32[fin].astype(np.float64), u[fin])
    for lv in sizes:
        for a in range(3):
            x32, i0, i1, w0, w1, _ = ue.tap32(u32[:, a], lv[a])
            with np.errstate(invalid="ignore"):
                x64 = np.clip((u[:, a] + 1.0) / 2.0 * (lv[a] - 1), 0.0, lv[a] - 1)
            ok = fin[:, a]
            assert np.array_equal(np.floor(x64[ok]).astype(np.int64), i0[ok])
            with np.errstate(invalid="ignore"):
                inside64 = (u[:, a] > -1.0) & (u[:, a] < 1.0)
            assert np.array_equal(ue.tap32(u32[:, a], lv[a])[5][ok] > 0, inside64[ok])      # the gmul decision


def test_time_values_reach_their_conditions():
    for T in sorted({r[3] for r in ue.RES}):
        hi = T - 1
        for t in ue.TIME_ENDS + ue.TIME_LINE:
            x, i0, i1, w0, w1, gmul = ue.tap32(np.float32(t), T)
            assert float(x) == (t + 1.0) / 2.0 * hi                        # exact in fp32
            if t >= 1.0:
                assert int(i0) == int(i1) == hi and float(w0) == 1.0 and float(w1) == 0.0
            if t <= -1.0:
                assert int(i0) == 0 and float(w0) == 1.0 and float(w1) == 0.0
        if T % 2 == 1:
            assert float(ue.tap32(np.float32(0.0), T)[0]) == hi / 2          # t = 0: the centre row is a texel line
        if hi in (4, 8):                                                  # t = 0.5 on a line away from the centre, neighbours
            xs = [float(ue.tap32(np.float32(t), T)[0]) for t in ue.TIME_LINE]   # one ulp of (t + 1) either side of it
            assert xs[0].is_integer() and xs[0] != hi / 2 and xs[1] < xs[0] < xs[2]
            assert int(np.floor(xs[1])) == int(xs[0]) - 1 and int(np.floor(xs[2])) == int(xs[0])


# --------------------------------------------------------------------------------------------------- oracle vs grid_sample
def _gs_features(planes, xyz, aabb, t):
    """hexplane.py:73-106 with F.grid_sample, as the reference computes it"""
    p = dr.normalize(xyz, aabb)
    q = torch.cat([p, t.reshape(-1, 1)], dim=-1)
    feats = []
    for lvl in planes:
        prod = None
        for k, (c0, c1) in enumerate(dr.PLANE_AXES):
            grid = torch.stack([q[:, c0], q[:, c1]], dim=-1).view(1, -1, 1, 2)
            s = F.grid_sample(lvl[k], grid, mode="bilinear", padding_mode="border", align_corners=True)[0, :, :, 0].t()
            prod = s if prod is None else prod * s
        feats.append(prod)
    return torch.cat(feats, dim=-1)


def _planes(res, multires, kind, seed):
    cfg = dr.DeformConfig(channels=4, resolution=res, multires=multires)
    g = torch.Generator().manual_seed(seed)
    out = []
    for l in range(cfg.levels):
        lvl = []
        for k in range(6):
            h, w = cfg.plane_hw(l, k)
            p = 0.1 + 0.4 * torch.rand(1, 4, h, w, generator=g, dtype=torch.float64)
            if kind == "zero" and l == 0 and k == 1:
                p[..., : (w + 1) // 2] = 0.0
            elif kind == "negative" and k % 2 == 1:
                p = -p
            elif kind == "wide" and k in (0, 1, 3):
                p = torch.pow(10.0, torch.rand(p.shape, generator=g, dtype=torch.float64) * 8 - 6) * \
                    torch.where(torch.rand(p.shape, generator=g) < 0.5, -1.0, 1.0).double()
            lvl.append(p)
        out.append(lvl)
    return out


def _per_row_grads(fn, planes, xyz, t, cot):
    """(features [n, F], d(xyz) [n, 3], d(planes) of each row [n][flat]) of <fn(...), cot> row by row"""
    leaves = [p.detach().clone().requires_grad_(True) for lvl in planes for p in lvl]
    lv = [leaves[6 * l:6 * l + 6] for l in range(len(planes))]
    x = xyz.clone().requires_grad_(True)
    aabb = torch.from_numpy(ue.AABB).double()
    feat = fn(lv, x, aabb, t)
    feat_np = feat.detach().numpy()
    (gx,) = torch.autograd.grad((feat * cot).sum(), [x], retain_graph=True)
    rows = []
    for i in range(xyz.shape[0]):
        g = torch.autograd.grad((feat[i] * cot[i]).sum(), leaves, retain_graph=True)
        rows.append(torch.cat([q.reshape(-1) for q in g]).numpy())
    return feat_np, gx.numpy(), np.stack(rows)


@pytest.mark.parametrize("res,multires", [(ue.RES[0], (1, 2)), (ue.RES[1], (1, 2, 4)), (ue.RES[2], (1, 2))])
@pytest.mark.parametrize("kind", ["default", "zero", "negative", "wide"])
@pytest.mark.parametrize("t", [0.25, 1.0, -1.5])
def test_oracle_equals_grid_sample_per_row(res, multires, kind, t):
    """forward features, d(xyz) and d(planes) per row: the oracle's restatement against ATen's grid_sample in fp64, on the
    face scene and the +-inf rows (NaN rows left out: ATen does not specify them)"""
    sc = ue.nonfinite_scene()
    keep = ~np.isnan(sc.xyz).any(axis=1)
    xyz = torch.from_numpy(np.concatenate([ue.face_scene().xyz, sc.xyz[keep]])).double()
    n = xyz.shape[0]
    planes = _planes(res, multires, kind, seed=len(res) + len(multires))
    tt = torch.full((n,), t, dtype=torch.float64)
    cot = torch.randn(n, 4 * len(multires), generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    f_o, gx_o, gp_o = _per_row_grads(dr.hexplane_features, planes, xyz, tt, cot)
    f_r, gx_r, gp_r = _per_row_grads(_gs_features, planes, xyz, tt, cot)
    assert np.allclose(f_o, f_r, rtol=1e-12, atol=0), float(np.abs(f_o - f_r).max())
    scale = np.maximum(np.abs(gx_r).max(axis=1, keepdims=True), 1e-300)
    assert np.all(np.abs(gx_o - gx_r) <= 1e-12 * scale), np.abs(gx_o - gx_r).max()
    scale = np.maximum(np.abs(gp_r).max(axis=1, keepdims=True), 1e-300)
    assert np.all(np.abs(gp_o - gp_r) <= 1e-12 * scale), np.abs(gp_o - gp_r).max()
    # the faces and everything outside take no coordinate gradient from the planes (ATen's clip_coordinates_set_grad)
    u = ue.u64(xyz.numpy())
    with np.errstate(invalid="ignore"):
        clipped = (u <= -1.0) | (u >= 1.0)
    assert clipped.any() and np.all(gx_o[clipped] == 0.0)
