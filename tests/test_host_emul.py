"""Host build of the product's per-Gaussian device math (csrc/g4d_math.cuh) vs the oracle.
Catches logic errors in the GPU-less container; the real parity tests are the -m gpu ones."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import raster_ref as rr
import util_raster_edges as ue
from util_scene import cam_tuple, raster_inputs, row_errors, synth

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "host_emul", "emul_math.cpp")
LIB = os.path.join(HERE, "host_emul", "libemul.so")


def _lib():
    hdr = os.path.join(os.path.dirname(HERE), "4dgaussians_b200", "csrc", "g4d_math.cuh")
    if not os.path.isfile(LIB) or os.path.getmtime(LIB) < max(os.path.getmtime(SRC), os.path.getmtime(hdr)):
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", LIB, SRC], check=True)
    return C.CDLL(LIB)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.mark.parametrize("seed,theta,radius,wh,deg", [(0, 10.0, 4.0, (400, 400), 3), (1, -100.0, 1.5, (1352, 1014), 2),
                                                       (2, 77.0, 2.2, (536, 960), 1), (3, 160.0, 3.0, (33, 17), 0)])
def test_preprocess_bit_exact_vs_oracle(seed, theta, radius, wh, deg):
    lib = _lib()
    cam = synth.make_camera(theta, wh[0], wh[1], radius=radius)
    rc, _ = cam_tuple(cam, (0, 0, 0), sh_degree=deg, scale_modifier=1.0 if seed != 2 else 0.7)
    m, s, r, o, sh = [t.numpy().astype(np.float32) for t in raster_inputs(5000, seed, scale_mean=0.03)]
    ref = rr.preprocess(rc, m, s, r, o, sh)
    n = m.shape[0]
    depth = np.zeros(n, np.float32); radii = np.zeros(n, np.int32); xy = np.zeros((n, 2), np.float32)
    co = np.zeros((n, 4), np.float32); rgb = np.zeros((n, 3), np.float32); cl = np.zeros((n, 3), np.uint8)
    rect = np.zeros((n, 4), np.int32); tiles = np.zeros(n, np.uint32)
    lib.emul_preprocess(C.byref(rc), n, _p(m), _p(s), _p(r), _p(o), _p(sh), _p(depth), _p(radii), _p(xy), _p(co), _p(rgb),
                        _p(cl), _p(rect), _p(tiles))
    assert (ref.radii > 0).sum() > 100
    for a, b in ((depth, ref.depth), (radii, ref.radii), (xy, ref.xy), (co, ref.conic_op), (rgb, ref.rgb),
                 (cl, ref.clamped), (rect, ref.rect), (tiles, ref.tiles_touched)):
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_gaussian_backward_vs_oracle():
    lib = _lib()
    cam = synth.make_camera(25.0, 200, 120, radius=2.0)
    rc, _ = cam_tuple(cam, (0, 0, 0), sh_degree=3, scale_modifier=1.3)
    m, s, r, o, sh = [t.numpy().astype(np.float32) for t in raster_inputs(3000, 4, scale_mean=0.05)]
    pr = rr.preprocess(rc, m, s, r, o, sh)
    n = m.shape[0]
    rng = np.random.default_rng(0)
    g2 = rng.standard_normal((n, 2)).astype(np.float32); gc = rng.standard_normal((n, 3)).astype(np.float32)
    grgb = rng.standard_normal((n, 3)).astype(np.float32)
    want = rr.preprocess_backward(rc, m, s, r, sh, pr, g2, gc, grgb)
    gm = np.zeros((n, 3), np.float32); gs = np.zeros((n, 3), np.float32); gr = np.zeros((n, 4), np.float32)
    gsh = np.zeros((n, 16, 3), np.float32)
    lib.emul_backward(C.byref(rc), n, _p(m), _p(s), _p(r), _p(sh), _p(pr.radii), _p(pr.clamped), _p(g2), _p(gc), _p(grgb),
                      _p(gm), _p(gs), _p(gr), _p(gsh))
    for got, ref, nm in zip((gm, gs, gr, gsh), want, ("mean", "scale", "rot", "sh")):
        # fp32 evaluation vs the oracle's fp64: relative to the per-row magnitude
        denom = np.maximum(np.abs(ref).reshape(n, -1).max(axis=1), 1e-2).reshape((n,) + (1,) * (ref.ndim - 1))
        err = (np.abs(got - ref) / denom).max()
        assert err < 5e-3, (nm, err)
        assert np.abs(ref).max() > 0


def test_depth_ordered_emission_plus_tile_sort_equals_the_reference_key_sort():
    """DESIGN §4 binning: stable-sorting the Gaussians by depth bits, emitting their (tile | depth) keys in that order and
    stable-sorting the keys on the TILE bits only must reproduce, entry for entry, the reference's stable sort of the keys
    emitted in Gaussian-index order on (tile, depth) -- including ties (equal depth bits keep Gaussian-index order)."""
    import numpy as np
    rng = np.random.default_rng(5)
    n, tiles = 4000, 37
    depth = rng.integers(0x3E4CCCCD, 0x3E4CCCCD + 60, size=n, dtype=np.uint64)          # few distinct values: many ties
    touched = rng.integers(0, 6, size=n)
    rects = [np.sort(rng.choice(tiles, size=k, replace=False)) for k in touched]         # tiles of Gaussian i, emission order
    # reference: emit in index order, stable sort on the full 64-bit key
    keys = np.concatenate([(t.astype(np.uint64) << np.uint64(32)) | depth[i] for i, t in enumerate(rects)])
    ids = np.concatenate([np.full(len(t), i, dtype=np.uint32) for i, t in enumerate(rects)])
    o = np.argsort(keys, kind="stable")
    ref_keys, ref_ids = keys[o], ids[o]
    # g4d: depth order first (invisible Gaussians last), emit in that order, stable sort on the tile bits alone
    dkey = np.where(touched > 0, depth, np.uint64(0xFFFFFFFF))
    perm = np.argsort(dkey, kind="stable")
    keys2 = np.concatenate([(rects[i].astype(np.uint64) << np.uint64(32)) | depth[i] for i in perm])
    ids2 = np.concatenate([np.full(len(rects[i]), i, dtype=np.uint32) for i in perm])
    o2 = np.argsort(keys2 >> np.uint64(32), kind="stable")
    assert np.array_equal(keys2[o2], ref_keys) and np.array_equal(ids2[o2], ref_ids)


def test_strip_cull_predicate_is_conservative():
    """The exact-cull predicate of the blend kernels / G4D_OPT_TIGHT_CULL (g4d_raster.cu rect_contributes), restated in
    float32 numpy: whenever it says 'cannot contribute', NO pixel centre of the rectangle reaches alpha >= 1/255."""
    import numpy as np
    f = np.float32
    rng = np.random.default_rng(11)

    def edge_min(a, b, c, fixed, lo, hi):
        t = f(-b * fixed / c)
        t = min(max(t, lo), hi)
        return f(a * fixed * fixed + f(2) * b * fixed * t + c * t * t)

    def rect_contributes(mx, my, A, B, C, op, x0, x1, y0, y1):
        dx0, dx1, dy0, dy1 = f(mx - x1), f(mx - x0), f(my - y1), f(my - y0)
        if dx0 <= 0 and dx1 >= 0 and dy0 <= 0 and dy1 >= 0:
            q = f(0)
        else:
            q = min(edge_min(A, B, C, dx0, dy0, dy1), edge_min(A, B, C, dx1, dy0, dy1),
                    edge_min(C, B, A, dy0, dx0, dx1), edge_min(C, B, A, dy1, dx0, dx1))
            q = max(q, f(0))
        return op * f(np.exp(f(-0.5) * q)) * f(1.0001) >= f(1.0 / 255.0)

    culled = kept = 0
    for _ in range(3000):
        # random positive-definite conic, mean near a 16 x 4 strip
        s1, s2, th = rng.uniform(0.8, 12.0), rng.uniform(0.8, 12.0), rng.uniform(0, np.pi)
        R = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
        con = np.linalg.inv(R @ np.diag([s1 * s1, s2 * s2]) @ R.T)
        A, B, C = f(con[0, 0]), f(con[0, 1]), f(con[1, 1])
        op = f(rng.uniform(0.02, 0.99))
        mx, my = f(rng.uniform(-30, 46)), f(rng.uniform(-30, 34))
        x0, x1, y0, y1 = f(0), f(15), f(0), f(3)
        xs, ys = np.meshgrid(np.arange(16, dtype=np.float32), np.arange(4, dtype=np.float32))
        dx, dy = mx - xs, my - ys
        power = f(-0.5) * (A * dx * dx + C * dy * dy) - B * dx * dy
        alpha = np.minimum(f(0.99), op * np.exp(power))
        reach = bool(((power <= 0) & (alpha >= f(1.0 / 255.0))).any())
        if rect_contributes(mx, my, A, B, C, op, x0, x1, y0, y1):
            kept += 1
        else:
            culled += 1
            assert not reach, (mx, my, A, B, C, op)
    assert culled > 300 and kept > 300      # the sample exercises both outcomes


def test_sub_segment_rank_fix_restores_the_depth_order():
    """DESIGN 4.2 step 5 (bin_fix_kernel) restated in numpy: the placement leaves the entries of a (tile, chunk) sub-segment in
    arbitrary order; the final position of an entry is lo + (number of smaller depth ranks in its sub-segment).  The three code
    paths -- per-lane register tiers padded with 0xFFFFFFFF, whole-warp ranking with S entries per lane, streaming of the keys past
    256 register-resident entries at a time -- give the depth-ordered list for every length."""
    import numpy as np
    rng = np.random.default_rng(3)
    PAD = np.uint32(0xFFFFFFFF)

    def rank_tier(keys, T):                          # one lane: T registers, padding never counts as smaller
        reg = np.full(T, PAD, np.uint32); reg[:len(keys)] = keys
        return [int(sum(reg[p] < reg[q] for p in range(T) if p != q)) for q in range(len(keys))]

    def coop_rank(keys, S):                          # one warp: lane l holds entries l, l + 32, ...; every key broadcast once
        n = len(keys)
        reg = np.full((S, 32), PAD, np.uint32); reg.reshape(-1)[:n] = keys
        r = np.zeros((S, 32), np.int64)
        for s2 in range(S):
            if 32 * s2 >= n:
                break
            for l in range(32):
                r += reg[s2, l] < reg
        return r.reshape(-1)[:n].tolist()

    def coop_rank_big(keys):                         # 256 entries at a time, the whole list streamed 32 keys per step
        n, out = len(keys), []
        for base in range(0, n, 256):
            reg = np.full(256, PAD, np.uint32); m = min(256, n - base); reg[:m] = keys[base:base + m]
            r = np.zeros(256, np.int64)
            for j0 in range(0, n, 32):
                cur = np.full(32, PAD, np.uint32); k = min(32, n - j0); cur[:k] = keys[j0:j0 + k]
                for l in range(32):
                    r += cur[l] < reg
            out += r[:m].tolist()
        return out

    for n in (1, 3, 4, 5, 8, 9, 12, 13, 16, 17, 24, 25, 32, 33, 64, 65, 128, 129, 200, 256, 257, 300, 700):
        ranks = np.sort(rng.choice(2_000_000, size=n, replace=False)).astype(np.uint32)     # unique depth ranks of the chunk
        ids = rng.integers(0, 1 << 31, size=n, dtype=np.int64)
        order = rng.permutation(n)                                                          # as the placement left them
        keys, vals = ranks[order], ids[order]
        if n <= 32:
            T = next(t for t in (4, 8, 12, 16, 24, 32) if n <= t)
            r = rank_tier(keys, T)
        elif n <= 256:
            r = coop_rank(keys, next(s for s in (2, 4, 8) if n <= 32 * s))
        else:
            r = coop_rank_big(keys)
        assert sorted(r) == list(range(n)), n                                              # a permutation: no two entries collide
        fixed = np.empty(n, np.int64); fixed[np.asarray(r)] = vals
        assert np.array_equal(fixed, ids), n


def _emul_preprocess(lib, rc, m, s, r, o, sh):
    n = m.shape[0]
    out = dict(depth=np.zeros(n, np.float32), radii=np.zeros(n, np.int32), xy=np.zeros((n, 2), np.float32),
               conic_op=np.zeros((n, 4), np.float32), rgb=np.zeros((n, 3), np.float32), clamped=np.zeros((n, 3), np.uint8),
               rect=np.zeros((n, 4), np.int32), tiles_touched=np.zeros(n, np.uint32))
    lib.emul_preprocess(C.byref(rc), n, _p(m), _p(s), _p(r), _p(o), _p(sh), *[_p(out[k]) for k in out])
    return out


@pytest.mark.parametrize("name", ue.names())
def test_edge_scenes_vs_oracle(name):
    """the scenes of test_raster_edge_scenes.py (guard band, near plane, clamped rects and colours, degenerate covariances,
    unnormalised quaternions): project_gaussian + sh_to_rgb bit for bit, gaussian_backward per row"""
    lib = _lib()
    sc = ue.scene(name)
    rc, _ = cam_tuple(sc.cam, sc.bg, sh_degree=sc.deg)
    m, s, r, o, sh = sc.ins
    ref = rr.preprocess(rc, m, s, r, o, sh)
    got = _emul_preprocess(lib, rc, m, s, r, o, sh)
    for k, v in got.items():
        assert np.array_equal(v.view(np.uint8), getattr(ref, k).view(np.uint8)), k
    # the cotangents of the oracle's blend backward under a random image gradient: their conic part has the size a real
    # backward gives it (unit random conic cotangents would hide the covariance terms behind the means2D term)
    n = m.shape[0]
    fwd = rr.rasterize_forward(rc, m, s, r, o, sh)
    dL = np.random.default_rng(len(name)).standard_normal((3, sc.H, sc.W)).astype(np.float32)
    g2, gc, _, grgb = rr.blend_backward(rc, fwd["proj"], fwd["bin"], fwd["final_T"], fwd["n_contrib"], dL)
    want = rr.preprocess_backward(rc, m, s, r, sh, ref, g2, gc, grgb)
    gm = np.zeros((n, 3), np.float32); gs = np.zeros((n, 3), np.float32); gr = np.zeros((n, 4), np.float32)
    gsh = np.zeros((n, 16, 3), np.float32)
    lib.emul_backward(C.byref(rc), n, _p(m), _p(s), _p(r), _p(sh), _p(ref.radii), _p(ref.clamped), _p(g2), _p(gc), _p(grgb),
                      _p(gm), _p(gs), _p(gr), _p(gsh))
    for g, w, nm in zip((gm, gs, gr, gsh), want, ("mean", "scale", "rot", "sh")):
        e = row_errors(g, w, 1e-4)
        assert float(e.max()) <= 2e-3, (nm, float(e.max()), int(np.argmax(e)))
