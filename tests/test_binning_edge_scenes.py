"""CPU companion of test_gpu_binning_edges.py: every scene it renders, checked on the oracle's projection alone to reach the
branch of g4d_bin.cu the GPU test names -- depth-bit span and kbits, visible count, tile counts, chunk lengths from the
placement's own cut formula, and rects crossing every band boundary.  G is an H100 SXM's SM count here; the GPU test uses
the device's."""
import numpy as np
import pytest

from oracle import raster_ref as rr
import util_binning as ub
from util_scene import cam_tuple

G = ub.H100_SXM_SMS


def _proj(cam, ins):
    rc, _ = cam_tuple(cam, (0.0, 0.0, 0.0), sh_degree=3)
    return rr.preprocess(rc, *ins)


def test_band_rows_follow_the_shared_memory_budgets():
    assert ub.band_rows(3840, 2160) == (135, 102) and ub.band_boundaries(3840, 2160) == ([], [102])
    assert ub.band_rows(5120, 2160) == (128, 76) and ub.band_boundaries(5120, 2160) == ([128], [76])
    assert ub.band_boundaries(1352, 1014) == ([], [])                   # C3: one band of each


@pytest.mark.parametrize("span", ub.PASS_SPANS)
def test_pass_scene_spans(span):
    cam, ins = ub.pass_scene(span)
    pr = _proj(cam, ins)
    vis = pr.tiles_touched > 0
    b = ub.depth_bits(pr.depth)[vis].astype(np.int64)
    assert vis.sum() >= (20_000 if span == 0 else 30_000)
    assert int(b.max() - b.min()) == span
    kbits, passes = ub.PASS_KBITS[span]
    assert ub.kbits_of(pr) == kbits and ub.passes_of(kbits) == passes
    if span:
        n = len(b)
        assert b[n // 3] == b.min() and b[2 * n // 3] == b.max() and (b == b.min()).sum() == 1 and (b == b.max()).sum() == 1


def test_four_pass_scene():
    pr = _proj(*ub.four_pass_scene())
    assert ub.passes_of(ub.kbits_of(pr)) == 4 and (pr.tiles_touched > 0).sum() >= 30_000


@pytest.mark.parametrize("n", ub.EXTREME_NS)
def test_extreme_layouts(n):
    lanes = [i for p in ub.extreme_layouts(n) for i in p]
    assert 0 in lanes and n - 1 in lanes
    if n > 32:
        assert any(i % 32 == 31 and i < n - 1 for i in lanes)             # lane 31 of a full warp, not the last Gaussian
    if n > 128:
        assert any(i % 128 == 127 and i < n - 1 for i in lanes)           # last Gaussian of a full 128-Gaussian tile
    for near, far in ub.extreme_layouts(n):
        pr = _proj(*ub.extreme_scene(n, near, far, seed=n))
        b = ub.depth_bits(pr.depth)
        assert (pr.tiles_touched > 0).all() and np.argmin(b) == near and np.argmax(b) == far
        assert n == 1 or ((b == b.min()).sum() == 1 and (b == b.max()).sum() == 1)


@pytest.mark.parametrize("nvis", [1, 2, 31, G - 1, G, G + 1, 2 * G + 1, 0])
def test_sparse_scene_visible_counts(nvis):
    n = 100_000 if nvis == 0 else 50_000
    pr = _proj(*ub.sparse_scene(nvis, n))
    assert int((pr.tiles_touched > 0).sum()) == nvis and int((pr.radii > 0).sum()) == nvis
    if nvis:
        perm, starts, _, _ = ub.chunk_starts(pr, G)
        assert (np.diff(starts) == 0).sum() >= G - nvis                    # at least G - nvis empty chunks


def test_chunk_cut_scene():
    pr = _proj(*ub.chunk_cut_scene())
    perm, starts, w, T = ub.chunk_starts(pr, G)
    k = int(np.argmax(w))
    assert w[k] >= 1000 and w[k] > 2 * T and int((starts == k + 1).sum()) >= 2
    assert 0 < k < len(perm) - 1


@pytest.mark.parametrize("L", ub.TIER_LENGTHS)
def test_tier_scene_sub_segments(L):
    pr = _proj(*ub.tier_scene(G, L, seed=L))
    assert (pr.tiles_touched == 1).all()
    b = ub.depth_bits(pr.depth)
    assert len(np.unique(b)) == G * L
    _, starts, _, T = ub.chunk_starts(pr, G)
    assert T == 5 * L and (np.diff(starts) == L).all()


@pytest.mark.parametrize("wh", ub.BAND_FRAMES)
def test_band_scene_crossings(wh):
    cam, ins = ub.band_scene(*wh)
    pr = _proj(cam, ins)
    cb, pb = ub.band_boundaries(*wh)
    for b in cb + pb:
        s, big, clipped = ub.straddlers(pr.rect, b)
        assert s >= 1000 and big >= 10 and clipped >= 1, (b, s, big, clipped)
    cl = ub.clone_exactly(ins, 0.3, seed=3)
    pr2 = _proj(cam, cl)
    tied, gap = ub.tie_groups(pr2)
    assert tied >= 30_000 and gap > len(cl[0]) // G


def test_tie_scene():
    cam, ins = ub.tie_scene()
    pr = _proj(cam, ins)
    n = len(ins[0])
    tied, gap = ub.tie_groups(pr)
    assert n >= 195_000 and tied >= 0.3 * int((pr.tiles_touched > 0).sum()) and gap > n // G
