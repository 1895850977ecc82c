"""CPU companion of test_gpu_train_kernels_edges.py: every case it runs, checked here to reach the condition it is named for
-- misaligned views, SSIM tile seams and clipped windows, Adam segments inside float4s and gaps, kNN clouds whose cell faces
round by more than the stopping rule's relative margin -- and the fp32-vs-fp64 distances of the plain restatements that set
the GPU tolerances."""
import numpy as np
import pytest
import torch

import util_train_kernels as ut


def test_l1_numels_take_every_tail():
    assert {n & 3 for n in ut.L1_NUMELS} == {0, 1, 2, 3}
    assert any(n > 4 * 256 and n & 3 for n in ut.L1_NUMELS)          # more than one block's float4s, then a tail
    assert int(np.prod(ut.L1_BATCH[1:])) % 4 == 0 and ut.L1_BATCH[:2] == (4, 3)


def test_offset_views_are_misaligned():
    seen = set()
    for name, out, gt in ut.offset_views():
        assert out.is_contiguous() and gt.is_contiguous() and out.dtype == torch.float32 and out.shape == gt.shape, name
        mo, mg = ut.misalignment(out), ut.misalignment(gt)
        side = name.rsplit(":", 1)[1]
        assert (mo != 0) == (side in ("out", "both")) and (mg != 0) == (side in ("gt", "both")), (name, mo, mg)
        seen |= {("out", mo), ("gt", mg)}
    assert {("out", 4), ("out", 8), ("out", 12), ("gt", 4), ("gt", 8), ("gt", 12)} <= seen     # 1, 2 and 3 floats off
    assert 3 * ut.ODD_HW[0] * ut.ODD_HW[1] % 2 == 1


def test_ssim_shapes_cross_every_seam():
    hs = {h for h, _ in ut.SSIM_HW}
    ws = {w for _, w in ut.SSIM_HW}
    assert set(ut.SSIM_SIDES) <= hs and set(ut.SSIM_SIDES) <= ws
    claims = [ut.ssim_claims(h, w) for h, w in ut.SSIM_HW]
    assert any(c["window_clipped_both_sides_x"] and c["window_clipped_both_sides_y"] for c in claims)
    for axis in "xy":
        assert {c["seams_" + axis] for c in claims} >= {0, 1, 2}                 # one tile, one seam, two seams
        assert any(c["seams_" + axis] and not c["partial_tile_" + axis] for c in claims)   # 32: tiles end on the edge
        assert any(c["seams_" + axis] and c["partial_tile_" + axis] for c in claims)
    assert (1, 77) in ut.SSIM_HW and (77, 1) in ut.SSIM_HW
    assert {len(ut.ssim_shape(i, 2, 2)) for i in range(3)} == {3, 4}
    assert ut.SSIM_MANY[0] * ut.SSIM_MANY[1] > 2048 and ut.SSIM_MANY[0] * ut.SSIM_MANY[1] <= 65535


def test_ssim_special_images_are_what_they_claim():
    x, y = ut.ssim_images((3, 12, 15), "same", 0)
    assert torch.equal(x, y)
    x, y = ut.ssim_images((3, 12, 15), "const", 0)
    assert x.unique().numel() == 1 and y.unique().numel() == 1
    x, y = ut.ssim_images((3, 32, 33), "bright", 0)
    assert float((x - 0.95).abs().max()) <= 1.0001e-3 and float(x.var()) < 1e-6
    # the cancellation the case is for: E[x^2] - mu^2 is ~3e-7, a few ulp of E[x^2] ~ 0.9 (ulp 6e-8) in fp32
    assert float(x.var()) < 1e-6 * float((x * x).mean())


def _ssim_cases():
    for i, (h, w) in enumerate(ut.SSIM_HW):
        yield ut.ssim_shape(i, h, w), "rand", i
    for kind in ("same", "const", "bright"):
        yield (3, 32, 33), kind, 7
        yield (4, 3, 17, 12), kind, 8


@pytest.mark.parametrize("shape,kind,seed", list(_ssim_cases()))
def test_ssim_fp32_restatement_distance(shape, kind, seed):
    """The distance loss_ref.ssim in fp32 keeps from fp64, per pixel: SSIM_K x this is the GPU tolerance.  It must stay below
    SSIM_FP32_BOUND, and only the near-flat bright images (E[x^2] - mu^2 cancels in fp32) come near it."""
    x, y = ut.ssim_images(shape, kind, seed)
    v64, g64 = ut.ssim_ref(x, y, torch.float64, 0.37)
    v32, g32 = ut.ssim_ref(x, y, torch.float32, 0.37)
    if kind == "same":
        assert abs(v64 - 1.0) < 1e-12 and np.abs(g64).max() < 1e-15
        return
    e = ut.pixel_err(g32, g64)
    assert e <= ut.SSIM_FP32_BOUND, e
    if kind != "bright":
        assert e <= 5e-3, e


@pytest.mark.parametrize("name", list(ut.REG_CONFIGS))
def test_regulariser_fp32_restatement_distance(name):
    a = ut.reg_args(**ut.REG_CONFIGS[name])
    planes = ut.reg_planes(a, 3)
    assert len(planes) == len(a.multires)
    if "4 levels" in name:
        assert len(planes) == 4 and sum(len(l) for l in planes) == 24
    if "time res 3" in name:
        assert all(planes[l][k].shape[-2] == 3 for l in range(len(planes)) for k in (2, 4, 5))
    for l in planes:                                   # time planes: |1 - p| of both signs and exact zeros
        r = 1.0 - l[2]
        assert (r > 0).any() and (r < 0).any() and (r == 0).any()
    for w in ut.REG_WEIGHTS:
        _, g64 = ut.reg_ref(planes, w, torch.float64, 1.7)
        _, g32 = ut.reg_ref(planes, w, torch.float32, 1.7)
        e = max(ut.texel_err(b, a_) for la, lb in zip(g64, g32) for a_, b in zip(la, lb))
        assert e <= ut.REG_FP32_BOUND, (w, e)


@pytest.mark.parametrize("name", list(ut.ADAM_LAYOUTS))
def test_adam_layouts_straddle_or_leave_gaps(name):
    numel, segs = ut.ADAM_LAYOUTS[name]
    assert numel % 4 == 0 and all(0 <= b <= e <= numel for b, e in segs)
    assert all(segs[i][0] >= segs[i - 1][1] for i in range(1, len(segs)))           # sorted and disjoint: a valid call
    c = ut.adam_claims(numel, segs)
    assert c["straddles"] or c["gaps"], c
    if name == "zero-length":
        assert c["zero_length"]
    if name == "sixteen":
        assert c["count"] == 16 and c["straddles"] and c["gaps"]
    if name in ("straddle", "gaps"):
        assert c["straddles"]
    g = ut.adam_grads(numel, 0)
    assert (g == 0).any() and (np.abs(g) == np.float32(1e-20)).any() and (np.abs(g) == np.float32(1e4)).any()


def test_adam_tiny_gradient_reaches_subnormal_second_moment():
    v = np.float32(1 - np.float32(0.999)) * np.float32(1e-20) * np.float32(1e-20)
    assert 0 < v < np.finfo(np.float32).tiny


@pytest.mark.parametrize("centre,n", ut.KNN_OFFSETS)
def test_knn_offset_clouds_round_their_faces_beyond_the_relative_margin(centre, n):
    p = ut.knn_offset_cloud(centre, n)
    assert p.shape == (n, 3) and abs(float(p.mean()) - centre) < 1e-3 * centre
    u = float(np.spacing(np.float32(centre)))
    k = (p.astype(np.float64) - centre) / u
    assert np.array_equal(k, np.round(k))                                          # on the fp32 lattice of the offset
    side = ut.KNN_SPACING_ULP * n ** (1 / 3)
    assert 100 <= side / n ** (1 / 3) <= 1000
    # the stopping rule keeps a relative margin face * 1e-4; the face position itself is off by up to ulp(centre) / 2
    assert max(ut.knn_face_rounding(p)) > 1e-4, ut.knn_face_rounding(p)


@pytest.mark.parametrize("kind", ut.KNN_KINDS)
def test_knn_degenerate_clouds(kind):
    p = ut.knn_cloud(kind)
    bmin, cs, dim = ut.knn_grid(p)
    ext = p.max(axis=0) - p.min(axis=0)
    if kind == "identical":
        assert (ext == 0).all() and (dim == 1).all()
    if kind == "two stacks":
        assert len(np.unique(p, axis=0)) == 2
    if kind == "collinear":
        assert ext[0] > 0 and ext[1] == 0 and ext[2] == 0 and dim[1] == dim[2] == 1
    if kind == "cluster + outliers":
        # the grid collapses: the 8000 points of the cluster share a handful of cells
        cell = np.floor((p[:-3] - bmin) / cs).astype(np.int64)
        assert len(np.unique(cell, axis=0)) <= 8
    if kind == "signed zeros":
        z = p == 0
        assert (z & np.signbit(p)).any() and (z & ~np.signbit(p)).any()
