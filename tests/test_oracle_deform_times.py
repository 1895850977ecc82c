"""Pins the oracle with one time per row -- oracle.deform_ref's HexPlane features with times [N] under the network of
util_deep_network.deform_forward -- against the reference's own deform_network run in fp64 with a times_sel whose rows differ
(oracle/make_golden_deform_times.py): the forward 5-tuple and the gradients w.r.t. the times, xyz, w0, a time plane and a
spatial plane.  The per-row GPU tests compare against this oracle."""
import os

import numpy as np
import torch

from oracle import deform_ref as dr
from oracle.make_golden_deform import param_checksum, synth_inputs
from util_deep_network import deform_forward

GOLD = os.path.join(os.path.dirname(__file__), "golden", "deform_times.npz")
AABB = torch.tensor([[1.31, 1.27, 1.3], [-1.29, -1.3, -1.22]])
NAMES = ("pts", "scales", "rot", "opacity", "shs")
TOL = 1e-9          # fp64 against fp64: summation order only


def _run():
    z = np.load(GOLD)
    cfg = dr.CONFIGS["tiny"]
    prm = dr.random_params(cfg, seed=int(z["seed"]), aabb=AABB)
    assert abs(param_checksum(prm) - float(z["param_checksum"])) <= 1e-6 * float(z["param_checksum"]), \
        "CPU RNG drift: regenerate the golden"
    p64 = prm.to(torch.float64)
    for q in p64.leaves():
        q.detach_().requires_grad_(True)
    n = int(z["n"])
    (xyz, sc, rot, op, shs), probes = synth_inputs(n, int(z["seed"]))
    x = xyz.double().requires_grad_(True)
    t = torch.from_numpy(z["times"]).double().requires_grad_(True)
    outs = deform_forward(cfg, p64, [], x, sc.double(), rot.double(), op.double(), shs.double(), t)
    sum((o * p.double()).sum() for o, p in zip(outs, probes)).backward()
    return z, p64, x, t, outs


def test_golden_rows_differ_and_cover_the_time_axis_edges():
    z = np.load(GOLD)
    tt = z["times"]
    T = dr.CONFIGS["tiny"].resolution[3]
    assert len(np.unique(tt)) > len(tt) // 2
    for v in [0.0, 1.0, -1.0] + [2.0 * k / (T - 1) - 1.0 for k in range(T)]:
        assert np.any(np.abs(tt - np.float32(v)) == 0), v
    assert np.any(tt > 1) and np.any(tt < -1)


def test_forward_matches_reference_golden():
    z, _, _, _, outs = _run()
    for nm, o in zip(NAMES, outs):
        ref = torch.from_numpy(z[nm])
        assert o.shape == ref.shape
        assert float((o.detach() - ref).abs().max()) <= TOL, nm


def test_backward_matches_reference_golden_including_dl_dt():
    z, p64, x, t, _ = _run()
    for got, key in ((t.grad, "g_times"), (x.grad, "g_xyz"), (p64.w0.grad, "g_w0"), (p64.planes[0][2].grad, "g_plane02"),
                     (p64.planes[1][0].grad, "g_plane10")):
        ref = torch.from_numpy(z[key])
        assert got.shape == ref.shape, key
        assert float((got - ref).abs().max()) <= TOL * max(1.0, float(ref.abs().max())), key
    # the time coordinate on or past the border: grid_sample's clamp gives dL/dt = 0 exactly
    clamped = np.abs(z["times"]) >= 1.0
    assert clamped.sum() >= 4 and np.all(z["g_times"][clamped] == 0)
    assert np.any(z["g_times"][~clamped] != 0)
