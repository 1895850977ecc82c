"""Generate golden vectors for deform_network with one time per row by running the REFERENCE's own module in fp64.

TEST INFRASTRUCTURE ONLY.  Run in the build container (needs /root/reference):
    python oracle/make_golden_deform_times.py
Writes tests/golden/deform_times.npz: the ``tiny`` configuration (SH and opacity heads on) with the weights of
``random_params(cfg, seed)`` (a parameter checksum guards against RNG drift), the inputs of ``synth_inputs`` and a
``times_sel`` [N, 1] whose rows differ -- rows at 0 and 1, on every time-grid line, outside [-1, 1] and random in between --
and that requires grad.  Stored: the forward 5-tuple and the autograd gradients of ``sum(out_i * probe_i)`` w.r.t. times_sel,
xyz, w0, a time plane (level 0, plane 2: (x, t)) and a spatial plane (level 1, plane 0: (x, y)).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import deform_ref as dr  # noqa: E402
from oracle.make_golden_deform import param_checksum, synth_inputs  # noqa: E402
from oracle.ref_loader import load_reference_deform_network  # noqa: E402

NAME, N, SEED = "tiny", 67, 5
AABB = torch.tensor([[1.31, 1.27, 1.3], [-1.29, -1.3, -1.22]])


def golden_times(n: int, T: int, seed: int) -> torch.Tensor:
    """[n] fp32: 0, 1, -1, every time-grid line, values outside [-1, 1], then uniform in [-1.2, 1.2]"""
    edge = [0.0, 1.0, -1.0, 1.5, -2.0, 1.0 + 2 ** -10] + [2.0 * k / (T - 1) - 1.0 for k in range(T)]
    g = torch.Generator().manual_seed(700 + seed)
    t = torch.rand(n, generator=g, dtype=torch.float64) * 2.4 - 1.2
    t[:len(edge)] = torch.tensor(edge, dtype=torch.float64)
    return t.float()


def main():
    cfg = dr.CONFIGS[NAME]
    prm = dr.random_params(cfg, seed=SEED, aabb=AABB)
    net = load_reference_deform_network(cfg)
    sd = net.state_dict()
    sd.update(dr.params_to_state_dict(prm))
    net.load_state_dict(sd)
    net = net.double()
    (xyz, sc, rot, op, shs), probes = synth_inputs(N, SEED)
    times = golden_times(N, cfg.resolution[3], SEED)
    xyz_r = xyz.double().requires_grad_(True)
    tsel = times.double().reshape(N, 1).requires_grad_(True)
    outs = net(xyz_r, sc.double(), rot.double(), op.double(), shs.double(), tsel)
    sum((o * p.double()).sum() for o, p in zip(outs, probes)).backward()
    grid = net.deformation_net.grid.grids
    blob = {"n": N, "seed": SEED, "times": times.numpy(), "param_checksum": param_checksum(prm),
            "g_times": tsel.grad.reshape(-1).numpy(), "g_xyz": xyz_r.grad.numpy(),
            "g_w0": net.deformation_net.feature_out[0].weight.grad.numpy(),
            "g_plane02": grid[0][2].grad.numpy(), "g_plane10": grid[1][0].grad.numpy()}
    for nm, o in zip(("pts", "scales", "rot", "opacity", "shs"), outs):
        blob[nm] = o.detach().numpy()
    out = os.path.join(os.path.dirname(HERE), "tests", "golden", "deform_times.npz")
    np.savez_compressed(out, **blob)
    print("wrote", out, os.path.getsize(out) // 1024, "KiB")


if __name__ == "__main__":
    main()
