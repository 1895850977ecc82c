"""Record the REFERENCE's outputs for the fp64 restatement checks of tests/test_oracle_deform.py and tests/test_oracle_loss.py.

TEST INFRASTRUCTURE ONLY.  Run where the reference tree is available (needs /root/reference or oracle/_ref):
    python oracle/make_golden_live.py
Writes tests/golden/reference_live.npz:
  * deform_<cfg>_<output>: the reference's deform_network in fp64 (``random_params(cfg, seed=11)`` weights, 129 points of
    ``synth_inputs(129, 7)``, t = 0.73) and the parameter checksum that guards against CPU RNG drift;
  * l1 / ssim / reg: the reference's l1_loss, ssim and compute_regulation on ``inputs(seed=5)``.
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
from oracle.make_golden_loss import inputs, load_reference_loss_modules, reference_compute_regulation  # noqa: E402
from oracle.ref_loader import load_reference_deform_network  # noqa: E402

AABB = torch.tensor([[1.31, 1.27, 1.3], [-1.29, -1.3, -1.22]])
NAMES = ("pts", "scales", "rot", "opacity", "shs")
REG_WEIGHTS = (0.01, 0.0001, 0.0001)


def main():
    out = {}
    for name in ("tiny", "dynerf"):
        cfg = dr.CONFIGS[name]
        prm = dr.random_params(cfg, seed=11, aabb=AABB, dtype=torch.float64)
        net = load_reference_deform_network(cfg).double()
        sd = net.state_dict()
        sd.update(dr.params_to_state_dict(prm))
        net.load_state_dict(sd)
        (xyz, sc, rot, op, shs), _ = synth_inputs(129, 7, dtype=torch.float64)
        with torch.no_grad():
            ref = net(xyz, sc, rot, op, shs, torch.tensor(0.73, dtype=torch.float64).repeat(129, 1))
        for nm, r in zip(NAMES, ref):
            out["deform_%s_%s" % (name, nm)] = r.numpy()
        out["deform_%s_checksum" % name] = np.array(param_checksum(prm))
    lu, reg = load_reference_loss_modules()
    img1, img2, grids = inputs(seed=5)
    out["l1"] = np.array(float(lu.l1_loss(img1, img2)))
    out["ssim"] = np.array(float(lu.ssim(img1.float(), img2.float())))
    out["reg"] = np.array(float(reference_compute_regulation(reg, grids, *REG_WEIGHTS)))
    out["reg_weights"] = np.array(REG_WEIGHTS)
    path = os.path.join(os.path.dirname(HERE), "tests", "golden", "reference_live.npz")
    np.savez_compressed(path, **out)
    print("wrote", path)


if __name__ == "__main__":
    main()
