"""Record the REFERENCE module's state_dict layout (keys, shapes, parameter groups) as golden data.

TEST INFRASTRUCTURE ONLY.  Run where the reference tree is available (needs /root/reference or oracle/_ref):
    python oracle/make_golden_state_dict.py
Writes tests/golden/reference_state_dicts.json: per config of ``deform_ref.CONFIGS`` used by the tests, the ordered
state_dict keys with their shapes and the shapes of ``get_mlp_parameters()`` / ``get_grid_parameters()`` -- what a
checkpoint written by one module must match to load in the other (load_state_dict is strict about both).
"""
from __future__ import annotations

import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import deform_ref as dr  # noqa: E402
from oracle.ref_loader import load_reference_deform_network  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "reference_state_dicts.json")


def main():
    out = {}
    for name in ("dnerf", "hypernerf", "dynerf"):
        ref = load_reference_deform_network(dr.CONFIGS[name])
        sd = ref.state_dict()
        out[name] = {"keys": list(sd.keys()), "shapes": [list(v.shape) for v in sd.values()],
                     "mlp_shapes": [list(p.shape) for p in ref.get_mlp_parameters()],
                     "grid_shapes": [list(p.shape) for p in ref.get_grid_parameters()]}
    with open(OUT, "w") as fh:
        json.dump(out, fh, indent=1)
    print(OUT)


if __name__ == "__main__":
    main()
