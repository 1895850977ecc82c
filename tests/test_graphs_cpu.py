"""CUDA-graph capture, the parts that need no device: the C mirrors of G4DGraphStatus and G4DAdamScalars, the new entry
points' argument checks, the host-computed Adam scalars, and GraphedRender's refusals that come before anything touches a GPU."""
import ctypes as C
import importlib
import os
import subprocess

import numpy as np

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_lib = importlib.import_module("4dgaussians_b200._lib")
build = importlib.import_module("4dgaussians_b200.build")
graphs = importlib.import_module("4dgaussians_b200.graphs")
synth = importlib.import_module("4dgaussians_b200.synth")


@pytest.fixture(scope="module")
def lib():
    build.build()
    return _lib.load()


def test_graph_status_struct_matches_c(tmp_path):
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "g4d.h"\nint main(){printf("%zu %zu %zu\\n", '
                    'sizeof(G4DGraphStatus), offsetof(G4DGraphStatus, max_instances), offsetof(G4DGraphStatus, f16_range));return 0;}')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(_lib.GraphStatus), _lib.GraphStatus.max_instances.offset, _lib.GraphStatus.f16_range.offset]


def test_entry_points_refuse_null_handles(lib):
    st = _lib.GraphStatus()
    assert lib.g4d_context_set_time_source(None, None) == -2
    assert lib.g4d_workspace_freeze(None, 1) == -2
    assert lib.g4d_workspace_graph_status(None, 0, C.byref(st)) == -2
    assert b"NULL" in lib.g4d_last_error()


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


class _DebugPipe(_Pipe):
    debug = True


def test_graphed_render_refuses_before_touching_a_device():
    pc = synth.SyntheticGaussianModel(synth.make_scene(16, seed=1), None, device="cpu")
    cam = synth.make_camera(0.0, 32, 32)
    with pytest.raises(ValueError, match="1..32 views"):
        graphs.GraphedRender(pc, _Pipe, torch.zeros(3), [])
    with pytest.raises(ValueError, match="1..32 views"):
        graphs.GraphedRender(pc, _Pipe, torch.zeros(3), [cam] * 33)
    with pytest.raises(NotImplementedError, match="g4d deformation network"):
        graphs.GraphedRender(pc, _Pipe, torch.zeros(3), cam)           # pc._deformation is None: not the g4d network
    with pytest.raises(ValueError, match="pipe.debug"):
        graphs.GraphedRender(pc, _DebugPipe, torch.zeros(3), cam, stage="coarse")


def test_adam_scalars_are_the_host_step_expressions(lib):
    """g4d_adam_scalars gives the float32 values g4d_adam_step computes in double: lr per segment, 1 / (1 - b1^t),
    1 / sqrt(1 - b2^t), grad_scale"""
    segs = (_lib.AdamSegment * 3)(_lib.AdamSegment(0, 8, 1.6e-4, 0.0), _lib.AdamSegment(8, 16, 2.5e-3, 0.0),
                                  _lib.AdamSegment(16, 24, 0.05, 0.0))
    b1, b2 = np.float32(0.9), np.float32(0.999)
    for step in (1, 2, 7, 1000, 30000):
        out = _lib.AdamScalars()
        assert lib.g4d_adam_scalars(segs, 3, float(b1), float(b2), step, 0.25, C.byref(out)) == 0
        assert list(out.lr[:3]) == [float(np.float32(x)) for x in (1.6e-4, 2.5e-3, 0.05)] and list(out.lr[3:]) == [0.0] * 13
        assert out.inv_bc1 == float(np.float32(1.0 / (1.0 - float(b1) ** step)))
        assert out.inv_sqrt_bc2 == float(np.float32(1.0 / np.sqrt(1.0 - float(b2) ** step)))
        assert out.grad_scale == 0.25
    assert lib.g4d_adam_scalars(segs, 3, 0.9, 0.999, 0, 1.0, C.byref(_lib.AdamScalars())) == -2
    assert lib.g4d_adam_scalars(segs, 17, 0.9, 0.999, 1, 1.0, C.byref(_lib.AdamScalars())) == -2


def test_adam_step_device_checks_its_arguments_before_touching_a_device(lib):
    segs = (_lib.AdamSegment * 1)(_lib.AdamSegment(0, 8, 1e-3, 0.0))
    assert lib.g4d_adam_step_device(None, None, None, None, None, 8, segs, 1, 0.9, 0.999, 1e-15, None, None) == -2
    assert b"g4d_adam_step_device" in lib.g4d_last_error()


def test_adam_scalars_struct_matches_c(tmp_path):
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "g4d.h"\nint main(){printf("%zu %zu\\n", '
                    'sizeof(G4DAdamScalars), offsetof(G4DAdamScalars, grad_scale));return 0;}')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(_lib.AdamScalars), _lib.AdamScalars.grad_scale.offset]
