"""The C-ABI library loads on a GPU-less box and exports every symbol include/g4d.h declares; the ctypes
mirrors have the sizes the C structs have; the product path refuses to run without a CUDA device."""
import ctypes as C
import os
import re
import subprocess
import sys
import importlib

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
g4d_lib = importlib.import_module("4dgaussians_b200._lib")
build = importlib.import_module("4dgaussians_b200.build")


@pytest.fixture(scope="module")
def lib():
    build.build()            # nvcc cross-compiles for sm_90a without a GPU
    return g4d_lib.load()


def _header_functions():
    src = open(os.path.join(ROOT, "include", "g4d.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(g4d_[a-z0-9_]+)\s*\(", src)))


def test_exports_every_declared_symbol(lib):
    names = _header_functions()
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), n
    assert sorted(g4d_lib.ABI_SYMBOLS) == names
    assert lib.g4d_abi_version() == 3


def test_struct_sizes_match_c(tmp_path):
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "g4d.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(G4DCamera),'
                    'sizeof(G4DDeformParams), sizeof(G4DDeformGrads), sizeof(G4DGaussians), sizeof(G4DGaussianGrads), sizeof(G4DStats));return 0;}')
    exe = tmp_path / "sz"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    sizes = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert sizes == [C.sizeof(g4d_lib.Camera), C.sizeof(g4d_lib.DeformParams), C.sizeof(g4d_lib.DeformGrads),
                     C.sizeof(g4d_lib.Gaussians), C.sizeof(g4d_lib.GaussianGrads), C.sizeof(g4d_lib.Stats)]


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the behaviour on a GPU-less box")
def test_no_cpu_fallback(lib):
    with pytest.raises(g4d_lib.G4DError):
        g4d_lib.Workspace(0)
    g4d = importlib.import_module("4dgaussians_b200")
    rs = g4d.GaussianRasterizationSettings(8, 8, 0.5, 0.5, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0, torch.zeros(3),
                                           False, False)
    r = g4d.GaussianRasterizer(rs)
    with pytest.raises(RuntimeError):
        r(means3D=torch.zeros(1, 3), means2D=torch.zeros(1, 3), shs=torch.zeros(1, 16, 3), colors_precomp=None,
          opacities=torch.zeros(1, 1), scales=torch.ones(1, 3), rotations=torch.ones(1, 4), cov3D_precomp=None)


def test_sass_is_sm90a(lib):
    out = subprocess.run(["cuobjdump", "--list-elf", g4d_lib.LIB_PATH], capture_output=True, text=True)
    if out.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    assert "sm_90a" in out.stdout


def test_option_constants_match_header():
    src = open(os.path.join(ROOT, "include", "g4d.h")).read()
    enum = src[src.index("enum { G4D_OPT_SYNC_MODE"):]
    enum = re.sub(r"/\*.*?\*/", "", enum[:enum.index("};")], flags=re.S)
    found = dict(re.findall(r"G4D_OPT_([A-Z_]+)\s*=\s*(\d+)", enum))
    assert len(found) >= 9 and len(set(found.values())) == len(found)
    for name, value in found.items():
        assert getattr(g4d_lib, "OPT_" + name) == int(value), name


def test_forward_chain_kernels_carry_the_dependent_launch_instructions(lib):
    """DESIGN.md 4.6: every kernel of the forward chain waits on / releases its programmatic dependents (SASS ACQBULK / PREEXIT)."""
    chain = {"_ZN3g4d16bin_place_kernelENS_12BinPlaceArgsE": ("ACQBULK", "PREEXIT"),
             "_ZN3g4d14bin_fix_kernelENS_12BinPlaceArgsEi": ("ACQBULK", "PREEXIT"),
             "_ZN3g4d15bin_sort_kernelENS_11BinSortArgsE": ("PREEXIT",)}
    for fn, needed in chain.items():
        out = subprocess.run(["cuobjdump", "-sass", "-fun", fn, g4d_lib.LIB_PATH], capture_output=True, text=True)
        if out.returncode != 0:
            pytest.skip("cuobjdump unavailable")
        assert "Function : " + fn in out.stdout, fn
        for ins in needed:
            assert ins in out.stdout, (fn, ins)
