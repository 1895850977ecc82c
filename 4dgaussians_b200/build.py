"""Build recipe for libg4d.so (hand-written sm_90a kernels behind the C-ABI of include/g4d.h).

In-tree build with plain nvcc (no torch dependency): the .so travels to the GPU box with the snapshot.
``g4d_geom.cu`` and ``g4d_deform_tc.cu`` -- the translation units that contain the projection maths (and ``g4d_knn.cu``:
exact distances) -- are compiled with -fmad=false (bit-exact index stages, see g4d_math.cuh); the others use the default FMA
contraction.  The wgmma building-block self test (``g4d_tc_selftest.cu``) goes into its own ``libg4d_selftest.so`` (tests only).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libg4d.so")
SELFTEST_OUT = os.path.join(HERE, "libg4d_selftest.so")     # wgmma building-block self test: tests only
OBJ = os.path.join(HERE, "build")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "--expt-extended-lambda",
          "-Xptxas", "-v"]
UNITS = {
    "g4d_geom.cu": ["-fmad=false"],
    "g4d_raster.cu": [],
    "g4d_bin.cu": [],
    "g4d_loss.cu": [],
    "g4d_knn.cu": ["-fmad=false"],
    "g4d_optim.cu": [],
    "g4d_backward.cu": [],
    "g4d_backward_depth.cu": [],
    "g4d_api.cu": [],
    "g4d_deform_tc.cu": ["-fmad=false"],
    "g4d_deform_tc_bwd.cu": [],
}


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.isfile(cand):
            return cand
    raise RuntimeError("nvcc not found: libg4d.so cannot be built (there is no CPU fallback)")


def _sources_mtime() -> float:
    m = 0.0
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for f in os.listdir(root):
            m = max(m, os.path.getmtime(os.path.join(root, f)))
    return max(m, os.path.getmtime(__file__))


def needs_build() -> bool:
    return not os.path.isfile(OUT) or not os.path.isfile(SELFTEST_OUT) or os.path.getmtime(OUT) < _sources_mtime()


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return OUT
    nvcc = _nvcc()
    os.makedirs(OBJ, exist_ok=True)
    logs = {}

    def compile_one(item):
        src, extra = item
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        cmd = [nvcc] + ARCH + COMMON + extra + ["-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        logs[src] = r.stdout + r.stderr
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s" % (src, logs[src]))
        return obj

    with ThreadPoolExecutor(max_workers=4) as ex:
        objs = list(ex.map(compile_one, list(UNITS.items()) + [("g4d_tc_selftest.cu", [])]))
    selftest_obj = objs.pop()
    for out, oo in ((OUT, objs), (SELFTEST_OUT, [selftest_obj])):
        cmd = [nvcc] + ARCH + ["-shared", "-o", out] + oo + ["-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    with open(os.path.join(OBJ, "ptxas.log"), "w") as f:
        for k, v in logs.items():
            f.write("==== %s ====\n%s\n" % (k, v))
    if verbose:
        for k, v in logs.items():
            print("====", k)
            print(v)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
