"""ctypes binding of libg4d.so (the C-ABI in include/g4d.h).

There is deliberately no fallback: if the library is missing or cannot be loaded, every product entry
point raises.  ``load()`` only dlopens (works on a GPU-less box; used by the `not gpu` ABI test);
workspaces need a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from typing import Dict, Optional

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libg4d.so")

MAX_LEVELS = 4
NUM_HEADS = 5
HEAD_POS, HEAD_SCALES, HEAD_ROT, HEAD_OPACITY, HEAD_SHS = 1, 2, 4, 8, 16

OPT_SYNC_MODE, OPT_INSTANCE_CAPACITY, OPT_TIGHT_CULL, OPT_STAGE_TIMING, OPT_TENSOR_CORES, OPT_TC_DEBUG, OPT_WARP_CULL = 1, 2, 3, 4, 5, 6, 7
OPT_KEEP_DEFORMED = 8
OPT_PDL = 9
STAGES = ("prep", "geom", "scan", "emit", "sort", "ranges", "blend", "blend_bwd", "geom_bwd", "deform_bwd")

BUF = dict(depth=1, rect=2, tiles_touched=3, xy=4, conic_opacity=5, rgb=6, sorted_keys=7, sorted_ids=8, ranges=9,
           final_T=10, n_contrib=11, clamped=12, deformed=13, deformed_shs=14, bin_phases=15)

# every symbol include/g4d.h declares (tests/test_abi.py checks the .so exports all of them)
ABI_SYMBOLS = [
    "g4d_abi_version", "g4d_last_error", "g4d_workspace_create", "g4d_workspace_destroy", "g4d_context_create",
    "g4d_context_destroy", "g4d_context_stats", "g4d_deform_forward", "g4d_deform_backward", "g4d_rasterize_forward",
    "g4d_rasterize_backward", "g4d_render_forward", "g4d_render_backward", "g4d_workspace_set_option", "g4d_context_read",
    "g4d_context_stage_times", "g4d_debug_tc_cycles", "g4d_l1_loss", "g4d_l1_loss_backward", "g4d_ssim", "g4d_ssim_backward",
    "g4d_plane_regulation", "g4d_dist2_knn3", "g4d_adam_step", "g4d_render_forward_cameras", "g4d_render_backward_cameras",
]

fp = C.c_void_p   # device pointers travel as integers
ABI_VERSION = 3
CAM_DEBUG, CAM_NO_GRAD = 1, 2      # G4DCamera.debug bits
MAX_CAMERAS = 32                   # G4D_MAX_CAMERAS: cameras of one g4d_render_forward_cameras call


def relu_bits_words(n: int) -> int:
    """G4D_RELU_BITS_WORDS (include/g4d.h)"""
    return 24 * int(n) + 4


class Camera(C.Structure):
    _fields_ = [("image_height", C.c_int32), ("image_width", C.c_int32), ("sh_degree", C.c_int32), ("debug", C.c_int32),
                ("tanfovx", C.c_float), ("tanfovy", C.c_float), ("scale_modifier", C.c_float), ("time", C.c_float),
                ("viewmatrix", C.c_float * 16), ("projmatrix", C.c_float * 16), ("campos", C.c_float * 3),
                ("bg", C.c_float * 3), ("d_viewmatrix", fp), ("d_projmatrix", fp), ("d_campos", fp), ("d_bg", fp)]


class DeformParams(C.Structure):
    _fields_ = [("levels", C.c_int32), ("channels", C.c_int32), ("net_width", C.c_int32), ("head_mask", C.c_int32),
                ("res", (C.c_int32 * 4) * MAX_LEVELS), ("planes", (fp * 6) * MAX_LEVELS), ("aabb", fp),
                ("w0", fp), ("b0", fp), ("w1", fp * NUM_HEADS), ("b1", fp * NUM_HEADS), ("w2", fp * NUM_HEADS),
                ("b2", fp * NUM_HEADS), ("version", C.c_uint64)]


class DeformGrads(C.Structure):
    _fields_ = [("planes", (fp * 6) * MAX_LEVELS), ("w0", fp), ("b0", fp), ("w1", fp * NUM_HEADS), ("b1", fp * NUM_HEADS),
                ("w2", fp * NUM_HEADS), ("b2", fp * NUM_HEADS)]


class Gaussians(C.Structure):
    _fields_ = [("n", C.c_int64), ("xyz", fp), ("scaling", fp), ("rotation", fp), ("opacity", fp), ("features_dc", fp),
                ("features_rest", fp)]


class GaussianGrads(C.Structure):
    _fields_ = [("xyz", fp), ("scaling", fp), ("rotation", fp), ("opacity", fp), ("features_dc", fp),
                ("features_rest", fp), ("means2D", fp)]


class AdamSegment(C.Structure):
    _fields_ = [("begin", C.c_int64), ("end", C.c_int64), ("lr", C.c_float), ("reserved", C.c_float)]


class Stats(C.Structure):
    _fields_ = [("num_rendered", C.c_int64), ("num_visible", C.c_int64), ("instance_capacity", C.c_int64),
                ("tiles_x", C.c_int32), ("tiles_y", C.c_int32)]


_lib = None
_lock = threading.Lock()


class G4DError(RuntimeError):
    pass


def load():
    """dlopen libg4d.so and declare prototypes.  Raises (never falls back) when the library is absent."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.isfile(LIB_PATH):
            raise G4DError(
                "libg4d.so is not built (%s). Run `python -c 'import __graft_entry__ as g; g.build()'` or "
                "`python 4dgaussians_b200/build.py`. The g4d render path has no CPU / PyTorch fallback." % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        lib.g4d_abi_version.restype = C.c_int
        lib.g4d_last_error.restype = C.c_char_p
        lib.g4d_workspace_create.restype = C.c_void_p
        lib.g4d_workspace_create.argtypes = [C.c_int]
        lib.g4d_workspace_destroy.argtypes = [C.c_void_p]
        lib.g4d_workspace_destroy.restype = None
        lib.g4d_context_create.restype = C.c_void_p
        lib.g4d_context_create.argtypes = [C.c_void_p]
        lib.g4d_context_destroy.argtypes = [C.c_void_p]
        lib.g4d_context_destroy.restype = None
        lib.g4d_context_stats.argtypes = [C.c_void_p, C.POINTER(Stats)]
        lib.g4d_workspace_set_option.argtypes = [C.c_void_p, C.c_int, C.c_int64]
        lib.g4d_context_read.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int64]
        lib.g4d_context_read.restype = C.c_int64
        lib.g4d_context_stage_times.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_int]
        lib.g4d_debug_tc_cycles.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        lib.g4d_deform_forward.argtypes = [C.c_void_p, C.POINTER(DeformParams), C.c_int64] + [fp] * 5 + [C.c_float] + \
            [fp] * 6 + [C.c_void_p]
        lib.g4d_deform_backward.argtypes = [C.c_void_p, C.POINTER(DeformParams), C.POINTER(DeformGrads), C.c_int64, fp,
                                            C.c_float] + [fp] * 11 + [C.c_void_p]
        lib.g4d_rasterize_forward.argtypes = [C.c_void_p, C.POINTER(Camera), C.c_int64] + [fp] * 8 + [C.c_void_p]
        lib.g4d_rasterize_backward.argtypes = [C.c_void_p, C.POINTER(Camera), C.c_int64] + [fp] * 12 + [C.c_void_p]
        lib.g4d_render_forward.argtypes = [C.c_void_p, C.POINTER(Camera), C.POINTER(DeformParams), C.POINTER(Gaussians),
                                           fp, fp, fp, C.c_void_p]
        lib.g4d_render_backward.argtypes = [C.c_void_p, C.POINTER(Camera), C.POINTER(DeformParams), C.POINTER(DeformGrads),
                                            C.POINTER(Gaussians), fp, C.POINTER(GaussianGrads), C.c_void_p]
        pp = C.POINTER(C.c_void_p)     # host array of device pointers / contexts
        lib.g4d_render_forward_cameras.argtypes = [pp, C.c_int32, C.POINTER(Camera), C.POINTER(DeformParams), C.POINTER(Gaussians),
                                                   pp, pp, pp, C.c_void_p]
        lib.g4d_render_backward_cameras.argtypes = [pp, C.c_int32, C.POINTER(Camera), C.POINTER(DeformParams), C.POINTER(DeformGrads),
                                                    C.POINTER(Gaussians), pp, C.POINTER(GaussianGrads), pp, C.c_void_p]
        lib.g4d_l1_loss.argtypes = [C.c_void_p, fp, fp, C.c_int64, C.c_float, fp, C.c_void_p]
        lib.g4d_l1_loss_backward.argtypes = [C.c_void_p, fp, fp, C.c_int64, C.c_float, fp, fp, C.c_void_p]
        lib.g4d_ssim.argtypes = [C.c_void_p, fp, fp, C.c_int32, C.c_int32, C.c_int32, C.c_float, fp, fp, C.c_void_p]
        lib.g4d_ssim_backward.argtypes = [C.c_void_p, fp, fp, C.c_int32, C.c_int32, C.c_int32, C.c_float, fp, fp, fp, C.c_void_p]
        lib.g4d_plane_regulation.argtypes = [C.c_void_p, C.POINTER(DeformParams), C.POINTER(DeformGrads), C.c_float, C.c_float,
                                             C.c_float, fp, fp, C.c_void_p]
        lib.g4d_adam_step.argtypes = [C.c_void_p, fp, fp, fp, fp, C.c_int64, C.POINTER(AdamSegment), C.c_int32, C.c_float, C.c_float,
                                      C.c_float, C.c_int64, C.c_float, C.c_void_p]
        lib.g4d_dist2_knn3.argtypes = [C.c_void_p, C.c_int64, fp, fp, C.c_void_p]
        if lib.g4d_abi_version() != ABI_VERSION:
            raise G4DError("libg4d.so ABI version mismatch")
        _lib = lib
        return lib


SELFTEST_LIB_PATH = os.path.join(HERE, "libg4d_selftest.so")


def load_selftest():
    """The wgmma building-block self test lives in its own tiny library (tests only; not in libg4d.so)."""
    if not os.path.isfile(SELFTEST_LIB_PATH):
        raise G4DError("libg4d_selftest.so is not built (run __graft_entry__.build())")
    lib = C.CDLL(SELFTEST_LIB_PATH)
    lib.g4d_selftest_wgmma.argtypes = [C.POINTER(C.c_int), fp, fp, fp, C.c_void_p]
    return lib


def check(rc: int, what: str = "g4d"):
    if rc != 0:
        msg = load().g4d_last_error().decode("utf-8", "replace")
        raise G4DError("%s failed (code %d): %s" % (what, rc, msg))


class Workspace:
    """One per (process, device).  Owns scratch memory and the packed-weight cache."""
    _by_device: Dict[int, "Workspace"] = {}

    def __init__(self, device: int):
        lib = load()
        self.device = int(device)
        self.handle = lib.g4d_workspace_create(self.device)
        if not self.handle:
            raise G4DError("g4d_workspace_create(%d): %s" % (device, lib.g4d_last_error().decode()))
        self._free_contexts = []

    @classmethod
    def get(cls, device: int) -> "Workspace":
        ws = cls._by_device.get(int(device))
        if ws is None:
            ws = cls(int(device))
            cls._by_device[int(device)] = ws
        return ws

    def set_option(self, option: int, value: int):
        check(load().g4d_workspace_set_option(self.handle, option, int(value)), "g4d_workspace_set_option")

    def acquire_context(self) -> "Context":
        while self._free_contexts:
            ctx = self._free_contexts.pop()
            if ctx.handle:
                return ctx
        return Context(self)

    def release_context(self, ctx: "Context"):
        if ctx.handle:      # (a context finalised in the same GC pass as its lease must not be resurrected into the pool)
            self._free_contexts.append(ctx)


class Context:
    """State one forward keeps for its backward (projected records, sorted instance list, final_T ...)."""

    def __init__(self, ws: Workspace):
        self.ws = ws
        self.handle = load().g4d_context_create(ws.handle)
        if not self.handle:
            raise G4DError("g4d_context_create: %s" % load().g4d_last_error().decode())

    def stats(self) -> Stats:
        s = Stats()
        check(load().g4d_context_stats(self.handle, C.byref(s)), "g4d_context_stats")
        return s

    def stage_times(self) -> Dict[str, float]:
        arr = (C.c_float * len(STAGES))()
        rc = load().g4d_context_stage_times(self.handle, arr, len(STAGES))
        if rc < 0:
            check(rc, "g4d_context_stage_times")
        return {k: float(arr[i]) for i, k in enumerate(STAGES)}

    def read(self, name: str):
        """Copy an internal buffer to a numpy array (tests / debugging)."""
        import numpy as np
        lib = load()
        which = BUF[name]
        nbytes = lib.g4d_context_read(self.handle, which, None, 0)
        if nbytes < 0:
            check(int(nbytes), "g4d_context_read")
        raw = np.zeros(max(int(nbytes), 1), dtype=np.uint8)
        got = lib.g4d_context_read(self.handle, which, raw.ctypes.data_as(C.c_void_p), int(nbytes))
        if got < 0:
            check(int(got), "g4d_context_read")
        raw = raw[:int(nbytes)]
        dt, shape = {
            "depth": (np.float32, (-1,)), "rect": (np.int32, (-1, 4)), "tiles_touched": (np.uint32, (-1,)),
            "xy": (np.float32, (-1, 2)), "conic_opacity": (np.float32, (-1, 4)), "rgb": (np.float32, (-1, 3)),
            "sorted_keys": (np.uint64, (-1,)), "sorted_ids": (np.uint32, (-1,)), "ranges": (np.uint32, (-1, 2)),
            "final_T": (np.float32, (-1,)), "n_contrib": (np.uint32, (-1,)), "clamped": (np.uint8, (-1, 3)),
            "deformed": (np.float32, (-1, 11)), "deformed_shs": (np.float32, (-1, 16, 3)),
            "bin_phases": (np.int64, (-1,))}[name]
        return raw.view(dt).reshape(shape)

    def __del__(self):
        try:
            if self.handle and _lib is not None:
                _lib.g4d_context_destroy(self.handle)
                self.handle = None
        except Exception:
            pass
