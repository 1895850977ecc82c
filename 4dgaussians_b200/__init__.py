"""g4d -- H100-native fused deform + rasterize render path for 4D Gaussian Splatting.

The package name starts with a digit (it is fixed by the project layout), so import it with
``importlib.import_module("4dgaussians_b200")`` or through ``4dgaussians_b200.dropin.install()`` which
registers the reference-facing module names (``diff_gaussian_rasterization`` ...).

Product path = the C-ABI library ``libg4d.so`` (hand-written sm_90a kernels, see include/g4d.h).  Importing
this package never compiles or falls back to anything: use ``__graft_entry__.build()`` / ``build.build()``.
"""
from . import _lib  # noqa: F401
from .deformation import deform_network  # noqa: F401
from .rasterizer import GaussianRasterizationSettings, GaussianRasterizer  # noqa: F401
from .renderer import render  # noqa: F401
from . import losses  # noqa: F401

__all__ = ["GaussianRasterizationSettings", "GaussianRasterizer", "deform_network", "render"]
