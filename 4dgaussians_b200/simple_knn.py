"""Drop-in for ``simple_knn._C`` (/root/reference/scene/gaussian_model.py:22 ``from simple_knn._C import distCUDA2``, used
at :148 to initialise the Gaussian scales).  The submodule is absent from the reference tree; this restates its published
behaviour (mean squared distance to the 3 nearest other points) on the g4d C-ABI.  ``dropin.install()`` registers it as
``simple_knn`` / ``simple_knn._C``."""
from __future__ import annotations

import torch

from . import _lib


def distCUDA2(points: torch.Tensor) -> torch.Tensor:
    if not points.is_cuda:
        raise RuntimeError("distCUDA2 needs a CUDA tensor (the g4d path has no CPU fallback)")
    p = _lib.cuda_f32(points, "points")
    if p.dim() != 2 or p.shape[1] != 3:
        raise RuntimeError("distCUDA2 expects an [N,3] tensor")
    n = p.shape[0]
    out = torch.empty(n, device=p.device, dtype=torch.float32)
    dev = p.device
    with torch.cuda.device(dev):
        _lib.check(_lib.load().g4d_dist2_knn3(_lib.workspace_of(dev).handle, n, p.data_ptr(), out.data_ptr(),
                                              _lib.stream_of(dev)), "g4d_dist2_knn3")
    return out
