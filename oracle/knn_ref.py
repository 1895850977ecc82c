"""CPU restatement of simple_knn._C.distCUDA2 (SURVEY.md 8f N4).  TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED by the reference: submodules/simple-knn is an empty directory in /root/reference (no source, no tests, no
binary).  Anchored on the call site scene/gaussian_model.py:148
(``dist2 = torch.clamp_min(distCUDA2(points), 0.0000001); scales = log(sqrt(dist2))``) and on the published algorithm of
graphdeco-inria/simple-knn (spatial.cu / simple_knn.cu): exact 3 nearest neighbours by squared Euclidean distance, self
excluded by index, result (d0 + d1 + d2) / 3 in fp32.
"""
from __future__ import annotations

import numpy as np


def dist2_knn3_bruteforce(xyz: np.ndarray, block: int = 512) -> np.ndarray:
    """O(N^2) in fp32 with the kernel's operation order: ((dx*dx + dy*dy) + dz*dz), then ((b0 + b1) + b2) / 3."""
    p = np.ascontiguousarray(xyz, dtype=np.float32)
    n = p.shape[0]
    out = np.empty(n, np.float32)
    for s in range(0, n, block):
        q = p[s:s + block]
        dx = p[None, :, 0] - q[:, None, 0]; dy = p[None, :, 1] - q[:, None, 1]; dz = p[None, :, 2] - q[:, None, 2]
        d = (dx * dx + dy * dy) + dz * dz
        d[np.arange(q.shape[0]), np.arange(s, s + q.shape[0])] = np.float32(np.finfo(np.float32).max)   # self, by index
        if n < 4:
            d = np.concatenate([d, np.full((q.shape[0], 3), np.finfo(np.float32).max, np.float32)], axis=1)
        b = np.sort(np.partition(d, 2, axis=1)[:, :3], axis=1)
        with np.errstate(over="ignore"):
            out[s:s + block] = ((b[:, 0] + b[:, 1]) + b[:, 2]) / np.float32(3.0)
    return out


def dist2_knn3_kdtree(xyz: np.ndarray) -> np.ndarray:
    """scipy cKDTree (fp64 search) for sizes brute force cannot reach; distances re-evaluated in fp32."""
    from scipy.spatial import cKDTree
    p = np.ascontiguousarray(xyz, dtype=np.float32)
    _, idx = cKDTree(p.astype(np.float64)).query(p.astype(np.float64), k=4)
    nb = p[idx[:, 1:4]]
    dx = nb[:, :, 0] - p[:, None, 0]; dy = nb[:, :, 1] - p[:, None, 1]; dz = nb[:, :, 2] - p[:, None, 2]
    d = np.sort((dx * dx + dy * dy) + dz * dz, axis=1)
    return ((d[:, 0] + d[:, 1]) + d[:, 2]) / np.float32(3.0)
