"""Synthetic Gaussians / cameras for tests and bench.py (SURVEY.md §8d).  No datasets exist offline.

Camera maths restates the reference's conventions:
  * pose_spherical            <- /root/reference/scene/dataset_readers.py:200-226 (D-NeRF orbit)
  * R/T extraction            <- /root/reference/scene/dataset_readers.py:243-247
  * world_view_transform etc. <- /root/reference/scene/cameras.py:53-64, utils/graphics_utils.py:38-71
Scene statistics follow SURVEY §8d (xyz ~ U(-1.3,1.3)^3, log-normal scales, un-normalised quats, ...).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional

import numpy as np
import torch


def focal2fov(focal: float, pixels: float) -> float:
    return 2.0 * math.atan(pixels / (2.0 * focal))


def fov2focal(fov: float, pixels: float) -> float:
    return pixels / (2.0 * math.tan(fov / 2.0))


def pose_spherical(theta_deg: float, phi_deg: float, radius: float) -> np.ndarray:
    th, ph = theta_deg / 180.0 * np.pi, phi_deg / 180.0 * np.pi
    trans_t = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, radius], [0, 0, 0, 1]], dtype=np.float32)
    rot_phi = np.array([[1, 0, 0, 0], [0, np.cos(ph), -np.sin(ph), 0], [0, np.sin(ph), np.cos(ph), 0],
                        [0, 0, 0, 1]], dtype=np.float32)
    rot_theta = np.array([[np.cos(th), 0, -np.sin(th), 0], [0, 1, 0, 0], [np.sin(th), 0, np.cos(th), 0],
                          [0, 0, 0, 1]], dtype=np.float32)
    flip = np.array([[-1, 0, 0, 0], [0, 0, 1, 0], [0, 1, 0, 0], [0, 0, 0, 1]], dtype=np.float32)
    return flip @ (rot_theta @ (rot_phi @ trans_t))


def projection_matrix(znear: float, zfar: float, fovx: float, fovy: float) -> torch.Tensor:
    ty, tx = math.tan(fovy / 2), math.tan(fovx / 2)
    top, right = ty * znear, tx * znear
    P = torch.zeros(4, 4)
    P[0, 0] = 2.0 * znear / (2 * right)
    P[1, 1] = 2.0 * znear / (2 * top)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


@dataclass
class SynthCamera:
    """Duck-types the fields of the reference's Camera / MiniCam that render() reads
    (scene/cameras.py:17-78; gaussian_renderer/__init__.py:36-52)."""
    FoVx: float
    FoVy: float
    image_width: int
    image_height: int
    world_view_transform: torch.Tensor   # [4,4] row-vector convention (transposed W2C)
    full_proj_transform: torch.Tensor    # [4,4]
    camera_center: torch.Tensor          # [3]
    time: float = 0.0
    znear: float = 0.01
    zfar: float = 100.0


def make_camera(theta_deg: float, width: int, height: int, *, phi_deg: float = -30.0, radius: float = 4.0,
                fovx: Optional[float] = None, focal: Optional[float] = None, time: float = 0.0) -> SynthCamera:
    if fovx is None:
        fovx = focal2fov(focal, width) if focal is not None else 0.6911112
    fovy = focal2fov(fov2focal(fovx, width), height)
    c2w = pose_spherical(theta_deg, phi_deg, radius)
    m = np.linalg.inv(c2w)
    R = -np.transpose(m[:3, :3])
    R[:, 0] = -R[:, 0]
    T = -m[:3, 3]
    Rt = np.zeros((4, 4), dtype=np.float64)
    Rt[:3, :3] = R.transpose()
    Rt[:3, 3] = T
    Rt[3, 3] = 1.0
    wvt = torch.tensor(np.float32(Rt)).transpose(0, 1).contiguous()
    proj = projection_matrix(0.01, 100.0, fovx, fovy).transpose(0, 1)
    full = (wvt.unsqueeze(0).bmm(proj.unsqueeze(0))).squeeze(0).contiguous()
    center = wvt.inverse()[3, :3].contiguous()
    return SynthCamera(FoVx=fovx, FoVy=fovy, image_width=width, image_height=height, world_view_transform=wvt,
                       full_proj_transform=full, camera_center=center, time=float(time))


def orbit_cameras(count: int, width: int, height: int, *, radius: float = 4.0, focal: Optional[float] = None,
                  timestamps: int = 1):
    thetas = np.linspace(-180, 180, count + 1)[:-1]
    cams = []
    for i, th in enumerate(thetas):
        t = 0.0 if timestamps <= 1 else (i % timestamps) / float(timestamps - 1)
        cams.append(make_camera(float(th), width, height, radius=radius, focal=focal, time=t))
    return cams


def make_scene(n: int, seed: int = 0, scale_mean: float = 0.02, extent: float = 1.3, sh_degree: int = 3) -> Dict[str, torch.Tensor]:
    """CPU fp32 tensors with the layouts GaussianModel holds (SURVEY §8a1); features_rest [N, (sh_degree + 1)^2 - 1, 3]: the
    first coefficients of the degree-3 scene of the same seed."""
    g = torch.Generator().manual_seed(seed)
    xyz = (torch.rand(n, 3, generator=g) * 2 - 1) * extent
    scaling = torch.log(scale_mean * torch.exp(0.5 * torch.randn(n, 3, generator=g)))
    rotation = torch.randn(n, 4, generator=g)
    opacity = torch.logit(0.05 + 0.9 * torch.rand(n, 1, generator=g))
    features_dc = ((torch.rand(n, 1, 3, generator=g) - 0.5) / 0.28209479177387814)
    features_rest = (torch.randn(n, 15, 3, generator=g) * 0.05)[:, :(sh_degree + 1) ** 2 - 1].contiguous()
    aabb = torch.stack([xyz.max(dim=0).values, xyz.min(dim=0).values]) if n > 0 else \
        torch.tensor([[extent] * 3, [-extent] * 3])
    return {"xyz": xyz, "scaling": scaling, "rotation": rotation, "opacity": opacity,
            "features_dc": features_dc, "features_rest": features_rest, "aabb": aabb}


# workloads named in BASELINE.json `configs` (SURVEY §8d "Config -> concrete inputs")
WORKLOADS = {
    "C0": dict(n=10_000, width=400, height=400, net="dnerf", radius=4.0, focal=None, scale_mean=0.02, bg=(1, 1, 1)),
    "C1": dict(n=70_000, width=800, height=800, net="dnerf", radius=4.0, focal=None, scale_mean=0.02, bg=(1, 1, 1)),
    "C2": dict(n=200_000, width=536, height=960, net="hypernerf", radius=2.2, focal=480.0, scale_mean=0.01, bg=(0, 0, 0)),
    "C3": dict(n=300_000, width=1352, height=1014, net="dynerf", radius=2.2, focal=729.0, scale_mean=0.01, bg=(0, 0, 0)),
    "C4": dict(n=2_000_000, width=1920, height=1080, net="dynerf", radius=2.2, focal=1200.0, scale_mean=0.01, bg=(0, 0, 0)),
}


class SyntheticGaussianModel:
    """Duck-types the GaussianModel attributes that render() reads (scene/gaussian_model.py:46-131):
    ``get_xyz, _scaling, _rotation, _opacity, _features_dc, _features_rest, get_features, active_sh_degree,
    max_sh_degree, _deformation, _deformation_table`` + the three activations."""

    def __init__(self, scene: Dict[str, torch.Tensor], deformation, device="cuda", sh_degree: int = 3, requires_grad=False):
        mk = lambda t: torch.nn.Parameter(t.to(device).contiguous(), requires_grad=requires_grad)
        self._xyz = mk(scene["xyz"])
        self._scaling = mk(scene["scaling"])
        self._rotation = mk(scene["rotation"])
        self._opacity = mk(scene["opacity"])
        self._features_dc = mk(scene["features_dc"])
        self._features_rest = mk(scene["features_rest"])
        self._deformation = deformation
        self._deformation_table = torch.ones(self._xyz.shape[0], dtype=torch.bool, device=device)
        self.active_sh_degree = sh_degree
        self.max_sh_degree = int(round(math.sqrt(self._features_rest.shape[1] + 1))) - 1
        self.scaling_activation = torch.exp
        self.opacity_activation = torch.sigmoid
        self.rotation_activation = torch.nn.functional.normalize

    @property
    def get_xyz(self):
        return self._xyz

    @property
    def get_features(self):
        return torch.cat((self._features_dc, self._features_rest), dim=1)

    def gaussian_parameters(self):
        return [self._xyz, self._scaling, self._rotation, self._opacity, self._features_dc, self._features_rest]


def hidden_args(net: str):
    """ModelHiddenParams (arguments/__init__.py:74-107) for the named reference config."""
    from argparse import Namespace
    cfgs = {
        "dnerf": dict(channels=32, resolution=[64, 64, 64, 75], multires=[1, 2], net_width=64, no_do=True, no_dshs=True),
        "hypernerf": dict(channels=16, resolution=[64, 64, 64, 100], multires=[1, 2, 4], net_width=128, no_do=True, no_dshs=True),
        "dynerf": dict(channels=16, resolution=[64, 64, 64, 150], multires=[1, 2], net_width=128, no_do=False, no_dshs=False),
        # small shapes for fast tests (same code paths as dnerf / dynerf)
        "small64": dict(channels=16, resolution=[12, 10, 9, 7], multires=[1, 2], net_width=64, no_do=True, no_dshs=True),
        "small128": dict(channels=16, resolution=[9, 12, 10, 8], multires=[1, 2], net_width=128, no_do=False, no_dshs=False),
        # head-mask / shape corner cases of the tensor-core kernels
        "pos128": dict(channels=16, resolution=[9, 12, 10, 8], multires=[1, 2], net_width=128, no_do=True, no_dshs=True,
                       no_ds=True, no_dr=True),                                                   # a single head
        "shs128": dict(channels=16, resolution=[8, 8, 8, 6], multires=[1, 2], net_width=128, no_do=True, no_dshs=False,
                       no_dx=True, no_ds=True, no_dr=True),                                       # only the 48-wide head
        "c32w128": dict(channels=32, resolution=[10, 9, 8, 6], multires=[1, 2], net_width=128, no_do=False, no_dshs=True),
        # F = 64 with all five heads: the largest shared-memory layout of the tensor-core kernels
        "c32w128sh": dict(channels=32, resolution=[10, 9, 8, 6], multires=[1, 2], net_width=128, no_do=False, no_dshs=False),
        # channel widths the tensor-core kernels do not take (FFMA network; the shared gather and scatter at C/4 = 1, 3, 5, 6)
        # and the widest feature vector, F = 128 (at net_width 64 without the SH head: the FFMA kernel's shared memory)
        "c4w64": dict(channels=4, resolution=[9, 8, 10, 5], multires=[1, 2], net_width=64, no_do=False, no_dshs=True),
        "c12w128": dict(channels=12, resolution=[8, 10, 9, 6], multires=[1, 2, 4], net_width=128, no_do=False, no_dshs=False),
        "c20w64": dict(channels=20, resolution=[10, 9, 8, 7], multires=[1, 2], net_width=64, no_do=True, no_dshs=False),
        "c24w128": dict(channels=24, resolution=[9, 10, 8, 6], multires=[1, 2], net_width=128, no_do=False, no_dshs=True),
        "f128w64": dict(channels=32, resolution=[6, 7, 5, 4], multires=[1, 2, 3, 4], net_width=64, no_do=False, no_dshs=True),
        # F = 60 with all five heads at net_width 128: the FFMA kernel's tile of 64 Gaussians only just fits (no room for trunk
        # biases: the half tile)
        "c20w128sh": dict(channels=20, resolution=[8, 10, 9, 6], multires=[1, 2, 4], net_width=128, no_do=False, no_dshs=False),
        # deformation networks with trunk layers (defor_depth 3): the dnerf heads at width 64, the dynerf heads at 128
        "deep64": dict(channels=32, resolution=[12, 10, 9, 7], multires=[1, 2], net_width=64, no_do=True, no_dshs=True,
                       defor_depth=3),
        "deep128": dict(channels=16, resolution=[9, 12, 10, 8], multires=[1, 2], net_width=128, no_do=False, no_dshs=False,
                        defor_depth=3),
    }
    c = cfgs[net]
    return Namespace(net_width=c["net_width"], timebase_pe=4, defor_depth=c.get("defor_depth", 1), posebase_pe=10, scale_rotation_pe=2, opacity_pe=2,
                     timenet_width=64, timenet_output=32, bounds=1.6, grid_pe=0,
                     kplanes_config={"grid_dimensions": 2, "input_coordinate_dim": 4, "output_coordinate_dim": c["channels"],
                                     "resolution": list(c["resolution"])},
                     multires=list(c["multires"]), no_dx=c.get("no_dx", False), no_grid=False, no_ds=c.get("no_ds", False),
                     no_dr=c.get("no_dr", False), no_do=c["no_do"],
                     no_dshs=c["no_dshs"], empty_voxel=False, static_mlp=False, apply_rotation=False)


def perturb_deformation(module, seed: int = 0):
    """Synthetic 'trained' weights (SURVEY §8d): time planes 1 + N(0, 0.05) so that the deformation is not constant;
    everything else keeps the reference initialisation."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for lvl in module.deformation_net.grid.grids:
            for k, p in enumerate(lvl):
                if k in (2, 4, 5):
                    p.add_((torch.randn(p.shape, generator=g) * 0.05).to(p.device))
    return module
