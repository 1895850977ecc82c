"""On-disk formats adjacent to the render path (SURVEY.md 8f N3), byte-compatible with the reference so that models trained
there render here and vice versa:

    save_ply / load_ply                 <- GaussianModel.save_ply / load_ply   scene/gaussian_model.py:250-314
    save_deformation / load_model       <- GaussianModel.save_deformation / load_model  scene/gaussian_model.py:233-249
    save_iteration / load_iteration     <- Scene.save / Scene.__init__ (loaded_iter branch)   scene/__init__.py:84-103
    export_perframe_3dgs                <- export_perframe_3DGS.py:55-106 + utils/render_utils.py get_state_at_time

The reference writes PLY through ``plyfile`` (not installed here): the same ``binary_little_endian 1.0`` vertex element
(float32 properties ``x y z nx ny nz f_dc_* f_rest_* opacity scale_* rot_*``) is written / parsed directly with numpy.
``deformation.pth`` is the module's ``state_dict()`` -- key- and shape-identical to the reference's (planes are saved as
ordinary contiguous ``[1,C,H,W]`` tensors; in memory they live channel-last).
"""
from __future__ import annotations

import os
from typing import Dict, Optional

import numpy as np
import torch

_PLY_TYPES = {"float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8", "uchar": "u1", "uint8": "u1", "char": "i1",
              "int8": "i1", "short": "<i2", "int16": "<i2", "ushort": "<u2", "uint16": "<u2", "int": "<i4", "int32": "<i4",
              "uint": "<u4", "uint32": "<u4"}


def list_of_attributes(n_dc: int = 3, n_rest: int = 45, n_scale: int = 3, n_rot: int = 4):
    """scene/gaussian_model.py:213-226 construct_list_of_attributes"""
    l = ['x', 'y', 'z', 'nx', 'ny', 'nz']
    l += ['f_dc_%d' % i for i in range(n_dc)]
    l += ['f_rest_%d' % i for i in range(n_rest)]
    l.append('opacity')
    l += ['scale_%d' % i for i in range(n_scale)]
    l += ['rot_%d' % i for i in range(n_rot)]
    return l


def write_ply_vertices(path: str, names, table: np.ndarray):
    """``table`` [N, len(names)] float32 -> binary little-endian PLY with one float property per column."""
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    table = np.ascontiguousarray(table, dtype="<f4")
    assert table.ndim == 2 and table.shape[1] == len(names)
    header = "ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % table.shape[0]
    header += "".join("property float %s\n" % n for n in names) + "end_header\n"
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(table.tobytes())


def read_ply_vertices(path: str) -> Dict[str, np.ndarray]:
    """Parses the first element of a PLY file (binary little-endian or ascii) into {property: array}."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError("%s is not a PLY file" % path)
        fmt, count, props, in_first, seen = None, 0, [], False, 0
        while True:
            line = f.readline()
            if not line:
                raise ValueError("unterminated PLY header")
            tok = line.decode("ascii").split()
            if not tok or tok[0] == "comment":
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                seen += 1
                in_first = seen == 1
                if in_first:
                    count = int(tok[2])
            elif tok[0] == "property" and in_first:
                if tok[1] == "list":
                    raise ValueError("list properties are not supported in the vertex element")
                props.append((tok[2], _PLY_TYPES[tok[1]]))
            elif tok[0] == "end_header":
                break
        if fmt == "binary_little_endian":
            dt = np.dtype(props)
            data = np.frombuffer(f.read(count * dt.itemsize), dtype=dt, count=count)
            return {n: np.asarray(data[n]) for n, _ in props}
        if fmt == "ascii":
            rows = np.loadtxt(f, max_rows=count, ndmin=2)
            return {n: rows[:, i].astype(t) for i, (n, t) in enumerate(props)}
        raise ValueError("unsupported PLY format %r" % fmt)


def save_ply(path: str, xyz, features_dc, features_rest, opacity, scaling, rotation):
    """GaussianModel.save_ply (scene/gaussian_model.py:250-268).  features are [N,1,3] / [N,M-1,3] with M = (max_sh_degree
    + 1)^2, written as 3M - 3 f_rest columns; f_dc / f_rest columns are channel-major (``transpose(1, 2).flatten(start_dim=1)``)."""
    t = lambda a: a.detach().float().cpu()
    xyz_, op, sc, rot = t(xyz).numpy(), t(opacity).numpy().reshape(-1, 1), t(scaling).numpy(), t(rotation).numpy()
    f_dc = t(features_dc).transpose(1, 2).flatten(start_dim=1).contiguous().numpy()
    f_rest = t(features_rest).transpose(1, 2).flatten(start_dim=1).contiguous().numpy()
    table = np.concatenate((xyz_, np.zeros_like(xyz_), f_dc, f_rest, op, sc, rot), axis=1)
    write_ply_vertices(path, list_of_attributes(f_dc.shape[1], f_rest.shape[1], sc.shape[1], rot.shape[1]), table)


def load_ply(path: str, max_sh_degree: int = 3, device="cuda") -> Dict[str, torch.Tensor]:
    """GaussianModel.load_ply (scene/gaussian_model.py:275-314): returns the six tensors in GaussianModel's layouts."""
    v = read_ply_vertices(path)
    n = v["x"].shape[0]
    xyz = np.stack((v["x"], v["y"], v["z"]), axis=1)
    dc = np.stack((v["f_dc_0"], v["f_dc_1"], v["f_dc_2"]), axis=1).reshape(n, 3, 1)
    rest_names = sorted((k for k in v if k.startswith("f_rest_")), key=lambda s: int(s.split('_')[-1]))
    if len(rest_names) != 3 * (max_sh_degree + 1) ** 2 - 3:
        raise ValueError("PLY holds %d f_rest columns, expected %d" % (len(rest_names), 3 * (max_sh_degree + 1) ** 2 - 3))
    rest = np.stack([v[k] for k in rest_names], axis=1).reshape(n, 3, (max_sh_degree + 1) ** 2 - 1) if rest_names else \
        np.zeros((n, 3, 0), np.float32)
    scale_names = sorted((k for k in v if k.startswith("scale_")), key=lambda s: int(s.split('_')[-1]))
    rot_names = sorted((k for k in v if k.startswith("rot")), key=lambda s: int(s.split('_')[-1]))
    mk = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float, device=device)
    return {"xyz": mk(xyz), "features_dc": mk(dc).transpose(1, 2).contiguous(), "features_rest": mk(rest).transpose(1, 2).contiguous(),
            "opacity": mk(v["opacity"][..., None]), "scaling": mk(np.stack([v[k] for k in scale_names], axis=1)),
            "rotation": mk(np.stack([v[k] for k in rot_names], axis=1))}


def save_deformation(path: str, deformation, deformation_table: Optional[torch.Tensor] = None,
                     deformation_accum: Optional[torch.Tensor] = None):
    """GaussianModel.save_deformation (scene/gaussian_model.py:246-249): deformation.pth (+ table / accum when given)."""
    os.makedirs(path, exist_ok=True)
    sd = {k: v.detach().contiguous().clone() for k, v in deformation.state_dict().items()}   # planes -> plain NCHW strides
    torch.save(sd, os.path.join(path, "deformation.pth"))
    if deformation_table is not None:
        torch.save(deformation_table, os.path.join(path, "deformation_table.pth"))
    if deformation_accum is not None:
        torch.save(deformation_accum, os.path.join(path, "deformation_accum.pth"))


def load_model(path: str, deformation, n_gaussians: int, device="cuda"):
    """GaussianModel.load_model (scene/gaussian_model.py:233-245): loads deformation.pth into ``deformation`` (a g4d or a
    reference deform_network) and returns (deformation_table, deformation_accum)."""
    sd = torch.load(os.path.join(path, "deformation.pth"), map_location=device)
    deformation.load_state_dict(sd)
    deformation.to(device)
    table = torch.gt(torch.ones(n_gaussians, device=device), 0)
    accum = torch.zeros(n_gaussians, 3, device=device)
    if os.path.exists(os.path.join(path, "deformation_table.pth")):
        table = torch.load(os.path.join(path, "deformation_table.pth"), map_location=device)
    if os.path.exists(os.path.join(path, "deformation_accum.pth")):
        accum = torch.load(os.path.join(path, "deformation_accum.pth"), map_location=device)
    return table, accum


def iteration_dir(model_path: str, iteration: int, stage: str = "fine") -> str:
    """Scene.save (scene/__init__.py:96-103)"""
    return os.path.join(model_path, "point_cloud", ("coarse_iteration_%d" if stage == "coarse" else "iteration_%d") % iteration)


def save_iteration(model_path: str, iteration: int, pc, stage: str = "fine") -> str:
    d = iteration_dir(model_path, iteration, stage)
    save_ply(os.path.join(d, "point_cloud.ply"), pc._xyz, pc._features_dc, pc._features_rest, pc._opacity, pc._scaling, pc._rotation)
    save_deformation(d, pc._deformation, getattr(pc, "_deformation_table", None), getattr(pc, "_deformation_accum", None))
    return d


def load_iteration(model_path: str, iteration: int, deformation, max_sh_degree: int = 3, device="cuda"):
    d = iteration_dir(model_path, iteration)
    g = load_ply(os.path.join(d, "point_cloud.ply"), max_sh_degree, device)
    table, accum = load_model(d, deformation, g["xyz"].shape[0], device)
    return g, table, accum


def get_state_at_time(pc, time: float):
    """utils/render_utils.py:3-19: the deformed Gaussians at one timestamp, in the PRE-activation parameterisation the PLY
    format stores (log-scales, raw quaternions, opacity logits).  Quirk kept: the reference returns the UN-deformed
    ``pc._opacity`` (":19" returns ``opacity``, not ``opacity_final``)."""
    with torch.no_grad():
        n = pc._xyz.shape[0]
        t = torch.tensor(float(time), device=pc._xyz.device).repeat(n, 1)
        m3, sc, rot, _op_final, shs = pc._deformation(pc._xyz, pc._scaling, pc._rotation, pc._opacity, pc.get_features, t)
        return m3, sc, rot, pc._opacity, shs


def export_perframe_3dgs(out_dir: str, pc, times) -> list:
    """export_perframe_3DGS.py:55-106: one static-3DGS PLY per timestamp (``time_%05d.ply``), loadable by any 3DGS viewer
    (standard pre-activation columns)."""
    os.makedirs(out_dir, exist_ok=True)
    paths = []
    n_dc = pc._features_dc.shape[1]
    for i, t in enumerate(times):
        m3, sc, rot, op, shs = get_state_at_time(pc, t)
        p = os.path.join(out_dir, "time_%05d.ply" % i)
        save_ply(p, m3, shs[:, :n_dc, :], shs[:, n_dc:, :], op, sc, rot)
        paths.append(p)
    return paths
