"""Models of SH degree 0..3 on the CPU: the G4DCamera tail that carries M = (max_sh_degree + 1)^2, PLY round trips at every
degree, the synthetic scene, GaussianSet's degrees, and the refusals raised in Python before the library is called."""
import ctypes as C
import importlib
import os
import subprocess

import numpy as np
import pytest
import torch

g4d = importlib.import_module("4dgaussians_b200")
synth = importlib.import_module("4dgaussians_b200.synth")
ck = importlib.import_module("4dgaussians_b200.checkpoint")
td = importlib.import_module("4dgaussians_b200.train_dp")
g4d_lib = importlib.import_module("4dgaussians_b200._lib")
rasterizer = importlib.import_module("4dgaussians_b200.rasterizer")
renderer = importlib.import_module("4dgaussians_b200.renderer")


def test_camera_tail_matches_the_header(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    prog = tmp_path / "cam.c"
    prog.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "g4d.h"\nint main(){printf("%zu %zu %zu %zu\\n", '
                    'sizeof(G4DCamera), offsetof(G4DCamera, d_bg), offsetof(G4DCamera, sh_coeffs), offsetof(G4DCamera, reserved));'
                    'return 0;}')
    exe = tmp_path / "cam"
    subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(prog), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    Cam = g4d_lib.Camera
    assert got == [C.sizeof(Cam), Cam.d_bg.offset, Cam.sh_coeffs.offset, Cam.reserved.offset]
    assert Cam().sh_coeffs == 0      # a zero-filled tail is the degree-3 model


@pytest.mark.parametrize("d", [0, 1, 2, 3])
def test_scene_and_settings_carry_the_degree(d):
    m = (d + 1) ** 2
    s, s3 = synth.make_scene(50, seed=4, sh_degree=d), synth.make_scene(50, seed=4)
    assert s["features_rest"].shape == (50, m - 1, 3) and s["features_rest"].is_contiguous()
    for k in s:   # the degree-d scene is the degree-3 scene of the same seed with the higher coefficients dropped
        assert torch.equal(s[k], s3[k][:, :m - 1] if k == "features_rest" else s3[k]), k
    assert g4d_lib.sh_coeffs(s["features_rest"], 50, "features_rest", skip=1) == m
    assert g4d_lib.sh_coeffs(torch.cat([s["features_dc"], s["features_rest"]], 1), 50, "shs") == m
    pc = synth.SyntheticGaussianModel(s, None, device="cpu", sh_degree=0)
    assert pc.max_sh_degree == d
    cam = synth.make_camera(10.0, 32, 24)
    rs, _ = renderer.settings_from_camera(cam, pc, type("P", (), {"debug": False}), torch.zeros(3))
    assert rasterizer.camera_from_settings(rs, sh_coeffs=m).sh_coeffs == m


@pytest.mark.parametrize("d", [0, 1, 2])
def test_ply_round_trip(tmp_path, d):
    m = (d + 1) ** 2
    s = synth.make_scene(23, seed=d, sh_degree=d)
    path = str(tmp_path / "point_cloud.ply")
    ck.save_ply(path, s["xyz"], s["features_dc"], s["features_rest"], s["opacity"], s["scaling"], s["rotation"])
    v = ck.read_ply_vertices(path)
    # scene/gaussian_model.py:213-226: 3 f_dc, 3 (M - 1) f_rest columns, channel-major
    assert list(v) == ck.list_of_attributes(3, 3 * (m - 1), 3, 4)
    assert [k for k in v if k.startswith("f_rest_")] == ["f_rest_%d" % i for i in range(3 * (m - 1))]
    for i in range(3 * (m - 1)):
        ch, k = divmod(i, m - 1)
        assert np.array_equal(v["f_rest_%d" % i], s["features_rest"][:, k, ch].numpy())
    g = ck.load_ply(path, max_sh_degree=d, device="cpu")
    assert g["features_dc"].shape == (23, 1, 3) and g["features_rest"].shape == (23, m - 1, 3)
    for k in ("xyz", "features_dc", "features_rest", "opacity", "scaling", "rotation"):
        assert torch.equal(g[k], s[k]), k
    with pytest.raises(ValueError, match="f_rest columns"):
        ck.load_ply(path, max_sh_degree=3, device="cpu")


@pytest.mark.parametrize("d", [0, 1, 2, 3])
def test_gaussian_set_degrees(d):
    gs = td.GaussianSet(synth.make_scene(40, seed=1, sh_degree=d), None, device="cpu", sh_degree=0)
    assert (gs.max_sh_degree, gs.active_sh_degree) == (d, 0)
    for want in range(1, 5):
        gs.oneupSHdegree()
        assert gs.active_sh_degree == min(want, d)
    assert td.GaussianSet(synth.make_scene(40, seed=1, sh_degree=d), None, device="cpu").active_sh_degree == d


def test_trainer_state_at_degree_1_and_0():
    for d in (1, 0):
        m = (d + 1) ** 2
        mod = g4d.deform_network(synth.hidden_args("small64"))
        tr = td.DPTrainer(td.GaussianSet(synth.make_scene(60, seed=2, sh_degree=d), mod, device="cpu"), td.default_opt())
        b, e = tr.state.segments["f_rest"]
        assert e - b == (60 * 3 * (m - 1) + 3) // 4 * 4
        assert tr.g._features_rest.shape == (60, m - 1, 3)
        # densify and prune rebuild the flat buffers at this M
        assert tr.prune_points(torch.arange(60) % 7 == 0)
        assert tr.g._features_rest.shape == (60 - 9, m - 1, 3)


def test_refusals_in_python():
    s = synth.make_scene(30, seed=3, sh_degree=1)
    with pytest.raises(ValueError, match="active SH degree 2"):
        g4d_lib.check_sh_degree(4, 2)
    with pytest.raises(ValueError, match="active SH degree 2"):
        td.GaussianSet(s, None, device="cpu", sh_degree=2)
    with pytest.raises(ValueError, match="SH head"):
        g4d_lib.check_sh_degree(9, 1, g4d_lib.HEAD_SHS)
    g4d_lib.check_sh_degree(16, 3, g4d_lib.HEAD_SHS | g4d_lib.HEAD_POS)
    for bad in (torch.zeros(30, 2, 3), torch.zeros(30, 16, 2), torch.zeros(30 * 3 * 5)):
        with pytest.raises(RuntimeError, match="no SH degree"):
            g4d_lib.sh_coeffs(bad, 30, "shs")
    with pytest.raises(RuntimeError, match="no SH degree"):
        g4d_lib.sh_coeffs(torch.zeros(30, 16, 3), 30, "features_rest", skip=1)
    assert g4d_lib.sh_coeffs(torch.zeros(30 * 27), 30, "shs") == 9
    assert g4d_lib.sh_coeffs(torch.zeros(30, 0, 3), 30, "features_rest", skip=1) == 1
