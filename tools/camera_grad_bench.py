"""Cost of camera gradients: render forward + backward of one weighted-sum loss, with and without the camera tensors
(world_view_transform, full_proj_transform, camera_center) requiring grad, for k = 1 (render) and k > 1 (render_cameras),
in the same process on the same scene and cameras.

CUDA events around every step, warm-up steps first, the L2 flushed (512 MiB write) between timed steps outside the event
pairs, the two arms alternate step by step.  Prints one JSON line: median [min, max] ms per step of each arm, with the GPU
name, power limit and SM clocks read by nvidia-smi in the same run; writes nothing else.

    python tools/camera_grad_bench.py [--workloads C1,C3] [--ks 1,4] [--steps 20]
"""
import argparse
import importlib
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from multicam_bench import Pipe, gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="C1,C3")
    ap.add_argument("--ks", default="1,4")
    ap.add_argument("--time", type=float, default=0.4)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20, help="timed steps per arm")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("camera_grad_bench measures the GPU: no CUDA device")
    g4d = importlib.import_module("4dgaussians_b200")
    synth = importlib.import_module("4dgaussians_b200.synth")
    dev = torch.device("cuda", 0)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
    result = {"unit": "ms per forward + backward step, median [min, max]", "l2": "flushed between timed steps (512 MiB write)",
              "arms": "plain = no camera tensor requires grad; camera = view, proj and campos of every camera require grad",
              **gpu_info(0), "runs": []}
    for wl in a.workloads.split(","):
        w = synth.WORKLOADS[wl]
        scene = synth.make_scene(w["n"], seed=0, scale_mean=w["scale_mean"])
        torch.manual_seed(1234)
        mod = g4d.deform_network(synth.hidden_args(w["net"]))
        synth.perturb_deformation(mod, 0)
        mod.deformation_net.set_aabb(scene["aabb"][0].tolist(), scene["aabb"][1].tolist())
        mod = mod.to(dev)
        pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
        params = pc.gaussian_parameters() + list(mod.flat_parameters())
        bg = torch.tensor([float(x) for x in w["bg"]], device=dev)
        for k in (int(x) for x in a.ks.split(",")):
            cams = synth.orbit_cameras(k, w["width"], w["height"], radius=w["radius"], focal=w["focal"])
            for c in cams:
                c.time = a.time
                for f in ("world_view_transform", "full_proj_transform", "camera_center"):
                    setattr(c, f, getattr(c, f).to(dev))
            leaf = [synth.SynthCamera(**{**c.__dict__, **{f: getattr(c, f).clone().requires_grad_(True) for f in
                                                           ("world_view_transform", "full_proj_transform", "camera_center")}})
                    for c in cams]
            gen = torch.Generator(device=dev).manual_seed(0)
            weights = [torch.rand(3, c.image_height, c.image_width, device=dev, generator=gen) for c in cams]

            def step(cs):
                for p in params:
                    p.grad = None
                outs = g4d.render(cs[0], pc, Pipe, bg) if k == 1 else None
                outs = [outs] if k == 1 else g4d.render_cameras(cs, pc, Pipe, bg)
                sum((o["render"] * wi).sum() for o, wi in zip(outs, weights)).backward()

            arms = {"plain": cams, "camera": leaf}
            times = {name: [] for name in arms}
            for _ in range(a.warmup):
                for cs in arms.values():
                    step(cs)
            torch.cuda.synchronize()
            for _ in range(a.steps):
                for name, cs in arms.items():
                    flush.fill_(1)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    step(cs)
                    e1.record()
                    torch.cuda.synchronize()
                    times[name].append(e0.elapsed_time(e1))
            assert all(c.world_view_transform.grad is not None for c in leaf)
            run = {"workload": wl, "n": w["n"], "width": w["width"], "height": w["height"], "k": k}
            for name, t in times.items():
                run[name] = [round(statistics.median(t), 4), round(min(t), 4), round(max(t), 4)]
            run["overhead_ms"] = round(run["camera"][0] - run["plain"][0], 4)
            result["runs"].append(run)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
