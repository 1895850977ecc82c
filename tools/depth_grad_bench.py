"""Cost of the depth gradient: render() forward + backward of a weighted-sum loss on the image, against the same loss plus a
weighted sum of the depth map (the depth instances of the blend and per-Gaussian backward, DESIGN.md §4.12), in the same
process on the same scene and camera.

CUDA events around every step, warm-up steps first, the L2 flushed (512 MiB write) between timed steps outside the event
pairs, the two arms alternate step by step until each has at least --min-seconds of device time and --steps steps.  Prints
one JSON line: median [min, max] ms per step of each arm, with the GPU name, power limit and SM clocks read by nvidia-smi in
the same run; writes nothing else.

    python tools/depth_grad_bench.py [--workloads C3,C1] [--min-seconds 1.0]
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
    ap.add_argument("--workloads", default="C3,C1")
    ap.add_argument("--time", type=float, default=0.4)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20, help="least timed steps per arm")
    ap.add_argument("--min-seconds", type=float, default=1.0, help="least device time per arm")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("depth_grad_bench measures the GPU: no CUDA device")
    g4d = importlib.import_module("4dgaussians_b200")
    synth = importlib.import_module("4dgaussians_b200.synth")
    dev = torch.device("cuda", 0)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
    result = {"unit": "ms per forward + backward step, median [min, max]", "l2": "flushed between timed steps (512 MiB write)",
              "arms": "colour = loss on the image; depth = the same loss plus a weighted sum of the depth map",
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
        cam = synth.orbit_cameras(1, w["width"], w["height"], radius=w["radius"], focal=w["focal"])[0]
        for f in ("world_view_transform", "full_proj_transform", "camera_center"):
            setattr(cam, f, getattr(cam, f).to(dev))
        cam = synth.SynthCamera(**{**cam.__dict__, "time": a.time})
        gen = torch.Generator(device=dev).manual_seed(0)
        weight = torch.rand(3, cam.image_height, cam.image_width, device=dev, generator=gen)
        dweight = torch.rand(1, cam.image_height, cam.image_width, device=dev, generator=gen)
        arms = {"colour": False, "depth": True}
        grad = {}

        def step(depth):
            for p in params:
                p.grad = None
            out = g4d.render(cam, pc, Pipe, bg)
            loss = (out["render"] * weight).sum()
            if depth:
                loss = loss + (out["depth"] * dweight).sum()
            loss.backward()
            grad[depth] = params[0].grad

        times = {name: [] for name in arms}
        for _ in range(a.warmup):
            for c in arms.values():
                step(c)
        torch.cuda.synchronize()
        while min(len(t) for t in times.values()) < a.steps or min(sum(t) for t in times.values()) < 1000.0 * a.min_seconds:
            for name, c in arms.items():
                flush.fill_(1)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                step(c)
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1))
        assert bool(torch.isfinite(grad[True]).all()) and not torch.equal(grad[True], grad[False])
        run = {"workload": wl, "n": w["n"], "width": w["width"], "height": w["height"], "steps": len(times["colour"]),
               "seconds_per_arm": [round(sum(t) / 1000.0, 3) for t in times.values()]}
        for name, t in times.items():
            run[name] = [round(statistics.median(t), 4), round(min(t), 4), round(max(t), 4)]
        run["overhead_ms"] = round(run["depth"][0] - run["colour"][0], 4)
        result["runs"].append(run)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
