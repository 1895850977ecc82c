"""Cost of the alpha map: render() / render_cameras() forward + backward of a weighted-sum loss on the images (colour), the same
with the alpha maps returned but outside the loss (alpha_out: the alpha write, DESIGN.md §4.13), and the same loss plus a
weighted sum of the alpha maps (alpha_loss: the alpha gradient folded into the blend backward), in the same process on the
same scene and cameras, for one camera and for --k cameras at one time.

CUDA events around every step, warm-up steps first, the L2 flushed (512 MiB write) between timed steps outside the event
pairs, the two arms alternate step by step until each has at least --min-seconds of device time and --steps steps.  Prints
one JSON line: median [min, max] ms per step of each arm, with the GPU name, power limit and SM clocks read by nvidia-smi in
the same run; writes nothing else.

    python tools/alpha_grad_bench.py [--workloads C3] [--k 3] [--min-seconds 1.0]
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
    ap.add_argument("--workloads", default="C3")
    ap.add_argument("--k", type=int, default=3, help="cameras of the render_cameras runs")
    ap.add_argument("--time", type=float, default=0.4)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20, help="least timed steps per arm")
    ap.add_argument("--min-seconds", type=float, default=1.0, help="least device time per arm")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("alpha_grad_bench measures the GPU: no CUDA device")
    g4d = importlib.import_module("4dgaussians_b200")
    synth = importlib.import_module("4dgaussians_b200.synth")
    dev = torch.device("cuda", 0)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
    result = {"unit": "ms per forward + backward step, median [min, max]", "l2": "flushed between timed steps (512 MiB write)",
              "arms": "colour = loss on the images; alpha_out = the same with the alpha maps returned; alpha_loss = the same "
                      "loss plus a weighted sum of the alpha maps",
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
        for k in sorted({1, a.k}):
            cams = []
            for cam in synth.orbit_cameras(k, w["width"], w["height"], radius=w["radius"], focal=w["focal"]):
                for f in ("world_view_transform", "full_proj_transform", "camera_center"):
                    setattr(cam, f, getattr(cam, f).to(dev))
                cams.append(synth.SynthCamera(**{**cam.__dict__, "time": a.time}))
            result["runs"].append(measure(a, g4d, wl, w, pc, params, bg, cams, flush, dev))
    print(json.dumps(result))


def measure(a, g4d, wl, w, pc, params, bg, cams, flush, dev):
    """one run: the three arms alternating step by step on cams (render() for one camera, render_cameras() for several)"""
    gen = torch.Generator(device=dev).manual_seed(0)
    H, W = cams[0].image_height, cams[0].image_width
    weight = torch.rand(3, H, W, device=dev, generator=gen)
    aweight = torch.rand(1, H, W, device=dev, generator=gen)
    arms = {"colour": (False, False), "alpha_out": (True, False), "alpha_loss": (True, True)}
    grad = {}

    def step(arm):
        want, in_loss = arms[arm]
        for p in params:
            p.grad = None
        if len(cams) == 1:
            outs = [g4d.render(cams[0], pc, Pipe, bg, return_alpha=want)]
        else:
            outs = g4d.render_cameras(cams, pc, Pipe, bg, return_alpha=want)
        loss = sum((o["render"] * weight).sum() for o in outs)
        if in_loss:
            loss = loss + sum((o["alpha"] * aweight).sum() for o in outs)
        loss.backward()
        grad[arm] = params[0].grad

    times = {name: [] for name in arms}
    for _ in range(a.warmup):
        for name in arms:
            step(name)
    torch.cuda.synchronize()
    while min(len(t) for t in times.values()) < a.steps or min(sum(t) for t in times.values()) < 1000.0 * a.min_seconds:
        for name in arms:
            flush.fill_(1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step(name)
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1))
    assert bool(torch.isfinite(grad["alpha_loss"]).all()) and not torch.equal(grad["alpha_loss"], grad["colour"])
    run = {"workload": wl, "k": len(cams), "n": w["n"], "width": W, "height": H, "steps": len(times["colour"]),
           "seconds_per_arm": [round(sum(t) / 1000.0, 3) for t in times.values()]}
    for name, t in times.items():
        run[name] = [round(statistics.median(t), 4), round(min(t), 4), round(max(t), 4)]
    run["alpha_out_overhead_ms"] = round(run["alpha_out"][0] - run["colour"][0], 4)
    run["alpha_loss_overhead_ms"] = round(run["alpha_loss"][0] - run["colour"][0], 4)
    return run


if __name__ == "__main__":
    main()
