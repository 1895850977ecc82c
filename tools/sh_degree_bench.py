"""Cost of the model's SH degree (max_sh_degree d, M = (d + 1)^2 coefficients per Gaussian): per view, the no-grad render,
render forward + backward and one DPTrainer step (one view, its image loss and the Adam update), for d = 0..3 at the active
degree d.

Each arm builds the workload's scene (its degree-d truncation: the first M coefficients of the same seed) and network with
the same seeds.  The SHS head deforms 16 coefficients, so every arm runs the network without it (no_dshs=True): at C3
(dynerf) that differs from the workload's own configuration.  Times are medians (with the range) of CUDA events around
single steps, with the L2 flushed (512 MiB write) between timed steps outside the event pairs, after --warmup steps, and at
least --min-seconds of device time per arm and mode.  Prints one JSON line (with the GPU name, power limit and SM clocks read
by nvidia-smi --query-gpu); writes nothing else.

    python tools/sh_degree_bench.py [--workloads C1,C3] [--degrees 0,1,2,3]
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
    ap.add_argument("--degrees", default="0,1,2,3")
    ap.add_argument("--time", type=float, default=0.4)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--min-seconds", type=float, default=0.3, help="device time per arm and mode")
    ap.add_argument("--min-steps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sh_degree_bench measures the GPU: no CUDA device")
    g4d = importlib.import_module("4dgaussians_b200")
    synth = importlib.import_module("4dgaussians_b200.synth")
    td = importlib.import_module("4dgaussians_b200.train_dp")
    dev = torch.device("cuda", 0)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
    result = {"unit": "ms per view (median, [min, max], steps)", "l2": "flushed between timed steps (512 MiB write)",
              "time": a.time, "network": "the workload's, without the SHS head (no_dshs=True)", "workloads": {}}
    for wname in a.workloads.split(","):
        w = synth.WORKLOADS[wname]
        cam = synth.orbit_cameras(1, w["width"], w["height"], radius=w["radius"], focal=w["focal"])[0]
        cam.time = a.time
        bg = torch.tensor([float(x) for x in w["bg"]], device=dev)
        weight = torch.rand(3, w["height"], w["width"], device=dev, generator=torch.Generator(device=dev).manual_seed(0))
        gt = torch.rand(3, w["height"], w["width"], device=dev, generator=torch.Generator(device=dev).manual_seed(1))
        entry = {"n": w["n"], "width": w["width"], "height": w["height"], "net": w["net"], "arms": {}}
        for d in (int(x) for x in a.degrees.split(",")):
            scene = synth.make_scene(w["n"], seed=0, scale_mean=w["scale_mean"], sh_degree=d)
            args = synth.hidden_args(w["net"])
            args.no_dshs = True

            def module():
                torch.manual_seed(1234)
                mod = g4d.deform_network(args)
                synth.perturb_deformation(mod, 0)
                mod.deformation_net.set_aabb(scene["aabb"][0].tolist(), scene["aabb"][1].tolist())
                return mod.to(dev)
            mod = module()
            pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=d, requires_grad=True)
            params = pc.gaussian_parameters() + list(mod.flat_parameters())
            opt = td.default_opt()
            opt.densify_until_iter = 0          # the step without densification bookkeeping: render, loss, backward, Adam
            trainer = td.DPTrainer(td.GaussianSet(scene, module(), device=dev), opt)

            def render():
                with torch.no_grad():
                    return g4d.render(cam, pc, Pipe, bg)

            def train():
                for p in params:
                    p.grad = None
                (g4d.render(cam, pc, Pipe, bg)["render"] * weight).sum().backward()

            def step():
                trainer.step([cam], [gt], bg, Pipe)

            def timed(fn):
                for _ in range(a.warmup):
                    fn()
                torch.cuda.synchronize()
                times = []
                while sum(times) < 1e3 * a.min_seconds or len(times) < a.min_steps:
                    flush.fill_(len(times) & 0xFF)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    fn()
                    e1.record()
                    torch.cuda.synchronize()
                    times.append(e0.elapsed_time(e1))
                return [round(statistics.median(times), 3), [round(min(times), 3), round(max(times), 3)], len(times)]

            entry["arms"]["d%d" % d] = {"sh_coeffs": (d + 1) ** 2, "sh_bytes_per_gaussian": 12 * (d + 1) ** 2,
                                        "render_no_grad": timed(render), "render_forward_backward": timed(train),
                                        "dp_trainer_step": timed(step)}
            del mod, pc, params, trainer
            torch.cuda.empty_cache()
        result["workloads"][wname] = entry
    result.update(gpu_info(0))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
