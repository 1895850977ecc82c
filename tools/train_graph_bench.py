"""DPTrainer steps, eager against CUDA-graph replays (DPTrainer(cuda_graph=True)), B views per step, in one process.

Both arms start from the same model and train on the same views (B cameras at B timestamps, ground truth a constant image);
densification is off (densify_until_iter = 0), so after its warm-up and capture the graphed arm only replays.  The arms
alternate in blocks of steps until each has run --min-seconds of steps.  Per step: the host clock from the call to
step() to a device synchronise after it (ms per step), and to the return of step() (host time per step: the Python,
library calls and host waits the caller spends on the step).  Reports median [min, max] of each and prints one JSON line
with the GPU name and power limit read by nvidia-smi; writes nothing else.

    python tools/train_graph_bench.py [--workloads C1,C3] [--views 2] [--min-seconds 1.0]
"""
import argparse
import importlib
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from multicam_bench import Pipe, gpu_info  # noqa: E402


def stat(xs):
    return {"median": round(statistics.median(xs), 4), "min": round(min(xs), 4), "max": round(max(xs), 4), "steps": len(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="C1,C3")
    ap.add_argument("--views", type=int, default=2)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    ap.add_argument("--block-seconds", type=float, default=0.2)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_graph_bench measures the GPU: no CUDA device")
    g4d = importlib.import_module("4dgaussians_b200")
    synth = importlib.import_module("4dgaussians_b200.synth")
    td = importlib.import_module("4dgaussians_b200.train_dp")
    dev = torch.device("cuda", 0)
    result = {"views_per_step": a.views, "min_seconds": a.min_seconds,
              "unit": "ms per step, median [min, max]; host_ms: until step() returns",
              "arms": "eager = DPTrainer(); graphed = DPTrainer(cuda_graph=True) replays", "workloads": {}}
    for wl in a.workloads.split(","):
        w = synth.WORKLOADS[wl]
        cams = synth.orbit_cameras(a.views, w["width"], w["height"], radius=w["radius"], focal=w["focal"])
        for i, c in enumerate(cams):
            c.time = i / max(1, a.views - 1)
        gts = [torch.full((3, w["height"], w["width"]), 0.25, device=dev) for _ in cams]
        bg = torch.tensor([float(x) for x in w["bg"]], device=dev)
        trainers = {}
        for name in ("eager", "graphed"):
            scene = synth.make_scene(w["n"], seed=0, scale_mean=w["scale_mean"])
            torch.manual_seed(1234)
            mod = g4d.deform_network(synth.hidden_args(w["net"]))
            synth.perturb_deformation(mod, 0)
            mod.deformation_net.set_aabb(scene["aabb"][0].tolist(), scene["aabb"][1].tolist())
            opt = td.default_opt()
            opt.densify_until_iter = 0
            trainers[name] = td.DPTrainer(td.GaussianSet(scene, mod.to(dev)), opt, cuda_graph=(name == "graphed"))
        for _ in range(a.warmup):
            for tr in trainers.values():
                tr.step(cams, gts, bg, Pipe)
        torch.cuda.synchronize()
        trainers["graphed"].check()
        wall = {k: [] for k in trainers}
        host = {k: [] for k in trainers}
        while min(sum(v) for v in wall.values()) < 1e3 * a.min_seconds:
            for name, tr in trainers.items():
                spent = 0.0
                while spent < 1e3 * a.block_seconds:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    tr.step(cams, gts, bg, Pipe)
                    t1 = time.perf_counter()
                    torch.cuda.synchronize()
                    t2 = time.perf_counter()
                    wall[name].append(1e3 * (t2 - t0))
                    host[name].append(1e3 * (t1 - t0))
                    spent += wall[name][-1]
        trainers["graphed"].check()
        actions = trainers["graphed"].last_action, trainers["graphed"].captures
        entry = {"n": w["n"], "width": w["width"], "height": w["height"], "net": w["net"],
                 "graphed_last_action": actions[0], "graphed_captures": actions[1]}
        for name in trainers:
            entry[name] = {"step_ms": stat(wall[name]), "host_ms": stat(host[name])}
        entry["speedup"] = round(entry["eager"]["step_ms"]["median"] / entry["graphed"]["step_ms"]["median"], 4)
        result["workloads"][wl] = entry
        del trainers
        torch.cuda.empty_cache()
    result.update(gpu_info(0))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
