"""Cost of the deformation network's trunk layers (defor_depth D): per view, the geometry stage, the no-grad render and render
forward + backward, for D = 1 on the default engine, D = 1 with the tensor cores off (the FFMA kernels every deeper trunk runs
on) and D in --depths.

Each arm builds the workload's scene and network with the same seeds; only the trunk differs.  Times are medians (with the
range) of CUDA events around single steps, with the L2 flushed (512 MiB write) between timed steps outside the event pairs,
after --warmup steps, and at least --min-seconds of device time per arm and mode.  The geometry stage is read from the
library's own per-stage events (G4D_OPT_STAGE_TIMING) in a pass of its own, so that the other two modes run without them.
Prints one JSON line (with the GPU name, power limit and SM clocks read by nvidia-smi --query-gpu); writes nothing else.

    python tools/deep_network_bench.py [--workloads C1,C3] [--depths 2,4,8]
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
    ap.add_argument("--depths", default="2,4,8")
    ap.add_argument("--time", type=float, default=0.4)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--min-seconds", type=float, default=0.3, help="device time per arm and mode")
    ap.add_argument("--min-steps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("deep_network_bench measures the GPU: no CUDA device")
    g4d = importlib.import_module("4dgaussians_b200")
    synth = importlib.import_module("4dgaussians_b200.synth")
    lib = g4d._lib
    dev = torch.device("cuda", 0)
    ws = lib.Workspace.get(0)
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
    arms = [("D1", 1, 2), ("D1_tc_off", 1, 0)] + [("D%d" % d, d, 2) for d in (int(x) for x in a.depths.split(","))]
    result = {"unit": "ms per view (median, [min, max])", "l2": "flushed between timed steps (512 MiB write)",
              "time": a.time, "workloads": {}}
    for wname in a.workloads.split(","):
        w = synth.WORKLOADS[wname]
        scene = synth.make_scene(w["n"], seed=0, scale_mean=w["scale_mean"])
        cam = synth.orbit_cameras(1, w["width"], w["height"], radius=w["radius"], focal=w["focal"])[0]
        cam.time = a.time
        bg = torch.tensor([float(x) for x in w["bg"]], device=dev)
        weight = torch.rand(3, w["height"], w["width"], device=dev, generator=torch.Generator(device=dev).manual_seed(0))
        entry = {"n": w["n"], "width": w["width"], "height": w["height"], "net": w["net"], "arms": {}}
        for name, depth, tc in arms:
            args = synth.hidden_args(w["net"])
            args.defor_depth = depth
            torch.manual_seed(1234)
            mod = g4d.deform_network(args)
            synth.perturb_deformation(mod, 0)
            mod.deformation_net.set_aabb(scene["aabb"][0].tolist(), scene["aabb"][1].tolist())
            mod = mod.to(dev)
            pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
            params = pc.gaussian_parameters() + list(mod.flat_parameters())
            ws.set_option(lib.OPT_TENSOR_CORES, tc)

            def render():
                with torch.no_grad():
                    return g4d.render(cam, pc, Pipe, bg)

            def train():
                for p in params:
                    p.grad = None
                (g4d.render(cam, pc, Pipe, bg)["render"] * weight).sum().backward()

            def geom():
                ws.set_option(lib.OPT_STAGE_TIMING, 1)
                try:
                    render()
                    return ws._free_contexts[-1].stage_times()["geom"]
                finally:
                    ws.set_option(lib.OPT_STAGE_TIMING, 0)

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
                return times

            def staged():
                for _ in range(a.warmup):
                    geom()
                times = []
                while sum(times) < 1e3 * a.min_seconds / 4 or len(times) < a.min_steps:
                    flush.fill_(len(times) & 0xFF)
                    times.append(geom())
                return times

            def summary(t):
                return [round(statistics.median(t), 3), [round(min(t), 3), round(max(t), 3)], len(t)]
            try:
                entry["arms"][name] = {"defor_depth": depth, "tensor_cores_option": tc, "geometry_stage": summary(staged()),
                                       "render_no_grad": summary(timed(render)), "render_forward_backward": summary(timed(train))}
            finally:
                ws.set_option(lib.OPT_TENSOR_CORES, 2)
            del mod, pc, params
            torch.cuda.empty_cache()
        result["workloads"][wname] = entry
    result.update(gpu_info(0))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
