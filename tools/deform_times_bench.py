"""Cost of deform_network with one time per Gaussian (times_sel rows that differ: g4d_deform_forward_times / _backward_times).

For each workload (C1: 70k Gaussians, dnerf network; C3: 300k, dynerf network), forward (no grad) and forward + backward:
  * scalar_xT  -- T calls at one time each over the N Gaussians (T frames of a trajectory the old way), T in --frames;
  * rows_T     -- one per-row call over the T*N rows (xyz.repeat(T, 1), times = t.repeat_interleave(N));
  * scalar_x1  -- one call at one time over N rows, and
  * uniform    -- one per-row call over the same N rows, every row at that time: the price of the per-row gather and scatter.
The per-row arms get a times tensor that requires grad, so that equal times still take the per-row path; forward + backward
then also computes dL/dt.  Times are medians (with the range) of CUDA events around single steps, after --warmup steps, over
at least --min-seconds of device time per arm.  Prints one JSON line (with the GPU name, power limit and SM clocks read by
nvidia-smi --query-gpu); writes nothing else.

    python tools/deform_times_bench.py [--workloads C1,C3] [--frames 8,32]
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

from multicam_bench import gpu_info  # noqa: E402


def _time_arm(step, warmup, min_seconds, min_steps):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    ms, total = [], 0.0
    while total < min_seconds * 1e3 or len(ms) < min_steps:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
        total += ms[-1]
    return {"ms": round(statistics.median(ms), 4), "min": round(min(ms), 4), "max": round(max(ms), 4), "steps": len(ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="C1,C3")
    ap.add_argument("--frames", default="8,32")
    ap.add_argument("--time", type=float, default=0.4)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=1.0, help="device time per arm and mode")
    ap.add_argument("--min-steps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("deform_times_bench measures the GPU: no CUDA device")
    g4d = importlib.import_module("4dgaussians_b200")
    synth = importlib.import_module("4dgaussians_b200.synth")
    dev = torch.device("cuda", 0)
    result = {"unit": "ms per call or per group of calls (median, [min, max])", **gpu_info(0), "workloads": {}}
    for wname in a.workloads.split(","):
        w = synth.WORKLOADS[wname]
        n = w["n"]
        scene = synth.make_scene(n, seed=0, scale_mean=w["scale_mean"])
        torch.manual_seed(1234)
        mod = g4d.deform_network(synth.hidden_args(w["net"]))
        synth.perturb_deformation(mod, 0)
        mod.deformation_net.set_aabb(scene["aabb"][0].tolist(), scene["aabb"][1].tolist())
        mod = mod.to(dev)
        base = [scene[k].to(dev).float().contiguous() for k in ("xyz", "scaling", "rotation", "opacity")]
        base.append(torch.cat([scene["features_dc"], scene["features_rest"]], dim=1).to(dev).float().contiguous())
        entry = {"n": n, "net": w["net"], "forward": {}, "forward_backward": {}}

        def arm(mode, name, ins, calls):
            """calls: list of times_sel values, one forward (+ backward) per entry, all over the tensors ins"""
            grad = mode == "forward_backward"
            leaves = [x.clone().requires_grad_(grad) for x in ins]

            def step():
                with torch.set_grad_enabled(grad):
                    for t in calls:
                        outs = mod(*leaves, t)
                        if grad:
                            sum(o.sum() for o in outs).backward()
                mod.zero_grad(set_to_none=True)
            try:
                entry[mode][name] = _time_arm(step, a.warmup, a.min_seconds, a.min_steps)
            except (torch.cuda.OutOfMemoryError, g4d._lib.G4DError) as e:   # the arm does not fit on this card
                torch.cuda.synchronize()
                entry[mode][name] = "not run: %s" % str(e).splitlines()[0][:160]
            mod.zero_grad(set_to_none=True)
            del leaves
            torch.cuda.empty_cache()

        for mode in ("forward", "forward_backward"):
            arm(mode, "scalar_x1", base, [a.time])
            arm(mode, "uniform", base, [torch.full((n, 1), a.time, device=dev, requires_grad=True)])
            for T in (int(x) for x in a.frames.split(",")):
                ts = torch.linspace(-1.0, 1.0, T).tolist()
                arm(mode, "scalar_x%d" % T, base, ts)
                big = [x.repeat((T,) + (1,) * (x.dim() - 1)) for x in base]
                times = torch.tensor(ts, device=dev).repeat_interleave(n).reshape(-1, 1).requires_grad_(True)
                arm(mode, "rows_%d" % T, big, [times])
                del big, times
                torch.cuda.empty_cache()
        result["workloads"][wname] = entry
    print(json.dumps(result))


if __name__ == "__main__":
    main()
