"""No-grad rendering of 32 views at 32 timestamps, three ways in one process: eager render() in exact sync mode (the default),
eager render() in no-sync mode, and replays of a CUDA graph (graphs.GraphedRender).

One step renders the 32 views one after the other and ends in a device synchronise; its time is the host clock around it
(what a caller waits for: enqueue work and host syncs included) and CUDA events around it (device time).  Warm-up steps
first; the arms alternate step by step.  Before timing, every view's image, depth and radii of each eager arm are compared
with the graphed arm's, byte for byte.  Prints one JSON line (with the GPU name and power limit read by nvidia-smi
--query-gpu); writes nothing else.

    python tools/graph_bench.py [--workloads C1,C3] [--views 32] [--rounds 20]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="C1,C3")
    ap.add_argument("--views", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("graph_bench measures the GPU: no CUDA device")
    g4d = importlib.import_module("4dgaussians_b200")
    synth = importlib.import_module("4dgaussians_b200.synth")
    graphs = importlib.import_module("4dgaussians_b200.graphs")
    _lib = g4d._lib
    dev = torch.device("cuda", 0)
    ws = _lib.Workspace.get(0)
    result = {"views": a.views, "rounds": a.rounds, "unit": "ms per step of all views (median)",
              "arms": "exact = eager render(), G4D_OPT_SYNC_MODE 1; nosync = eager render(), mode 0; graphed = GraphedRender replays",
              "workloads": {}}
    for wl in a.workloads.split(","):
        w = synth.WORKLOADS[wl]
        scene = synth.make_scene(w["n"], seed=0, scale_mean=w["scale_mean"])
        torch.manual_seed(1234)
        mod = g4d.deform_network(synth.hidden_args(w["net"]))
        synth.perturb_deformation(mod, 0)
        mod.deformation_net.set_aabb(scene["aabb"][0].tolist(), scene["aabb"][1].tolist())
        mod = mod.to(dev)
        pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3)
        bg = torch.tensor([float(x) for x in w["bg"]], device=dev)
        cams = synth.orbit_cameras(a.views, w["width"], w["height"], radius=w["radius"], focal=w["focal"])
        for i, c in enumerate(cams):
            c.time = i / max(1, a.views - 1)
        with torch.no_grad():
            graphed = graphs.GraphedRender(pc, Pipe, bg, cams[0])

            def eager(sync):
                def run():
                    ws.set_option(_lib.OPT_SYNC_MODE, sync)
                    return [g4d.render(c, pc, Pipe, bg) for c in cams]
                return run

            def replay():
                return [graphed(c) for c in cams]

            arms = {"exact": eager(1), "nosync": eager(0), "graphed": replay}
            # ---- the same bytes: every view of each eager arm against the graphed replay of that view
            identical = {}
            for name in ("exact", "nosync"):
                ref = arms[name]()
                same = True
                for c, r in zip(cams, ref):
                    g = graphed(c)
                    same = same and all(torch.equal(g[k], r[k]) for k in ("render", "depth", "radii"))
                identical[name] = bool(same)
                del ref
            graphed.check()
            for _ in range(a.warmup):
                for fn in arms.values():
                    fn()
            torch.cuda.synchronize()
            wall = {k: [] for k in arms}
            devt = {k: [] for k in arms}
            for _ in range(a.rounds):
                for name, fn in arms.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    e0.record()
                    fn()
                    e1.record()
                    torch.cuda.synchronize()
                    wall[name].append(1e3 * (time.perf_counter() - t0))
                    devt[name].append(e0.elapsed_time(e1))
            graphed.check()
            ws.set_option(_lib.OPT_SYNC_MODE, 1)
        entry = {"n": w["n"], "width": w["width"], "height": w["height"], "net": w["net"],
                 "byte_identical_to_graphed": identical}
        for name in arms:
            entry[name] = {"wall_ms": round(statistics.median(wall[name]), 3),
                           "wall_ms_range": [round(min(wall[name]), 3), round(max(wall[name]), 3)],
                           "device_ms": round(statistics.median(devt[name]), 3),
                           "device_ms_range": [round(min(devt[name]), 3), round(max(devt[name]), 3)]}
        entry["speedup_wall_vs_exact"] = round(entry["exact"]["wall_ms"] / entry["graphed"]["wall_ms"], 3)
        entry["speedup_wall_vs_nosync"] = round(entry["nosync"]["wall_ms"] / entry["graphed"]["wall_ms"], 3)
        result["workloads"][wl] = entry
        del graphed, pc, mod
        torch.cuda.empty_cache()
    result.update(gpu_info(0))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
