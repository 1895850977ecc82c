"""Kernel time of the HexPlane gather (deform_features_kernel) and of the tensor-core MLP that follows it (deform_tc_kernel),
with the Gaussians visited in index order (G4D_OPT_GATHER_ORDER = 0) and in the spatial walk order (1), in one process on one
scene.

No-grad fused forwards of the workload, back to back as bench.py renders them (a view moves more than the L2 holds, so
consecutive views evict one another).  Rounds alternate between the two orders; every round is one torch.profiler run with
CUDA activities over --views views after a warm-up view, and the kernel times are read from the profile.  The
rebuild of the order (order_*_kernel) happens on the first spatial view only, outside the profiled views.  The two orders'
images must be bit-identical.  Prints one JSON line (with the GPU name, power limit and SM clocks read by
nvidia-smi --query-gpu); writes nothing else.

    python tools/gather_order_bench.py [--workload C3] [--views 32] [--rounds 3]
"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KERNELS = {"gather": "deform_features_kernel", "mlp": "deform_tc_kernel"}


class Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


def gpu_info(index=0):
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, sm, smax = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit_w": float(plim), "sm_clock_mhz": float(sm), "sm_max_clock_mhz": float(smax)}
    except Exception as e:      # the numbers still stand; say why the card's settings are missing
        return {"gpu": torch.cuda.get_device_name(index), "nvidia_smi": "unavailable: %s" % e}


def kernel_us(prof, views):
    """mean device time per view (us) of every kernel whose name contains one of KERNELS' values"""
    tot = {k: 0.0 for k in KERNELS}
    for e in prof.key_averages():
        t = getattr(e, "self_device_time_total", None)
        if t is None:
            t = e.self_cuda_time_total
        for k, pat in KERNELS.items():
            if pat in e.key:
                tot[k] += t
    return {k: v / views for k, v in tot.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="C3")
    ap.add_argument("--views", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gather_order_bench measures the GPU: no CUDA device")
    g4d = importlib.import_module("4dgaussians_b200")
    lib = importlib.import_module("4dgaussians_b200._lib")
    synth = importlib.import_module("4dgaussians_b200.synth")
    dev = torch.device("cuda", 0)
    w = synth.WORKLOADS[a.workload]
    scene = synth.make_scene(w["n"], seed=0, scale_mean=w["scale_mean"])
    torch.manual_seed(1234)
    mod = g4d.deform_network(synth.hidden_args(w["net"]))
    synth.perturb_deformation(mod, 0)
    mod.deformation_net.set_aabb(scene["aabb"][0].tolist(), scene["aabb"][1].tolist())
    mod = mod.to(dev)
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3)
    bg = torch.tensor([float(x) for x in w["bg"]], device=dev)
    cams = synth.orbit_cameras(a.views, w["width"], w["height"], radius=w["radius"], focal=w["focal"], timestamps=300)
    ws = lib.Workspace.get(0)

    def views():
        with torch.no_grad():
            return [g4d.render(c, pc, Pipe, bg)["render"] for c in cams]

    images, per = {}, {0: [], 1: []}
    try:
        for r in range(a.rounds):
            for order in (0, 1):
                ws.set_option(lib.OPT_GATHER_ORDER, order)
                with torch.no_grad():
                    g4d.render(cams[0], pc, Pipe, bg)
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    imgs = views()
                    torch.cuda.synchronize()
                per[order].append(kernel_us(prof, len(cams)))
                if r == 0:
                    images[order] = imgs
    finally:
        ws.set_option(lib.OPT_GATHER_ORDER, 1)
    identical = all(torch.equal(x, y) for x, y in zip(images[0], images[1]))
    res = {"workload": a.workload, "n": w["n"], "width": w["width"], "height": w["height"], "net": w["net"],
           "unit": "us per view (device time from torch.profiler, median over rounds)", "views_per_round": len(cams),
           "rounds": a.rounds, "images_bit_identical": identical}
    for order, name in ((0, "index"), (1, "spatial")):
        res[name] = {k: round(statistics.median(p[k] for p in per[order]), 2) for k in KERNELS}
        res[name + "_range"] = {k: [round(min(p[k] for p in per[order]), 2), round(max(p[k] for p in per[order]), 2)]
                                for k in KERNELS}
    C, L = mod.args.kplanes_config["output_coordinate_dim"], len(mod.args.multires)
    # loads of the gather: per level 3 spatial planes x 4 taps + 3 collapsed time rows x 2 taps, C fp32 channels each
    res["gather_load_bytes_per_view"] = w["n"] * L * (3 * 4 + 3 * 2) * C * 4
    res["gather_speedup"] = round(res["index"]["gather"] / res["spatial"]["gather"], 3) if res["spatial"]["gather"] else None
    res.update(gpu_info(0))
    print(json.dumps(res))
    if not identical:
        raise SystemExit("the two orders rendered different images")


if __name__ == "__main__":
    main()
