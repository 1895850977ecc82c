"""One timestamp from k cameras: render_cameras (deformation once, forward and backward) against k back-to-back render()
calls, both in the same process, on the same scene and cameras.

For each k: the no-grad forward, and forward + backward of one weighted-sum loss over the k images.  CUDA events around
every step, warm-up steps first, the L2 flushed (512 MiB write) between timed steps outside the event pairs, steps alternate
between the two arms and each arm gets at least --min-seconds of device time.  Before timing, the two arms' images and
gradients are compared at the same sizes (gradients to 2e-5 of their max; where the network's BF16x2 tensor-core backward
misses that, the comparison is repeated with its FP32 backward, which must meet it).  Prints one JSON line (with the GPU name, power limit and SM clocks read by
nvidia-smi --query-gpu); writes nothing else.

    python tools/multicam_bench.py [--workload C3] [--ks 1,2,4,8,20]
"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="C3")
    ap.add_argument("--ks", default="1,2,4,8,20")
    ap.add_argument("--time", type=float, default=0.4)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--min-seconds", type=float, default=0.5, help="device time per arm and mode")
    ap.add_argument("--min-steps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multicam_bench measures the GPU: no CUDA device")
    g4d = importlib.import_module("4dgaussians_b200")
    synth = importlib.import_module("4dgaussians_b200.synth")
    dev = torch.device("cuda", 0)
    w = synth.WORKLOADS[a.workload]
    scene = synth.make_scene(w["n"], seed=0, scale_mean=w["scale_mean"])
    torch.manual_seed(1234)
    mod = g4d.deform_network(synth.hidden_args(w["net"]))
    synth.perturb_deformation(mod, 0)
    mod.deformation_net.set_aabb(scene["aabb"][0].tolist(), scene["aabb"][1].tolist())
    mod = mod.to(dev)
    pc = synth.SyntheticGaussianModel(scene, mod, sh_degree=3, requires_grad=True)
    params = pc.gaussian_parameters() + list(mod.flat_parameters())
    bg = torch.tensor([float(x) for x in w["bg"]], device=dev)
    ks = [int(x) for x in a.ks.split(",")]
    cams = synth.orbit_cameras(max(ks), w["width"], w["height"], radius=w["radius"], focal=w["focal"])
    for c in cams:
        c.time = a.time
    gen = torch.Generator(device=dev).manual_seed(0)
    weights = [torch.rand(3, c.image_height, c.image_width, device=dev, generator=gen) for c in cams]
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)

    def fwd_multi(cs):
        with torch.no_grad():
            return [o["render"] for o in g4d.render_cameras(cs, pc, Pipe, bg)]

    def fwd_sep(cs):
        with torch.no_grad():
            return [g4d.render(c, pc, Pipe, bg)["render"] for c in cs]

    def train_multi(cs):
        outs = g4d.render_cameras(cs, pc, Pipe, bg)
        sum((o["render"] * wi).sum() for o, wi in zip(outs, weights)).backward()
        return outs

    def train_sep(cs):
        outs = [g4d.render(c, pc, Pipe, bg) for c in cs]
        sum((o["render"] * wi).sum() for o, wi in zip(outs, weights)).backward()
        return outs

    def zero():
        for p in params:
            p.grad = None

    n_gauss = len(pc.gaussian_parameters())

    def grads_of(fn, cs):
        zero()
        outs = fn(cs)
        torch.cuda.synchronize()
        g = [p.grad.clone() if p.grad is not None else None for p in params]
        return g, [o["viewspace_points"].grad.clone() for o in outs]

    def rel(xs, ys):
        return max(float((x - y).abs().max()) / max(1e-3, float(y.abs().max())) for x, y in zip(xs, ys))

    def compare(cs):
        """max |a - b| / max |b| of the two arms' gradients: Gaussian parameters, network parameters, viewspace points"""
        (ga, pa), (gb, pb) = grads_of(train_multi, cs), grads_of(train_sep, cs)
        assert [x is None for x in ga] == [x is None for x in gb]
        net = [(x, y) for x, y in zip(ga[n_gauss:], gb[n_gauss:]) if x is not None]
        return {"gaussians": rel(ga[:n_gauss], gb[:n_gauss]), "network": rel(*zip(*net)), "viewspace": rel(pa, pb)}

    result = {"workload": a.workload, "n": w["n"], "width": w["width"], "height": w["height"], "net": w["net"],
              "time": a.time, "unit": "ms per step (median)", "l2": "flushed between timed steps (512 MiB write)",
              "arms": "multi = render_cameras(k cameras); separate = k back-to-back render() calls", "k": {}}
    ok = True
    for k in ks:
        cs = cams[:k]
        # ---- the two arms compute the same thing at the timed size
        ia, ib = fwd_multi(cs), fwd_sep(cs)
        img_err = max(float((x - y).abs().max()) for x, y in zip(ia, ib))
        img0_equal = bool(torch.equal(ia[0], ib[0]))
        grad_err = compare(cs)
        agree = img0_equal and img_err <= 1e-6 and max(grad_err.values()) <= 2e-5
        del ia, ib
        entry = {"image_linf": img_err, "image0_bit_identical": img0_equal, "grad_rel_max": grad_err}
        if not agree and img0_equal and img_err <= 1e-6 and grad_err["viewspace"] <= 2e-5:
            # the same comparison with the network's backward in FP32 (FFMA kernels) instead of BF16x2 tensor-core operands
            # (~16 mantissa bits): one backward on the gradients summed over k cameras rounds differently from k backward
            # passes.  When the FP32 network agrees to 2e-5, the difference is that precision, not an error of the path.
            ws = g4d._lib.Workspace.get(0)
            ws.set_option(g4d._lib.OPT_TENSOR_CORES, 0)
            try:
                entry["grad_rel_max_fp32_network"] = fp32 = compare(cs)
            finally:
                ws.set_option(g4d._lib.OPT_TENSOR_CORES, 2)
            agree = max(fp32.values()) <= 2e-5
        entry["agree"] = agree
        ok = ok and agree
        zero()
        for mode, arms in (("forward", (("multi", fwd_multi), ("separate", fwd_sep))),
                           ("forward_backward", (("multi", train_multi), ("separate", train_sep)))):
            times = {name: [] for name, _ in arms}
            for _ in range(a.warmup):
                for _, fn in arms:
                    zero(); fn(cs)
            torch.cuda.synchronize()
            step = 0
            while min(sum(t) for t in times.values()) < 1e3 * a.min_seconds or step < a.min_steps:
                for name, fn in arms:
                    zero()
                    flush.fill_(step & 0xFF)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    fn(cs)
                    e1.record()
                    torch.cuda.synchronize()
                    times[name].append(e0.elapsed_time(e1))
                step += 1
            med = {name: statistics.median(t) for name, t in times.items()}
            entry[mode] = {"multi_ms": round(med["multi"], 3), "separate_ms": round(med["separate"], 3),
                           "speedup": round(med["separate"] / med["multi"], 3), "steps": step,
                           "multi_ms_range": [round(min(times["multi"]), 3), round(max(times["multi"]), 3)],
                           "separate_ms_range": [round(min(times["separate"]), 3), round(max(times["separate"]), 3)]}
        zero()
        result["k"][str(k)] = entry
    result["results_agree"] = ok
    result.update(gpu_info(0))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
