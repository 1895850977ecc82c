"""Debug: tensor-core vs FFMA backward of the deformation network, per-parameter error table."""
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from util_scene import make_module, rel_err, rel_err_bulk  # noqa: E402

g4d = importlib.import_module("4dgaussians_b200")


def inputs(n, seed):
    from oracle.make_golden_deform import synth_inputs
    (xyz, sc, rot, op, shs), probes = synth_inputs(n, seed)
    return [t.cuda() for t in (xyz, sc, rot, op, shs)], probes


for net, n in [("small128", 700), ("dynerf", 21000), ("hypernerf", 40000)]:
    mod = make_module(net, seed=5)
    ins, probes = inputs(n, 3)
    ws = g4d._lib.Workspace.get(0)
    t = torch.tensor(0.27).repeat(n, 1).cuda()
    res = []
    for tc in (2, 0, 2):
        ws.set_option(g4d._lib.OPT_TENSOR_CORES, tc)
        mod.zero_grad(set_to_none=True)
        dev_in = [x.clone().requires_grad_(True) for x in ins]
        outs = mod(*dev_in, t)
        sum((o * p.cuda()).sum() for o, p in zip(outs, probes)).backward()
        res.append(([x.grad.clone() for x in dev_in], {k: p.grad.clone() for k, p in mod.named_parameters() if p.grad is not None}))
    ws.set_option(g4d._lib.OPT_TENSOR_CORES, 2)
    print("====", net, n)
    for nm, a, b, c in zip(("xyz", "scales", "rot", "opacity", "shs"), res[0][0], res[1][0], res[2][0]):
        print("  in  %-10s tc-vs-ffma bulk/max %.2e %.2e   tc-vs-tc %.2e" % ((nm,) + rel_err_bulk(a.cpu().numpy(), b.cpu().numpy())
                                                                              + (rel_err(a.cpu().numpy(), c.cpu().numpy()),)))
    for k in res[1][1]:
        a, b, c = res[0][1][k].cpu().numpy(), res[1][1][k].cpu().numpy(), res[2][1][k].cpu().numpy()
        eb, em = rel_err_bulk(a, b)
        i = int(np.abs(a - b).argmax())
        print("  par %-48s norm %.2e bulk %.2e max %.2e @%d (tc %.5g ffma %.5g, |ref|max %.3g)  tc-vs-tc %.2e" %
              (k[-48:], rel_err(a, b), eb, em, i, a.reshape(-1)[i], b.reshape(-1)[i], np.abs(b).max(), rel_err(a, c)))
