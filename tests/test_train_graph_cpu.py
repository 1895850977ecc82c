"""DPTrainer(cuda_graph=True), the parts that need no device: the eager / capture / replay schedule around densification,
SH-degree and stage changes, the scoped workspace routing a captured step runs under, and the refusals that come before
anything touches a GPU."""
import importlib

import pytest
import torch

td = importlib.import_module("4dgaussians_b200.train_dp")
synth = importlib.import_module("4dgaussians_b200.synth")
_lib = importlib.import_module("4dgaussians_b200._lib")
g4d = importlib.import_module("4dgaussians_b200")


def _schedule(opt, steps, rebuild_at=(), sh_raise_at=(), fine_from=None):
    """The actions of `steps` steps, with the inputs DPTrainer derives: the template (N, SH degree, stage, statistics on)
    against the previous step's, and whether a graph of it survives (a rebuild at an eager step drops it)."""
    n, sh, stage = 1000, 0, "coarse"
    last_key, graph_key, out = None, None, []
    for it in range(1, steps + 1):
        sh += it in sh_raise_at
        stage = "fine" if fine_from is not None and it >= fine_from else stage
        key = (n, sh, stage, it < opt.densify_until_iter)
        a = td.graph_action(it, opt, key != last_key, graph_key == key)
        last_key = key
        if a == "capture":
            graph_key = key
        if a == "eager" and it in rebuild_at:
            n, graph_key = n + 1, None
        out.append(a[0].upper())
    return "".join(out)


def test_graph_action_schedule_around_densify_prune_reset_sh_and_stage():
    opt = td.default_opt()
    opt.densification_interval, opt.pruning_interval, opt.opacity_reset_interval, opt.densify_until_iter = 10, 15, 25, 45
    got = _schedule(opt, 50, rebuild_at=(10, 30), sh_raise_at=(22,), fine_from=36)
    want = ("EC" + "R" * 7 +        # 1: first template (warm-up), 2: capture
            "EEC" + "RR" +          # 10: densify with a rebuild, 11: new N (warm-up), 12: recapture
            "E" + "RRRR" +          # 15: prune, nothing replaced: the graph stays
            "E" + "R" +             # 20: densify without a change
            "EC" + "R" +            # 22: SH degree raised: one eager step, one recapture
            "E" + "RRRR" +          # 25: opacity reset (in place: the graph stays)
            "EEC" + "RRR" +         # 30: rebuild again
            "EC" + "RR" +           # 36: coarse -> fine
            "E" + "RRRR" +          # 40: densify
            "EC" + "RRRR")          # 45: densify_until_iter reached: the statistics update leaves the step
    assert got == want


def test_graph_action_without_densification_only_warms_up_and_captures_once():
    opt = td.default_opt()
    opt.densify_until_iter = 0
    assert _schedule(opt, 300) == "EC" + "R" * 298
    assert td.densifies(100, td.default_opt()) and td.densifies(3000, td.default_opt())
    assert not td.densifies(15_000, td.default_opt()) and not td.densifies(101, td.default_opt())


class _FakeWorkspace(_lib.Workspace):
    def __init__(self, device):         # (no library, no device)
        self.device, self.handle, self._free_contexts, self._fixed = device, None, [], None


def test_routed_hands_out_the_fixed_contexts_in_order_and_only_inside_the_block():
    ws, ctxs = _FakeWorkspace(7), [object(), object()]
    dev = torch.device("cuda", 7)
    with _lib.routed(ws, ctxs):
        assert _lib.workspace_of(dev) is ws
        a, b = ws.acquire_context(), ws.acquire_context()
        assert (a, b) == tuple(ctxs)
        ws.release_context(a)
        assert ws._free_contexts == []                   # fixed contexts never go back to a pool
        with pytest.raises(_lib.G4DError, match="more forwards"):
            ws.acquire_context()
        with pytest.raises(_lib.G4DError, match="already active"):
            with _lib.routed(_FakeWorkspace(7), ctxs):
                pass
    assert 7 not in _lib._routed and ws._fixed is None


class _Pipe:
    convert_SHs_python = False
    compute_cov3D_python = False
    debug = False


class _DebugPipe(_Pipe):
    debug = True


class _Gloo:
    @staticmethod
    def get_backend():
        return "gloo"


def _gaussians(module=None):
    scene = synth.make_scene(64, seed=1, scale_mean=0.05)
    return td.GaussianSet(scene, module if module is not None else g4d.deform_network(synth.hidden_args("small128")),
                          device="cpu")


def test_refusals_before_anything_runs():
    with pytest.raises(ValueError, match="NCCL"):
        td.DPTrainer(_gaussians(), dist=_Gloo(), world_size=2, cuda_graph=True)
    with pytest.raises(NotImplementedError, match="g4d deformation network"):
        td.DPTrainer(_gaussians(torch.nn.Linear(3, 3)), cuda_graph=True)
    tr = td.DPTrainer(_gaussians(), cuda_graph=True)
    cam = synth.make_camera(0.0, 32, 32)
    gt = torch.zeros(3, 32, 32)
    with pytest.raises(ValueError, match="pipe.debug"):
        tr.step([cam], [gt], torch.zeros(3), _DebugPipe)
    with pytest.raises(NotImplementedError, match="PanopticSports"):
        tr.step([{"camera": None, "time": 0.0}], [gt], torch.zeros(3), _Pipe)
    assert tr.iteration == 0 and tr.captures == 0 and tr.last_action is None
    assert not td.DPTrainer(_gaussians()).cuda_graph                  # off by default
