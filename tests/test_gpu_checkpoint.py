"""-m gpu: saving and resuming the captured training step (TrainStep.state_dict / load_state_dict, checkpoint.py).

A run resumed from a checkpoint into a fresh step (other initial weights, its graph captured before the load) continues
bit for bit like the run that never stopped, on the fused optimizer (graphed and eager) and on DFOLD_TORCH_ADAM=1; the
optimizer state moves to torch.optim.Adam(amsgrad=True) and back; refused loads change nothing."""
import copy

import pytest
import torch

from dynamicpdb_b200 import checkpoint as C
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from dynamicpdb_b200.train_step import TrainStep
from tests.test_cpu_checkpoint import REFUSALS, dead_indices
from tests.test_gpu_simt import _adam_ref

pytestmark = pytest.mark.gpu
K_STEPS, M_STEPS, LR = 3, 2, 1e-4
PRESETS = {"tiny": (syn.PRESET_TINY, 3, 24), "A": (syn.PRESET_A, 8, 64)}
ROUTES = {"graph": (True, "0"), "eager": (False, "0"), "torch_adam": (True, "1")}       # graph, DFOLD_TORCH_ADAM


def _net(preset, seed):
    p, nf, _ = PRESETS[preset]
    torch.manual_seed(seed)
    net = FullScoreNetwork(syn.model_conf(nf, **p), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd, seed=seed + 1)
    net.load_state_dict(sd)
    return net.cuda()


def _windows(preset):
    _, nf, N = PRESETS[preset]
    return [{k: v.cuda() for k, v in syn.make_feats(nf, N, seed=30 + i).items()} for i in range(K_STEPS + M_STEPS)]


def _step(preset, seed, windows, graph):
    ts = TrainStep(_net(preset, seed), syn.surrogate_loss, windows[0], lr=LR, graph=graph, warmup=2)
    assert (ts.graph is not None) == graph, ts.graph_error
    return ts


def _run(ts, windows):
    losses = []
    for w in windows:
        ts.load(w)
        losses.append(ts().clone())
    torch.cuda.synchronize()
    return torch.stack(losses).cpu()


def _snapshot(ts):
    """Every tensor of the optimisation state, copied to the host."""
    if ts.opt is None:
        return [t.detach().cpu() for t in (ts.flat_param, ts.exp_avg, ts.exp_avg_sq, ts.max_exp_avg_sq, ts.step_count)]
    out = [p.detach().cpu() for p in ts.params]
    for p in ts.params:
        out += [v.detach().cpu() for v in ts.opt.state[p].values() if torch.is_tensor(v)]
    return out


def _assert_same(a, b, what):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.dtype == y.dtype and torch.equal(x.view(torch.int32), y.view(torch.int32)), f"{what}: tensor {i} differs"


@pytest.mark.parametrize("preset,route", [("tiny", r) for r in ROUTES] + [("A", "graph")])
def test_resume_is_bit_exact(preset, route, monkeypatch, tmp_path):
    graph, torch_adam = ROUTES[route]
    monkeypatch.setenv("DFOLD_TORCH_ADAM", torch_adam)
    windows = _windows(preset)
    ts = _step(preset, 0, windows, graph)                       # run A: k + m steps without stopping
    _run(ts, windows[:K_STEPS])
    losses_a = _run(ts, windows[K_STEPS:])
    state_a = _snapshot(ts)
    del ts
    ts = _step(preset, 0, windows, graph)                       # run B: k steps, save ...
    _run(ts, windows[:K_STEPS])
    path = str(tmp_path / "step_3.pth")
    C.save_checkpoint(path, ts, syn.model_conf(PRESETS[preset][1], **PRESETS[preset][0]), 0, K_STEPS)
    del ts
    torch.cuda.empty_cache()
    ts = _step(preset, 5, windows, graph)                       # ... and resume in a fresh step from other weights
    captured = ts.graph
    assert not torch.equal(_snapshot(ts)[0], state_a[0])
    assert C.load_checkpoint(path, ts) == (0, K_STEPS)
    losses_b = _run(ts, windows[K_STEPS:])
    assert ts.graph is captured
    assert torch.equal(losses_a, losses_b), (losses_a, losses_b)
    _assert_same(state_a, _snapshot(ts), "state after resuming")


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _torch_flat(layout, tensors):
    flat = torch.zeros(layout.numel, dtype=torch.float64, device="cuda")
    for v, t in zip((v for v in C.views(layout, flat) if v is not None), tensors):
        v.copy_(t)
    return flat


def _next_step_agrees(ts, ref, opt, window, t):
    """One eager fused step of `ts` and one torch.optim.Adam step of `opt` over `ref` from the same state, on the gradient
    the fused step computed, against float64 of the update (tests/test_gpu_simt.py _adam_ref and its bound).  torch runs
    this step with the fp32 values of lr, betas and eps that the fused kernel receives: with the Python doubles,
    1 - beta2 alone differs by 1.3e-5 relative and would swamp a per-element bound."""
    L = ts.layout
    before = [b.double() for b in (ts.flat_param, ts.exp_avg, ts.exp_avg_sq, ts.max_exp_avg_sq)]
    assert torch.equal(before[0], _torch_flat(L, [p.detach() for p in ref.parameters()]))
    ts.load(window)
    ts()
    torch.cuda.synchronize()
    grad = ts.flat_grad.clone()
    for p, g in zip(ref.parameters(), (v for v in C.views(L, grad) if v is not None)):
        p.grad = g.clone()
    opt.param_groups[0].update(lr=_f32(LR), betas=(_f32(0.9), _f32(0.999)), eps=_f32(1e-8))
    opt.step()
    refs, errs = _adam_ref(before[0], grad.double(), *before[1:], t, _f32(LR), _f32(0.9), _f32(0.999), _f32(1e-8), 1.0)
    fused = (ts.flat_param, ts.exp_avg, ts.exp_avg_sq, ts.max_exp_avg_sq)
    params = list(ref.parameters())
    torch_side = [_torch_flat(L, [p.detach() for p in params])] + [_torch_flat(L, [opt.state[p][k] for p in params])
                                                                   for k in C.MOMENTS]
    for name, f, tt, r, e in zip(("p", "m", "v", "vmax"), fused, torch_side, refs, errs):
        f = f.double()
        assert bool(((f - r).abs() <= e).all()), f"fused {name} outside the float64 bound"
        assert bool(((f - tt).abs() <= 2 * e).all()), f"fused and torch {name} differ by more than twice the bound"


def test_state_moves_to_torch_adam():
    windows = _windows("tiny")
    ts = _step("tiny", 0, windows, graph=False)
    _run(ts, windows[:K_STEPS])
    sd = ts.state_dict()
    ref = _net("tiny", 7)
    ref.load_state_dict(sd["model"], strict=True)
    opt = torch.optim.Adam(ref.parameters(), lr=LR, amsgrad=True)
    opt.load_state_dict(copy.deepcopy(sd["optimizer"]))
    _next_step_agrees(ts, ref, opt, windows[K_STEPS], K_STEPS + 1)


def test_torch_adam_checkpoint_resumes(tmp_path):
    """k steps of the reference trainer's optimizer (non-capturable, CPU step, no state for the dead parameters), written
    in du.write_checkpoint's layout under DDP's module. prefix, then loaded into a fresh step."""
    windows = _windows("tiny")
    ref = _net("tiny", 0)
    opt = torch.optim.Adam(ref.parameters(), lr=LR, amsgrad=True)
    for w in windows[:K_STEPS]:
        opt.zero_grad()
        syn.surrogate_loss(ref(dict(w))).backward()
        opt.step()
    layout = C.flat_layout(ref)
    assert sorted(set(range(len(layout.names))) - set(opt.state_dict()["state"])) == dead_indices(layout)
    path = str(tmp_path / "ref.pth")
    torch.save({"model": {"module." + k: v for k, v in ref.state_dict().items()}, "conf": None,
                "optimizer": opt.state_dict(), "epoch": 4, "step": K_STEPS}, path)
    ts = _step("tiny", 5, windows, graph=False)
    assert C.load_checkpoint(path, ts) == (4, K_STEPS)
    assert float(ts.step_count) == K_STEPS
    _next_step_agrees(ts, ref, opt, windows[K_STEPS], K_STEPS + 1)


@pytest.mark.parametrize("route", ["graph", "torch_adam"])
def test_refused_load_changes_nothing(route, monkeypatch):
    graph, torch_adam = ROUTES[route]
    monkeypatch.setenv("DFOLD_TORCH_ADAM", torch_adam)
    windows = _windows("tiny")
    ts = _step("tiny", 0, windows, graph)
    _run(ts, windows[:2])
    sd = ts.state_dict()
    before = _snapshot(ts)
    for case, (mutate, msg) in sorted(REFUSALS.items()):
        bad = copy.deepcopy(sd)
        mutate(bad)
        with pytest.raises(ValueError, match=msg):
            ts.load_state_dict(bad)
        _assert_same(before, _snapshot(ts), f"after the refused '{case}' load")
    ts.load_state_dict(sd)                                      # the unmodified dict loads and the step goes on
    _assert_same(before, _snapshot(ts), "after reloading its own state")
    assert torch.isfinite(_run(ts, windows[2:3])).all()


def test_dead_parameters_without_state_resume_like_zero_state():
    windows = _windows("tiny")
    ts = _step("tiny", 0, windows, graph=True)
    _run(ts, windows[:K_STEPS])
    full = ts.state_dict()
    del ts
    dead = dead_indices(C.flat_layout(_net("tiny", 0)))
    for i in dead:
        assert all(not full["optimizer"]["state"][i][k].any() for k in C.MOMENTS), i
    sparse = copy.deepcopy(full)
    for i in dead:
        del sparse["optimizer"]["state"][i]
    runs = []
    for sd in (full, sparse):
        ts = _step("tiny", 5, windows, graph=True)
        ts.load_state_dict(sd)
        runs.append((_run(ts, windows[K_STEPS:]), _snapshot(ts)))
        del ts
    assert torch.equal(runs[0][0], runs[1][0])
    _assert_same(runs[0][1], runs[1][1], "state after resuming without dead-parameter entries")


def test_weights_only_load_zeroes_the_optimizer():
    windows = _windows("tiny")
    ts = _step("tiny", 0, windows, graph=True)
    _run(ts, windows[:K_STEPS])
    sd = ts.state_dict()
    ts.load_state_dict({"model": {"module." + k: v for k, v in sd["model"].items()}, "optimizer": None})
    assert float(ts.step_count) == 0.0
    assert not any(bool(b.any()) for b in (ts.exp_avg, ts.exp_avg_sq, ts.max_exp_avg_sq))
    for k, v in ts.net.state_dict().items():
        assert torch.equal(v.cpu(), sd["model"][k]), k
