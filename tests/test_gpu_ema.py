"""-m gpu: OpenFold's exponential moving average of the weights in the captured training step (TrainStep(ema_decay=...),
csrc/simt.cu dfold_ema_update), its checkpoint entry and evaluation on it.

OpenFold's update (ExponentialMovingAverage._update_state_dict_) is restated here as the three torch ops it runs:
``diff = stored - param; diff *= 1 - decay; stored -= diff``.

  * the kernel gives the bits of those ops on random data of mixed sign and magnitude, for decay 0.999, 0.5, 0 and 1;
  * a step with the average trains bit for bit like one without (loss, weights, all three moments, step), graphed and
    eager, with clipping, with the AlphaFold schedule and with accumulate=2, batched=True; its average equals the
    restated recurrence over the weights of the run without it after every step, and the weights handed in right after
    construction (warm-up and capture do not leak into it);
  * a run saved after 3 steps and resumed into a fresh step for 2 more equals 5 uninterrupted steps bit for bit,
    average included; the checkpoint has OpenFold's ``ema`` layout; a checkpoint without ``ema`` starts the average from
    its weights; a refused ``ema`` changes nothing;
  * Evaluator(ema=True) gives the rows of an evaluation of the averaged weights saved as the checkpoint's model."""
import copy

import numpy as np
import pytest
import torch

from dynamicpdb_b200 import checkpoint as C
from dynamicpdb_b200 import kernels as K
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.evaluator import Evaluator
from dynamicpdb_b200.input_pipeline import TrajectoryStore, WindowPrefetcher
from dynamicpdb_b200.loss import score_network_loss
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from dynamicpdb_b200.train_step import AlphaFoldSchedule, TrainStep
from tests.test_gpu_checkpoint import _assert_same
from tests.test_gpu_evaluator import DEV, NF as EVAL_NF, _conf, _Exp, _split, rows_of
from tests.test_gpu_evaluator import _net as _eval_net

pytestmark = pytest.mark.gpu
NF, N, LR, DECAY = 3, 24, 1e-4, 0.999
K_STEPS, M_STEPS = 3, 2


def _openfold_update(stored, param, decay):
    """ExponentialMovingAverage._update_state_dict_ on one tensor, in place."""
    diff = stored - param
    diff *= 1 - decay
    stored -= diff


def _bits(t):
    return t.contiguous().view(torch.int32)


def _preset_a_numel():
    with torch.device("meta"):
        net = FullScoreNetwork(syn.model_conf(64, **syn.PRESET_A), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    return C.flat_layout(net).numel


def _mixed(n, seed):
    """fp32 values of both signs over magnitudes 2^-30 .. 2^30, some exact zeros and some pairs of equal values."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, generator=g, device="cuda") * torch.exp2(torch.randint(-30, 31, (n,), generator=g, device="cuda").float())
    x[torch.rand(n, generator=g, device="cuda") < 0.01] = 0.0
    return x


@pytest.mark.parametrize("n", [4, 1028, "A"])
def test_kernel_gives_the_bits_of_openfolds_update(n):
    n = _preset_a_numel() if n == "A" else n
    assert n % 4 == 0
    param = _mixed(n, 1)
    for j, decay in enumerate((0.999, 0.5, 0.0, 1.0)):
        stored = _mixed(n, 10 + j)
        stored[::7] = param[::7]                                 # equal pairs: diff exactly 0
        stored[1::11] = param[1::11] * -1.0
        want = stored.clone()
        _openfold_update(want, param, decay)
        got = stored.clone()
        K.launch("dfold_ema_update", got, param, n, 1.0 - decay)
        torch.cuda.synchronize()
        assert torch.equal(_bits(got), _bits(want)), (n, decay, int((_bits(got) != _bits(want)).sum()))
        if decay == 1.0:                      # the same values; a -0 average of a +0 weight becomes +0, as in torch
            assert torch.equal(got, stored)


def _net(seed):
    torch.manual_seed(seed)
    net = FullScoreNetwork(syn.model_conf(NF, **syn.PRESET_TINY), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd, seed=seed + 1)
    net.load_state_dict(sd)
    return net.cuda()


def _windows(count):
    return [{k: v.cuda() for k, v in syn.make_feats(NF, N, seed=30 + i).items()} for i in range(count)]


def _step(seed, windows, **kw):
    graph = kw.setdefault("graph", True)
    ts = TrainStep(_net(seed), syn.surrogate_loss, windows[0], lr=LR, warmup=2, **kw)
    assert (ts.graph is not None) == graph, ts.graph_error
    return ts


def _state(ts):
    return [t.detach().clone() for t in (ts.flat_param, ts.exp_avg, ts.exp_avg_sq, ts.max_exp_avg_sq, ts.step_count)]


def _train(ts, windows, steps, after=None):
    """`steps` optimizer steps, each on the next ts.accumulate windows; returns the losses."""
    losses, k = [], ts.accumulate
    for s in range(steps):
        for i in range(k):
            ts.load(windows[(s * k + i) % len(windows)], slot=i)
        losses.append(ts().clone())
        if after is not None:
            after(ts)
    torch.cuda.synchronize()
    return torch.stack(losses)


CASES = {
    "graph": dict(graph=True),
    "eager": dict(graph=False),
    "clip": dict(max_grad_norm=1e-3),
    "schedule": dict(lr_schedule=AlphaFoldSchedule(base_lr=1e-5, max_lr=1e-3, warmup_no_steps=3,
                                                   start_decay_after_n_steps=4, decay_every_n_steps=1, decay_factor=0.5)),
    "batched": dict(accumulate=2, batched=True),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_average_follows_openfold_without_perturbing_training(case):
    steps = K_STEPS + M_STEPS
    windows = _windows(2 * steps)
    plain = _step(0, windows, **CASES[case])
    assert plain.ema is None
    weights = []
    losses_plain = _train(plain, windows, steps, after=lambda ts: weights.append(ts.flat_param.clone()))
    state_plain = _state(plain)
    del plain
    ts = _step(0, windows, ema_decay=DECAY, **CASES[case])
    want = ts.flat_param.clone()
    assert torch.equal(_bits(ts.ema), _bits(want)), "the average is not the weights handed in after construction"
    averages = []
    losses = _train(ts, windows, steps, after=lambda t: averages.append(t.ema.clone()))
    assert torch.equal(_bits(losses), _bits(losses_plain))
    _assert_same(state_plain, _state(ts), f"{case}: optimisation state with the average")
    for s, (w, got) in enumerate(zip(weights, averages)):
        _openfold_update(want, w, DECAY)
        assert torch.equal(_bits(got), _bits(want)), f"{case}: average after step {s + 1}"
    assert not torch.equal(want, weights[-1])                    # the average lags the weights


def test_resume_restores_the_average(tmp_path):
    windows = _windows(K_STEPS + M_STEPS)
    ts = _step(0, windows, ema_decay=DECAY)
    losses_a = _train(ts, windows, K_STEPS + M_STEPS)
    state_a, ema_a = _state(ts), ts.ema.clone()
    del ts
    ts = _step(0, windows, ema_decay=DECAY)
    _train(ts, windows, K_STEPS)
    path = str(tmp_path / "step_3.pth")
    C.save_checkpoint(path, ts, None, 0, K_STEPS)
    del ts
    ck = torch.load(path, map_location="cpu", weights_only=False)
    assert list(ck) == ["model", "conf", "optimizer", "epoch", "step", "ema"]
    assert list(ck["ema"]) == ["params", "decay"] and ck["ema"]["decay"] == DECAY
    assert list(ck["ema"]["params"]) == list(ck["model"])
    for k, v in ck["ema"]["params"].items():
        assert v.dtype == torch.float32 and v.shape == ck["model"][k].shape, k

    ts = _step(5, windows[K_STEPS:], ema_decay=DECAY)
    captured = ts.graph
    assert C.load_checkpoint(path, ts) == (0, K_STEPS)
    losses_b = _train(ts, windows[K_STEPS:], M_STEPS)
    assert ts.graph is captured
    assert torch.equal(_bits(losses_a[K_STEPS:]), _bits(losses_b))
    _assert_same(state_a, _state(ts), "state after resuming")
    assert torch.equal(_bits(ts.ema), _bits(ema_a)), "average after resuming"

    # a checkpoint without an average (a reference checkpoint, or a run without one) starts it from its weights
    del ck["ema"]
    ts.load_state_dict(ck)
    assert torch.equal(_bits(ts.ema), _bits(ts.flat_param))
    assert not torch.equal(ts.ema, ema_a)

    # a step without an average loads a checkpoint that has one, as before
    plain = _step(6, windows)
    plain.load_state_dict(torch.load(path, map_location="cpu", weights_only=False))
    assert torch.equal(_bits(plain.flat_param), _bits(ts.flat_param))


def test_refused_average_changes_nothing():
    windows = _windows(3)
    ts = _step(0, windows, ema_decay=DECAY)
    _train(ts, windows, 2)
    sd = ts.state_dict()
    before = _state(ts) + [ts.ema.clone()]
    first = next(iter(sd["ema"]["params"]))
    for mutate, msg in ((lambda d: d["ema"].update(decay=0.99), "ema decay 0.99 differs"),
                        (lambda d: d["ema"]["params"].update({first: d["ema"]["params"][first].double()}), "float32"),
                        (lambda d: d["ema"]["params"].pop(first), "missing keys")):
        bad = copy.deepcopy(sd)
        mutate(bad)
        with pytest.raises(ValueError, match=msg):
            ts.load_state_dict(bad)
        _assert_same(before, _state(ts) + [ts.ema.clone()], f"after a refused load ({msg})")


@pytest.mark.timeout(600)
def test_evaluator_runs_on_the_average(tmp_path, capsys):
    csv_path, rows = _split(tmp_path, [17, 23])
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    example, = list(WindowPrefetcher(TrajectoryStore(frame_time=EVAL_NF), rows[:1], DEV, diffuser=diffuser))
    step = TrainStep(_eval_net(seed=3), lambda out, w: score_network_loss(out, w, _Exp), example, lr=1e-3, graph=False,
                     loss_reads_window=True, ema_decay=0.5)
    for _ in range(2):
        step()
    ours = str(tmp_path / "step_2.pth")
    C.save_checkpoint(ours, step, {"model": "conf"}, 0, 2)
    ck = torch.load(ours, map_location="cpu", weights_only=False)
    assert any(not torch.equal(ck["ema"]["params"][k], v) for k, v in ck["model"].items())
    swapped = str(tmp_path / "swapped.pth")
    torch.save(dict(ck, model=ck["ema"]["params"]), swapped)
    a = rows_of(Evaluator(_conf(csv_path, ours), _eval_net(seed=1), diffuser, seed=4, ema=True).evaluate())
    b = rows_of(Evaluator(_conf(csv_path, swapped), _eval_net(seed=2), diffuser, seed=4).evaluate())
    assert np.array_equal(a, b)
    assert np.isfinite(a).all()
    capsys.readouterr()
