"""The AlphaFold learning-rate schedule of the captured training step on the host: the float64 restatement
(oracle/lr_schedule_oracle.py) and the package's own (train_step.AlphaFoldSchedule.lr) equal the reference's
AlphaFoldLRScheduler bit for bit (tests/golden/lr_schedule.pt); settings on which the reference fails or means nothing are
refused; TrainStep refuses a bad schedule or window count before it touches a device; and a checkpoint is accepted under a
schedule exactly when its lr is the schedule's lr at its step."""
import copy
import math
import os

import pytest
import torch

from dynamicpdb_b200 import checkpoint as C
from dynamicpdb_b200.train_step import AlphaFoldSchedule, TrainStep
from oracle.lr_schedule_oracle import alphafold_lr
from tests.test_cpu_checkpoint import _net, host_state

GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lr_schedule.pt"))


def _bits(x: float) -> int:
    return torch.tensor(x, dtype=torch.float64).view(torch.int64).item()


@pytest.mark.parametrize("setting", sorted(GOLD["settings"]))
def test_restatements_equal_the_reference(setting):
    g = GOLD["settings"][setting]
    sched = AlphaFoldSchedule(**g["kwargs"])
    for s, want in zip(g["steps"], g["lr"]):
        assert _bits(alphafold_lr(s, **g["kwargs"])) == _bits(want), (setting, s)
        assert _bits(sched.lr(s)) == _bits(want), (setting, s)


def test_fixture_covers_every_phase_and_boundary():
    af = GOLD["settings"]["alphafold"]
    w, s, e = (af["kwargs"][k] for k in ("warmup_no_steps", "start_decay_after_n_steps", "decay_every_n_steps"))
    assert {0, w, w + 1, s, s + 1, s + e - 1, s + e, 10 ** 6} <= set(af["steps"])
    assert {st["kwargs"]["decay_factor"] for st in GOLD["settings"].values()} >= {0.95, 1.0, 0.5}


@pytest.mark.parametrize("kw,needle", [
    (dict(warmup_no_steps=0), "warmup_no_steps must be positive"),
    (dict(decay_every_n_steps=0), "decay_every_n_steps must be positive"),
    (dict(decay_every_n_steps=-3), "decay_every_n_steps"),
    (dict(warmup_no_steps=11, start_decay_after_n_steps=10), "must not exceed"),
    (dict(warmup_no_steps=-1), "warmup_no_steps"),
    (dict(start_decay_after_n_steps=-1), "start_decay_after_n_steps"),
    (dict(max_lr=0.0), "max_lr must be positive"),
    (dict(max_lr=-1e-3), "max_lr must be positive"),
    (dict(max_lr=math.inf), "max_lr"),
    (dict(max_lr=math.nan), "max_lr"),
    (dict(base_lr=math.nan), "base_lr"),
    (dict(decay_factor=math.inf), "decay_factor"),
    (dict(warmup_no_steps=2.5), "warmup_no_steps"),
    (dict(decay_every_n_steps=True), "decay_every_n_steps"),
    (dict(max_lr="1e-3"), "max_lr"),
])
def test_bad_schedules_are_refused(kw, needle):
    with pytest.raises(ValueError, match=needle):
        AlphaFoldSchedule(**kw)


def test_good_schedules():
    s = AlphaFoldSchedule(base_lr=0, max_lr=1, warmup_no_steps=3, start_decay_after_n_steps=3, decay_every_n_steps=1)
    assert isinstance(s.base_lr, float) and isinstance(s.max_lr, float)
    assert [s.lr(k) for k in range(6)] == [0.0, 1 / 3, 2 / 3, 1.0, 0.95 ** 2, 0.95 ** 3]     # (k - 3) // 1 + 1 factors


def _make(**kw):
    return TrainStep(torch.nn.Linear(4, 4), lambda out: out, {}, **kw)


@pytest.mark.parametrize("kw,needle", [
    (dict(lr_schedule={"max_lr": 1e-3}), "AlphaFoldSchedule"),
    (dict(accumulate=0), "accumulate"),
    (dict(accumulate=-2), "accumulate"),
    (dict(accumulate=2.0), "accumulate"),
    (dict(accumulate=True), "accumulate"),
])
def test_train_step_refuses_before_device_work(kw, needle):
    with pytest.raises(ValueError, match=needle):
        _make(**kw)


def test_mid_warmup_param_groups_match_the_reference():
    """TrainStep.state_dict()'s param_groups under a schedule (checkpoint.optimizer_state_dict with the schedule's lr at
    the step and initial_lr) equal what Adam + the reference's scheduler hold at the same step."""
    mid = GOLD["mid_warmup"]
    g = GOLD["settings"][mid["setting"]]
    layout = C.FlatLayout(["p"], [torch.Size([4])], [0], 4)
    z = torch.zeros(4)
    sd = C.optimizer_state_dict(layout, z, z, z, float(mid["step"]), AlphaFoldSchedule(**g["kwargs"]).lr(mid["step"]),
                                initial_lr=GOLD["adam_lr"])
    assert sd["param_groups"] == mid["param_groups"]


def _scheduled_state(net, sched, step, initial_lr=1e-4):
    sd, _ = host_state(net, lr=sched.lr(int(step)), step=step)
    sd["optimizer"]["param_groups"][0]["initial_lr"] = initial_lr
    return sd


def _check(net, sd, lr=1e-4, schedule=None):
    return C.check_state(sd, C.flat_layout(net), {k: v.shape for k, v in net.state_dict().items()}, lr, schedule)


def test_checkpoint_lr_follows_the_schedule():
    net = _net()
    sched = AlphaFoldSchedule(max_lr=1e-3, warmup_no_steps=4, start_decay_after_n_steps=7, decay_every_n_steps=2)
    for step in (0.0, 2.0, 4.0, 7.0, 8.0, 9.0, 30.0):
        sd = _scheduled_state(net, sched, step)
        _, entries, got = _check(net, sd, schedule=sched)
        assert got == step and entries
        del sd["optimizer"]["param_groups"][0]["initial_lr"]          # initial_lr is allowed, not required
        _check(net, sd, schedule=sched)
    sd = _scheduled_state(net, sched, 2.0)
    other = AlphaFoldSchedule(max_lr=1e-3, warmup_no_steps=5, start_decay_after_n_steps=7, decay_every_n_steps=2)
    with pytest.raises(ValueError, match="different schedule"):
        _check(net, sd, schedule=other)
    with pytest.raises(ValueError, match="lr"):                     # and without a schedule, today's rule
        _check(net, sd, lr=1e-4)
    plain, _ = host_state(net, lr=1e-4, step=2.0)
    with pytest.raises(ValueError, match="different schedule"):     # a run without a schedule
        _check(net, plain, schedule=sched)
    fractional = copy.deepcopy(sd)
    for st in fractional["optimizer"]["state"].values():
        st["step"] = torch.tensor(2.5)
    with pytest.raises(ValueError, match="whole number"):
        _check(net, fractional, schedule=sched)
    _, entries, step = _check(net, {"model": sd["model"], "optimizer": None}, schedule=sched)   # weights only
    assert entries is None and step == 0.0
