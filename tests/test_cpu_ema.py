"""The host side of the moving average of the weights (TrainStep(ema_decay=...), checkpoint.check_ema,
evaluator.load_weights(ema=True)): OpenFold's ``ema`` checkpoint entry validates, maps back to the flat buffer bit for bit
and loads into a network; what would resume or evaluate another average is refused before anything is written; invalid
settings raise before any device work."""
import collections
import copy
import math
import re

import pytest
import torch

from dynamicpdb_b200 import checkpoint as C
from dynamicpdb_b200.evaluator import Evaluator, load_weights
from dynamicpdb_b200.train_step import TrainStep, check_ema_decay
from dynamicpdb_b200.trainer import Trainer
from tests.test_cpu_checkpoint import GOLD, _HostStep, _net, host_state
from tests.test_cpu_trainer import _conf, _csv

DECAY = 0.999


def _with_ema(net, seed=0, decay=DECAY):
    """host_state's dict with the ``ema`` entry TrainStep.state_dict() adds, and the average's flat buffer."""
    sd, _ = host_state(net, seed=seed)
    layout = C.flat_layout(net)
    flat = torch.zeros(layout.numel)
    n = sum(s.numel() for s, o in zip(layout.shapes, layout.offsets) if o is not None)
    flat[:n] = torch.randn(n, generator=torch.Generator().manual_seed(seed + 100))
    avg = {k: v for k, v in zip(layout.names, C.views(layout, flat)) if v is not None}
    params = collections.OrderedDict((k, avg[k]) for k in sd["model"])
    sd["ema"] = collections.OrderedDict(params=params, decay=decay)
    return sd, flat


def _shapes(net):
    return {k: v.shape for k, v in net.state_dict().items()}


def test_ema_round_trips_to_the_flat_buffer():
    net = _net()
    sd, flat = _with_ema(net)
    sd = copy.deepcopy(sd)
    for prefix in ("", "module."):
        d = dict(sd, ema=dict(sd["ema"], params={prefix + k: v for k, v in sd["ema"]["params"].items()}))
        params = C.check_ema(d, _shapes(net), DECAY)
        assert torch.equal(C.model_to_flat(C.flat_layout(net), params).view(torch.int32), flat.view(torch.int32))
    assert C.check_ema({"model": sd["model"]}, _shapes(net), DECAY) is None


def _first(sd):
    return next(iter(sd["ema"]["params"]))


# (mutation of a state dict with an ema entry, text the ValueError must contain)
REFUSALS = {
    "decay": (lambda sd: sd["ema"].update(decay=0.99), r"ema decay 0\.99 differs .* TrainStep\(ema_decay=0\.99\)"),
    "decay_type": (lambda sd: sd["ema"].update(decay="0.999"), "decay must be a number"),
    "no_params": (lambda sd: sd["ema"].pop("params"), "no 'params'"),
    "not_a_dict": (lambda sd: sd.update(ema=[1, 2]), "no 'params'"),
    "unknown_key": (lambda sd: sd["ema"]["params"].update({"score_model.extra.weight": torch.zeros(2)}),
                    r"checkpoint ema does not match the network: unknown keys \[score_model.extra"),
    "missing_key": (lambda sd: sd["ema"]["params"].pop(_first(sd)), r"missing keys \[embedding_layer"),
    "wrong_shape": (lambda sd: sd["ema"]["params"].update({_first(sd): torch.zeros(3, 3)}), "checkpoint ema '.*' has shape"),
    "float64": (lambda sd: sd["ema"]["params"].update({_first(sd): sd["ema"]["params"][_first(sd)].double()}),
                "torch.float64; the average is kept in torch.float32"),
    "bfloat16": (lambda sd: sd["ema"]["params"].update({_first(sd): sd["ema"]["params"][_first(sd)].bfloat16()}),
                 "torch.bfloat16"),
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_validation_refuses(case):
    net = _net()
    sd, _ = _with_ema(net)
    C.check_ema(copy.deepcopy(sd), _shapes(net), DECAY)
    bad = copy.deepcopy(sd)
    mutate, msg = REFUSALS[case]
    mutate(bad)
    with pytest.raises(ValueError, match=msg):
        C.check_ema(bad, _shapes(net), DECAY)


def test_checkpoint_layout_adds_ema_after_the_references_keys(tmp_path):
    net = _net()
    sd, _ = _with_ema(net)
    path = str(tmp_path / "step_2.pth")
    C.save_checkpoint(path, _HostStep(sd), None, 1, 2)
    ck = torch.load(path, map_location="cpu", weights_only=False)
    assert list(ck) == GOLD["top_keys"] + ["ema"]
    assert list(ck["ema"]) == ["params", "decay"] and ck["ema"]["decay"] == DECAY
    assert [(k, tuple(v.shape), v.dtype) for k, v in ck["ema"]["params"].items()] == \
           [(k, tuple(v.shape), torch.float32) for k, v in ck["model"].items()]


def test_load_weights_ema(tmp_path):
    src = _net()
    sd, _ = _with_ema(src)
    path = str(tmp_path / "ema.pth")
    torch.save(dict(sd, ema=dict(sd["ema"], params={"module." + k: v for k, v in sd["ema"]["params"].items()})), path)
    net = _net()
    load_weights(net, path, ema=True)
    for k, v in net.state_dict().items():
        assert torch.equal(v, sd["ema"]["params"][k]), k
    load_weights(net, path)
    for k, v in net.state_dict().items():
        assert torch.equal(v, sd["model"][k]), k

    plain = str(tmp_path / "plain.pth")
    torch.save({"model": sd["model"], "conf": None}, plain)
    before = {k: v.clone() for k, v in net.state_dict().items()}
    with pytest.raises(ValueError, match=re.escape(plain) + ".*no 'ema'"):
        load_weights(net, plain, ema=True)
    assert all(torch.equal(v, before[k]) for k, v in net.state_dict().items())
    bad = str(tmp_path / "bad.pth")
    torch.save(dict(sd, ema=dict(sd["ema"], params={k: v.double() for k, v in sd["ema"]["params"].items()})), bad)
    with pytest.raises(ValueError, match="float32"):
        load_weights(net, bad, ema=True)
    assert all(torch.equal(v, before[k]) for k, v in net.state_dict().items())


@pytest.mark.parametrize("v", [0.0, 0.5, DECAY, 1.0, 1, 0])
def test_decay_in_the_unit_interval_is_accepted(v):
    assert check_ema_decay(v) == float(v) and isinstance(check_ema_decay(v), float)
    assert check_ema_decay(None) is None


BAD_DECAYS = [True, False, -0.1, 1.001, math.nan, math.inf, "0.999"]


@pytest.mark.parametrize("v", BAD_DECAYS)
def test_trainer_refuses_a_bad_decay_before_device_work(v, tmp_path):
    with pytest.raises(ValueError, match="ema_decay must be None or a number in"):
        Trainer(_conf(_csv(tmp_path / "train.csv", [64] * 3)), None, None, ema_decay=v)


@pytest.mark.parametrize("v", BAD_DECAYS)
def test_train_step_refuses_a_bad_decay_before_device_work(v):
    with pytest.raises(ValueError, match="ema_decay must be None or a number in"):
        TrainStep(_net(), None, {}, ema_decay=v)


def test_torch_adam_refuses_the_average_before_device_work(monkeypatch):
    monkeypatch.setenv("DFOLD_TORCH_ADAM", "1")
    with pytest.raises(ValueError, match="DFOLD_TORCH_ADAM=1"):
        TrainStep(_net(), None, {}, ema_decay=DECAY)


def test_evaluator_refuses_a_non_bool_ema():
    with pytest.raises(ValueError, match="ema must be True or False"):
        Evaluator({}, None, None, ema=1)
