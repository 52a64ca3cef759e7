"""The checkpoint format of the captured training step (dynamicpdb_b200/checkpoint.py) on the host: the dict built from
flat buffers has the structure of a checkpoint the reference trainer writes (tests/golden/checkpoint_layout.pt), maps
back to the same flat buffers bit for bit, loads into the network and into torch.optim.Adam, and the validation refuses
what would resume a different optimisation.  The save is atomic."""
import copy
import os

import pytest
import torch

from dynamicpdb_b200 import checkpoint as C
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser

GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "checkpoint_layout.pt"))
LR = GOLD["lr"]


def _net():
    torch.manual_seed(0)
    return FullScoreNetwork(syn.model_conf(3, **syn.PRESET_TINY), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))


def dead_indices(layout):
    """Parameters that never receive a gradient: the output-less embedder and linear_rbf."""
    return [i for i, n in enumerate(layout.names) if n.startswith("embedding_layer.") or "linear_rbf" in n]


def _flats(layout, seed=0):
    """Random host flat buffers (parameters, exp_avg, exp_avg_sq, max_exp_avg_sq) with zero padding."""
    g = torch.Generator().manual_seed(seed)
    n = sum(s.numel() for s, o in zip(layout.shapes, layout.offsets) if o is not None)
    out = []
    for k in range(4):
        f = torch.zeros(layout.numel)
        r = torch.randn(n, generator=g)
        f[:n] = r if k < 2 else r * r * (1 + k)
        out.append(f)
    return out


def host_state(net, lr=LR, indices=None, step=7.0, seed=0):
    """What TrainStep.state_dict() returns, built from host flat buffers."""
    layout = C.flat_layout(net)
    flat = _flats(layout, seed)
    trained = {n: v for n, v in zip(layout.names, C.views(layout, flat[0])) if v is not None}
    model = {k: trained.get(k, v.detach()) for k, v in net.state_dict().items()}
    return {"model": model, "optimizer": C.optimizer_state_dict(layout, *flat[1:], step, lr, indices)}, flat


class _HostStep:
    def __init__(self, sd):
        self.sd = sd

    def state_dict(self):
        return self.sd


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_layout_matches_reference_checkpoint(tmp_path):
    net = _net()
    layout = C.flat_layout(net)
    dead = dead_indices(layout)
    sd, _ = host_state(net, indices=[i for i in range(len(layout.names)) if i not in dead])
    path = str(tmp_path / "step_2.pth")
    C.save_checkpoint(path, _HostStep(sd), {"model": "conf"}, 1, 2)
    ck = torch.load(path, map_location="cpu", weights_only=False)
    assert list(ck) == GOLD["top_keys"]
    assert [(k, tuple(v.shape)) for k, v in ck["model"].items()] == list(GOLD["model"].items())
    opt = ck["optimizer"]
    assert list(opt) == GOLD["state_keys"]
    assert [{k: (list(v) if k == "params" else v) for k, v in g.items()} for g in opt["param_groups"]] == GOLD["param_groups"]
    desc = lambda t: (str(t.dtype), str(t.device), tuple(t.shape))
    got = {i: {k: desc(v) for k, v in st.items()} for i, st in opt["state"].items()}
    assert list(got) == list(GOLD["state"]) and got == GOLD["state"]
    for i in got:
        assert list(got[i]) == list(GOLD["state"][i]), i
    assert [i for i in range(len(layout.names)) if i not in opt["state"]] == GOLD["missing"] == dead
    assert ck["epoch"] == 1 and ck["step"] == 2


@pytest.mark.parametrize("frozen", [False, True])
def test_flat_dict_flat_round_trip(frozen):
    net = _net()
    if frozen:                                         # parameters the step does not train sit outside the flat buffers
        for name, p in net.named_parameters():
            if "ipa_1." in name:
                p.requires_grad_(False)
    layout = C.flat_layout(net)
    assert any(o is None for o in layout.offsets) == frozen and layout.numel % 4 == 0
    sd, flat = host_state(net, step=5.0)
    sd = copy.deepcopy(sd)                             # no longer views of the source buffers
    model, entries, step = C.check_state(sd, layout, {k: v.shape for k, v in net.state_dict().items()}, LR)
    assert step == 5.0 and len(entries) == sum(o is not None for o in layout.offsets)
    for a, b in zip([C.model_to_flat(layout, model)] + C.optimizer_to_flat(layout, entries), flat):
        assert _bits_equal(a, b)


def test_model_loads_into_network_strict():
    sd, _ = host_state(_net(), seed=3)
    for prefix in ("", "module."):
        model = {prefix + k: v for k, v in sd["model"].items()}
        net = _net()
        net.load_state_dict(C.strip_module_prefix(model), strict=True)
        for k, v in net.state_dict().items():
            assert torch.equal(v, sd["model"][k]), k


def test_torch_adam_state_dict_loads():
    """A non-capturable torch.optim.Adam(amsgrad=True) over the network, stepped with gradients on all but the dead
    parameters (which then have no state entry), validates and maps to the moments torch holds; dead ones get zeros."""
    net = _net()
    layout = C.flat_layout(net)
    dead = set(dead_indices(layout))
    opt = torch.optim.Adam(net.parameters(), lr=LR, amsgrad=True)
    g = torch.Generator().manual_seed(4)
    for _ in range(3):
        for i, p in enumerate(net.parameters()):
            p.grad = None if i in dead else torch.randn(p.shape, generator=g)
        opt.step()
    sd = {"model": {"module." + k: v for k, v in net.state_dict().items()}, "conf": None,
          "optimizer": copy.deepcopy(opt.state_dict()), "epoch": 0, "step": 3}
    model, entries, step = C.check_state(sd, layout, {k: v.shape for k, v in net.state_dict().items()}, LR)
    assert step == 3.0 and set(entries) == set(range(len(layout.names))) - dead
    flats = C.optimizer_to_flat(layout, entries)
    for k, flat in zip(C.MOMENTS, flats):
        for i, (p, v) in enumerate(zip(net.parameters(), C.views(layout, flat))):
            want = torch.zeros_like(p) if i in dead else opt.state[p][k]
            assert torch.equal(v, want), (k, layout.names[i])
    assert _bits_equal(C.model_to_flat(layout, model), torch.cat([torch.cat([p.detach().reshape(-1) for p in net.parameters()]),
                                                                   torch.zeros(layout.numel - sum(p.numel() for p in net.parameters()))]))


def test_weights_only_checkpoint():
    net = _net()
    layout = C.flat_layout(net)
    sd, _ = host_state(net)
    for opt in ("none", "absent"):
        d = dict(sd, optimizer=None) if opt == "none" else {"model": sd["model"]}
        model, entries, step = C.check_state(d, layout, {k: v.shape for k, v in net.state_dict().items()}, LR)
        assert entries is None and step == 0.0
        assert all(not f.any() for f in C.optimizer_to_flat(layout, entries))


def _group(sd):
    return sd["optimizer"]["param_groups"][0]


def _first_key(sd):
    return next(iter(sd["model"]))


def _set(d, k, v):
    d[k] = v


# (mutation of a state dict, text the ValueError must contain); tests/test_gpu_checkpoint.py loads the same cases
REFUSALS = {
    "lr": (lambda sd: _set(_group(sd), "lr", _group(sd)["lr"] * 2), r"TrainStep\(lr="),
    "amsgrad": (lambda sd: _set(_group(sd), "amsgrad", False), "amsgrad"),
    "weight_decay": (lambda sd: _set(_group(sd), "weight_decay", 1e-3), "weight_decay"),
    "betas": (lambda sd: _set(_group(sd), "betas", (0.9, 0.99)), "betas"),
    "eps": (lambda sd: _set(_group(sd), "eps", 1e-6), "eps"),
    "maximize": (lambda sd: _set(_group(sd), "maximize", True), "maximize"),
    "two_groups": (lambda sd: _set(sd["optimizer"], "param_groups",
                                   [dict(_group(sd), params=_group(sd)["params"][:70]),
                                    dict(_group(sd), params=_group(sd)["params"][70:])]), "2 param groups"),
    "unequal_steps": (lambda sd: _set(sd["optimizer"]["state"][20], "step", sd["optimizer"]["state"][20]["step"] + 1),
                      "different step counts"),
    "unknown_key": (lambda sd: _set(sd["model"], "score_model.extra.weight", torch.zeros(2)), r"unknown keys \[score_model.extra"),
    "missing_key": (lambda sd: sd["model"].pop(_first_key(sd)), r"missing keys \[embedding_layer"),
    "wrong_shape": (lambda sd: _set(sd["model"], _first_key(sd), torch.zeros(3, 3)), "has shape"),
    "moment_shape": (lambda sd: _set(sd["optimizer"]["state"][20], "exp_avg", torch.zeros(5)), "'exp_avg' of"),
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_validation_refuses(case):
    net = _net()
    layout = C.flat_layout(net)
    sd, _ = host_state(net)
    C.check_state(copy.deepcopy(sd), layout, {k: v.shape for k, v in net.state_dict().items()}, LR)
    bad = copy.deepcopy(sd)
    mutate, msg = REFUSALS[case]
    mutate(bad)
    with pytest.raises(ValueError, match=msg):
        C.check_state(bad, layout, {k: v.shape for k, v in net.state_dict().items()}, LR)


def test_refuses_state_for_untrained_parameter():
    net = _net()
    sd, _ = host_state(net)
    next(net.parameters()).requires_grad_(False)
    with pytest.raises(ValueError, match="does not train"):
        C.check_state(sd, C.flat_layout(net), {k: v.shape for k, v in net.state_dict().items()}, LR)


def test_save_is_atomic(tmp_path, monkeypatch):
    net = _net()
    path = str(tmp_path / "ckpt.pth")
    C.save_checkpoint(path, _HostStep(host_state(net, seed=1)[0]), None, 0, 10)
    before = open(path, "rb").read()
    real_save = torch.save

    def failing_save(obj, f, **kw):
        f.write(before[: len(before) // 3])            # part of a file, then the process is interrupted
        raise KeyboardInterrupt

    monkeypatch.setattr(torch, "save", failing_save)
    with pytest.raises(KeyboardInterrupt):
        C.save_checkpoint(path, _HostStep(host_state(net, seed=2)[0]), None, 0, 20)
    assert open(path, "rb").read() == before
    assert os.listdir(tmp_path) == ["ckpt.pth"]
    monkeypatch.setattr(torch, "save", real_save)
    C.save_checkpoint(path, _HostStep(host_state(net, seed=2)[0]), None, 0, 20)
    assert torch.load(path, weights_only=False)["step"] == 20 and os.listdir(tmp_path) == ["ckpt.pth"]
