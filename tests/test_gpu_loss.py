"""-m gpu: the training-loss kernel (csrc/loss.cu, SURVEY.md §8 f3) against the fixtures generated from the unmodified
Experiment.loss_fn (tests/golden/loss.pt) and against the oracle restatement."""
import pytest
import torch

from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.loss import score_network_loss
from oracle import dfold_oracle as O
from tests.test_cpu_oracle import close, load

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _run(name, device_fn):
    feats, out, separate = syn.loss_variant(name)
    feats = {k: v.to(DEV) for k, v in feats.items()}
    leaves = {k: out[k].to(DEV).requires_grad_(True) for k in ("angles", "rot_score", "rigids")}
    model_out = dict({k: v.to(DEV) for k, v in out.items()}, **leaves)
    loss, aux = device_fn(model_out, feats, O.default_exp_conf(separate_rot_loss=separate))
    grads = torch.autograd.grad(loss, list(leaves.values()), allow_unused=True)
    return loss.detach().cpu(), {k: v.cpu() for k, v in aux.items()}, {k: (g.cpu() if g is not None else None) for k, g in zip(leaves, grads)}


@pytest.mark.parametrize("name", list(syn.LOSS_VARIANTS))
def test_loss_kernel_matches_reference_golden(name):
    gold = load("loss")[name]
    loss, aux, grads = _run(name, score_network_loss)
    assert loss.dtype == gold["loss"].dtype == torch.float64
    assert close(loss, gold["loss"], 1e-6)
    assert set(aux) == set(gold["aux"])
    for k in aux:
        assert aux[k].shape == gold["aux"][k].shape and aux[k].dtype == gold["aux"][k].dtype, k
        assert close(aux[k], gold["aux"][k], 1e-6), k
    for k, g in grads.items():
        ref = gold["grads"][k]
        ref = torch.zeros_like(g) if ref is None else ref
        assert g.dtype == ref.dtype and close(g, ref, 1e-6), k


def test_loss_kernel_is_capturable_and_refuses_cpu():
    """No host synchronisation (t and the score scaling are read on the device): the loss can sit inside a CUDA graph."""
    feats, out, _ = syn.loss_variant("plain")
    with pytest.raises(RuntimeError):
        score_network_loss(out, feats, O.default_exp_conf())
    feats = {k: v.to(DEV) for k, v in feats.items()}
    out = {k: v.to(DEV) for k, v in out.items()}
    score_network_loss(out, feats, O.default_exp_conf())              # warm-up (library load, allocator)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    static = {}
    with torch.cuda.graph(g):
        static["loss"], _ = score_network_loss(out, feats, O.default_exp_conf())
    feats["t"].fill_(0.1)                                             # replays see the new t: the gate is evaluated on the device
    g.replay()
    torch.cuda.synchronize()
    assert close(static["loss"].cpu(), load("loss")["t_low"]["loss"], 1e-6)
