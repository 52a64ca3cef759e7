"""-m gpu: the CUDA-graph training step (dynamicpdb_b200/train_step.py) replays to the same parameters as eager
stepping, leaves gradient-free parameters untouched, and the long-chain configuration (N_res=1024) runs."""
import copy

import pytest
import torch

from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from dynamicpdb_b200.train_step import TrainStep

pytestmark = pytest.mark.gpu


def _net(nf, preset):
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(nf, **preset), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    return net.cuda()


def test_graph_replay_matches_eager_steps(monkeypatch):
    nf, N = 3, 24
    feats = {k: v.cuda() for k, v in syn.make_feats(nf, N, seed=4).items()}
    base = _net(nf, syn.PRESET_TINY)
    runs = {}
    for graph in (True, False):
        net = copy.deepcopy(base)
        ts = TrainStep(net, syn.surrogate_loss, feats, lr=1e-3, graph=graph, warmup=2)
        assert (ts.graph is not None) == graph, ts.graph_error
        losses, grads = [], []
        for _ in range(3):
            losses.append(float(ts()))
            grads.append(ts.flat_grad.clone())
        runs[graph] = (losses, {k: v.detach().clone() for k, v in net.state_dict().items()}, grads)
    for a, b in zip(runs[True][0], runs[False][0]):
        assert abs(a - b) < 1e-4 * max(1.0, abs(b)), (runs[True][0], runs[False][0])
    # gradients of every step agree (parameters themselves are not compared element-wise: Adam turns the noise-level
    # gradients of mathematically gradient-free parameters, e.g. linear_b.bias, into +-lr moves of arbitrary sign)
    for ga, gb in zip(runs[True][2], runs[False][2]):
        assert ((ga - gb).norm() / gb.norm()).item() < 5e-3
    # parameters that receive no gradient (dead-output embedder, linear_rbf) are not moved by Adam
    for k, v in base.state_dict().items():
        if k.startswith("embedding_layer.") or "linear_rbf" in k:
            assert torch.equal(runs[True][1][k], v), k
    assert runs[True][0][-1] < runs[True][0][0]            # the loss goes down


def test_training_steps_are_reproducible():
    """Two runs of the same captured training steps from the same weights and inputs give bit-identical losses, gradients
    and parameters.  Preset A at 8 frames has the small, long-K launches (the last layers of the dead-frame pyramid, the
    IPA dV over frames) and the bias-gradient / d(gamma) reductions that an order-dependent (atomic) reduction would
    make differ; Adam would amplify such differences of noise-level gradients to +-lr moves."""
    nf, N = 8, 64
    feats = {k: v.cuda() for k, v in syn.make_feats(nf, N, seed=3).items()}
    runs = []
    for _ in range(2):
        net = _net(nf, syn.PRESET_A)
        ts = TrainStep(net, syn.surrogate_loss, feats, lr=1e-4, graph=True, warmup=2)
        losses = [ts().clone() for _ in range(3)]
        torch.cuda.synchronize()
        runs.append((torch.stack(losses).cpu(), ts.flat_grad.cpu(), ts.flat_param.cpu()))
        del net, ts
        torch.cuda.empty_cache()
    for a, b, what in zip(runs[0], runs[1], ("loss", "gradients", "parameters")):
        assert torch.equal(a, b), f"{what} differ between two identical runs: max |diff| {(a - b).abs().max().item():.3e}"


def test_long_chain_1024_residues_forward_backward():
    """BASELINE.json configs[4]: N_res=1024, 8 frames — the O(N^2) attention rows (131 KB of shared memory per CTA)."""
    nf, N = 8, 1024
    net = _net(nf, syn.PRESET_A)
    feats = {k: v.cuda() for k, v in syn.make_feats(nf, N, seed=1).items()}
    out = net(feats)
    loss = syn.surrogate_loss(out)
    loss.backward()
    torch.cuda.synchronize()
    assert torch.isfinite(loss)
    assert out["rigids"].shape == (nf, N, 7) and out["atom37"].shape == (nf, N, 37, 3)
    g = net.score_model.trunk["ipa_0"].linear_q.weight.grad
    assert g is not None and torch.isfinite(g).all() and float(g.abs().max()) > 0


def test_fused_adam_matches_torch_adam_amsgrad():
    """csrc/simt.cu adam_amsgrad_kernel == torch.optim.Adam(amsgrad=True) (the reference trainer's optimizer,
    train_DFOLD_dynamics.py:412) over several steps, including zero gradients (parameters stay put)."""
    from dynamicpdb_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(0)
    n = 4096 + 8
    p0 = torch.randn(n, device="cuda", generator=g)
    ref = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=1e-3, amsgrad=True)
    p = p0.clone()
    m, v, vm = torch.zeros_like(p), torch.zeros_like(p), torch.zeros_like(p)
    step = torch.zeros((), device="cuda")
    for it in range(6):
        grad = torch.randn(n, device="cuda", generator=g) * (10.0 ** (it - 3))
        grad[:100] = 0
        ref.grad = grad.clone()
        opt.step()
        K._check(K.lib().dfold_adam_amsgrad(K._ptr(p), K._ptr(grad), K._ptr(m), K._ptr(v), K._ptr(vm), n, K._ptr(step), 1,
                                            1e-3, 0.9, 0.999, 1e-8, 1.0, K._stream()), "dfold_adam_amsgrad")
        assert (p - ref.detach()).abs().max().item() < 2e-6 * max(1.0, ref.abs().max().item()), it
    assert torch.equal(p[:100], p0[:100]) and float(step) == 6.0


def test_train_step_gradients_equal_plain_autograd(monkeypatch):
    """The step accumulates the shared ConvNet's weight gradients in place (kernels.GRAD_ACCUMULATE_INPLACE) and updates flat
    parameter views: its gradient buffer must equal what loss.backward() gives on an untouched copy of the network."""
    nf, N = 3, 24
    feats = {k: v.cuda() for k, v in syn.make_feats(nf, N, seed=4).items()}
    base = _net(nf, syn.PRESET_TINY)
    ref = copy.deepcopy(base)
    syn.surrogate_loss(ref(dict(feats))).backward()
    ts = TrainStep(base, syn.surrogate_loss, feats, lr=1e-3, graph=False, warmup=1)
    ts()
    off = 0
    for (name, p), q in zip(base.named_parameters(), ref.parameters()):
        n = p.numel()
        g = ts.flat_grad[off:off + n].view_as(p)
        off += n
        want = torch.zeros_like(g) if q.grad is None else q.grad
        assert (g - want).abs().max().item() <= 2e-5 * max(1e-6, want.abs().max().item()) + 1e-9, name
