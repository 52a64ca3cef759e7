"""-m gpu: the training step's backward with the convolution weight gradients on a side stream.

* Eager TrainStep steps with the weight gradients overlapped on the side stream give the same losses, flat gradient and
  flat parameters, bit for bit, as the same steps taken with kernels.PROFILE set, where every launch stays on one stream:
  preset A at 8 x 64 (the dead-frame pyramid's small grids), the tiny preset at 20 x 16 with accumulate=2 and gradient
  clipping (the norm kernel reads the joined buffer), and preset A at the benchmark's 64 x 256.
* The captured step (fork and join inside the graph) equals the same single-stream eager steps at 8 x 64.
* dfold_split2d_residual_gate gives the planes and column sums of the torch emulation with gate = out - residual, bit for
  bit, including elements where out == residual and where out - residual is subnormal.
"""
import pytest
import torch

from dynamicpdb_b200 import kernels as K
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from dynamicpdb_b200.train_step import TrainStep
from tests.test_gpu_simt import DEV, SENT16, _colsum_emul, _gen, _ok, _planes, _same_bits, _twice, _wide

pytestmark = pytest.mark.gpu
PRESETS = {"A": syn.PRESET_A, "tiny": syn.PRESET_TINY}


def _steps(preset, nf, N, *, steps, accumulate=1, max_grad_norm=None, graph=False, single_stream=False):
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(nf, **PRESETS[preset]), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    net = net.cuda()
    windows = [{k: v.cuda() for k, v in syn.make_feats(nf, N, seed=60 + i).items()} for i in range(accumulate)]
    prev = K.PROFILE
    K.PROFILE = [] if single_stream else None
    try:
        ts = TrainStep(net, syn.surrogate_loss, windows[0], lr=1e-3, graph=graph, warmup=1, accumulate=accumulate,
                       max_grad_norm=max_grad_norm)
        assert (ts.graph is not None) == graph, ts.graph_error
        for i, w in enumerate(windows):
            ts.load(w, slot=i)
        losses = []
        for _ in range(steps):
            losses.append(ts().clone())
            if K.PROFILE is not None:
                K.PROFILE.clear()
        torch.cuda.synchronize()
    finally:
        K.PROFILE = prev
    out = (torch.stack(losses).cpu(), ts.flat_grad.cpu(), ts.flat_param.cpu())
    del ts, net
    torch.cuda.empty_cache()
    return out


def _assert_equal(a, b):
    for x, y, what in zip(a, b, ("losses", "flat_grad", "flat_param")):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), \
            f"{what}: {int((x != y).sum())} elements differ, max |diff| {(x - y).abs().max().item():.3e}"


@pytest.mark.parametrize("preset,nf,N,steps,accumulate,max_grad_norm", [
    ("A", 8, 64, 3, 1, None),
    ("tiny", 20, 16, 3, 2, 1e-2),
    ("A", 64, 256, 1, 1, None),
], ids=["A-8x64", "tiny-20x16-acc2-clip", "A-64x256"])
def test_overlapped_eager_step_equals_single_stream(preset, nf, N, steps, accumulate, max_grad_norm):
    kw = dict(steps=steps, accumulate=accumulate, max_grad_norm=max_grad_norm)
    _assert_equal(_steps(preset, nf, N, **kw), _steps(preset, nf, N, single_stream=True, **kw))


def test_captured_overlapped_step_equals_single_stream():
    _assert_equal(_steps("A", 8, 64, steps=3, graph=True), _steps("A", 8, 64, steps=3, single_stream=True))


def _residual_gate_values(R, C, seed):
    """(out, residual) [R, C] whose difference is positive, zero (out == residual), negative, and subnormal of both signs."""
    g = _gen(seed)
    res = _wide(R * C, seed + 1, lo_exp=-126, hi_exp=20).view(R, C)
    kind = torch.randint(0, 6, (R, C), generator=g, device=DEV)
    step = torch.rand(R, C, generator=g, device=DEV) + 0.5
    out = torch.where(kind == 0, res + step * res.abs().clamp(min=1.0), res)             # clearly open
    out = torch.where(kind == 1, res - step * res.abs().clamp(min=1.0), out)             # clearly closed
    out = torch.where(kind == 2, res, out)                                               # out == residual: closed
    # around a subnormal residual, out one ulp (2^-149) above / below it: out - residual = +-2^-149
    tiny = torch.full_like(res, 2.0 ** -140)
    base = torch.where(kind >= 3, tiny, res)
    res = torch.where(kind >= 3, base, res)
    out = torch.where(kind == 3, torch.nextafter(base, torch.full_like(base, 1.0)), out)
    out = torch.where(kind == 4, torch.nextafter(base, torch.full_like(base, -1.0)), out)
    out = torch.where(kind == 5, base - 2.0 ** -140 * 0.75, out)                         # a subnormal difference
    d = out - res
    assert (d == 0).any() and ((d != 0) & (d.abs() < 2.0 ** -126)).any()
    return out.contiguous(), res.contiguous()


@pytest.mark.parametrize("R,C,trans,pre_relu", [(515, 1280, False, False), (515, 1280, False, True), (67, 37, True, False),
                                                 (67, 40, True, True)])
def test_split2d_residual_gate(R, C, trans, pre_relu):
    """[R, C] contiguous rows take the vectorised kernel; with transposed planes (and odd C) the tile kernel runs."""
    seed = R + C
    x = _wide(R * C, seed).view(R, C)
    out, res = _residual_gate_values(R, C, seed + 5)
    v = x.clamp(min=0) if pre_relu else x
    v = torch.where((out - res) > 0, v, torch.zeros_like(v))
    hi, lo = _planes(v)
    c8 = -(-C // 8) * 8
    r8 = -(-R // 8) * 8
    init = torch.randn(C, generator=_gen(seed + 2), device=DEV)
    exp = [torch.zeros(R, c8, dtype=torch.int16, device=DEV) for _ in range(2)]
    exp[0][:, :C], exp[1][:, :C] = hi, lo
    if trans:
        for p, t in ((hi, 0), (lo, 1)):
            e = torch.zeros(C, r8, dtype=torch.int16, device=DEV)
            e[:, :R] = p.T
            exp.append(e)
    exp.append(_colsum_emul(v, init))

    def make():
        return [torch.full_like(e, SENT16) for e in exp[:-1]] + [init.clone()]

    def launch(b):
        ht, lt = (b[2], b[3]) if trans else (None, None)
        return K.lib().dfold_split2d_residual_gate(K._ptr(x), R, C, C, int(pre_relu), K._ptr(out), K._ptr(res), C,
                                                   K._ptr(b[0]), K._ptr(b[1]), c8, c8, K._ptr(ht), K._ptr(lt),
                                                   r8 if trans else 0, r8 if trans else 0, K._ptr(b[-1]), K._stream())
    got = _twice(make, launch)
    for i, (g_, e_) in enumerate(zip(got, exp)):
        _same_bits(f"split2d_residual_gate R{R} C{C} trans{int(trans)} relu{int(pre_relu)} output {i}", g_, e_)
    # the same as dfold_split2d with the difference computed first
    gate = out - res
    (h2, l2), _ = K._split2d(x, pre_relu=pre_relu, gate=gate)
    cs = init.clone()
    K._split2d(x, pre_relu=pre_relu, gate=gate, want=False, colsum=cs)
    torch.cuda.synchronize()
    _same_bits("vs dfold_split2d hi", got[0], h2)
    _same_bits("vs dfold_split2d lo", got[1], l2)
    _same_bits("vs dfold_split2d colsum", got[-1], cs)


def test_split2d_residual_gate_needs_both_operands():
    x = torch.zeros(8, 8, device=DEV)
    o = torch.zeros(2, 64, dtype=torch.int16, device=DEV)
    L = K.lib()
    for a, b in ((x, None), (None, x)):
        assert L.dfold_split2d_residual_gate(K._ptr(x), 8, 8, 8, 0, K._ptr(a), K._ptr(b), 8, K._ptr(o[0]), K._ptr(o[1]),
                                             8, 8, None, None, 0, 0, None, K._stream()) != 0
        assert b"out and residual" in L.dfold_last_error()
    _ok(L.dfold_split2d_residual_gate(K._ptr(x), 8, 8, 8, 0, K._ptr(x), K._ptr(x), 8, K._ptr(o[0]), K._ptr(o[1]), 8, 8,
                                      None, None, 0, 0, None, K._stream()))
