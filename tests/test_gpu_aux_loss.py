"""-m gpu: the backbone-atom and pair-distance losses (``score_network_loss(aux_losses=True)``, csrc/aux_loss.cu).

  a. the kernel pair against oracle.aux_loss_oracle.aux_structure_losses in float64, per frame and d loss / d atoms, at the
     training shapes and at the edges: masked and fixed residues, glycine CBs at the origin with coincident predicted
     atoms, a ground-truth pair at exactly 6 A, frames with an empty loss mask;
  b. the objective over the product network against the unmodified reference (tests/golden/aux_loss.pt), including the
     20-frame window where the product runs its dead-frame pyramid;
  c. aux_losses=False against a call without the argument, bit for bit;
  d. the captured step on the aux objective: graph replay against eager steps, reproducibility, and peak memory.

Bounds of a.  Kernel and oracle read the same fp32 coordinates and both work in fp64 from there; they differ only in
the order of their sums (the kernel's rows stream column tiles, torch reduces its own way) and in sqrt / division
rounding, a few ulp per term.  A frame's sums have at most (5N)^2 = 26.2M terms of one sign, so the relative difference
of a value is below 26.2M x 2^-52 = 5.8e-9: the bound is 1e-8.  A gradient row sums up to 2 x 5N terms of either sign, so
its error is bounded relative to the largest gradient component: 1e-9.  Both sides also form the distances in fp64 from
the same coordinates, a few ulp (< 1e-14 A) apart, so a pair is classified alike when its ground-truth distance lies at
least 1e-9 A away from 6 A, which the test asserts of every random case.  (With (5N)^2 pairs, a margin of 1e-4 A, which an
fp32 distance would need, cannot be kept at N = 1024: random cases there hold pairs within 1e-6 A of 6 A.)
"""
import copy
import os
from types import SimpleNamespace

import pytest
import torch

from dynamicpdb_b200 import loss as L
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.loss import score_network_loss
from dynamicpdb_b200.train_step import TrainStep
from oracle import aux_loss_oracle as A
from oracle import dfold_oracle as O
from oracle import make_aux_loss_golden as G
from tests.test_cpu_oracle import close
from tests.test_gpu_training_objective import _network, _to, _window

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "aux_loss.pt")
CONF = SimpleNamespace(bb_atom_loss_weight=1.0, bb_atom_loss_t_filter=0.25, dist_mat_loss_weight=1.0,
                       dist_mat_loss_t_filter=0.25, aux_loss_weight=0.25)
CONSTS = tuple(getattr(CONF, k) for k in L.AUX_KEYS)
VALUE_BAR, GRAD_BAR = 1e-8, 1e-9


# ---------------------------------------------------------------------------------------------------------------------
# a. the kernels against float64
# ---------------------------------------------------------------------------------------------------------------------
def _inputs(nf, N, seed, edges=True):
    """(pred atom37 [nf,N,37,3] fp64 holding fp32 values, gt atom37 fp32, res_mask, fixed_mask) on DEV.  The ground truth
    is the alanine backbone of a synthetic trajectory, the prediction that plus 0.6 A noise; `edges` adds masked and fixed
    residues, glycines (CB at the origin, so several predicted CBs coincide), a predicted atom placed on another one, and
    two frames with an empty loss mask (all residues masked, all fixed)."""
    g = torch.Generator().manual_seed(seed)
    feats = _to(syn.make_feats(nf, N, seed=seed, loader_dtypes=True, node_dim=4, edge_dim=4), DEV)
    gt = L.ground_truth_backbone(feats)
    pred = torch.zeros(nf, N, 37, 3, dtype=torch.float32)
    pred[:, :, :5] = gt[:, :, :5].cpu() + torch.randn(nf, N, 5, 3, generator=g) * 0.6
    res = torch.ones(nf, N, dtype=torch.float64)
    fixed = torch.zeros(nf, N, dtype=torch.float64)
    if edges:
        res[:, torch.randperm(N, generator=g)[:max(1, N // 8)]] = 0
        fixed[:, torch.randperm(N, generator=g)[:max(1, N // 10)]] = 1
        gly = torch.randperm(N, generator=g)[:max(2, N // 6)]
        pred[:, gly, 3] = 0
        pred[:, 1, 0] = pred[:, 0, 2]
        if nf >= 3:
            res[1] = 0
            fixed[2] = 1
    return pred.double().to(DEV), gt, res.to(DEV), fixed.to(DEV)


def _kernel(pred, gt, res, fixed, t):
    """(per-frame bb, per-frame dist, normalised bb, normalised dist, d bb / d atoms, d dist / d atoms) of the kernels."""
    nf = res.shape[0]
    p = pred.clone().requires_grad_(True)
    out = L._AuxLossFn.apply(p, gt, res, fixed, t, CONSTS)
    g_bb, = torch.autograd.grad(out[0], p, retain_graph=True)
    g_dm, = torch.autograd.grad(out[1], p)
    return out[2:2 + nf].detach(), out[2 + nf:].detach(), out[0].detach(), out[1].detach(), g_bb[:, :, :5], g_dm[:, :, :5]


def _oracle(pred, gt, res, fixed, t, chunk):
    """The same six values from the float64 restatement, `chunk` frames at a time (its (5N)^2 tensors are large)."""
    nf = res.shape[0]
    n = float(torch.any(res != 0, dim=-1).sum()) + float(torch.tensor(1e-10, dtype=torch.float32))
    bb, dm, g_bb, g_dm = [], [], [], []
    for f0 in range(0, nf, chunk):
        sl = slice(f0, f0 + chunk)
        p = pred[sl, :, :5].clone().requires_grad_(True)
        b, d = A.aux_structure_losses(p, gt[sl, :, :5].double(), res[sl], fixed[sl], t, CONF)
        g_bb.append(torch.autograd.grad(b.sum() / n, p, retain_graph=True)[0])
        g_dm.append(torch.autograd.grad(d.sum() / n, p)[0])
        bb.append(b.detach())
        dm.append(d.detach())
    bb, dm = torch.cat(bb), torch.cat(dm)
    return bb, dm, bb.sum() / n, dm.sum() / n, torch.cat(g_bb), torch.cat(g_dm)


def _gt_distances_clear_of_6(gt, res):
    for f in range(gt.shape[0]):
        x = gt[f, :, :5].double().reshape(-1, 3)
        d = torch.cdist(x, x)
        assert float((d - 6).abs().min()) >= 1e-9, "a ground-truth distance lies within 1e-9 A of 6 A"


def _compare(got, want, what):
    names = ("bb per frame", "dist per frame", "bb", "dist", "d bb / d atoms", "d dist / d atoms")
    for a, b, name in zip(got, want, names):
        assert torch.isfinite(a).all(), (what, name)
        if name.startswith("d "):
            assert (a - b).abs().max().item() <= GRAD_BAR * max(1e-30, b.abs().max().item()), (what, name)
            assert not bool(a[b == 0].any()), (what, name, "non-zero where torch's gradient is 0")
        else:
            assert (a - b).abs().max().item() <= VALUE_BAR * max(1.0, b.abs().max().item()), (what, name, a, b)


SHAPES = [(nf, N) for nf in (2, 20, 64) for N in (16, 130, 256)] + [(8, 1024)]


@pytest.mark.parametrize("nf,N", SHAPES)
def test_aux_kernels_match_float64(nf, N):
    pred, gt, res, fixed = _inputs(nf, N, seed=nf * 1000 + N)
    _gt_distances_clear_of_6(gt, res)
    t = torch.tensor([0.1], dtype=torch.float64, device=DEV)
    got = _kernel(pred, gt, res, fixed, t)
    want = _oracle(pred, gt, res, fixed, t, chunk=max(1, 2 ** 22 // (5 * N) ** 2 * 2))
    assert float(want[2]) > 0 and float(want[3]) > 0
    _compare(got, want, (nf, N))
    if nf >= 3:             # the empty-loss-mask frames contribute nothing and raise nothing
        assert got[0][1:3].abs().max().item() == 0 and got[1][1:3].abs().max().item() == 0
        assert not got[4][1:3].any() and not got[5][1:3].any()


@pytest.mark.parametrize("t,on", [(0.2499, True), (0.25, False), (0.9, False)])
def test_aux_gates_are_strict_and_read_on_the_device(t, on):
    pred, gt, res, fixed = _inputs(3, 40, seed=5)
    tt = torch.tensor([t], dtype=torch.float64, device=DEV)
    got = _kernel(pred, gt, res, fixed, tt)
    _compare(got, _oracle(pred, gt, res, fixed, tt, chunk=3), t)
    assert bool(got[2] != 0) == on and bool(got[3] != 0) == on and bool(got[4].any()) == on


def test_ground_truth_pair_at_exactly_6_angstrom_is_excluded():
    """Every atom on a line 6 A from its neighbours but one pair 5.5 A apart: only that pair and the diagonal count."""
    nf, N = 2, 4
    x = torch.arange(5 * N, dtype=torch.float32) * 6.0
    x[7] = x[6] + 5.5
    gt = torch.zeros(nf, N, 37, 3)
    gt[:, :, :5, 0] = x.reshape(N, 5) + 1.0
    gt = gt.to(DEV)
    pred = gt.double().clone()
    pred[:, :, :5] += torch.randn(nf, N, 5, 3, generator=torch.Generator().manual_seed(2), dtype=torch.float64).to(DEV)
    pred = pred.float().double()
    res, fixed = torch.ones(nf, N, dtype=torch.float64, device=DEV), torch.zeros(nf, N, dtype=torch.float64, device=DEV)
    t = torch.tensor([0.1], dtype=torch.float64, device=DEV)
    got, want = _kernel(pred, gt, res, fixed, t), _oracle(pred, gt, res, fixed, t, chunk=nf)
    _compare(got, want, "6 A")
    # two counted off-diagonal pairs over 5N + 2 - N in the denominator
    gf, pf = gt[0, :, :5].double().reshape(-1, 3), pred[0, :, :5].reshape(-1, 3)
    e = torch.linalg.norm(gf[6] - gf[7]) - torch.linalg.norm(pf[6] - pf[7])
    assert close(got[1][0].cpu(), (2 * e * e / (5 * N + 2 - N) * 0.25).cpu(), 1e-12)


# ---------------------------------------------------------------------------------------------------------------------
# b. the reference's own numbers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(G.CASES))
def test_aux_objective_matches_reference_golden(name):
    """Loss, aux_data (keys, order, dtypes, values) and every parameter gradient of the reference's loss_fn with the
    auxiliary terms in final_loss.  The fixtures hold the reference's own fp32 ReLU gates, which the kernels' rounding
    flips on a few activations; the bar is 1e-2 (measured worst on an H100: 5.4e-3, t_high, conv_0.conv4.0.bias)."""
    g = torch.load(GOLD)[name]
    c = G.CASES[name]
    net = _network(syn.PRESET_TINY, c["nf"], c["coordinate_scaling"], c["seed"] + 100, angle_bias=0.0)[0].to(DEV)
    batch = _to(G.case_batch(c), DEV)
    out = net(dict(batch))
    out["atom37"].retain_grad()
    loss, aux = score_network_loss(out, batch, G.exp_conf(c), aux_losses=True)
    loss.backward()
    gt = L.ground_truth_backbone(batch)[:, :, :5].cpu()
    assert (gt - g["gt_atom37"]).abs().max().item() < 1e-4 * max(1.0, g["gt_atom37"].abs().max().item())
    assert torch.equal(torch.any(gt != 0, dim=-1), g["atom37_mask"])
    live = c["t"] < 0.25
    assert bool(out["atom37"].grad[:, :, :5].any()) == live and not out["atom37"].grad[:, :, 5:].any()
    if live:                # every frame is trained on, not the last one only
        assert all(bool(out["atom37"].grad[f].any()) for f in range(c["nf"]))
    assert loss.dtype == g["loss"].dtype and close(loss.detach().cpu(), g["loss"], 1e-4)
    assert list(aux) == list(g["aux"])
    for k, ref in g["aux"].items():
        v = aux[k].cpu()
        assert v.shape == ref.shape and v.dtype == ref.dtype and close(v, ref, 1e-4), k
    grads = {k: p.grad.cpu() for k, p in net.named_parameters() if p.grad is not None}
    assert set(grads) == set(g["grad_norms"]) and len(grads) > 50
    for k, ref in g["grads"].items():
        if ref.norm() < 1e-7:
            continue
        assert ((grads[k] - ref).norm() / ref.norm()).item() < 1e-2, f"{name}: grad {k}"
    for k, n in g["grad_norms"].items():
        if n > 1e-6:
            assert abs(grads[k].norm().item() - n) < 1e-2 * n, f"{name}: |grad {k}|"


# ---------------------------------------------------------------------------------------------------------------------
# c. the default stays as it was
# ---------------------------------------------------------------------------------------------------------------------
def test_aux_losses_false_is_the_default_bit_for_bit():
    c = G.CASES["t_low"]
    batch = _to(G.case_batch(c), DEV)
    runs = []
    for kw in ({}, {"aux_losses": False}):
        net = _network(syn.PRESET_TINY, c["nf"], 1.0, 7)[0].to(DEV)
        loss, aux = score_network_loss(net(dict(batch)), batch, G.exp_conf(c), **kw)
        loss.backward()
        runs.append((loss.detach(), aux, [p.grad for p in net.parameters()]))
    (l0, a0, g0), (l1, a1, g1) = runs
    assert torch.equal(l0, l1) and l0.dtype == l1.dtype
    assert list(a0) == list(a1)
    for k in a0:
        assert a0[k].dtype == a1[k].dtype and torch.equal(a0[k], a1[k]), k
    for x, y in zip(g0, g1):
        assert (x is None) == (y is None) and (x is None or torch.equal(x, y))


# ---------------------------------------------------------------------------------------------------------------------
# d. the captured step
# ---------------------------------------------------------------------------------------------------------------------
def _aux_loss(batch):
    conf = O.default_exp_conf(**vars(CONF))
    return lambda out: score_network_loss(out, batch, conf, aux_losses=True)[0]


@pytest.mark.parametrize("s", [pytest.param(dict(preset=syn.PRESET_TINY, nf=20, N=16), id="tiny_nf20"),
                               pytest.param(dict(preset=syn.PRESET_A, nf=8, N=64), id="A_nf8")])
def test_graph_replay_of_the_aux_objective_equals_eager_steps(s):
    """One graph captured at t = 0.5 (aux terms gated off), replayed on windows below and above the filters, gives the
    eager step's loss, gradient and updated parameters bit for bit."""
    base = _network(s["preset"], s["nf"], 1.0, 7)[0].to(DEV)
    steps = []
    for graph in (True, False):
        b = _window(s, 4, 0.5)
        ts = TrainStep(copy.deepcopy(base), _aux_loss(b), b, lr=1e-4, graph=graph, warmup=2)
        assert (ts.graph is not None) == graph, ts.graph_error
        steps.append(ts)
    losses = []
    for i, t in enumerate((0.1, 0.6, 0.05)):
        new = _window(s, 30 + i, t)
        out = []
        for ts in steps:
            ts.load(new)
            out.append((ts().clone(), ts.flat_grad.clone(), ts.flat_param.clone()))
        (la, ga, pa), (lb, gb, pb) = out
        assert torch.equal(la, lb), (t, float(la), float(lb))
        assert torch.equal(ga, gb) and torch.equal(pa, pb), t
        losses.append(float(la))
    assert len(set(losses)) == 3


def test_aux_training_steps_are_reproducible():
    s = dict(preset=syn.PRESET_A, nf=8, N=64)
    batch = _window(s, 3, 0.1)
    runs = []
    for _ in range(2):
        net = _network(s["preset"], s["nf"], 1.0, 7)[0].to(DEV)
        b = {k: v.clone() for k, v in batch.items()}
        ts = TrainStep(net, _aux_loss(b), b, lr=1e-4, graph=True, warmup=2)
        assert ts.graph is not None, ts.graph_error
        losses = [ts().clone() for _ in range(3)]
        torch.cuda.synchronize()
        runs.append((torch.stack(losses).cpu(), ts.flat_grad.cpu(), ts.flat_param.cpu()))
        del net, ts
        torch.cuda.empty_cache()
    for a, b, what in zip(runs[0], runs[1], ("loss", "gradients", "parameters")):
        assert torch.equal(a, b), what


def _peak_step_bytes(aux_losses, nf, N):
    torch.manual_seed(0)
    s = dict(preset=syn.PRESET_A, nf=nf, N=N)
    batch = _window(s, 3, 0.1)
    net = _network(s["preset"], nf, 1.0, 7)[0].to(DEV)
    conf = O.default_exp_conf(**vars(CONF))
    loss_fn = (lambda out: score_network_loss(out, batch, conf, aux_losses=aux_losses)[0])
    ts = TrainStep(net, loss_fn, batch, lr=1e-4, graph=False, warmup=1)
    ts()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ts()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del ts, net
    torch.cuda.empty_cache()
    return peak


def test_aux_objective_allocates_no_pair_buffer():
    """At 64 x 256 the reference's (5N)^2 fp32 matrices are 420 MB each; the step's peak grows by less than 32 MB."""
    default = _peak_step_bytes(False, 64, 256)
    aux = _peak_step_bytes(True, 64, 256)
    print(f"[aux] peak step memory 64 x 256: default {default / 2**20:.1f} MiB, aux {aux / 2**20:.1f} MiB")
    assert aux - default < 32 * 2 ** 20, (default, aux)
