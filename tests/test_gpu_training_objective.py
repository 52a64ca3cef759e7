"""-m gpu: one training step of the reference's objective through the CUDA kernels: FullScoreNetwork ->
dynamicpdb_b200.loss.score_network_loss (csrc/loss.cu) -> backward through the score epilogue, the frame updates, the
ConvNet (the dead-frame pyramid when nf > 17) and the IPA blocks -> every parameter gradient.

  a. against the unmodified reference's Experiment.loss_fn over its own network (tests/golden/boundary.pt, objective.pt);
  b. against the oracle (oracle.dfold_oracle full_forward + loss_fn on the CPU) at the shapes, diffusion times,
     coordinate_scaling, loss options, masks and batch field forms of CASES, through the ReLU gates the CUDA forward
     applied (as tests/test_gpu_model.py), so no outlier allowance is needed;
  c. the captured TrainStep driving the real loss: gradient buffer against plain autograd, graph replay on windows with
     different t against eager steps, and bit-reproducibility.

The oracle's trunk casts to float32 in place (dfold_oracle.trunk), so it cannot run in float64 by casting its inputs: the
oracle side is fp32 at every shape, and the reported gradient errors contain its rounding as well as the kernels'.
"""
import copy
import os

import pytest
import torch

from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.loss import score_network_loss
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from dynamicpdb_b200.train_step import TrainStep
from oracle import dfold_oracle as O
from oracle import make_objective_golden as G
from tests.test_cpu_boundary import EXP_CONF as BOUNDARY_EXP_CONF, _batch as boundary_batch
from tests.test_cpu_oracle import close
from tests.test_gpu_model import _record, _record_gates

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ANGLE_BIAS = "score_model.angle_resnet.linear_out.bias"


def _network(preset, nf, cs, seed, angle_bias=0.5):
    """(FullScoreNetwork on the host, its state) with random_state weights: every 'final' layer is non-zero.  angles =
    u / |u| has the gradient w / |u|, so `angle_bias` is added to AngleResnet's output bias to keep every |u| of order
    one: the comparison is then of the kernels and not of an ill-conditioned division (_preconditions asserts it)."""
    net = FullScoreNetwork(syn.model_conf(nf, coordinate_scaling=cs, **preset), SE3ScoreDiffuser(syn.diffuser_conf(cs)))
    state = syn.random_state({k: v.shape for k, v in net.state_dict().items()}, seed=seed)
    state[ANGLE_BIAS] = state[ANGLE_BIAS] + angle_bias
    net.load_state_dict(state, strict=True)
    return net, state


def _to(d, dev):
    return {k: v.to(dev) for k, v in d.items()}


def _forward_loss_backward(net, batch, exp_conf, diffuse_rot=True):
    """Product forward, real loss, backward on DEV -> (out with the gradients of the loss w.r.t. it retained, loss, aux)."""
    out = net(dict(batch))
    for k in ("angles", "unorm_angles", "rot_score", "trans_score", "rigids", "atom37"):
        out[k].retain_grad()
    loss, aux = score_network_loss(out, batch, exp_conf, diffuse_rot=diffuse_rot)
    loss.backward()
    if DEV == "cuda":
        torch.cuda.synchronize()
    return out, loss.detach().cpu(), {k: v.cpu() for k, v in aux.items()}


def _check_output_gradients(out, angles=True, rot_score=True, rigids=True):
    """What the loss hands back to the network: the last frame of angles / rot_score / the translation of rigids only,
    each non-zero exactly when its term counts."""
    for k, live in (("angles", angles), ("rot_score", rot_score), ("rigids", rigids)):
        g = out[k].grad
        assert g is not None and g.shape == out[k].shape, k
        assert not bool(g[:-1].any()), f"d loss / d {k} is non-zero outside the trained-on frame"
        assert bool(g[-1].any()) == live, (k, live)
    assert not bool(out["rigids"].grad[..., :4].any())
    for k in ("trans_score", "unorm_angles", "atom37"):
        assert out[k].grad is None, f"{k} is not part of the objective"


# ---------------------------------------------------------------------------------------------------------------------
# a. the reference's own numbers
# ---------------------------------------------------------------------------------------------------------------------
def _golden_case(name):
    if name == "boundary":
        g = torch.load(os.path.join(GOLD, "boundary.pt"))
        return g, dict(nf=3, coordinate_scaling=1.0, t=0.5), 131, boundary_batch(), O.default_exp_conf(**BOUNDARY_EXP_CONF)
    c = G.CASES[name]
    return torch.load(os.path.join(GOLD, "objective.pt"))[name], c, c["seed"] + 100, G.case_batch(c), G.exp_conf(c)


@pytest.mark.parametrize("name", ["boundary"] + list(G.CASES))
def test_training_objective_matches_reference_loss_fn_golden(name):
    """Loss, aux_data and parameter gradients of Experiment.loss_fn over the reference network, from the CUDA kernels.
    The fixtures hold the reference's own ReLU gates, so the gradient bar is that of tests/test_gpu_goldens.py: 5e-3."""
    g, c, weight_seed, batch, exp_conf = _golden_case(name)
    net = _network(syn.PRESET_TINY, c["nf"], c["coordinate_scaling"], weight_seed, angle_bias=0.0)[0].to(DEV)
    out, loss, aux = _forward_loss_backward(net, _to(batch, DEV), exp_conf)
    _check_output_gradients(out, rot_score=c["t"] > 0.2)
    assert loss.dtype == g["loss"].dtype == torch.float64 and close(loss, g["loss"], 1e-4)
    assert set(aux) == set(g["aux"]), (sorted(aux), sorted(g["aux"]))
    for k, ref in g["aux"].items():
        ref = torch.as_tensor(ref)
        assert aux[k].shape == ref.shape and aux[k].dtype == ref.dtype and close(aux[k], ref, 1e-4), k
    grads = {k: p.grad.cpu() for k, p in net.named_parameters() if p.grad is not None}
    assert set(grads) == set(g["grad_norms"]) and len(grads) > 50          # the dead-output embedder, linear_rbf: none
    worst = 0.0
    for k, ref in g["grads"].items():
        if ref.norm() < 1e-7:
            continue
        e = ((grads[k] - ref).norm() / ref.norm()).item()
        worst = max(worst, e)
        assert e < 5e-3, f"{name}: grad {k} rel L2 {e:.3e}"
    for k, n in g["grad_norms"].items():
        if n > 1e-6:
            assert abs(grads[k].norm().item() - n) < 5e-3 * n, f"{name}: |grad {k}|"
    _record("objective_golden_" + name, {"loss_rel": abs(float(loss) - float(g["loss"])) / max(1.0, abs(float(g["loss"]))),
                                         "worst_grad_rel_l2": worst})


# ---------------------------------------------------------------------------------------------------------------------
# b. the oracle at the shapes and settings that matter
# ---------------------------------------------------------------------------------------------------------------------
# relative L2 error per parameter tensor.  The bar of tests/test_gpu_model.py; the denominator is floored at 1e-4 of the
# largest tensor gradient of the case: linear_b.bias and the like have a mathematically zero gradient (a shift the softmax
# cancels), both sides hold rounding noise there, and a ratio of two noises is not an error of either
GRAD_BAR = 2e-3            # measured worst 1.6e-3 (tiny_masked, ipa_0.head_weights); unmasked cases <= 3.3e-4
GRAD_FLOOR = 1e-4
# A fully masked frame: every logit of it carries the reference's -1e5, whose fp32 spacing is 2^-7, so what is left of the
# logits after the row maximum is subtracted is quantised to 7.8e-3 on BOTH sides, each rounding its own sum; the
# attention of that frame, and the d(head_weights) it feeds, agree to that spacing's order only.  Measured 3.8e-3 (tiny).
GRAD_BAR_MASKED_FRAME = 1e-2


def _case(name, preset, nf, N, **kw):
    c = dict(preset=preset, nf=nf, N=N, t=0.5, cs=1.0, separate=False, diffuse_rot=True, masks="none", form="loader",
             w_tor=1.0, far=False, bar=GRAD_BAR)
    assert set(kw) <= set(c), kw
    c.update(kw)
    return pytest.param(c, id=name)


TINY, A4x40, A19x24 = (syn.PRESET_TINY, 3, 12), (syn.PRESET_A, 4, 40), (syn.PRESET_A, 19, 24)
CASES = [
    # every shape of tests/test_gpu_model.py at the default setting
    _case("tiny", *TINY),
    _case("B", syn.PRESET_B, 2, 24),
    _case("A", *A4x40),
    _case("A130", syn.PRESET_A, 2, 130),                                  # ragged tiles
    _case("tiny_nf20", syn.PRESET_TINY, 20, 16),                          # dead-frame pyramid: built for the last-frame loss
    _case("A_nf19", *A19x24),                                             # dead-frame pyramid, preset A
    _case("A256_nf8", syn.PRESET_A, 8, 256),                              # the benched residue count
    _case("A1024_nf2", syn.PRESET_A, 2, 1024),                            # the long chain
    # the big shapes at the shipped coordinate_scaling and min_t: scores at their largest, rotation term gated off
    _case("A256_nf8_cs0.1_tmin", syn.PRESET_A, 8, 256, cs=0.1, t=0.01),
    _case("A1024_nf2_cs0.1_tmin", syn.PRESET_A, 2, 1024, cs=0.1, t=0.01),
    # diffusion time: min_t, exactly the rotation threshold (a strict comparison), the end of the schedule
    _case("tiny_tmin", *TINY, t=0.01),
    _case("tiny_t0.2", *TINY, t=0.2),
    _case("tiny_t1", *TINY, t=1.0),
    _case("A_tmin", *A4x40, t=0.01),
    _case("A_t0.2_separate", *A4x40, t=0.2, separate=True),               # the angle half gated off, the axis half not
    _case("A_nf19_t1", *A19x24, t=1.0),
    # coordinate_scaling 0.1: fused_scores sees the translation before the unscale, the loss after it
    _case("tiny_cs0.1", *TINY, cs=0.1),
    # (the axis / angle loss is not crossed with min_t: make_feats draws rigids_t uniformly, and angles of order pi at
    # sigma(min_t) = 0.1 put the IGSO(3) series where it cancels to e^-100, so the SIGN of the predicted score, and with
    # it the axis term, is rounding noise on both sides; tests/test_gpu_residue_kernels.py bounds that regime)
    _case("tiny_cs0.1_t0.2_separate", *TINY, cs=0.1, t=0.2, separate=True),
    _case("A_cs0.1", *A4x40, cs=0.1),
    _case("A_cs0.1_separate_masked", *A4x40, cs=0.1, separate=True, masks="loss_case"),
    _case("A_nf19_cs0.1_tmin", *A19x24, cs=0.1, t=0.01),
    # loss options
    _case("tiny_separate", *TINY, separate=True),
    _case("A_separate", *A4x40, separate=True),
    _case("A_nf19_separate_masked", *A19x24, separate=True, masks="loss_case"),
    _case("tiny_no_diffuse_rot", *TINY, diffuse_rot=False),               # the rotation term switched off by the config
    _case("tiny_no_torsion", *TINY, w_tor=0.0),                           # rotation and translation paths without u / |u|
    _case("A_no_torsion", *A4x40, w_tor=0.0),
    # masks: two masked residues and a fixed one; the trained-on frame fully masked (the rotation term has no residue)
    _case("tiny_masked", *TINY, masks="loss_case"),
    _case("A_masked_t1", *A4x40, masks="loss_case", t=1.0),
    _case("tiny_last_frame_masked", *TINY, masks="last_frame", bar=GRAD_BAR_MASKED_FRAME),
    _case("A_nf19_last_frame_masked", *A19x24, masks="last_frame", bar=GRAD_BAR_MASKED_FRAME),
    # batch field forms: the prefetcher hands 0-dim scalings, add_loss_targets [1]; fp32 fields instead of the loader's fp64
    _case("tiny_0dim", *TINY, form="0dim"),
    _case("A_0dim_separate", *A4x40, form="0dim", separate=True),
    _case("tiny_fp32", *TINY, form="fp32"),
    _case("A_nf19_fp32", *A19x24, form="fp32"),
    # the translation term over the loss's `< 100` gate: it and the rotation term are exactly zero with their gradients;
    # the torsion term stays, because the reference gates it on the translation term it has just zeroed (:1337-1339)
    _case("tiny_far", *TINY, far=True),
    _case("A_nf19_far", *A19x24, far=True),
]


def _batch(c, seed=11):
    """(the batch the product gets, the same batch in the reference's [1]-shaped form for the oracle), on the host."""
    feats = syn.make_feats(c["nf"], c["N"], seed=seed, t=c["t"], coordinate_scaling=c["cs"], loader_dtypes=c["form"] != "fp32")
    feats = syn.add_loss_targets(feats, seed=seed, loader_dtypes=c["form"] != "fp32")
    if c["masks"] == "loss_case":
        feats["fixed_mask"][:, 1] = 1
        feats["res_mask"][:, -2:] = 0
    elif c["masks"] == "last_frame":
        feats["res_mask"][-1] = 0
    G.target_in_output_units(feats, c["cs"])
    if c["far"]:
        feats["rigids_0"][-1, :, 4:] += 30.0
    product = dict(feats)
    if c["form"] == "0dim":
        product["t"], product["rot_score_scaling"] = feats["t"].reshape(()), feats["rot_score_scaling"].reshape(())
    return product, feats


def _preconditions(c, out, aux, batch):
    """The case exercises what it is meant to: gate open (or closed on purpose), every term that should count non-zero,
    and the torsion normalisation well conditioned.  -> whether the rotation term counts."""
    if c["far"]:
        assert float(aux["trans_loss"]) == 0.0 and not bool(aux["batch_trans_loss"].any())
    else:
        assert 0 < float(aux["trans_loss"]) < 100, aux["trans_loss"]
    rot_on = c["diffuse_rot"] and c["masks"] != "last_frame" and (c["t"] > 0.2 or c["separate"]) and not c["far"]
    assert (float(aux["rot_loss"]) > 0) == rot_on, (aux["rot_loss"], rot_on)
    assert (float(aux["torsion_loss"]) > 0) == (c["w_tor"] > 0), aux["torsion_loss"]
    counted = (batch["torsion_angles_mask"][-1] * (1 - batch["fixed_mask"][-1])[:, None]) > 0
    u = out["unorm_angles"][-1].detach().norm(dim=-1).cpu()
    assert float(u[counted].min()) > 0.05, f"min |u| over counted torsions {float(u[counted].min()):.3e}"
    return rot_on


@pytest.mark.parametrize("c", CASES)
def test_training_objective_matches_oracle(c, request, monkeypatch):
    """Loss, aux and EVERY parameter gradient of one step of the real objective against the fp32 oracle through the same
    ReLU gates: loss and aux within 1e-4 max(1, |oracle|), gradients within the case's bar (GRAD_BAR) relative L2 per tensor."""
    name = request.node.callspec.id
    net, state = _network(c["preset"], c["nf"], c["cs"], 7)
    batch, batch_o = _batch(c)
    exp_conf = O.default_exp_conf(separate_rot_loss=c["separate"], torsion_loss_weight=c["w_tor"])
    # ---- product, recording the ReLU gates its kernels applied ----
    net = net.to(DEV)
    gates = _record_gates(net, monkeypatch)
    out, loss, aux = _forward_loss_backward(net, _to(batch, DEV), exp_conf, c["diffuse_rot"])
    monkeypatch.undo()
    rot_on = _preconditions(c, out, aux, batch)
    _check_output_gradients(out, angles=c["w_tor"] > 0, rot_score=rot_on, rigids=not c["far"])
    grads = {k: (None if p.grad is None else p.grad.cpu()) for k, p in net.named_parameters()}
    # ---- oracle (CPU, fp32), same weights, inputs and gates ----
    p = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point) for k, v in state.items()}
    O.set_gates(gates)
    try:
        out_o = O.full_forward(p, batch_o, O.default_conf(coordinate_scaling=c["cs"], **c["preset"]), O.default_diffuser_conf(c["cs"]))
    finally:
        O.set_gates(None)
    loss_o, aux_o = O.loss_fn(out_o, batch_o, exp_conf, diffuse_rot=c["diffuse_rot"])
    names = [k for k in p if p[k].requires_grad]
    g_o = dict(zip(names, torch.autograd.grad(loss_o, [p[k] for k in names], allow_unused=True)))
    loss_o = loss_o.detach()
    assert loss.dtype == torch.float64 and close(loss, loss_o, 1e-4), (float(loss), float(loss_o))
    assert set(aux) == set(aux_o)
    # dtypes as the reference arithmetic gives them for the loader's float64 targets (an all-fp32 batch, which the loader
    # never emits, would leave the reference's loss in float32; the kernel's stays float64)
    same_dtypes = c["form"] != "fp32"
    assert not same_dtypes or loss_o.dtype == torch.float64
    for k, ref in aux_o.items():
        assert aux[k].shape == ref.shape and close(aux[k], ref, 1e-4), (k, aux[k], ref)
        assert not same_dtypes or aux[k].dtype == ref.dtype, (k, aux[k].dtype, ref.dtype)
    # the outputs the objective reads, and trans_score, which it does not (so only this line holds fused_scores to the
    # translation BEFORE the unscale): per-residue L2 within 1e-4 of the largest residue, the bar of
    # tests/test_gpu_model.py made relative because the score grows as 1 / t and 1 / coordinate_scaling.  rot_score is held
    # through the loss where it counts; on its own it is ill-conditioned at small sigma(t) for make_feats' uniformly drawn
    # rigids_t, the regime tests/test_gpu_residue_kernels.py bounds
    for k, tol in (("rigids", 1e-4), ("trans_score", 1e-4)):
        ref = out_o[k].detach().double().flatten(2)
        err = (ref - out[k].detach().cpu().double().flatten(2)).norm(dim=-1).max().item()
        assert err <= tol * max(1.0, ref.norm(dim=-1).max().item()), f"{name}: {k} per-residue L2 {err:.3e}"
    norms = [float(g.norm()) for g in g_o.values() if g is not None]
    assert sum(n * n for n in norms) > 0
    floor = GRAD_FLOOR * max(norms)
    worst = ("", 0.0)
    for k, gg in grads.items():
        go = g_o.get(k)
        if go is None or gg is None:
            assert (go is None or float(go.abs().max()) < 1e-7) and (gg is None or float(gg.abs().max()) < 1e-7), k
            continue
        e = ((go - gg).norm() / max(float(go.norm()), floor)).item()
        if e > worst[1]:
            worst = (k, e)
    _record("objective_" + name, {"loss_rel": abs(float(loss) - float(loss_o)) / max(1.0, abs(float(loss_o))),
                                  "worst_grad_rel_l2": worst[1], "worst_grad_name": worst[0]})
    assert worst[1] < c["bar"], f"{name}: gradient of {worst[0]} rel L2 err {worst[1]:.3e}"


# ---------------------------------------------------------------------------------------------------------------------
# c. the captured step with the real loss
# ---------------------------------------------------------------------------------------------------------------------
STEP_SHAPES = [pytest.param(dict(preset=syn.PRESET_TINY, nf=20, N=16), id="tiny_nf20"),     # three cropped ConvNet calls
               pytest.param(dict(preset=syn.PRESET_A, nf=8, N=64), id="A_nf8")]


def _window(s, seed, t):
    c = dict(s, t=t, cs=1.0, form="loader", masks="loss_case", far=False)
    batch = _batch(c, seed=seed)[0]
    batch["rot_score_scaling"] = batch["rot_score_scaling"] * 0 + 0.5 + t       # as t, read on the device by the loss
    return _to(batch, DEV)


def _train_step(net, batch, **kw):
    exp_conf = O.default_exp_conf()
    return TrainStep(net, lambda out: score_network_loss(out, batch, exp_conf)[0], batch, **kw)


@pytest.mark.parametrize("s", STEP_SHAPES)
def test_train_step_gradients_of_the_objective_equal_plain_autograd(s):
    """tests/test_gpu_trainstep.py test_train_step_gradients_equal_plain_autograd for the real loss: the shared ConvNet's
    four weight gradients are accumulated in place, from cropped calls when nf > 17."""
    batch = _window(s, 4, 0.5)
    base = _network(s["preset"], s["nf"], 1.0, 7)[0].to(DEV)
    ref = copy.deepcopy(base)
    score_network_loss(ref(dict(batch)), batch, O.default_exp_conf())[0].backward()
    ts = _train_step(base, batch, lr=1e-3, graph=False, warmup=1)
    ts()
    assert float(ts.flat_grad.norm()) > 0
    off = 0
    for (name, p), q in zip(base.named_parameters(), ref.parameters()):
        n = p.numel()
        g = ts.flat_grad[off:off + n].view_as(p)
        off += n
        want = torch.zeros_like(g) if q.grad is None else q.grad
        assert (g - want).abs().max().item() <= 2e-5 * max(1e-6, want.abs().max().item()) + 1e-9, name


@pytest.mark.parametrize("s", STEP_SHAPES)
def test_graph_replay_of_the_objective_follows_new_windows(s):
    """A graph captured on one window (t = 0.5), replayed on three others with t below, on and above the rotation
    threshold, gives the loss and the gradient that plain autograd gives from the same weights on the same window: t and
    rot_score_scaling are read on the device, so nothing of the capture window is baked in."""
    batch = _window(s, 4, 0.5)
    net = _network(s["preset"], s["nf"], 1.0, 7)[0].to(DEV)
    ref = copy.deepcopy(net)
    ts = _train_step(net, batch, lr=1e-4, graph=True, warmup=2)
    assert ts.graph is not None, ts.graph_error
    losses = []
    for i, t in enumerate((0.05, 0.2, 0.9)):
        new = _window(s, 20 + i, t)
        with torch.no_grad():
            for q, p in zip(ref.parameters(), net.parameters()):
                q.copy_(p)
                q.grad = None
        want = score_network_loss(ref(dict(new)), new, O.default_exp_conf())[0]
        want.backward()
        want_grad = torch.cat([(torch.zeros_like(q) if q.grad is None else q.grad).reshape(-1) for q in ref.parameters()])
        ts.load(new)
        for k in batch:
            batch[k].copy_(new[k])
        got = float(ts())
        got_grad = ts.flat_grad[:want_grad.numel()]
        assert abs(got - float(want)) <= 1e-6 * max(1.0, abs(float(want))), (t, got, float(want))
        assert float(want_grad.norm()) > 0 and ((got_grad - want_grad).norm() / want_grad.norm()).item() < 5e-3, t
        losses.append(got)
    assert len({round(l, 6) for l in losses}) == 3, losses                     # the three windows are told apart


def test_training_steps_on_the_objective_are_reproducible():
    """tests/test_gpu_trainstep.py test_training_steps_are_reproducible for the real loss: two identical runs of captured
    steps give bit-identical loss, gradient and parameters."""
    s = dict(preset=syn.PRESET_A, nf=8, N=64)
    batch = _window(s, 3, 0.5)
    runs = []
    for _ in range(2):
        net = _network(s["preset"], s["nf"], 1.0, 7)[0].to(DEV)
        ts = _train_step(net, {k: v.clone() for k, v in batch.items()}, lr=1e-4, graph=True, warmup=2)
        assert ts.graph is not None, ts.graph_error
        losses = [ts().clone() for _ in range(3)]
        torch.cuda.synchronize()
        runs.append((torch.stack(losses).cpu(), ts.flat_grad.cpu(), ts.flat_param.cpu()))
        del net, ts
        torch.cuda.empty_cache()
    for a, b, what in zip(runs[0], runs[1], ("loss", "gradients", "parameters")):
        assert torch.equal(a, b), f"{what} differ between two identical runs: max |diff| {(a - b).abs().max().item():.3e}"
