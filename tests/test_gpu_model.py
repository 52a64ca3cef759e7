"""-m gpu: the whole FullScoreNetwork on the GPU (product path, C-ABI kernels) against the CPU oracle on the same
seeded inputs and weights — outputs and parameter gradients.  Stated tolerance (BASELINE.json north_star):
per-residue L2 error of the rotation / translation updates < 1e-4."""
import json
import os

import pytest
import torch

from dynamicpdb_b200 import kernels as K
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from oracle import dfold_oracle as O

pytestmark = pytest.mark.gpu


def _per_residue_l2(a, b):
    return (a.double() - b.double()).flatten(2).norm(dim=-1).max().item()


def _record(case, errs):
    """Measured parity errors -> the JSON file named by $DFOLD_PARITY_ERRORS, when set (DESIGN.md §2)."""
    path = os.environ.get("DFOLD_PARITY_ERRORS")
    if not path:
        return
    try:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        d = json.load(open(path)) if os.path.exists(path) else {}
        d[case] = errs
        json.dump(d, open(path, "w"), indent=1, sort_keys=True)
    except OSError:
        pass


def _record_gates(net, monkeypatch):
    """Wrap the product's ReLU-carrying operators so that every gate the CUDA kernels applied is recorded (from the
    kernels' own outputs, exactly as their backward derives it), keyed by the owning layer's state_dict name."""
    names = {id(p): n for n, p in net.named_parameters()}
    rec = {}
    conv0, lin0 = K.conv5x5, K.linear

    def conv(x, weight, bias=None, relu=True, residual=None, crop=0):
        out = conv0(x, weight, bias, relu, residual, crop)
        if relu:
            pre = out if residual is None else out - residual
            rec.setdefault(names[id(weight)], []).append((pre.detach() > 0).cpu())
        return out

    def lin(x, weight, bias=None, act=None, residual=None, pre_relu=False):
        if pre_relu:
            rec.setdefault(names[id(weight)] + ":in", []).append((x.detach() > 0).cpu())
        out = lin0(x, weight, bias, act, residual, pre_relu)
        if act == "relu":
            pre = out if residual is None else out - residual
            rec.setdefault(names[id(weight)] + ":out", []).append((pre.detach() > 0).cpu())
        return out

    monkeypatch.setattr(K, "conv5x5", conv)
    monkeypatch.setattr(K, "linear", lin)
    return rec


@pytest.mark.parametrize("name,preset,nf,N", [("tiny", syn.PRESET_TINY, 3, 12), ("B", syn.PRESET_B, 2, 24),
                                               ("A", syn.PRESET_A, 4, 40), ("A130", syn.PRESET_A, 2, 130),
                                               # nf > 17: the middle blocks run the dead-frame pyramid (cropped convs)
                                               ("tiny_nf20", syn.PRESET_TINY, 20, 16), ("A_nf19", syn.PRESET_A, 19, 24),
                                               # the BENCHED residue count (BASELINE.json configs[2]) and the long chain
                                               # (configs[4]); the 64-frame shape itself: test_gpu_goldens.py::net_A256
                                               ("A256_nf8", syn.PRESET_A, 8, 256), ("A1024_nf2", syn.PRESET_A, 2, 1024)])
def test_full_network_matches_oracle(name, preset, nf, N, monkeypatch):
    """Outputs and EVERY parameter gradient.  The oracle back-propagates through the ReLU gates the CUDA forward applied
    (oracle.set_gates), so a pre-activation within rounding of zero cannot gate differently on the two sides; the
    gradient comparison then has no outlier allowance: relative L2 per parameter tensor <= 2e-3 (measured <= 1e-3)."""
    torch.manual_seed(0)
    conf = syn.model_conf(nf, **preset)
    dconf = syn.diffuser_conf(1.0)
    net = FullScoreNetwork(conf, SE3ScoreDiffuser(dconf))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    feats = syn.make_feats(nf, N, seed=11)
    feats["res_mask"][:, -2:] = 0
    # ---- product (GPU), recording the ReLU gates its kernels applied ----
    net = net.cuda()
    gates = _record_gates(net, monkeypatch)
    out_g = net({k: v.cuda() for k, v in feats.items()})
    loss_g = syn.surrogate_loss(out_g)
    loss_g.backward()
    torch.cuda.synchronize()
    monkeypatch.undo()
    # ---- oracle (CPU, fp32), same gates ----
    p = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
    oc = O.default_conf(**preset)
    O.set_gates(gates)
    try:
        out_o = O.full_forward(p, feats, oc, O.default_diffuser_conf(1.0))
    finally:
        O.set_gates(None)
    loss_o = O.surrogate_loss(out_o)
    names = [k for k in p if p[k].requires_grad]
    g_o = dict(zip(names, torch.autograd.grad(loss_o, [p[k] for k in names], allow_unused=True)))
    problems = []
    errs = {}
    for k, tol in (("rigid_update", 1e-4), ("rigids", 1e-4), ("trans_score", 1e-4), ("rot_score", 5e-4), ("unorm_angles", 5e-4)):
        err = _per_residue_l2(out_o[k], out_g[k].cpu())
        errs[k] = err
        if not err < tol:
            problems.append(f"{k} per-residue L2 {err:.3e} >= {tol}")
    # angles = u / |u| is ill-conditioned where |u| ~ 0 (the reference's own fp32 noise shows the same): weigh the error
    # of every angle by its |u|, i.e. compare in the units of the un-normalised prediction
    u = out_o["unorm_angles"].double()
    w = u.norm(dim=-1, keepdim=True)
    err = ((out_o["angles"].double() - out_g["angles"].cpu().double()) * w).flatten(2).norm(dim=-1).max().item()
    errs["angles_u_weighted"] = err
    if not err < 5e-4:
        problems.append(f"angles (|u|-weighted) per-residue L2 {err:.3e} >= 5e-4")
    # atom positions inherit that conditioning through the torsion frames: residues with a well-defined direction only
    ok = (w.squeeze(-1).min(dim=-1).values > 0.05)                       # [nf, N]
    d = (out_o["atom37"].double() - out_g["atom37"].cpu().double()).flatten(2).norm(dim=-1)
    err = float((d * ok).max())
    errs["atom37_conditioned"] = err
    if not err < 2e-3:
        problems.append(f"atom37 per-residue L2 {err:.3e} >= 2e-3 (residues with |u| > 0.05)")
    errs["loss_rel"] = abs(loss_o.item() - loss_g.item()) / max(1.0, abs(loss_o.item()))
    # gradients: relative L2 per parameter tensor (a max-norm would be dominated by the handful of ReLU gates whose
    # pre-activation lies within rounding of zero and flips between the fp32 oracle and the split-bf16 kernels)
    worst = ("", 0.0)
    for k, prm in net.named_parameters():
        go = g_o.get(k)
        if go is None or prm.grad is None:
            assert (go is None or float(go.abs().max()) < 1e-7) and (prm.grad is None or float(prm.grad.abs().max()) < 1e-7), k
            continue
        if go.norm().item() < 1e-7:
            continue
        e = ((go - prm.grad.cpu()).norm() / go.norm()).item()
        if e > worst[1]:
            worst = (k, e)
    errs["worst_grad_rel_l2"] = worst[1]
    errs["worst_grad_name"] = worst[0]
    _record(name, errs)
    assert not problems, f"{name}: " + "; ".join(problems)
    assert errs["loss_rel"] < 1e-4
    assert worst[1] < 2e-3, f"{name}: gradient of {worst[0]} rel L2 err {worst[1]:.3e}"
