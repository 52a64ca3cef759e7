"""-m gpu: the product on CUDA against outputs of the UNMODIFIED reference (tests/golden/*.pt, written by
oracle/make_golden.py from a checkout of the reference).  No oracle in between: these are the
reference's own numbers.

  * net_tiny / net_B / net_A      FullScoreNetwork outputs + selected gradients (masked residues, one fixed residue)
  * net_A256                      the BENCHED shape, BASELINE.json configs[2]: preset A, 64 frames x 256 residues, forward
  * vanilla                       openfold.model.structure_module.InvariantPointAttention / StructureModule (rows a4, a16)
  * transitions                   StructureModuleTransition / EdgeTransition / TorsionAngles / ScoreLayer (row a15)
  * rigid                         the rigid_utils API on CUDA tensors (rows a8-a10)
"""
import pytest
import torch

from dynamicpdb_b200 import rigid_utils as ru
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from tests.test_cpu_oracle import case_inputs, load
from tests.test_gpu_model import _per_residue_l2, _record

pytestmark = pytest.mark.gpu
DEV = "cuda"


def close(a, b, tol):
    a, b = a.detach().double().cpu(), b.double()
    return (a - b).abs().max().item() <= tol * max(1.0, b.abs().max().item())


def _net_on_gpu(g):
    feats, state, preset = case_inputs(g)
    net = FullScoreNetwork(syn.model_conf(g["case"]["nf"], **preset), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    net.load_state_dict(state, strict=True)
    return net.to(DEV), {k: v.to(DEV) for k, v in feats.items()}


@pytest.mark.parametrize("name", ["net_tiny", "net_B", "net_A"])
def test_network_matches_reference_golden_on_gpu(name):
    g = load(name)
    net, feats = _net_on_gpu(g)
    out = net(feats)
    errs = {}
    for k, tol in (("rigid_update", 1e-4), ("rigids", 1e-4), ("trans_score", 1e-4), ("rot_score", 1e-4), ("unorm_angles", 1e-4)):
        assert out[k].dtype == g["out"][k].dtype, (k, out[k].dtype)
        errs[k] = _per_residue_l2(g["out"][k], out[k].detach().cpu())
        assert errs[k] < tol, f"{name}: {k} per-residue L2 {errs[k]:.3e}"
    for k in ("angles", "atom37", "atom14"):
        errs[k] = _per_residue_l2(g["out"][k], out[k].detach().cpu())
    loss = syn.surrogate_loss(out)
    loss.backward()
    assert abs(loss.item() - g["loss"]) < 1e-4 * max(1.0, abs(g["loss"]))
    params = dict(net.named_parameters())
    worst = 0.0
    for k, ref in g["grads"].items():
        if ref.abs().max() < 1e-7:
            continue
        e = ((params[k].grad.cpu() - ref).norm() / ref.norm()).item()
        worst = max(worst, e)
        assert e < 5e-3, f"{name}: grad {k} rel L2 {e:.3e}"
    for k, n in g["grad_norms"].items():
        if n > 1e-6:
            assert abs(params[k].grad.norm().item() - n) < 5e-3 * n, f"{name}: |grad {k}|"
    errs["worst_grad_rel_l2"] = worst
    _record("golden_" + name, errs)
    assert all(params[k].grad is None for k in params if k.startswith("embedding_layer."))


def test_benched_shape_matches_reference_golden():
    """Preset A, 64 frames x 256 residues (the shape bench.py times): every output of the unmodified reference's forward.
    The reference itself shows 1.4e-6 / 4.7e-6 / 1.5e-5 / 3.3e-5 per-residue noise on rigid_update / rigids / rot_score /
    atom37 between thread counts (SURVEY.md 8c)."""
    g = load("net_A256")
    net, feats = _net_on_gpu(g)
    with torch.no_grad():
        out = net(feats)
    torch.cuda.synchronize()
    errs = {}
    fr = g["frames"]                                   # the fixture keeps a fixed sample of the 64 frames
    assert fr[-2:] == [62, 63]
    for k, tol in (("rigid_update", 1e-4), ("rigids", 1e-4), ("trans_score", 1e-4), ("rot_score", 2e-4), ("unorm_angles", 2e-4)):
        ref = g["out"][k]
        assert tuple(out[k].shape[1:]) == tuple(ref.shape[1:]) and out[k].shape[0] == 64 and out[k].dtype == ref.dtype, k
        errs[k] = _per_residue_l2(ref, out[k][fr].cpu())
    # normalised angles / atoms: conditioned on |u| as in test_gpu_model.py
    u = g["out"]["unorm_angles"].double()
    w = u.norm(dim=-1, keepdim=True)
    errs["angles_u_weighted"] = ((g["out"]["angles"].double() - out["angles"][fr].cpu().double()) * w).flatten(2).norm(dim=-1).max().item()
    ok = (w.squeeze(-1).min(dim=-1).values > 0.05)[-2:]
    d = (g["out"]["atom37"].double() - out["atom37"][-2:].cpu().double()).flatten(2).norm(dim=-1)
    errs["atom37_conditioned"] = float((d * ok).max())
    loss = float(syn.surrogate_loss(out))
    errs["loss_rel"] = abs(loss - g["loss"]) / max(1.0, abs(g["loss"]))
    _record("golden_net_A256_nf64", errs)
    for k, tol in (("rigid_update", 1e-4), ("rigids", 1e-4), ("trans_score", 1e-4), ("rot_score", 2e-4), ("unorm_angles", 2e-4),
                   ("angles_u_weighted", 5e-4), ("atom37_conditioned", 2e-3), ("loss_rel", 1e-4)):
        assert errs[k] < tol, f"net_A256: {k} {errs[k]:.3e} >= {tol}"


def test_vanilla_ipa_and_structure_module_on_gpu():
    """Rows a4 / a16: the vendored OpenFold modules with their own signatures, on CUDA."""
    from dynamicpdb_b200 import structure_module as SM
    g = load("vanilla")
    d = g["dims"]
    gen = torch.Generator().manual_seed(22)
    s = torch.randn(d["B"], d["N"], d["c_s"], generator=gen)
    z = torch.randn(d["B"], d["N"], d["N"], d["c_z"], generator=gen)
    rig7 = torch.cat([torch.nn.functional.normalize(torch.randn(d["B"], d["N"], 4, generator=gen), dim=-1),
                      torch.randn(d["B"], d["N"], 3, generator=gen) * 5], dim=-1)
    mask = torch.ones(d["B"], d["N"])
    mask[:, -1] = 0
    ipa = SM.InvariantPointAttention(d["c_s"], d["c_z"], d["c_h"], d["H"], d["Pq"], d["Pv"])
    ipa.load_state_dict(syn.random_state(g["ipa_shapes"], seed=21), strict=True)
    ipa = ipa.to(DEV)
    s_g, z_g, mask_g = s.to(DEV).requires_grad_(True), z.to(DEV).requires_grad_(True), mask.to(DEV)
    y = ipa(s_g, z_g, ru.Rigid.from_tensor_7(rig7.to(DEV)), mask_g)
    assert close(y, g["ipa_out"], 5e-5)
    y.square().sum().backward()                     # the autograd path of the module API runs on CUDA too
    assert torch.isfinite(s_g.grad).all() and torch.isfinite(z_g.grad).all() and float(z_g.grad.abs().max()) > 0
    # inplace_safe / offload keywords are accepted (ref structure_module.py:231-260)
    y2 = ipa(s_g, None, ru.Rigid.from_tensor_7(rig7.to(DEV)), mask_g, inplace_safe=True, _offload_inference=True,
             _z_reference_list=[z_g])
    assert close(y2, g["ipa_out"], 5e-5)

    sm = SM.StructureModule(c_s=d["c_s"], c_z=d["c_z"], c_ipa=d["c_h"], c_resnet=16, no_heads_ipa=d["H"], no_qk_points=d["Pq"],
                            no_v_points=d["Pv"], dropout_rate=0.0, no_blocks=2, no_transition_layers=1, no_resnet_blocks=2,
                            no_angles=7, trans_scale_factor=10, epsilon=1e-8, inf=1e5)
    sm.eval()
    sm.load_state_dict(syn.random_state(g["sm_shapes"], seed=23), strict=True)
    sm = sm.to(DEV)
    aatype = torch.randint(0, 20, (d["B"], d["N"]), generator=gen)
    with torch.no_grad():
        out = sm({"single": s.to(DEV), "pair": z.to(DEV)}, aatype.to(DEV), mask=mask_g)
    assert set(out) == set(g["sm_out"])
    for k, ref in g["sm_out"].items():
        assert close(out[k], ref, 1e-4), k


def test_transition_modules_on_gpu():
    """Row a15: the fork's transition modules on CUDA against the reference's outputs."""
    from dynamicpdb_b200 import ipa_pytorch_dynamic as ipd
    g = load("transitions")
    d = g["dims"]
    gen = torch.Generator().manual_seed(41)
    s = torch.randn(d["B"], d["N"], d["c"], generator=gen).to(DEV)
    e = torch.randn(d["B"], d["N"], d["N"], d["cz"], generator=gen).to(DEV)
    mods = {
        "sm_transition": ipd.StructureModuleTransition(d["c"]),
        "edge_transition": ipd.EdgeTransition(node_embed_size=d["c"], edge_embed_in=d["cz"], edge_embed_out=d["cz"]),
        "torsion_angles": ipd.TorsionAngles(d["c"], 7),
        "score_layer": ipd.ScoreLayer(d["c"], d["c"], 6),
    }
    for i, (k, m) in enumerate(mods.items()):
        m.load_state_dict(syn.random_state(g[k + "_shapes"], seed=50 + i), strict=True)
        m = m.to(DEV)
        sg = s.clone().requires_grad_(True)
        y = m(sg, e) if k == "edge_transition" else m(sg)
        ys = list(y) if isinstance(y, tuple) else [y]
        refs = g[k] if isinstance(g[k], list) else [g[k]]
        for a, b in zip(ys, refs):
            assert close(a, b, 5e-5), k
        sum(t.square().sum() for t in ys).backward()
        assert torch.isfinite(sg.grad).all() and float(sg.grad.abs().max()) > 0, k
    # the OpenFold StructureModuleTransition (structure_module.py:489-512)
    from dynamicpdb_b200 import structure_module as SM
    t = SM.StructureModuleTransition(d["c"], 2, 0.0).to(DEV).eval()
    assert t(s).shape == s.shape


def test_rigid_utils_api_on_gpu():
    """Rows a8-a10: every rigid_utils entry point of the golden on CUDA tensors."""
    g = load("rigid")
    gen = torch.Generator().manual_seed(31)
    q = (torch.randn(5, 7, 4, generator=gen) * 1.3).to(DEV)
    t = (torch.randn(5, 7, 3, generator=gen) * 4).to(DEV)
    pts = (torch.randn(5, 7, 6, 3, generator=gen) * 3).to(DEV)
    upd = (torch.randn(5, 7, 6, generator=gen) * 0.4).to(DEV)
    m = (torch.rand(5, 7, 1, generator=gen) > 0.3).float().to(DEV)
    r = ru.Rigid.from_tensor_7(torch.cat([q, t], -1))
    rn = ru.Rigid.from_tensor_7(torch.cat([q, t], -1), normalize_quats=True)
    got = {
        "quat_to_rot": ru.quat_to_rot(q),
        "apply": r[..., None].apply(pts),
        "invert_apply": r[..., None].invert_apply(pts),
        "compose_q_update": r.compose_q_update_vec(upd, m).to_tensor_7(),
        "compose_q_update_nomask": r.compose_q_update_vec(upd).to_tensor_7(),
        "quat_multiply": ru.quat_multiply(q, q.flip(0)),
        "quat_multiply_by_vec": ru.quat_multiply_by_vec(q, upd[..., :3]),
        "invert_quat": ru.invert_quat(q),
        "rotvec": rn.get_rots().get_rotvec(),
        "compose": rn.compose(ru.Rigid.from_tensor_7(torch.cat([q.flip(1), t.flip(1)], -1), normalize_quats=True)).to_tensor_4x4(),
        "invert": rn.invert().to_tensor_7(),
        "from_3_points": ru.Rigid.from_3_points(pts[..., 0, :], pts[..., 1, :], pts[..., 2, :]).to_tensor_4x4(),
        "make_transform_from_reference": ru.Rigid.make_transform_from_reference(pts[..., 0, :], pts[..., 1, :], pts[..., 2, :]).to_tensor_4x4(),
        "rot_to_quat_abs": ru.rot_to_quat(ru.quat_to_rot(torch.nn.functional.normalize(q, dim=-1))).abs(),
    }
    for k, ref in g.items():
        assert got[k].is_cuda, k
        assert close(got[k], ref, 2e-5), k
