"""Generate tests/golden/*.pt from the UNMODIFIED reference (a checkout of it at $DFOLD_REFERENCE_ROOT):

    python oracle/make_golden.py

Each fixture stores, for one seeded case, the reference's outputs (and selected gradients); the inputs and the
weights are NOT stored — they are regenerated from the seed by dynamicpdb_b200.synthetic (make_feats,
random_state) in the tests, which keeps the fixtures small.  Cases cover the network (tiny / preset B / preset A
geometry, with masked residues and a fixed residue), the vanilla OpenFold IPA and StructureModule, and the rigid
algebra on non-unit quaternions.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402

ref_shims.install()
from src.model import Dfold_network_dynamic as RefNet  # noqa: E402
from src.data import se3_diffuser  # noqa: E402
from openfold.model import structure_module as RefSM  # noqa: E402
from openfold.utils import rigid_utils as RefRU  # noqa: E402
from dynamicpdb_b200 import synthetic as syn  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
os.makedirs(OUT, exist_ok=True)

NET_CASES = {
    "net_tiny": dict(preset="PRESET_TINY", nf=3, N=12, seed=3),
    "net_B": dict(preset="PRESET_B", nf=2, N=20, seed=4),
    "net_A": dict(preset="PRESET_A", nf=2, N=16, seed=5),
}


def case_feats(c):
    feats = syn.make_feats(c["nf"], c["N"], seed=c["seed"], loader_dtypes=True)
    feats["res_mask"][:, -2:] = 0
    feats["fixed_mask"][:, 0] = 1
    return feats


def run_net(name, c):
    preset = getattr(syn, c["preset"])
    conf = syn.model_conf(c["nf"], **preset)
    net = RefNet.FullScoreNetwork(conf, se3_diffuser.SE3Diffuser(syn.diffuser_conf(1.0)))
    sd = syn.random_state({k: v.shape for k, v in net.state_dict().items()}, seed=c["seed"] + 100)
    net.load_state_dict(sd)
    out = net(case_feats(c))
    loss = syn.surrogate_loss(out)
    params = dict(net.named_parameters())
    grads = torch.autograd.grad(loss, list(params.values()), allow_unused=True)
    gsel = {}
    for (k, _), g in zip(params.items(), grads):
        if g is None:
            continue
        keep = g.numel() <= 4096 or any(s in k for s in ("bb_update_3", "head_weights", "ipa_0.linear_b.weight"))
        gsel[k] = g.detach().clone() if keep else None
    gnorm = {k: float(g.norm()) for (k, _), g in zip(params.items(), grads) if g is not None}
    torch.save({"case": c, "shapes": {k: tuple(v.shape) for k, v in sd.items()},
                "out": {k: v.detach() for k, v in out.items()}, "loss": float(loss),
                "grads": {k: v for k, v in gsel.items() if v is not None}, "grad_norms": gnorm},
               os.path.join(OUT, name + ".pt"))
    print(name, "loss", float(loss), "params", len(sd))


FRAMES_A256 = [0, 31, 62, 63]


def run_net_big(name="net_A256", nf=64, N=256, seed=7):
    """The BENCHED shape (BASELINE.json configs[2]: preset A, 64 frames x 256 residues), forward only under no_grad
    (the unmodified reference materialises [nf,N,N,H,Pq,3] tensors; ~25 GB peak).  Stores the frames FRAMES_A256 of every
    output but the atom tensors, the last two frames of those, and the surrogate loss over all frames (under 1 MB)."""
    c = dict(preset="PRESET_A", nf=nf, N=N, seed=seed)
    conf = syn.model_conf(nf, **syn.PRESET_A)
    net = RefNet.FullScoreNetwork(conf, se3_diffuser.SE3Diffuser(syn.diffuser_conf(1.0)))
    sd = syn.random_state({k: v.shape for k, v in net.state_dict().items()}, seed=seed + 100)
    net.load_state_dict(sd)
    with torch.no_grad():
        out = net(case_feats(c))
    keep = {}
    for k, v in out.items():
        v = v.detach()
        keep[k] = v[-2:].clone() if k in ("atom37", "atom14") else v[FRAMES_A256].clone()
    torch.save({"case": c, "shapes": {k: tuple(v.shape) for k, v in sd.items()}, "out": keep, "frames": FRAMES_A256,
                "loss": float(syn.surrogate_loss(out))}, os.path.join(OUT, name + ".pt"))
    print(name, "loss", float(syn.surrogate_loss(out)))


def reverse_case():
    """Inputs of the reverse-step fixture (shared with the tests): noised frames, scores, mask; the normal draws come from
    numpy's legacy global stream seeded with 77 — so3 first, then r3, as SE3Diffuser.reverse consumes them."""
    import numpy as np
    F, N = 3, 11
    g = torch.Generator().manual_seed(71)
    rig = syn.make_feats(F, N, seed=9)["rigids_t"]
    rig = torch.cat([rig[..., :4], rig[..., 4:] * 6.0], dim=-1)
    rot_score = torch.randn(F, N, 3, generator=g, dtype=torch.float64) * 0.8
    trans_score = torch.randn(F, N, 3, generator=g, dtype=torch.float64) * 0.5
    mask = (torch.rand(F, N, generator=g) > 0.25).double()
    return dict(rig=rig, rot_score=rot_score, trans_score=trans_score, mask=mask, t=0.37, dt=0.01, noise_scale=0.7, cs=0.1, seed=77)


def run_reverse():
    """SE3Diffuser.reverse of the unmodified reference (se3_diffuser.py:160-215)."""
    import numpy as np
    c = reverse_case()
    diff = se3_diffuser.SE3Diffuser(syn.diffuser_conf(c["cs"]))
    np.random.seed(c["seed"])
    out = diff.reverse(rigid_t=RefRU.Rigid.from_tensor_7(c["rig"]), rot_score=c["rot_score"].numpy(), trans_score=c["trans_score"].numpy(),
                       diffuse_mask=c["mask"].numpy(), t=c["t"], dt=c["dt"], center=True, noise_scale=c["noise_scale"])
    t7 = out.to_tensor_7()
    t7 = torch.cat([torch.where(t7[..., :1] < 0, -t7[..., :4], t7[..., :4]), t7[..., 4:]], dim=-1)     # eigh sign is arbitrary
    torch.save({"rigids_t_1": t7.float()}, os.path.join(OUT, "reverse.pt"))
    print("reverse ok")


def run_vanilla():
    torch.manual_seed(0)
    c_s, c_z, c_h, H, Pq, Pv, N, B = 32, 16, 8, 4, 4, 8, 14, 2
    ipa = RefSM.InvariantPointAttention(c_s, c_z, c_h, H, Pq, Pv)
    sd = syn.random_state({k: v.shape for k, v in ipa.state_dict().items()}, seed=21)
    ipa.load_state_dict(sd)
    g = torch.Generator().manual_seed(22)
    s = torch.randn(B, N, c_s, generator=g)
    z = torch.randn(B, N, N, c_z, generator=g)
    rig7 = torch.cat([torch.nn.functional.normalize(torch.randn(B, N, 4, generator=g), dim=-1),
                      torch.randn(B, N, 3, generator=g) * 5], dim=-1)
    mask = torch.ones(B, N)
    mask[:, -1] = 0
    out = ipa(s, z, RefRU.Rigid.from_tensor_7(rig7), mask)
    sm = RefSM.StructureModule(c_s=c_s, c_z=c_z, c_ipa=c_h, c_resnet=16, no_heads_ipa=H, no_qk_points=Pq, no_v_points=Pv,
                               dropout_rate=0.0, no_blocks=2, no_transition_layers=1, no_resnet_blocks=2, no_angles=7,
                               trans_scale_factor=10, epsilon=1e-8, inf=1e5)
    sm.eval()
    sd2 = syn.random_state({k: v.shape for k, v in sm.state_dict().items()}, seed=23)
    sm.load_state_dict(sd2)
    aatype = torch.randint(0, 20, (B, N), generator=g)
    with torch.no_grad():
        smo = sm({"single": s, "pair": z}, aatype, mask=mask)
    torch.save({"ipa_shapes": {k: tuple(v.shape) for k, v in sd.items()}, "ipa_out": out.detach(),
                "sm_shapes": {k: tuple(v.shape) for k, v in sd2.items()},
                "sm_out": {k: v.detach() for k, v in smo.items()},
                "dims": dict(c_s=c_s, c_z=c_z, c_h=c_h, H=H, Pq=Pq, Pv=Pv, N=N, B=B)},
               os.path.join(OUT, "vanilla.pt"))
    print("vanilla ok")


def run_rigid():
    g = torch.Generator().manual_seed(31)
    q = torch.randn(5, 7, 4, generator=g) * 1.3          # non-unit on purpose
    t = torch.randn(5, 7, 3, generator=g) * 4
    pts = torch.randn(5, 7, 6, 3, generator=g) * 3
    upd = torch.randn(5, 7, 6, generator=g) * 0.4
    m = (torch.rand(5, 7, 1, generator=g) > 0.3).float()
    r = RefRU.Rigid.from_tensor_7(torch.cat([q, t], -1))
    rn = RefRU.Rigid.from_tensor_7(torch.cat([q, t], -1), normalize_quats=True)
    out = {
        "quat_to_rot": RefRU.quat_to_rot(q),
        "apply": r[..., None].apply(pts),
        "invert_apply": r[..., None].invert_apply(pts),
        "compose_q_update": r.compose_q_update_vec(upd, m).to_tensor_7(),
        "compose_q_update_nomask": r.compose_q_update_vec(upd).to_tensor_7(),
        "quat_multiply": RefRU.quat_multiply(q, q.flip(0)),
        "quat_multiply_by_vec": RefRU.quat_multiply_by_vec(q, upd[..., :3]),
        "invert_quat": RefRU.invert_quat(q),
        "rotvec": rn.get_rots().get_rotvec(),
        "compose": rn.compose(RefRU.Rigid.from_tensor_7(torch.cat([q.flip(1), t.flip(1)], -1), normalize_quats=True)).to_tensor_4x4(),
        "invert": rn.invert().to_tensor_7(),
        "from_3_points": RefRU.Rigid.from_3_points(pts[..., 0, :], pts[..., 1, :], pts[..., 2, :]).to_tensor_4x4(),
        "make_transform_from_reference": RefRU.Rigid.make_transform_from_reference(pts[..., 0, :], pts[..., 1, :], pts[..., 2, :]).to_tensor_4x4(),
        "rot_to_quat_abs": RefRU.rot_to_quat(RefRU.quat_to_rot(torch.nn.functional.normalize(q, dim=-1))).abs(),
    }
    torch.save({k: v.detach() for k, v in out.items()}, os.path.join(OUT, "rigid.pt"))
    print("rigid ok")


def run_transitions():
    """§8 row a15: the transition modules the fork defines (ipa_pytorch_dynamic.py:175-239, 519-572)."""
    from src.model import ipa_pytorch_dynamic as RefIpa
    g = torch.Generator().manual_seed(41)
    c, B, N, cz = 32, 2, 9, 16
    s = torch.randn(B, N, c, generator=g)
    e = torch.randn(B, N, N, cz, generator=g)
    mods = {
        "sm_transition": RefIpa.StructureModuleTransition(c),
        "edge_transition": RefIpa.EdgeTransition(node_embed_size=c, edge_embed_in=cz, edge_embed_out=cz),
        "torsion_angles": RefIpa.TorsionAngles(c, 7),
        "score_layer": RefIpa.ScoreLayer(c, c, 6),
    }
    out = {"dims": dict(c=c, B=B, N=N, cz=cz)}
    for i, (k, m) in enumerate(mods.items()):
        sd = syn.random_state({n: v.shape for n, v in m.state_dict().items()}, seed=50 + i)
        m.load_state_dict(sd)
        out[k + "_shapes"] = {n: tuple(v.shape) for n, v in sd.items()}
        with torch.no_grad():
            y = m(s, e) if k == "edge_transition" else m(s)
        out[k] = [t.detach() for t in y] if isinstance(y, tuple) else y.detach()
    torch.save(out, os.path.join(OUT, "transitions.pt"))
    print("transitions ok")


def run_loss():
    """tests/golden/loss.pt: value, aux_data and gradients of the UNMODIFIED Experiment.loss_fn (train_DFOLD_dynamics.py:
    1181-1400) on seeded model outputs, for the plain / separate-rotation / t-below-threshold / gated (>100) variants."""
    from types import SimpleNamespace
    from oracle import dfold_oracle as O
    res = {}
    for name in syn.LOSS_VARIANTS:
        feats, out, separate = syn.loss_variant(name)
        leaves = {k: out[k].clone().requires_grad_(True) for k in ("angles", "rot_score", "rigids")}
        model_out = dict(out, **leaves)
        exp_conf = O.default_exp_conf(separate_rot_loss=separate, bb_atom_loss_weight=1.0,
                                      bb_atom_loss_t_filter=0.25, dist_mat_loss_weight=1.0, dist_mat_loss_t_filter=0.25,
                                      aux_loss_weight=0.25)
        model_conf = SimpleNamespace(cfg_drop_in_train=True, cfg_drop_rate=0.0, embed=SimpleNamespace(embed_self_conditioning=False))
        exp = ref_shims.reference_experiment(lambda batch, drop_ref=False: model_out, None, model_conf, exp_conf,
                                             SimpleNamespace(diffuse_rot=True))
        loss, aux = exp.loss_fn(dict(feats))
        grads = torch.autograd.grad(loss, list(leaves.values()), allow_unused=True)
        res[name] = {"loss": loss.detach(), "aux": {k: a.detach() for k, a in aux.items()},
                     "grads": {k: (g_.detach() if g_ is not None else None) for k, g_ in zip(leaves, grads)}}
        print(f"[golden] loss/{name}: {float(loss):.6f}")
    torch.save(res, os.path.join(OUT, "loss.pt"))


def run_loader():
    """tests/golden/loader.pt: what the UNMODIFIED loader computes for one window of a synthetic trajectory written in the
    reference's on-disk formats: PdbDataset._process_csv_row (src/data/Dfold_data_loader_dynamic.py:192-259) and the
    rigids_0 lines of __getitem__ (:323-330), training-mode window selection with numpy seed 5."""
    import tempfile
    from types import SimpleNamespace
    import numpy as np
    from oracle import synth_traj
    ref_shims.install_trainer_stubs()
    from src.data import Dfold_data_loader_dynamic as L
    traj = synth_traj.make_trajectory()
    with tempfile.TemporaryDirectory() as d:
        row = synth_traj.write_files(traj, d)
        ds = object.__new__(L.PdbDataset)
        ds._is_training = True
        ds._data_conf = SimpleNamespace(frame_time=3, keep_first=8, frame_sample_step=2, fix_sample_start=0)
        np.random.seed(5)
        feats = ds._process_csv_row(row[0], row[1], row[2], None)
    rig = RefRU.Rigid.from_tensor_4x4(feats["rigidgroups_0"])[:, :, 0]
    res = {k: feats[k].clone() for k in ("aatype", "seq_idx", "res_mask", "torsion_angles_sin_cos", "alt_torsion_angles_sin_cos",
                                         "torsion_angles_mask", "force", "vel")}
    res["rigids_0"] = rig.to_tensor_7()
    res["rot_0"] = rig.get_rots().get_rot_mats()
    torch.save(res, os.path.join(OUT, "loader.pt"))
    print("[golden] loader:", {k: tuple(v.shape) for k, v in res.items()})


def boundary_batch():
    """The batch of the boundary fixture (shared with tests/test_cpu_boundary.py)."""
    feats = syn.add_loss_targets(syn.make_feats(3, 12, seed=21, loader_dtypes=True), seed=21)
    feats["fixed_mask"][:, 2] = 1
    return feats


def run_boundary():
    """The reference's own caller: Experiment.loss_fn (train_DFOLD_dynamics.py:1181) driving the reference network on
    boundary_batch() (loss, aux_data, every parameter gradient), and one plain forward of the reference network on
    loader-dtype features (tiny preset, 3 frames x 14 residues).  Weights: synthetic.random_state, seeds 131 / 132."""
    from types import SimpleNamespace
    from oracle import dfold_oracle as O
    ref_shims.install_trainer_stubs()
    diffuser = se3_diffuser.SE3Diffuser(syn.diffuser_conf(1.0))
    net = RefNet.FullScoreNetwork(syn.model_conf(3, **syn.PRESET_TINY), diffuser)
    net.load_state_dict(syn.random_state({k: v.shape for k, v in net.state_dict().items()}, seed=131))
    model_conf = SimpleNamespace(cfg_drop_in_train=True, cfg_drop_rate=0.0, embed=SimpleNamespace(embed_self_conditioning=False))
    exp = ref_shims.reference_experiment(net, diffuser, model_conf, O.default_exp_conf(**BOUNDARY_EXP_CONF),
                                         SimpleNamespace(diffuse_rot=True))
    exp._conf = SimpleNamespace(model=SimpleNamespace(cfg_drop_rate=0.0, cfg_gamma=1.0))
    exp._data_conf = SimpleNamespace(num_t=4, min_t=0.01)
    loss, aux = exp.loss_fn(boundary_batch())
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}
    grad_norms = {k: float(g.norm()) for k, g in grads.items()}
    grads = {k: g for k, g in grads.items() if g.numel() <= 4096}           # small gradients whole, norms of all
    net2 = RefNet.FullScoreNetwork(syn.model_conf(3, **syn.PRESET_TINY), diffuser)
    net2.load_state_dict(syn.random_state({k: v.shape for k, v in net2.state_dict().items()}, seed=132))
    with torch.no_grad():
        fwd = net2(syn.make_feats(3, 14, seed=9, loader_dtypes=True))
    torch.save({"loss": loss.detach(), "aux": {k: v.detach() if torch.is_tensor(v) else v for k, v in aux.items()},
                "grads": grads, "grad_norms": grad_norms, "forward": {k: v.detach() for k, v in fwd.items()}}, os.path.join(OUT, "boundary.pt"))
    print("[golden] boundary: loss", float(loss.detach()), "grads", len(grad_norms))


BOUNDARY_EXP_CONF = dict(bb_atom_loss_weight=1.0, bb_atom_loss_t_filter=0.25, dist_mat_loss_weight=1.0,
                         dist_mat_loss_t_filter=0.25, aux_loss_weight=0.25)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "boundary":
        run_boundary()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "loader":
        run_loader()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "loss":
        run_loss()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "big":
        run_net_big()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "reverse":
        run_reverse()
        sys.exit(0)
    run_reverse()
    run_loss()
    run_loader()
    run_transitions()
    for n, c in NET_CASES.items():
        run_net(n, c)
    run_vanilla()
    run_rigid()
    run_boundary()
