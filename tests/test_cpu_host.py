"""CPU: the product's host-side logic (module wiring, autograd plumbing, state_dict ABI, rigid_utils API, C-ABI
surface) — the arithmetic is routed to the oracle through the `oracle_ops` test fixture; no CUDA kernel runs here."""
import ctypes
import os
import re
import subprocess
import sys

import pytest
import torch

from dynamicpdb_b200 import kernels
from dynamicpdb_b200 import rigid_utils as ru
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from tests.test_cpu_oracle import NET_CASES, case_inputs, close, load

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name", NET_CASES)
def test_network_host_logic_matches_reference_golden(name, oracle_ops):
    g = load(name)
    feats, state, preset = case_inputs(g)
    net = FullScoreNetwork(syn.model_conf(g["case"]["nf"], **preset), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    net.load_state_dict(state, strict=True)                      # state_dict ABI: same 142 names and shapes
    assert {k: tuple(v.shape) for k, v in net.state_dict().items()} == g["shapes"]
    out = net(dict(feats))
    for k, ref in g["out"].items():
        assert out[k].dtype == ref.dtype, (k, out[k].dtype, ref.dtype)
        assert close(out[k], ref, 2e-5), f"{name}: output {k}"
    loss = syn.surrogate_loss(out)
    loss.backward()
    params = dict(net.named_parameters())
    for k, ref in g["grads"].items():
        if ref.abs().max() < 1e-7:
            continue
        assert ((params[k].grad - ref).norm() / ref.norm()).item() < 2e-3, f"{name}: grad {k}"
    for k, n in g["grad_norms"].items():
        if n > 1e-6:
            assert abs(params[k].grad.norm().item() - n) < 5e-3 * n, f"{name}: |grad {k}|"
    # parameters the reference leaves without gradient (dead-output embedder, linear_rbf) stay without one
    assert all(params[k].grad is None for k in params if k.startswith("embedding_layer."))


def test_rigid_utils_api_matches_reference_golden():
    g = load("rigid")
    gen = torch.Generator().manual_seed(31)
    q = torch.randn(5, 7, 4, generator=gen) * 1.3
    t = torch.randn(5, 7, 3, generator=gen) * 4
    pts = torch.randn(5, 7, 6, 3, generator=gen) * 3
    upd = torch.randn(5, 7, 6, generator=gen) * 0.4
    m = (torch.rand(5, 7, 1, generator=gen) > 0.3).float()
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
        assert close(got[k], ref, 1e-5), k
    with pytest.raises(ValueError):
        ru.Rotation(rot_mats=None, quats=None)
    with pytest.raises(ValueError):
        ru.Rigid.from_tensor_7(torch.zeros(3, 6))
    with pytest.raises(ValueError):
        ru.rot_to_quat(torch.zeros(3, 4))
    assert r[2, 3:5].shape == (2,) and r.unsqueeze(-1).shape == (5, 7, 1)
    assert ru.Rigid.cat([r, r], dim=0).shape == (10, 7)


def test_vanilla_structure_module_matches_reference_golden(oracle_ops):
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
    assert close(ipa(s, z, ru.Rigid.from_tensor_7(rig7), mask), g["ipa_out"], 2e-5)
    sm = SM.StructureModule(c_s=d["c_s"], c_z=d["c_z"], c_ipa=d["c_h"], c_resnet=16, no_heads_ipa=d["H"], no_qk_points=d["Pq"],
                            no_v_points=d["Pv"], dropout_rate=0.0, no_blocks=2, no_transition_layers=1, no_resnet_blocks=2,
                            no_angles=7, trans_scale_factor=10, epsilon=1e-8, inf=1e5)
    sm.eval()
    sm.load_state_dict(syn.random_state(g["sm_shapes"], seed=23), strict=True)
    aatype = torch.randint(0, 20, (d["B"], d["N"]), generator=gen)
    with torch.no_grad():
        out = sm({"single": s, "pair": z}, aatype, mask=mask)
    for k, ref in g["sm_out"].items():
        assert close(out[k], ref, 5e-5), k


def test_c_abi_exports_every_declared_symbol():
    header = open(os.path.join(ROOT, "include", "dfold_b200.h")).read()
    declared = set(re.findall(r"\b(dfold_\w+)\s*\(", header))
    assert len(declared) >= 20
    L = kernels.lib()                                 # loads without a GPU
    for name in declared:
        assert isinstance(getattr(L, name), ctypes._CFuncPtr), name
    assert declared == set(kernels.exported_symbols())
    assert L.dfold_abi_version() == 4


def test_ctypes_signatures_match_the_header():
    """kernels._SIGS (p pointer, l long, i int, f float, d double) must agree, argument by argument, with include/dfold_b200.h."""
    header = open(os.path.join(ROOT, "include", "dfold_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    for name, args in re.findall(r"\bint\s+(dfold_\w+)\s*\((.*?)\)\s*;", header, flags=re.S):
        sig = ""
        for a in [x.strip() for x in args.split(",")]:
            if a == "void":
                continue
            sig += "p" if "*" in a else ("l" if a.startswith("long") else ("i" if a.startswith("int") else ("f" if a.startswith("float") else ("d" if a.startswith("double") else "?"))))
        assert kernels._SIGS[name] == sig, (name, kernels._SIGS[name], sig)


def test_ops_refuse_cpu_tensors():
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        kernels.linear(torch.zeros(4, 8), torch.zeros(3, 8))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        kernels.global_layernorm(torch.zeros(2, 3, 4))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        kernels.conv5x5(torch.zeros(2, 8, 8), torch.zeros(8, 8, 5, 5))
    # the widened rows (loss, input featurisation) have no host path either
    from dynamicpdb_b200 import synthetic as syn
    from dynamicpdb_b200.input_pipeline import featurize_window
    from dynamicpdb_b200.loss import score_network_loss
    from oracle import dfold_oracle as O
    feats, out, _ = syn.loss_variant("plain")
    with pytest.raises(RuntimeError, match="no CPU path"):
        score_network_loss(out, feats, O.default_exp_conf())
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        featurize_window(torch.zeros(2, 5, 37, 3), torch.ones(5, 37), torch.zeros(5, dtype=torch.long))


def _skeleton_reference(root):
    """A stand-in for the original project's package layout (namespace packages src / src.model / src.data /
    openfold.utils, regular packages openfold / openfold.model / openfold.np): one marker module per file."""
    files = ["src/model/ipa_pytorch_dynamic.py", "src/model/Dfold_network_dynamic.py", "src/model/utils.py",
             "src/data/se3_diffuser.py", "openfold/__init__.py", "openfold/model/__init__.py",
             "openfold/model/structure_module.py", "openfold/np/__init__.py", "openfold/np/residue_constants.py",
             "openfold/utils/rigid_utils.py", "openfold/utils/tensor_utils.py"]
    for f in files:
        path = os.path.join(root, f)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "w") as fh:
            fh.write("SKELETON = True\n")


def test_import_overlay_shadows_only_the_hot_path(tmp_path):
    """overlay/ first on sys.path: the four hot-path modules resolve to the overlay, everything else of the reference
    (here a skeleton of its layout) still resolves to the reference tree."""
    ref = str(tmp_path / "reference")
    _skeleton_reference(ref)
    code = ("import sys; sys.path[:0]=[%r, %r]; from oracle import ref_shims; ref_shims.install();"
            "import src.model.ipa_pytorch_dynamic as a, src.model.Dfold_network_dynamic as b, openfold.utils.rigid_utils as c,"
            "openfold.model.structure_module as d, src.data.se3_diffuser as e, openfold.np.residue_constants as f,"
            "openfold.utils.tensor_utils as g, src.model.utils as h; "
            "print(a.__file__, b.__file__, c.__file__, d.__file__, e.__file__, f.__file__, g.__file__, h.__file__)"
            ) % (os.path.join(ROOT, "overlay"), ROOT)
    env = dict(os.environ, DFOLD_REFERENCE_ROOT=ref)
    out = subprocess.run([sys.executable, "-W", "ignore", "-c", code], capture_output=True, text=True, timeout=300, env=env)
    assert out.returncode == 0, out.stderr[-2000:]
    paths = out.stdout.split()[-8:]
    overlay = os.path.join(ROOT, "overlay") + os.sep
    assert all(p.startswith(overlay) for p in paths[:4]), paths
    assert all(p.startswith(ref + os.sep) for p in paths[4:]), paths


def test_dead_frame_elimination_is_exact(oracle_ops, monkeypatch):
    """Cropping the ConvNet input of the middle blocks to the last 17 frames changes neither outputs nor gradients."""
    from dynamicpdb_b200 import ipa_pytorch_dynamic as ipd
    nf, N = 21, 6
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(nf, **syn.PRESET_TINY), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    feats = syn.make_feats(nf, N, seed=2)
    res = {}
    for skip in (True, False):
        monkeypatch.setattr(ipd, "_DEAD_FRAME_SKIP", skip)
        net.zero_grad(set_to_none=True)
        out = net(dict(feats))
        syn.surrogate_loss(out).backward()
        res[skip] = ({k: v.detach().clone() for k, v in out.items()},
                     {k: p.grad.clone() for k, p in net.named_parameters() if p.grad is not None})
    for k in res[True][0]:
        assert close(res[True][0][k], res[False][0][k], 1e-6), k
    for k in res[False][1]:
        a, b = res[True][1][k], res[False][1][k]
        assert (a - b).norm() <= 1e-5 * (b.norm() + 1e-12), k


def test_memoized_inference_matches_repeated_forward(oracle_ops):
    """Trunk memoisation across reverse-diffusion steps (only t / rigids_t change) reproduces the full forward."""
    from dynamicpdb_b200.inference import MemoizedScoreNetwork
    nf, N = 3, 10
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(nf, **syn.PRESET_TINY), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    memo = MemoizedScoreNetwork(net)
    feats = syn.make_feats(nf, N, seed=6)
    for step, tval in enumerate((1.0, 0.6, 0.05)):
        feats = dict(feats)
        feats["t"] = torch.tensor([tval])
        feats["rigids_t"] = syn.make_feats(nf, N, seed=100 + step)["rigids_t"]
        with torch.no_grad():
            full = net(dict(feats))
        fast = memo(dict(feats))
        for k in full:
            assert close(fast[k], full[k], 1e-6), (step, k)


def test_transition_modules_match_reference_golden(oracle_ops):
    """SURVEY.md §8 row a15: StructureModuleTransition / EdgeTransition / TorsionAngles / ScoreLayer of the fork."""
    from dynamicpdb_b200 import ipa_pytorch_dynamic as ipd
    from oracle import dfold_oracle as O
    g = load("transitions")
    d = g["dims"]
    gen = torch.Generator().manual_seed(41)
    s = torch.randn(d["B"], d["N"], d["c"], generator=gen)
    e = torch.randn(d["B"], d["N"], d["N"], d["cz"], generator=gen)
    mods = {
        "sm_transition": ipd.StructureModuleTransition(d["c"]),
        "edge_transition": ipd.EdgeTransition(node_embed_size=d["c"], edge_embed_in=d["cz"], edge_embed_out=d["cz"]),
        "torsion_angles": ipd.TorsionAngles(d["c"], 7),
        "score_layer": ipd.ScoreLayer(d["c"], d["c"], 6),
    }
    for i, (k, m) in enumerate(mods.items()):
        sd = syn.random_state(g[k + "_shapes"], seed=50 + i)
        m.load_state_dict(sd, strict=True)
        with torch.no_grad():
            y = m(s, e) if k == "edge_transition" else m(s)
        ys = list(y) if isinstance(y, tuple) else [y]
        refs = g[k] if isinstance(g[k], list) else [g[k]]
        for a, b in zip(ys, refs):
            assert close(a, b, 2e-5), k
        # the oracle restatement of the same modules
        if k == "sm_transition":
            assert close(O.sm_transition({"m." + n: v for n, v in sd.items()}, "m", s), g[k], 2e-5)
        if k == "edge_transition":
            assert close(O.edge_transition({"m." + n: v for n, v in sd.items()}, "m", s, e), g[k], 2e-5)
