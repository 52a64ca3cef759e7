"""Seeded synthetic inputs and configs for the DFOLDv2 score network (SURVEY.md §8d, Appendix B).

Used by bench.py, __graft_entry__.smoke() and the tests; no dynamicPDB data exists in the container.
Shapes follow the batch dict that reaches ``FullScoreNetwork.forward`` after the trainer's
``[B,F,...] -> [B*F,...]`` flatten with B=1 (train_DFOLD_dynamics.py:680-684).
"""
import math
from types import SimpleNamespace
from typing import Dict

import torch


def model_conf(nf: int, *, c_s=256, c_z=128, c_hidden=256, no_heads=8, no_qk_points=8, no_v_points=12,
               num_blocks=4, coordinate_scaling=1.0) -> SimpleNamespace:
    """Attribute-style config with the fields the model reads (config/train_DFOLDv2.yaml:65-104)."""
    ipa = SimpleNamespace(c_s=c_s, c_z=c_z, c_hidden=c_hidden, no_heads=no_heads, no_qk_points=no_qk_points,
                          no_v_points=no_v_points, num_blocks=num_blocks, coordinate_scaling=coordinate_scaling)
    embed = SimpleNamespace(DFOLDv2_embedder=True, index_embed_size=32)
    return SimpleNamespace(node_embed_size=c_s, edge_embed_size=c_z, frame_time=nf, embed=embed, ipa=ipa)


PRESET_A = dict(c_s=256, c_z=128, c_hidden=256, no_heads=8, no_qk_points=8, no_v_points=12)   # train_DFOLDv2.yaml
PRESET_B = dict(c_s=256, c_z=128, c_hidden=16, no_heads=12, no_qk_points=4, no_v_points=8)    # train_DFOLDv2_new.yaml
PRESET_TINY = dict(c_s=32, c_z=16, c_hidden=8, no_heads=2, no_qk_points=2, no_v_points=3)     # fast CPU tests


def diffuser_conf(coordinate_scaling: float = 1.0) -> SimpleNamespace:
    """config/train_DFOLDv2.yaml:43-63 (run_train.sh:24 overrides coordinate_scaling to 1.0)."""
    so3 = SimpleNamespace(num_omega=1000, num_sigma=1000, min_sigma=0.1, max_sigma=1.5,
                          schedule="logarithmic", cache_dir="/tmp/dfold_igso3_cache", use_cached_score=False)
    r3 = SimpleNamespace(min_b=0.1, max_b=20.0, coordinate_scaling=coordinate_scaling)
    return SimpleNamespace(diffuse_trans=True, diffuse_rot=True, r3=r3, so3=so3)


def _unit(x):
    return x / torch.linalg.norm(x, dim=-1, keepdim=True)


def _quat_mul(a, b):
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                        aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], dim=-1)


def make_feats(nf: int, n_res: int, *, seed: int = 0, node_dim: int = 256, edge_dim: int = 128, t: float = 0.5,
               coordinate_scaling: float = 1.0, device="cpu", loader_dtypes: bool = False) -> Dict[str, torch.Tensor]:
    """One protein window of ``nf`` consecutive trajectory frames.

    Frame 0: random unit quaternions on a 3.8 A C-alpha random walk (centred); frame f = frame f-1 composed with a
    small rigid motion (rotvec sigma 0.02 rad, translation sigma 0.1 A), i.e. ~1 ps MD spacing.
    ``loader_dtypes=True`` reproduces the float64 fields the reference's loader emits (Appendix B).
    """
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)
    q = _unit(rn(n_res, 4))
    steps = _unit(rn(n_res, 3)) * 3.8
    ca = torch.cumsum(steps, dim=0)
    ca = ca - ca.mean(0, keepdim=True)
    rig = [torch.cat([q, ca], dim=-1)]
    for _ in range(1, nf):
        rv = rn(n_res, 3) * 0.02
        ang = torch.linalg.norm(rv, dim=-1, keepdim=True)
        dq = torch.cat([torch.cos(ang / 2), rv / ang * torch.sin(ang / 2)], dim=-1)
        q = _unit(_quat_mul(q, dq))
        ca = ca + rn(n_res, 3) * 0.1
        rig.append(torch.cat([q, ca], dim=-1))
    rigids_0 = torch.stack(rig, dim=0)
    rigids_t = torch.cat([_unit(rn(nf, n_res, 4)), rn(nf, n_res, 3) / coordinate_scaling], dim=-1)
    ang = rn(nf, n_res, 7) * math.pi
    f64 = torch.float64 if loader_dtypes else torch.float32
    feats = {
        "res_mask": torch.ones(nf, n_res),
        "fixed_mask": torch.zeros(nf, n_res),
        "seq_idx": torch.arange(1, n_res + 1).unsqueeze(0).repeat(nf, 1),
        "t": torch.tensor([t], dtype=f64),
        "rigids_0": rigids_0,
        "rigids_t": rigids_t,
        "force": rn(nf, n_res, 3).to(f64),
        "vel": rn(nf, n_res, 3).to(f64),
        "node_repr": rn(n_res, node_dim),
        "edge_repr": rn(n_res, n_res, edge_dim),
        "torsion_angles_sin_cos": torch.stack([torch.sin(ang), torch.cos(ang)], dim=-1).to(f64),
        "torsion_angles_mask": torch.ones(nf, n_res, 7, dtype=f64),
        "aatype": torch.randint(0, 20, (nf, n_res), generator=g),
        "sc_ca_t": torch.zeros(nf, n_res, 3),
    }
    return {k: v.to(device) for k, v in feats.items()}


def random_state(shapes: Dict[str, tuple], seed: int = 0) -> Dict[str, torch.Tensor]:
    """Deterministic weights for every tensor of a ``state_dict`` given only names and shapes (so golden fixtures
    need not store weights): weights ~ N(0, 1/fan_in) (x0.1 for the reference's zero-initialised 'final' layers),
    biases ~ N(0, 0.1^2), LayerNorm weights 1 + N(0, 0.1^2), IPA head weights around softplus^-1(1)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k in sorted(shapes):
        shp = tuple(shapes[k])
        r = torch.randn(shp, generator=g)
        if k.endswith("head_weights"):
            v = 0.5413 + 0.2 * r
        elif k.endswith(".bias"):
            v = 0.1 * r
        elif len(shp) == 1:                                   # LayerNorm weight
            v = 1.0 + 0.1 * r
        else:
            fan_in = 1
            for d in shp[1:]:
                fan_in *= d
            v = r / math.sqrt(max(1, fan_in))
            if any(s in k for s in ("bb_update", "linear_out", "linear_2", "linear_3", "final_layer")):
                v = v * 0.1
        out[k] = v
    return out


def dezero_(state: Dict[str, torch.Tensor], seed: int = 1, std: float = 0.02) -> None:
    """Redraw every all-zero *weight* (the reference's 'final' init: IPA linear_out, bb_update, AngleResnet
    linear_2) from N(0, std^2) so parity is not vacuous (SURVEY.md §8d)."""
    g = torch.Generator().manual_seed(seed)
    for k in sorted(state):
        v = state[k]
        if k.endswith("weight") and v.dtype.is_floating_point and v.numel() > 0 and not bool(v.any()):
            v.copy_(torch.randn(v.shape, generator=g) * std)


def surrogate_loss(out: Dict[str, torch.Tensor]) -> torch.Tensor:
    """Mean squares of the trained-on outputs (SURVEY.md §8d); the reference's loss_fn needs the trainer.
    The L2-normalised ``angles`` are left out: u/|u| is ill-conditioned where |u| ~ 0 and would dominate the
    gradient comparison."""
    return ((out["rigids"] ** 2).mean() + (out["unorm_angles"] ** 2).mean()
            + (out["rot_score"].float() ** 2).mean() + (out["trans_score"].float() ** 2).mean())


def add_loss_targets(feats: Dict[str, torch.Tensor], *, seed: int = 0, loader_dtypes: bool = True) -> Dict[str, torch.Tensor]:
    """The extra batch fields ``Experiment.loss_fn`` reads (SURVEY.md Appendix B): alternative torsion targets, the
    ground-truth scores and their scalings (float64 from the numpy diffuser in the reference's loader)."""
    g = torch.Generator().manual_seed(1000 + seed)
    nf, n_res = feats["res_mask"].shape
    f64 = torch.float64 if loader_dtypes else torch.float32
    out = dict(feats)
    sc = feats["torsion_angles_sin_cos"].cpu()
    flip = (torch.rand(nf, n_res, 7, generator=g) > 0.5).to(sc.dtype)[..., None]
    dev = feats["res_mask"].device
    out["alt_torsion_angles_sin_cos"] = (sc * (1 - 2 * flip)).to(dev)          # pi-periodic alternative (openfold convention)
    out["rot_score"] = (torch.randn(nf, n_res, 3, generator=g) * 0.7).to(f64).to(dev)
    out["trans_score"] = torch.randn(nf, n_res, 3, generator=g).to(f64).to(dev)
    out["rot_score_scaling"] = torch.tensor([0.8], dtype=f64, device=dev)
    out["trans_score_scaling"] = torch.tensor([1.3], dtype=f64, device=dev)
    return out


def loss_case(seed: int = 11, nf: int = 3, N: int = 14):
    """Seeded (batch, model_out) pair for the loss fixtures tests/golden/loss.pt (oracle/make_golden.py run_loss): a fixed
    residue, masked residues, masked torsions and one zero-length predicted torsion vector."""
    g = torch.Generator().manual_seed(seed)
    feats = add_loss_targets(make_feats(nf, N, seed=seed, loader_dtypes=True), seed=seed)
    feats["fixed_mask"][:, 1] = 1
    feats["res_mask"][:, -2:] = 0
    feats["torsion_angles_mask"][:, :, 5:] = 0
    out = {"angles": torch.randn(nf, N, 7, 2, generator=g) * 0.8, "rot_score": torch.randn(nf, N, 3, generator=g, dtype=torch.float64),
           "rigids": torch.cat([torch.randn(nf, N, 4, generator=g), feats["rigids_0"][..., 4:] + torch.randn(nf, N, 3, generator=g)], dim=-1),
           "trans_score": torch.randn(nf, N, 3, generator=g), "atom37": torch.randn(nf, N, 37, 3, generator=g)}
    out["angles"][-1, 0, 0] = 0.0                                     # |u| = 0: the reference's eps-guarded normalisation
    return feats, out


# variants of the loss case: separate axis / angle rotation loss, t below rot_loss_t_threshold, translation loss above the 100 gate
LOSS_VARIANTS = {"plain": dict(), "separate": dict(separate_rot_loss=True), "t_low": dict(t=0.1), "far": dict(shift=30.0)}


def loss_variant(name: str):
    """(batch, model_out, separate_rot_loss) of one variant."""
    v = LOSS_VARIANTS[name]
    feats, out = loss_case()
    if "t" in v:
        feats["t"] = torch.tensor([v["t"]], dtype=torch.float64)
    if "shift" in v:
        out["rigids"][..., 4:] += v["shift"]
    return feats, out, v.get("separate_rot_loss", False)


# edge cases of the loss (tests/golden/loss_edges.pt, oracle/make_loss_edges_golden.py), each an edit of one variant:
#   zero_torsion_alt_gt   the zero-length predicted torsion [-1, 0, 0] with alternative == target (torsions 0-2 and chis
#                         that are not pi-periodic): the reference's gradient there is w / 1e-8
#   zero_torsion_alt_neg  the same torsion with alternative == -target: torch.minimum's tie split cancels it to 0
#   zero_rot_score        separate loss, a counted residue whose predicted rotation score is exactly 0
#   t_at_threshold        t == rot_loss_t_threshold: the rotation gate is a strict comparison
#   last_frame_masked     every residue of the trained-on frame masked out; the normaliser counts the other frames
#   all_masked            every residue of every frame masked out
LOSS_EDGES = ("zero_torsion_alt_gt", "zero_torsion_alt_neg", "zero_rot_score", "t_at_threshold", "last_frame_masked", "all_masked")


def loss_edge(name: str):
    """(batch, model_out, separate_rot_loss) of one edge case."""
    assert name in LOSS_EDGES, name
    feats, out, separate = loss_variant("separate" if name == "zero_rot_score" else "plain")
    if name == "zero_torsion_alt_gt":
        feats["alt_torsion_angles_sin_cos"] = feats["torsion_angles_sin_cos"].clone()
    elif name == "zero_torsion_alt_neg":
        feats["alt_torsion_angles_sin_cos"][-1, 0, 0] = -feats["torsion_angles_sin_cos"][-1, 0, 0]
    elif name == "zero_rot_score":
        out["rot_score"][-1, 4] = 0.0
    elif name == "t_at_threshold":
        feats["t"] = torch.tensor([0.2], dtype=torch.float64)
    elif name == "last_frame_masked":
        feats["res_mask"][-1] = 0
    else:
        feats["res_mask"][:] = 0
    return feats, out, separate
