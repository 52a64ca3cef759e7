"""Host-side mirror of the reference's ``src/model/ipa_pytorch_dynamic.py`` (SURVEY.md §8 rows a2, a3, a5-a7, a14, a15).

Same class names, constructor arguments, forward signatures and ``state_dict`` layout as the reference, so the
reference's ``train_DFOLD_dynamics.py`` / ``eval_DFOLD_dynamics.py`` run unchanged against it (through the import
overlay in ``overlay/``).  All arithmetic is dispatched to the hand-written sm_90a kernels in ``csrc/`` through
``kernels`` (C-ABI, ctypes); there is no CPU fallback — the ops raise if the extension or a CUDA device is missing.

GPU-first restructuring that keeps results identical to the reference:
  * activations stay channels-last ``[frames, residues, C]`` end to end — the reference permutes to NCHW for its
    ``Conv2d`` stack (ipa_pytorch_dynamic.py:694); here the 5x5 frame x residue convolution is an implicit GEMM
    over TMA halo tiles of the channels-last tensor;
  * the single representation ``s`` fed to IPA is the same for every trajectory frame in DFOLDv2
    (ipa_pytorch_dynamic.py:829-833: ``index_embeder(...).expand(nf)`` + broadcast ``expand_node_repr``), so q, k, v,
    the raw point projections and the scalar logits ``q.k/sqrt(3C) + b/sqrt(3)`` are computed once per sample and
    shared by all frames; only the frame-dependent part (rigid application, point distances, softmax, value / point
    / pair aggregation) runs per frame inside the fused attention kernel;
  * the pair tensor ``z`` is un-batched and shared by all frames (:834,857).
"""
import math
import os
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch
import torch.nn as nn

from . import kernels as K
from .layers import (Linear, _lin, ipa_forward, permute_final_dims, flatten_final_dims,  # noqa: F401
                     ipa_point_weights_init_, _calculate_fan, trunc_normal_init_, lecun_normal_init_,
                     he_normal_init_, glorot_uniform_init_, final_init_, gating_init_, normal_init_)
from .rigid_utils import Rigid
from .structure_module import AngleResnet


# --------------------------------------------------------------------------------------------------
# transitions (defined by the reference, not instantiated by DFOLDv2; kept as drop-in modules) — row a15
# --------------------------------------------------------------------------------------------------
class StructureModuleTransition(nn.Module):
    """ref :175-197."""

    def __init__(self, c):
        super().__init__()
        self.c = c
        self.linear_1 = Linear(c, c, init="relu")
        self.linear_2 = Linear(c, c, init="relu")
        self.linear_3 = Linear(c, c, init="final")
        self.relu = nn.ReLU()
        self.ln = nn.LayerNorm(c)

    def forward(self, s):
        h = _lin(self.linear_1, s, act="relu")
        h = _lin(self.linear_2, h, act="relu")
        h = K.linear(h, self.linear_3.weight, self.linear_3.bias, residual=s)
        return K.layer_norm(h, self.ln.weight, self.ln.bias, self.ln.eps)


class EdgeTransition(nn.Module):
    """ref :200-239."""

    def __init__(self, *, node_embed_size, edge_embed_in, edge_embed_out, num_layers=2, node_dilation=2):
        super().__init__()
        bias_embed_size = node_embed_size // node_dilation
        self.initial_embed = Linear(node_embed_size, bias_embed_size, init="relu")
        hidden_size = bias_embed_size * 2 + edge_embed_in
        trunk_layers = []
        for _ in range(num_layers):
            trunk_layers.append(Linear(hidden_size, hidden_size, init="relu"))
            trunk_layers.append(nn.ReLU())
        self.trunk = nn.Sequential(*trunk_layers)
        self.final_layer = Linear(hidden_size, edge_embed_out, init="final")
        self.layer_norm = nn.LayerNorm(edge_embed_out)

    def forward(self, node_embed, edge_embed):
        node_embed = _lin(self.initial_embed, node_embed)
        batch_size, num_res, _ = node_embed.shape
        edge_bias = torch.cat([
            node_embed[:, :, None, :].expand(-1, -1, num_res, -1),
            node_embed[:, None, :, :].expand(-1, num_res, -1, -1),
        ], dim=-1)
        e = torch.cat([edge_embed, edge_bias], dim=-1).reshape(batch_size * num_res ** 2, -1)
        h = e
        for layer in self.trunk:
            if isinstance(layer, nn.Linear):
                h = _lin(layer, h, act="relu")
        h = K.linear(h + e, self.final_layer.weight, self.final_layer.bias)
        h = K.layer_norm(h, self.layer_norm.weight, self.layer_norm.bias, self.layer_norm.eps)
        return h.reshape(batch_size, num_res, num_res, -1)


# --------------------------------------------------------------------------------------------------
# Invariant point attention, DFOLD fork — row a3
# --------------------------------------------------------------------------------------------------
class InvariantPointAttention(nn.Module):
    """Algorithm 22 with the DFOLD changes (ref :242-516): config-object constructor, ``down_z`` pair projection
    (c_z -> c_z/4), extra global-frame point features; concat width H*(c_z/4 + C + 8*Pv)."""

    def __init__(self, ipa_conf, inf: float = 1e5, eps: float = 1e-8):
        super().__init__()
        self._ipa_conf = ipa_conf
        self.c_s = ipa_conf.c_s
        self.c_z = ipa_conf.c_z
        self.c_hidden = ipa_conf.c_hidden
        self.no_heads = ipa_conf.no_heads
        self.no_qk_points = ipa_conf.no_qk_points
        self.no_v_points = ipa_conf.no_v_points
        self.inf = inf
        self.eps = eps

        hc = self.c_hidden * self.no_heads
        self.linear_q = Linear(self.c_s, hc)
        self.linear_kv = Linear(self.c_s, 2 * hc)
        self.linear_q_points = Linear(self.c_s, self.no_heads * self.no_qk_points * 3)
        self.linear_kv_points = Linear(self.c_s, self.no_heads * (self.no_qk_points + self.no_v_points) * 3)
        self.linear_b = Linear(self.c_z, self.no_heads)
        self.down_z = Linear(self.c_z, self.c_z // 4)
        self.head_weights = nn.Parameter(torch.zeros((ipa_conf.no_heads)))
        ipa_point_weights_init_(self.head_weights)
        concat_out_dim = self.c_z // 4 + self.c_hidden + self.no_v_points * 8
        self.linear_out = Linear(self.no_heads * concat_out_dim, self.c_s, init="final")
        self.softmax = nn.Softmax(dim=-1)
        self.softplus = nn.Softplus()
        # carried by published checkpoints, never used (ref :310-311)
        self.linear_rbf = Linear(20, 1)

    def forward(self, s: torch.Tensor, z: Optional[torch.Tensor], r: Rigid, mask: torch.Tensor,
                _offload_inference: bool = False,
                _z_reference_list: Optional[Sequence[torch.Tensor]] = None) -> torch.Tensor:
        """s [*,N,c_s]; z [N,N,c_z] or [*,N,N,c_z]; r Rigid[*,N]; mask [*,N] -> [*,N,c_s]."""
        if _offload_inference:
            z = _z_reference_list[0]
        return ipa_forward(self, s, z, r, mask, dfold=True)


# --------------------------------------------------------------------------------------------------
# ConvNet / MyLayerNorm / BackboneUpdate — rows a5, a6, a7
# --------------------------------------------------------------------------------------------------
class TorsionAngles(nn.Module):
    """ref :519-552 (unused by DFOLDv2)."""

    def __init__(self, c, num_torsions, eps=1e-8):
        super().__init__()
        self.c = c
        self.eps = eps
        self.num_torsions = num_torsions
        self.linear_1 = Linear(c, c, init="relu")
        self.linear_2 = Linear(c, c, init="relu")
        self.linear_3 = Linear(c, c, init="final")
        self.linear_final = Linear(c, num_torsions * 2, init="final")
        self.relu = nn.ReLU()

    def forward(self, s):
        h = _lin(self.linear_1, s, act="relu")
        h = K.linear(h, self.linear_2.weight, self.linear_2.bias, residual=s)
        unnormalized_s = _lin(self.linear_final, h)
        norm_denom = torch.sqrt(torch.clamp(torch.sum(unnormalized_s ** 2, dim=-1, keepdim=True), min=self.eps))
        return unnormalized_s, unnormalized_s / norm_denom


class ScoreLayer(nn.Module):
    """ref :555-572 (unused by DFOLDv2)."""

    def __init__(self, dim_in, dim_hid, dim_out):
        super().__init__()
        self.linear_1 = Linear(dim_in, dim_hid, init="relu")
        self.linear_2 = Linear(dim_hid, dim_hid)
        self.linear_3 = Linear(dim_hid, dim_out, init="final")
        self.relu = nn.ReLU()

    def forward(self, s):
        h = _lin(self.linear_1, s, act="relu")
        h = K.linear(h, self.linear_2.weight, self.linear_2.bias, residual=s)
        return _lin(self.linear_3, h)


class BackboneUpdate(nn.Module):
    """Algorithm 23 update head: Linear(c_s -> 6), zero ('final') init (ref :575-602)."""

    def __init__(self, c_s):
        super().__init__()
        self.c_s = c_s
        self.linear = Linear(self.c_s, 6, init="final")

    def forward(self, s: torch.Tensor):
        return _lin(self.linear, s)


class ConvNet(nn.Module):
    """Four residual stages of Conv2d(dim->dim/2,5,pad 2)+ReLU+Conv2d(dim/2->dim,5,pad 2)+ReLU over the
    (frame, residue) image (ref :664-706).  Parameters keep the reference's ``convK.{0,2}.{weight,bias}`` names and
    ``[C_out, C_in, 5, 5]`` layout; the arithmetic is the channels-last implicit GEMM ``kernels.conv5x5``."""

    def __init__(self, dim):
        super().__init__()
        for st in range(1, 5):
            setattr(self, f"conv{st}", nn.Sequential(
                nn.Conv2d(dim, dim // 2, kernel_size=5, padding=2), nn.ReLU(True),
                nn.Conv2d(dim // 2, dim, kernel_size=5, padding=2), nn.ReLU(True)))

    def forward(self, x, last_frame_only: bool = False, windows: Optional[int] = None):
        """x [frames, residues, dim] -> same shape.

        ``last_frame_only`` (needs >= 17 frames): returns [1, residues, dim], the LAST frame of the full result, computing
        for each of the eight layers only the frames that last frame still depends on (15, 13, ... 1).

        ``windows=W``: x stacks W windows of equal frame counts, each convolved on its own (``kernels.conv5x5``); with
        ``last_frame_only`` the result is [W, residues, dim], the last frame of each window."""
        # the plain calls keep the operators' plain signatures (the CPU tests route them to the oracle's ops)
        win = {} if windows is None else {"windows": windows}
        for st in range(1, 5):
            seq = getattr(self, f"conv{st}")
            if last_frame_only:
                h = K.conv5x5(x, seq[0].weight, seq[0].bias, relu=True, crop=2, **win)
                res = x[4:] if windows is None else x.unflatten(0, (windows, -1))[:, 4:].flatten(0, 1)
                x = K.conv5x5(h, seq[2].weight, seq[2].bias, relu=True, residual=res, crop=2, **win)
            else:
                h = K.conv5x5(x, seq[0].weight, seq[0].bias, relu=True, **win)
                x = K.conv5x5(h, seq[2].weight, seq[2].bias, relu=True, residual=x, **win)
        return x


class MyLayerNorm(nn.Module):
    """(x - mean) / sqrt(var_unbiased + 1e-4) with ONE mean/variance over the whole [frames, residues, C] tensor,
    no affine (ref :709-724)."""

    def __init__(self):
        super().__init__()
        self.eps = 1e-4

    def forward(self, x, segments: Optional[int] = None):
        """``segments=W``: x stacks W windows along its leading axis, each normalised on its own."""
        return K.global_layernorm(x, self.eps, **({} if segments is None else {"segments": segments}))


class TimeBlock(nn.Module):
    """ref :604-633 (unused by DFOLDv2)."""

    def __init__(self, node_dim, time_embed_dim, hidden_dim=None):
        super().__init__()
        self.node_dim = node_dim
        self.time_embed_dim = time_embed_dim
        self.hidden_dim = hidden_dim if hidden_dim is not None else node_dim // 2
        self.time_proj = nn.Sequential(nn.Linear(time_embed_dim, 4 * time_embed_dim), nn.SiLU(),
                                       nn.Linear(4 * time_embed_dim, self.hidden_dim))
        self.node_proj = nn.Sequential(nn.LayerNorm(node_dim), nn.SiLU(), nn.Linear(node_dim, self.hidden_dim))
        self.out_prj = nn.Sequential(nn.LayerNorm(self.hidden_dim), nn.SiLU(), nn.Linear(self.hidden_dim, node_dim))

    def forward(self, node_feature, time_embeddings):
        return node_feature + self.out_prj(self.time_proj(time_embeddings) + self.node_proj(node_feature))


class PositionalEncoding(nn.Module):
    """ref :636-661 (unused by DFOLDv2)."""

    def __init__(self, d_model, dropout=0.0, max_len=40):
        super().__init__()
        self.dropout = nn.Dropout(p=dropout)
        position = torch.arange(max_len).unsqueeze(1)
        div_term = torch.exp(torch.arange(0, d_model, 2) * (-math.log(10000.0) / d_model))
        pe = torch.zeros(1, max_len, d_model)
        pe[0, :, 0::2] = torch.sin(position * div_term)
        pe[0, :, 1::2] = torch.cos(position * div_term)
        self.register_buffer("pe", pe)

    def forward(self, x):
        return self.dropout(x + self.pe[:, : x.size(1)])


# set DFOLD_NO_DEAD_FRAME_SKIP=1 to run the ConvNet on every frame in every block, as the reference does
_DEAD_FRAME_SKIP = os.environ.get("DFOLD_NO_DEAD_FRAME_SKIP", "0") != "1"


def _embedder(in_dim: int, width: int) -> nn.Sequential:
    return nn.Sequential(nn.Linear(in_dim, width), nn.SiLU(), nn.Linear(width, width), MyLayerNorm(), nn.SiLU())


def _run_embedder(seq: nn.Sequential, x: torch.Tensor, windows: Optional[int] = None) -> torch.Tensor:
    """Linear-SiLU-Linear-MyLayerNorm-SiLU (ref :757-796) on the fused kernels; ``windows=W``: x stacks W windows along
    its leading axis and the layer norm takes one mean / variance per window."""
    h = K.linear(x, seq[0].weight, seq[0].bias, act="silu")
    h = K.linear(h, seq[2].weight, seq[2].bias)
    return K.global_layernorm(h, seq[3].eps, silu=True, **({} if windows is None else {"segments": windows}))


def _shift_last(x: torch.Tensor) -> torch.Tensor:
    """cat(x[:-1], x[-2:-1]): the last frame's input is its predecessor's (ref :819,822,826,842)."""
    return torch.cat([x[:-1], x[-2:-1]], dim=0)


# --------------------------------------------------------------------------------------------------
# the trunk — row a2
# --------------------------------------------------------------------------------------------------
class DFOLDIpaScore(nn.Module):
    """ref :726-907."""

    def __init__(self, model_conf, diffuser):
        super().__init__()
        self._model_conf = model_conf
        ipa_conf = model_conf.ipa
        self._ipa_conf = ipa_conf
        self.diffuser = diffuser
        # device-resident twin of the caller's diffuser for the fused score epilogue (None: use the object as handed in)
        from .score_epilogue import SE3ScoreDiffuser
        self._fused_scores = diffuser if isinstance(diffuser, SE3ScoreDiffuser) else SE3ScoreDiffuser.from_reference(diffuser)

        self.scale_pos = lambda x: x * ipa_conf.coordinate_scaling
        self.scale_rigids = lambda x: x.apply_trans_fn(self.scale_pos)
        self.unscale_pos = lambda x: x / ipa_conf.coordinate_scaling
        self.unscale_rigids = lambda x: x.apply_trans_fn(self.unscale_pos)

        self.trunk = nn.ModuleDict()
        for b in range(ipa_conf.num_blocks):
            self.trunk[f"ipa_{b}"] = InvariantPointAttention(ipa_conf)
            self.trunk[f"ln_{b}"] = MyLayerNorm()
            self.trunk[f"bb_update_{b}"] = BackboneUpdate(ipa_conf.c_s * 5)
        self.trunk["conv_0"] = ConvNet(ipa_conf.c_s * 5)

        self.angle_resnet = AngleResnet(c_in=ipa_conf.c_s * 5, c_hidden=ipa_conf.c_s * 5, no_blocks=2,
                                        no_angles=7, epsilon=1e-12)
        w = model_conf.node_embed_size
        self.force_embeder = _embedder(3, w)
        self.vel_embeder = _embedder(3, w)
        self.index_embeder = _embedder(1, w)
        self.rigid_embeder = _embedder(7, w)
        self.angle_embeder = _embedder(14, w)

    def forward(self, init_node_embed, edge_embed, input_feats, drop_ref=False):
        """``init_node_embed`` / ``edge_embed`` / ``drop_ref`` are accepted and unused, as in the reference."""
        t = input_feats["t"]
        node_mask = input_feats["res_mask"].type(torch.float32)
        diffuse_mask = (1 - input_feats["fixed_mask"].type(torch.float32)) * node_mask
        init_rigids = Rigid.from_tensor_7(input_feats["rigids_t"].type(torch.float32))

        rigids_0 = input_feats["rigids_0"]
        dt = rigids_0.dtype
        nf = rigids_0.shape[0]
        curr = _shift_last(rigids_0).to(torch.float32)

        force_embed = _run_embedder(self.force_embeder, _shift_last(input_feats["force"].to(dt)))
        vel_embed = _run_embedder(self.vel_embeder, _shift_last(input_feats["vel"].to(dt)))

        idx = input_feats["seq_idx"][0:1].unsqueeze(-1).to(input_feats["node_repr"].dtype)
        node_1 = _run_embedder(self.index_embeder, idx)[0] + input_feats["expand_node_repr"]     # [N,c_s]
        node_embed = node_1.unsqueeze(0).expand(nf, -1, -1)       # frame-invariant; stays a stride-0 view
        edge_embed = input_feats["expand_edge_repr"]

        angle = input_feats["torsion_angles_sin_cos"].to(dt)
        angle = (angle * input_feats["torsion_angles_mask"].to(dt).unsqueeze(-1)).to(dt)
        angle = _shift_last(angle).reshape(nf, -1, angle.shape[-2] * 2)
        angle_embed = _run_embedder(self.angle_embeder, angle)

        node_feat = init_node_feat = rigid_update = None
        for b in range(self._ipa_conf.num_blocks):
            rigids_embed = _run_embedder(self.rigid_embeder, curr)
            ipa_embed = self.trunk[f"ipa_{b}"](node_embed, edge_embed, Rigid.from_tensor_7(curr), node_mask)
            ipa_embed = self.trunk[f"ln_{b}"](ipa_embed)
            node_feat = torch.cat([rigids_embed, ipa_embed, force_embed, vel_embed, angle_embed], dim=-1)
            # Dead-frame elimination (exact): only the LAST frame's update survives `rigid_update[:-1] *= 0`
            # (ref :869), block 0's features feed AngleResnet.s_initial (:875-878) and the last block's feed
            # AngleResnet (:878); for the blocks in between, every other frame of the ConvNet output is dead.
            # Eight 5x5 convolutions reach 8*2 = 16 frames back, so the last 17 input frames reproduce the last
            # output frame exactly (the cropped edge's zero padding cannot reach it), and layer k of the stack only
            # needs to produce the 17 - 2k frames the last one still depends on.
            halo = 2 * 8
            middle = (0 < b < self._ipa_conf.num_blocks - 1) and nf > halo + 1 and _DEAD_FRAME_SKIP
            if middle:
                node_feat = self.trunk["conv_0"](node_feat[-(halo + 1):], last_frame_only=True)     # [1,N,5c]
            else:
                node_feat = self.trunk["conv_0"](node_feat)

            upd_last = self.trunk[f"bb_update_{b}"](node_feat[-1:])        # [1,N,6]
            rigid_update = torch.cat([upd_last.new_zeros((nf - 1,) + upd_last.shape[1:]), upd_last], dim=0)   # ref :869
            new_rigids = Rigid.from_tensor_7(curr).compose_q_update_vec(rigid_update, diffuse_mask[..., None])
            curr = new_rigids.to_tensor_7()
            if b == 0:
                init_node_feat = node_feat

        unorm_angles, angles = self.angle_resnet(node_feat, init_node_feat)
        curr_rigids = Rigid.from_tensor_7(curr)
        if self._fused_scores is not None:
            # ref :883-897 in one kernel: rotation score (IGSO(3) series, fp64), unscale, translation score, masks
            rot_score, trans_score = self._fused_scores.fused_scores(init_rigids, curr_rigids, t, node_mask,
                                                                     self._ipa_conf.coordinate_scaling)
            curr_rigids = self.unscale_rigids(curr_rigids)
        else:
            rot_score = self.diffuser.calc_rot_score(init_rigids.get_rots(), curr_rigids.get_rots(), t)
            rot_score = rot_score * node_mask[..., None]
            curr_rigids = self.unscale_rigids(curr_rigids)
            trans_score = self.diffuser.calc_trans_score(init_rigids.get_trans(), curr_rigids.get_trans(),
                                                         t[:, None, None], use_torch=True)
            trans_score = trans_score * node_mask[..., None]
        return {
            "angles": angles,
            "unorm_angles": unorm_angles,
            "rot_score": rot_score,
            "trans_score": trans_score,
            "final_rigids": curr_rigids,
            "rigid_update": rigid_update,
        }

    def forward_windows(self, feats_list):
        """``forward`` over W windows of equal frame and residue counts in one pass (checked by the caller,
        ``FullScoreNetwork.forward_windows``).  The per-frame inputs are stacked along the frame axis, and the row-wise
        layers run once on all W * nf frames.  What couples frames stays within a window: ``_shift_last``, the
        last-frame-only ``rigid_update``, each window's own index embedding and node / edge representations, one
        MyLayerNorm mean and variance per window, the ConvNet's frame halo (and the dead-frame crop), and ``t`` in the
        score epilogue.  IPA runs once per window.  Returns the stacked trunk outputs, with ``final_rigids`` a Rigid over
        all W * nf frames; window i owns frames [i * nf, (i + 1) * nf) of every entry."""
        W = len(feats_list)
        f0 = feats_list[0]
        nf = f0["rigids_0"].shape[0]
        cat = lambda xs: torch.cat(xs, dim=0)
        node_mask = [f["res_mask"].type(torch.float32) for f in feats_list]
        diffuse_mask = cat([(1 - f["fixed_mask"].type(torch.float32)) * m for f, m in zip(feats_list, node_mask)])
        init_rigids = [Rigid.from_tensor_7(f["rigids_t"].type(torch.float32)) for f in feats_list]
        dt = f0["rigids_0"].dtype
        curr = cat([_shift_last(f["rigids_0"]).to(torch.float32) for f in feats_list])

        force_embed = _run_embedder(self.force_embeder, cat([_shift_last(f["force"].to(dt)) for f in feats_list]), W)
        vel_embed = _run_embedder(self.vel_embeder, cat([_shift_last(f["vel"].to(dt)) for f in feats_list]), W)

        idx = cat([f["seq_idx"][0:1].unsqueeze(-1).to(f["node_repr"].dtype) for f in feats_list])      # [W,N,1]
        node_1 = _run_embedder(self.index_embeder, idx, W)
        node_embed = [(node_1[i] + f["expand_node_repr"]).unsqueeze(0).expand(nf, -1, -1) for i, f in enumerate(feats_list)]

        angle = []
        for f in feats_list:
            a = f["torsion_angles_sin_cos"].to(dt)
            a = (a * f["torsion_angles_mask"].to(dt).unsqueeze(-1)).to(dt)
            angle.append(_shift_last(a).reshape(nf, -1, a.shape[-2] * 2))
        angle_embed = _run_embedder(self.angle_embeder, cat(angle), W)

        node_feat = init_node_feat = rigid_update = None
        for b in range(self._ipa_conf.num_blocks):
            rigids_embed = _run_embedder(self.rigid_embeder, curr, W)
            ipa = self.trunk[f"ipa_{b}"]
            ipa_embed = cat([ipa(node_embed[i], f["expand_edge_repr"], Rigid.from_tensor_7(curr[i * nf:(i + 1) * nf]),
                                 node_mask[i]) for i, f in enumerate(feats_list)])
            ipa_embed = self.trunk[f"ln_{b}"](ipa_embed, segments=W)
            node_feat = torch.cat([rigids_embed, ipa_embed, force_embed, vel_embed, angle_embed], dim=-1)
            halo = 2 * 8                        # dead-frame elimination, per window (see forward)
            middle = (0 < b < self._ipa_conf.num_blocks - 1) and nf > halo + 1 and _DEAD_FRAME_SKIP
            if middle:
                tail = node_feat.unflatten(0, (W, nf))[:, -(halo + 1):].flatten(0, 1)
                node_feat = self.trunk["conv_0"](tail, last_frame_only=True, windows=W)                  # [W,N,5c]
                last = node_feat
            else:
                node_feat = self.trunk["conv_0"](node_feat, windows=W)
                last = node_feat.unflatten(0, (W, nf))[:, -1]
            upd_last = self.trunk[f"bb_update_{b}"](last)                                                 # [W,N,6]
            rigid_update = torch.cat([upd_last.new_zeros((W, nf - 1) + upd_last.shape[1:]), upd_last[:, None]],
                                     dim=1).flatten(0, 1)
            new_rigids = Rigid.from_tensor_7(curr).compose_q_update_vec(rigid_update, diffuse_mask[..., None])
            curr = new_rigids.to_tensor_7()
            if b == 0:
                init_node_feat = node_feat

        unorm_angles, angles = self.angle_resnet(node_feat, init_node_feat)
        rot_score, trans_score = [], []
        for i, f in enumerate(feats_list):
            cr = Rigid.from_tensor_7(curr[i * nf:(i + 1) * nf])
            if self._fused_scores is not None:
                rs, ts = self._fused_scores.fused_scores(init_rigids[i], cr, f["t"], node_mask[i],
                                                         self._ipa_conf.coordinate_scaling)
            else:
                rs = self.diffuser.calc_rot_score(init_rigids[i].get_rots(), cr.get_rots(), f["t"]) * node_mask[i][..., None]
                ts = self.diffuser.calc_trans_score(init_rigids[i].get_trans(), self.unscale_rigids(cr).get_trans(),
                                                    f["t"][:, None, None], use_torch=True) * node_mask[i][..., None]
            rot_score.append(rs)
            trans_score.append(ts)
        return {
            "angles": angles,
            "unorm_angles": unorm_angles,
            "rot_score": cat(rot_score),
            "trans_score": cat(trans_score),
            "final_rigids": self.unscale_rigids(Rigid.from_tensor_7(curr)),
            "rigid_update": rigid_update,
        }
