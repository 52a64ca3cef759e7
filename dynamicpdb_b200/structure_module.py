"""Host-side mirror of ``openfold/model/structure_module.py`` (SURVEY.md §8 rows a4, a12, a16): ``AngleResnet``
(the only class DFOLDv2 executes, ipa_pytorch_dynamic.py:10,754), the vanilla ``InvariantPointAttention``,
``BackboneUpdate``, the transition blocks and ``StructureModule`` with the reference's constructor arguments,
forward signatures and parameter names.  Arithmetic runs on the sm_90a kernels through ``kernels``.
"""
from typing import Optional, Sequence, Tuple

import torch
import torch.nn as nn

from . import kernels as K
from . import feats as _feats
from .layers import LayerNorm, Linear, _lin, ipa_forward, ipa_point_weights_init_
from .rigid_utils import Rigid, Rotation


class AngleResnetBlock(nn.Module):
    """structure_module.py:47-72."""

    def __init__(self, c_hidden):
        super().__init__()
        self.c_hidden = c_hidden
        self.linear_1 = Linear(c_hidden, c_hidden, init="relu")
        self.linear_2 = Linear(c_hidden, c_hidden, init="final")
        self.relu = nn.ReLU()

    def forward(self, a: torch.Tensor) -> torch.Tensor:
        h = K.linear(a, self.linear_1.weight, self.linear_1.bias, pre_relu=True, act="relu")
        return K.linear(h, self.linear_2.weight, self.linear_2.bias, residual=a)


class AngleResnet(nn.Module):
    """Algorithm 20 lines 11-14 (structure_module.py:75-158)."""

    def __init__(self, c_in, c_hidden, no_blocks, no_angles, epsilon):
        super().__init__()
        self.c_in = c_in
        self.c_hidden = c_hidden
        self.no_blocks = no_blocks
        self.no_angles = no_angles
        self.eps = epsilon
        self.linear_in = Linear(c_in, c_hidden)
        self.linear_initial = Linear(c_in, c_hidden)
        self.layers = nn.ModuleList([AngleResnetBlock(c_hidden=c_hidden) for _ in range(no_blocks)])
        self.linear_out = Linear(c_hidden, no_angles * 2)
        self.relu = nn.ReLU()

    def forward(self, s: torch.Tensor, s_initial: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """s, s_initial [*, c_in] -> (unnormalised, normalised) [*, no_angles, 2]."""
        a0 = K.linear(s_initial, self.linear_initial.weight, self.linear_initial.bias, pre_relu=True)
        a = K.linear(s, self.linear_in.weight, self.linear_in.bias, pre_relu=True, residual=a0)
        for l in self.layers:
            a = l(a)
        u = K.linear(a, self.linear_out.weight, self.linear_out.bias, pre_relu=True)
        u = u.view(u.shape[:-1] + (-1, 2))
        denom = torch.sqrt(torch.clamp(torch.sum(u ** 2, dim=-1, keepdim=True), min=self.eps))
        return u, u / denom


class InvariantPointAttention(nn.Module):
    """Vanilla Algorithm 22 (structure_module.py:161-431): full-width pair aggregation, 4*Pv point features."""

    def __init__(self, c_s: int, c_z: int, c_hidden: int, no_heads: int, no_qk_points: int, no_v_points: int,
                 inf: float = 1e5, eps: float = 1e-8):
        super().__init__()
        self.c_s, self.c_z, self.c_hidden = c_s, c_z, c_hidden
        self.no_heads, self.no_qk_points, self.no_v_points = no_heads, no_qk_points, no_v_points
        self.inf, self.eps = inf, eps
        hc = c_hidden * no_heads
        self.linear_q = Linear(c_s, hc)
        self.linear_kv = Linear(c_s, 2 * hc)
        self.linear_q_points = Linear(c_s, no_heads * no_qk_points * 3)
        self.linear_kv_points = Linear(c_s, no_heads * (no_qk_points + no_v_points) * 3)
        self.linear_b = Linear(c_z, no_heads)
        self.head_weights = nn.Parameter(torch.zeros((no_heads)))
        ipa_point_weights_init_(self.head_weights)
        self.linear_out = Linear(no_heads * (c_z + c_hidden + no_v_points * 4), c_s, init="final")
        self.softmax = nn.Softmax(dim=-1)
        self.softplus = nn.Softplus()

    def forward(self, s: torch.Tensor, z: Optional[torch.Tensor], r: Rigid, mask: torch.Tensor,
                inplace_safe: bool = False, _offload_inference: bool = False,
                _z_reference_list: Optional[Sequence[torch.Tensor]] = None) -> torch.Tensor:
        """``inplace_safe`` selects an in-place softmax in upstream OpenFold; the fused kernel never materialises
        the attention matrix, so the flag changes nothing here."""
        if _offload_inference and inplace_safe:
            z = _z_reference_list[0]
        return ipa_forward(self, s, z, r, mask, dfold=False)


class BackboneUpdate(nn.Module):
    """structure_module.py:434-461."""

    def __init__(self, c_s):
        super().__init__()
        self.c_s = c_s
        self.linear = Linear(c_s, 6, init="final")

    def forward(self, s: torch.Tensor):
        return _lin(self.linear, s)


class StructureModuleTransitionLayer(nn.Module):
    """structure_module.py:464-486."""

    def __init__(self, c):
        super().__init__()
        self.c = c
        self.linear_1 = Linear(c, c, init="relu")
        self.linear_2 = Linear(c, c, init="relu")
        self.linear_3 = Linear(c, c, init="final")
        self.relu = nn.ReLU()

    def forward(self, s):
        h = _lin(self.linear_1, s, act="relu")
        h = _lin(self.linear_2, h, act="relu")
        return K.linear(h, self.linear_3.weight, self.linear_3.bias, residual=s)


class StructureModuleTransition(nn.Module):
    """structure_module.py:489-512."""

    def __init__(self, c, num_layers, dropout_rate):
        super().__init__()
        self.c, self.num_layers, self.dropout_rate = c, num_layers, dropout_rate
        self.layers = nn.ModuleList([StructureModuleTransitionLayer(c) for _ in range(num_layers)])
        self.dropout = nn.Dropout(dropout_rate)
        self.layer_norm = LayerNorm(c)

    def forward(self, s):
        for l in self.layers:
            s = l(s)
        return self.layer_norm(self.dropout(s))


def _stack_dicts(dicts):
    return {k: torch.stack([d[k] for d in dicts]) for k in dicts[0]}


class StructureModule(nn.Module):
    """structure_module.py:515-820."""

    def __init__(self, c_s, c_z, c_ipa, c_resnet, no_heads_ipa, no_qk_points, no_v_points, dropout_rate, no_blocks,
                 no_transition_layers, no_resnet_blocks, no_angles, trans_scale_factor, epsilon, inf, **kwargs):
        super().__init__()
        self.c_s, self.c_z, self.c_ipa, self.c_resnet = c_s, c_z, c_ipa, c_resnet
        self.no_heads_ipa, self.no_qk_points, self.no_v_points = no_heads_ipa, no_qk_points, no_v_points
        self.dropout_rate, self.no_blocks = dropout_rate, no_blocks
        self.no_transition_layers, self.no_resnet_blocks = no_transition_layers, no_resnet_blocks
        self.no_angles, self.trans_scale_factor, self.epsilon, self.inf = no_angles, trans_scale_factor, epsilon, inf

        self.layer_norm_s = LayerNorm(c_s)
        self.layer_norm_z = LayerNorm(c_z)
        self.linear_in = Linear(c_s, c_s)
        self.ipa = InvariantPointAttention(c_s, c_z, c_ipa, no_heads_ipa, no_qk_points, no_v_points,
                                           inf=inf, eps=epsilon)
        self.ipa_dropout = nn.Dropout(dropout_rate)
        self.layer_norm_ipa = LayerNorm(c_s)
        self.transition = StructureModuleTransition(c_s, no_transition_layers, dropout_rate)
        self.bb_update = BackboneUpdate(c_s)
        self.angle_resnet = AngleResnet(c_s, c_resnet, no_resnet_blocks, no_angles, epsilon)

    def forward(self, evoformer_output_dict, aatype, mask=None, inplace_safe=False, _offload_inference=False):
        s = evoformer_output_dict["single"]
        if mask is None:
            mask = s.new_ones(s.shape[:-1])
        s = self.layer_norm_s(s)
        z = self.layer_norm_z(evoformer_output_dict["pair"])
        s_initial = s
        s = _lin(self.linear_in, s)
        rigids = Rigid.identity(s.shape[:-1], s.dtype, s.device, self.training, fmt="quat")
        outputs = []
        for _ in range(self.no_blocks):
            s = s + self.ipa(s, z, rigids, mask)
            s = self.ipa_dropout(s)
            s = self.layer_norm_ipa(s)
            s = self.transition(s)
            rigids = rigids.compose_q_update_vec(self.bb_update(s))
            # rotation-matrix form, as AlphaFold (structure_module.py:701-714)
            backb_to_global = Rigid(Rotation(rot_mats=rigids.get_rots().get_rot_mats(), quats=None),
                                    rigids.get_trans()).scale_translation(self.trans_scale_factor)
            unnormalized_angles, angles = self.angle_resnet(s, s_initial)
            # torsion_angles_to_frames + frames_and_literature_positions_to_atom14_pos (:716-727) in one kernel
            pred_xyz, _, sidechain_frames = _feats.frames_to_atoms(backb_to_global, angles, aatype, want_frames=True)
            scaled_rigids = rigids.scale_translation(self.trans_scale_factor)
            outputs.append({
                "frames": scaled_rigids.to_tensor_7(),
                "sidechain_frames": sidechain_frames,
                "unnormalized_angles": unnormalized_angles,
                "angles": angles,
                "positions": pred_xyz,
                "states": s,
            })
            rigids = rigids.stop_rot_gradient()
        outputs = _stack_dicts(outputs)
        outputs["single"] = s
        return outputs

    def torsion_angles_to_frames(self, r, alpha, f):
        return _feats.torsion_angles_to_frames(r, alpha, f, _feats.table("default_frames", alpha.device, alpha.dtype))

    def frames_and_literature_positions_to_atom14_pos(self, r, f):
        return _feats.frames_to_atom14_pos(r, f)
