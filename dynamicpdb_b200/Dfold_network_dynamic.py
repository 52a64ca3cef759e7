"""Host-side mirror of ``src/model/Dfold_network_dynamic.py`` (SURVEY.md §8 row a1): ``FullScoreNetwork`` with the
reference's constructor, ``forward(input_feats, drop_ref=False) -> dict`` contract, output keys and ``state_dict``
layout (``embedding_layer.*``, ``score_model.*``, ``expand_node``, ``expand_edge``).

Differences that leave every returned value identical:
  * the ``DFOLDv2_Embeder`` call (ref :478-484) produces tensors nothing consumes (SURVEY.md §8 a1: it materialises
    the frame-expanded edge tensor three times, ~10 GB of traffic at nf=64); its parameters are kept (checkpoint
    ABI, ``find_unused_parameters=True`` as in the reference trainer) but the dead computation is not run unless
    ``DFOLD_RUN_DEAD_EMBEDDER=1``;
  * residue tables are device-resident, so the epilogue has no host synchronisation.
"""
import functools as fn
import os
from typing import Tuple

import torch
from torch import nn

from . import feats
from . import ipa_pytorch_dynamic
from . import kernels as K
from .feats import atom14_to_atom37  # noqa: F401  (public name in the reference module)

Tensor = torch.Tensor


def get_timestep_embedding(timesteps, embedding_dim, max_positions=10000):
    """src/model/utils.py:46-58."""
    import math
    assert len(timesteps.shape) == 1
    timesteps = timesteps * max_positions
    half_dim = embedding_dim // 2
    emb = math.log(max_positions) / (half_dim - 1)
    emb = torch.exp(torch.arange(half_dim, dtype=torch.float32, device=timesteps.device) * -emb)
    emb = timesteps.float()[:, None] * emb[None, :]
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=1)
    if embedding_dim % 2 == 1:
        emb = torch.nn.functional.pad(emb, (0, 1), mode="constant")
    return emb


class DFOLDv2_Embeder(nn.Module):
    """ref :19-88.  Owns checkpoint parameters; its outputs are not consumed by the trunk."""

    def __init__(self, model_conf):
        super().__init__()
        self._model_conf = model_conf
        self._embed_conf = model_conf.embed
        node_embed_size = model_conf.node_embed_size
        edge_embed_size = model_conf.edge_embed_size
        time_embed_size = node_embed_size
        self.timestep_embed = fn.partial(get_timestep_embedding, embedding_dim=time_embed_size)
        self.node_timestep_proj = nn.Sequential(nn.Linear(time_embed_size, node_embed_size // 2), nn.SiLU(),
                                                nn.Linear(node_embed_size // 2, node_embed_size))
        self.node_ln = nn.LayerNorm(node_embed_size)
        self.edge_timestep_proj = nn.Sequential(nn.Linear(time_embed_size, edge_embed_size // 2), nn.SiLU(),
                                                nn.Linear(edge_embed_size // 2, edge_embed_size))
        self.edge_ln = nn.LayerNorm(edge_embed_size)

    def forward(self, node_repr, edge_repr, seq_idx, t):
        num_batch, num_res = seq_idx.shape
        t_embed = self.timestep_embed(t)
        node_embed = K.layer_norm(node_repr, self.node_ln.weight, self.node_ln.bias, self.node_ln.eps)
        edge_embed = K.layer_norm(edge_repr.reshape(num_batch, num_res * num_res, -1),
                                  self.edge_ln.weight, self.edge_ln.bias, self.edge_ln.eps)
        ref_edge = edge_embed[0].reshape(num_res, num_res, -1)
        return node_embed, edge_embed.reshape(num_batch, num_res, num_res, -1), node_embed[0], ref_edge, t_embed


def check_windows(feats_list) -> None:
    """The windows ``FullScoreNetwork.forward_windows`` takes: a non-empty list of input dicts with the same keys and,
    key by key, the same shape and dtype; in particular the same residue and frame counts.  Raises ValueError."""
    if not isinstance(feats_list, (list, tuple)) or not feats_list:
        raise ValueError("forward_windows: needs a non-empty list of window dicts")
    if not all(isinstance(f, dict) for f in feats_list):
        raise ValueError("forward_windows: every window must be a dict of input tensors")
    f0 = feats_list[0]
    for k in ("node_repr", "rigids_0"):
        if k not in f0:
            raise ValueError(f"forward_windows: window 0 has no '{k}'")
    n0, nf0 = f0["node_repr"].shape[0], f0["rigids_0"].shape[0]
    for i, f in enumerate(feats_list[1:], start=1):
        if set(f) != set(f0):
            raise ValueError(f"forward_windows: window {i} has keys {sorted(set(f) ^ set(f0))} that window 0 "
                             "has not, or the reverse")
        n, nf = f["node_repr"].shape[0], f["rigids_0"].shape[0]
        if n != n0:
            raise ValueError(f"forward_windows: window {i} has {n} residues and window 0 has {n0}; one pass takes "
                             "windows of one residue count")
        if nf != nf0:
            raise ValueError(f"forward_windows: window {i} has {nf} frames and window 0 has {nf0}; one pass takes "
                             "windows of one frame count")
        for k, v in f.items():
            if torch.is_tensor(v) and (v.shape != f0[k].shape or v.dtype != f0[k].dtype):
                raise ValueError(f"forward_windows: '{k}' of window {i} is {tuple(v.shape)} {v.dtype}, of window 0 "
                                 f"{tuple(f0[k].shape)} {f0[k].dtype}")


class FullScoreNetwork(nn.Module):
    """ref :429-569."""

    def __init__(self, model_conf, diffuser):
        super().__init__()
        self._model_conf = model_conf
        self.embedding_layer = DFOLDv2_Embeder(model_conf)
        self.diffuser = diffuser
        self.score_model = ipa_pytorch_dynamic.DFOLDIpaScore(model_conf, diffuser)
        self.expand_node = nn.Linear(256, model_conf.node_embed_size)
        self.expand_edge = nn.Linear(128, model_conf.edge_embed_size)

    def _apply_mask(self, aatype_diff, aatype_0, diff_mask):
        return diff_mask * aatype_diff + (1 - diff_mask) * aatype_0

    def forward(self, input_feats, drop_ref=False):
        fixed_mask = input_feats["fixed_mask"].type(torch.float32)
        num_res = input_feats["node_repr"].shape[0]

        input_feats["expand_node_repr"] = K.linear(input_feats["node_repr"], self.expand_node.weight,
                                                   self.expand_node.bias)
        input_feats["expand_edge_repr"] = K.linear(
            input_feats["edge_repr"].reshape(num_res * num_res, -1), self.expand_edge.weight,
            self.expand_edge.bias).reshape(num_res, num_res, -1)

        if os.environ.get("DFOLD_RUN_DEAD_EMBEDDER") == "1":
            ft = self._model_conf.frame_time
            _, _, ref_node, ref_edge, t_embed = self.embedding_layer(
                node_repr=input_feats["expand_node_repr"].unsqueeze(0).expand(ft, -1, -1),
                edge_repr=input_feats["expand_edge_repr"].unsqueeze(0).expand(ft, -1, -1, -1),
                seq_idx=input_feats["seq_idx"], t=input_feats["t"])
            input_feats.update({"ref_node_repr": ref_node, "ref_edge_repr": ref_edge, "t_embed": t_embed})

        model_out = self.score_model(None, None, input_feats, drop_ref=drop_ref)

        gt_angles = input_feats["torsion_angles_sin_cos"]
        dm = 1 - fixed_mask[..., None, None]
        angles_pred = self._apply_mask(model_out["angles"], gt_angles, dm)
        unorm_angles = self._apply_mask(model_out["unorm_angles"], gt_angles, dm)
        pred_out = {
            "angles": angles_pred,
            "unorm_angles": unorm_angles,
            "rot_score": model_out["rot_score"],
            "trans_score": model_out["trans_score"],
        }
        rigids_pred = model_out["final_rigids"]
        pred_out["rigids"] = rigids_pred.to_tensor_7()
        # torsion frames -> atom14 -> atom37 (ref :532-538) in one kernel
        atom14_pos, atom37_pos = feats.frames_to_atoms(rigids_pred, angles_pred, input_feats["aatype"])
        pred_out["atom37"] = atom37_pos
        pred_out["atom14"] = atom14_pos
        pred_out["rigid_update"] = model_out["rigid_update"]
        return pred_out

    def forward_windows(self, feats_list):
        """``[forward(f) for f in feats_list]`` in one pass: the windows' per-frame inputs are stacked along the frame axis,
        so every row-wise layer (``expand_*``, the embedders' linears, AngleResnet, BackboneUpdate, ``frames_to_atoms``)
        and every convolution runs once for all of them, while each window is normalised, convolved and scored on its own
        (``DFOLDIpaScore.forward_windows``).  IPA runs once per window.  The windows may come from different proteins, but
        must share their residue count, frame count and the shape and dtype of every input; anything else raises
        ValueError before any device work.  Returns one output dict per window, with ``forward``'s keys; its tensors are
        views of the stacked results.  Like ``forward``, it stores ``expand_node_repr`` / ``expand_edge_repr`` in each
        window's dict."""
        check_windows(feats_list)
        W = len(feats_list)
        f0 = feats_list[0]
        num_res = f0["node_repr"].shape[0]
        nf = f0["rigids_0"].shape[0]
        node = K.linear(torch.cat([f["node_repr"] for f in feats_list], dim=0), self.expand_node.weight,
                        self.expand_node.bias)
        edge = K.linear(torch.cat([f["edge_repr"].reshape(num_res * num_res, -1) for f in feats_list], dim=0),
                        self.expand_edge.weight, self.expand_edge.bias)
        for i, f in enumerate(feats_list):
            f["expand_node_repr"] = node[i * num_res:(i + 1) * num_res]
            f["expand_edge_repr"] = edge[i * num_res * num_res:(i + 1) * num_res * num_res].reshape(num_res, num_res, -1)

        model_out = self.score_model.forward_windows(feats_list)

        gt_angles = torch.cat([f["torsion_angles_sin_cos"] for f in feats_list], dim=0)
        dm = 1 - torch.cat([f["fixed_mask"] for f in feats_list], dim=0).type(torch.float32)[..., None, None]
        angles_pred = self._apply_mask(model_out["angles"], gt_angles, dm)
        unorm_angles = self._apply_mask(model_out["unorm_angles"], gt_angles, dm)
        rigids_pred = model_out["final_rigids"]
        atom14_pos, atom37_pos = feats.frames_to_atoms(rigids_pred, angles_pred,
                                                       torch.cat([f["aatype"] for f in feats_list], dim=0))
        stacked = {
            "angles": angles_pred,
            "unorm_angles": unorm_angles,
            "rot_score": model_out["rot_score"],
            "trans_score": model_out["trans_score"],
            "rigids": rigids_pred.to_tensor_7(),
            "atom37": atom37_pos,
            "atom14": atom14_pos,
            "rigid_update": model_out["rigid_update"],
        }
        return [{k: v[i * nf:(i + 1) * nf] for k, v in stacked.items()} for i in range(W)]

    def debug_foward(self, input_feats, drop_ref=False):
        """ref :549-569: forward + the set of parameters whose module ran."""
        used_params = set()

        def hook(module, _inp, _out):
            for param in module.parameters():
                used_params.add(param)

        hooks = [m.register_forward_hook(hook) for m in self.modules()]
        output = self.forward(input_feats, drop_ref)
        for h in hooks:
            h.remove()
        return output, used_params
