"""Float64-capable restatement of the backbone-atom and pair-distance losses of Experiment.loss_fn
(train_DFOLD_dynamics.py:1316-1364), which the reference computes on every step but leaves out of final_loss.

TEST INFRASTRUCTURE, as oracle/dfold_oracle.py: plain torch, written from the reference's lines, pinned to the unmodified
reference by tests/golden/aux_loss.pt (oracle/make_aux_loss_golden.py, tests/test_cpu_aux_loss.py), and the yardstick of
csrc/aux_loss.cu in tests/test_gpu_aux_loss.py.
"""
from typing import Dict

import torch

from oracle.dfold_oracle import atom14_to_atom37, frames_to_atom14, loss_fn, torsion_angles_to_frames


def compute_backbone(rigids_0: torch.Tensor, psi: torch.Tensor) -> torch.Tensor:
    """all_atom.compute_backbone (all_atom.py:157-180) as Experiment.loss_fn calls it (train_DFOLD_dynamics.py:1318-1320):
    rigids_0 [F,N,7], psi [F,N,2] -> [F,N,5,3] N, CA, C, CB, O of alanine (aatype 0 for every residue) with psi as all
    seven torsions, in the dtype of rigids_0."""
    aatype = torch.zeros(rigids_0.shape[:-1], dtype=torch.long, device=rigids_0.device)
    alpha = psi.to(rigids_0.dtype)[..., None, :].expand(psi.shape[:-1] + (7, 2))
    a37, _ = atom14_to_atom37(frames_to_atom14(torsion_angles_to_frames(rigids_0, alpha, aatype), aatype), aatype)
    return a37[..., :5, :]


def aux_structure_losses(pred_atoms: torch.Tensor, gt_atoms: torch.Tensor, res_mask: torch.Tensor,
                         fixed_mask: torch.Tensor, t: torch.Tensor, exp_conf):
    """The backbone-atom and pair-distance losses of Experiment.loss_fn (train_DFOLD_dynamics.py:1323-1364), per frame:
    pred_atoms / gt_atoms [F,N,5,3] (N, CA, C, CB, O), masks [F,N], t broadcast over frames -> (bb_atom_loss [F],
    dist_mat_loss [F]), weighted and gated by t < *_t_filter, in the promoted dtype of the inputs."""
    F_, N = res_mask.shape
    loss_mask = res_mask * (1 - fixed_mask)
    bm = torch.any(gt_atoms != 0, dim=-1) * loss_mask[..., None]
    bb = torch.sum((pred_atoms - gt_atoms) ** 2 * bm[..., None], dim=(-1, -2, -3)) / (bm.sum(dim=(-1, -2)) + 1e-10)
    bb = bb * exp_conf.bb_atom_loss_weight * (t < exp_conf.bb_atom_loss_t_filter) * exp_conf.aux_loss_weight
    gt_flat, pred_flat = gt_atoms.reshape(F_, 5 * N, 3), pred_atoms.reshape(F_, 5 * N, 3)
    gt_d = torch.linalg.norm(gt_flat[:, :, None, :] - gt_flat[:, None, :, :], dim=-1)
    pred_d = torch.linalg.norm(pred_flat[:, :, None, :] - pred_flat[:, None, :, :], dim=-1)
    flat_loss = loss_mask[:, :, None].expand(F_, N, 5).reshape(F_, 5 * N)
    flat_res = res_mask[:, :, None].expand(F_, N, 5).reshape(F_, 5 * N)
    gt_d = gt_d * flat_loss[..., None]
    pred_d = pred_d * flat_loss[..., None]
    pair = flat_loss[..., None] * flat_res[:, None, :] * (gt_d < 6)
    dm = torch.sum((gt_d - pred_d) ** 2 * pair, dim=(1, 2)) / (torch.sum(pair, dim=(1, 2)) - N)
    dm = dm * exp_conf.dist_mat_loss_weight * (t < exp_conf.dist_mat_loss_t_filter) * exp_conf.aux_loss_weight
    return bb, dm


def loss_fn_aux(out: Dict[str, torch.Tensor], batch: Dict[str, torch.Tensor], exp_conf, diffuse_rot: bool = True):
    """loss_fn with the backbone-atom and pair-distance terms in final_loss, as uncommenting train_DFOLD_dynamics.py:
    1370-1371 and the aux_data lines :1380-1381, :1388-1389 makes it.  Both terms cover every frame."""
    loss, aux = loss_fn(out, batch, exp_conf, diffuse_rot)
    gt = compute_backbone(batch["rigids_0"].to(torch.float32), batch["torsion_angles_sin_cos"][..., 2, :]).to(torch.float32)
    bb, dm = aux_structure_losses(out["atom37"][:, :, :5], gt, batch["res_mask"], batch["fixed_mask"], batch["t"], exp_conf)
    n = torch.any(batch["res_mask"], dim=-1).sum() + 1e-10
    final = aux["batch_rot_loss"] + aux["batch_trans_loss"] + bb.detach() + dm.detach() + aux["batch_torsion_loss"]
    keys = ("batch_train_loss", "batch_rot_loss", "batch_trans_loss", "batch_bb_atom_loss", "batch_dist_mat_loss",
            "batch_torsion_loss", "total_loss", "rot_loss", "trans_loss", "bb_atom_loss", "dist_mat_loss", "torsion_loss")
    vals = dict(aux, batch_train_loss=final, batch_bb_atom_loss=bb.detach(), batch_dist_mat_loss=dm.detach(),
                bb_atom_loss=(bb.sum() / n).detach(), dist_mat_loss=(dm.sum() / n).detach())
    total = loss + bb.sum() / n + dm.sum() / n
    vals["total_loss"] = total.detach()
    return total, {k: vals[k] for k in keys}
