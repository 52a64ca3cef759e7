"""Training loss of the DFOLDv2 score network on the device (SURVEY.md §8 f3).

``score_network_loss(model_out, batch, exp_conf)`` returns what ``Experiment.loss_fn`` returns after its model call
(reference train_DFOLD_dynamics.py:1206-1400): ``(loss, aux_data)`` with the same keys and dtypes (float64: its loader hands
float64 targets, which promotes every expression they enter) and the same gradients.  Only the last trajectory
frame is trained on (:1222, :1248, :1312), so the whole loss is ONE kernel over the N residues of that frame
(csrc/loss.cu) that also emits the gradients w.r.t. ``angles``, ``rot_score`` and the translation of ``rigids``; the
backward pass only scales them.  ``t`` and ``rot_score_scaling`` are read on the device (no host synchronisation, so the
step stays CUDA-graph capturable).  The reference additionally builds two O((5N)^2) pair-distance tensors and a
ground-truth backbone (:1316-1365) that never reach ``final_loss`` (:1367-1373) — they are not computed here.
"""
from typing import Dict, Tuple

import torch
from torch.autograd import Function

from . import kernels as K


class _LossFn(Function):
    @staticmethod
    @K._on_device
    def forward(ctx, angles, rot_score, rigids, fixed, consts):
        """fixed: the non-differentiated fp64 tensors (a_gt, a_alt, a_mask, gt_rot, x0, res_mask, fixed_mask, t, rot_scaling)."""
        K._need_cuda(angles, rot_score, rigids)
        a_gt, a_alt, a_mask, gt_rot, x0, res_mask, fixed_mask, t, scaling = fixed
        nf, N = res_mask.shape
        dev = angles.device
        f64 = lambda v: v.detach().to(torch.float64).contiguous()
        ang, rs, x = f64(angles[-1]), f64(rot_score[-1]), f64(rigids[-1, :, 4:])
        out = torch.empty(8, dtype=torch.float64, device=dev)
        d_ang, d_rs, d_x = torch.empty_like(ang), torch.empty_like(rs), torch.empty_like(x)
        w_tor, w_rot, w_trans, t_thr, rot_on, separate = consts
        K.launch("dfold_loss_fwd", ang, a_gt, a_alt, a_mask, rs, gt_rot, x, x0, res_mask, fixed_mask, t, scaling,
                 nf, N, float(w_tor), float(w_rot), float(w_trans), float(t_thr), int(rot_on), int(separate), out, d_ang, d_rs, d_x)
        ctx.save_for_backward(d_ang, d_rs, d_x)
        ctx.meta = (angles.shape, angles.dtype, rot_score.shape, rot_score.dtype, rigids.shape, rigids.dtype)
        return out

    @staticmethod
    @K._on_device
    def backward(ctx, g):
        d_ang, d_rs, d_x = ctx.saved_tensors
        sa, da, sr, dr, sx, dx = ctx.meta
        dev = d_ang.device
        ga = torch.zeros(sa, dtype=da, device=dev)
        gr = torch.zeros(sr, dtype=dr, device=dev)
        gx = torch.zeros(sx, dtype=dx, device=dev)
        ga[-1] = (g[0] * d_ang).to(da)          # only out[0] (the loss) carries gradient; out[1:] are logging values
        gr[-1] = (g[0] * d_rs).to(dr)
        gx[-1, :, 4:] = (g[0] * d_x).to(dx)
        return ga, gr, gx, None, None


def score_network_loss(model_out: Dict[str, torch.Tensor], batch: Dict[str, torch.Tensor], exp_conf, diffuse_rot: bool = True
                       ) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """``Experiment.loss_fn`` after the model call.  `exp_conf` needs torsion_loss_weight, rot_loss_weight,
    trans_loss_weight, rot_loss_t_threshold, separate_rot_loss (config/train_DFOLDv2.yaml:145-156)."""
    res_mask = batch["res_mask"]
    if not res_mask.is_cuda:
        raise RuntimeError("dynamicpdb_b200.loss has no CPU path (the reference's loss_fn runs on host tensors)")
    f64 = lambda v: v.detach().to(torch.float64).contiguous()
    batch_size = res_mask.shape[0]
    fixed = (f64(batch["torsion_angles_sin_cos"][-1]), f64(batch["alt_torsion_angles_sin_cos"][-1]),
             f64(batch["torsion_angles_mask"][-1]), f64(batch["rot_score"][-1]), f64(batch["rigids_0"][-1, :, 4:]),
             f64(res_mask), f64(batch["fixed_mask"]), f64(batch["t"]).reshape(-1)[-1:],
             f64(batch["rot_score_scaling"]).reshape(-1)[-1:])
    consts = (exp_conf.torsion_loss_weight, exp_conf.rot_loss_weight, exp_conf.trans_loss_weight,
              exp_conf.rot_loss_t_threshold, 1 if diffuse_rot else 0, 1 if exp_conf.separate_rot_loss else 0)
    out = _LossFn.apply(model_out["angles"], model_out["rot_score"], model_out["rigids"], fixed, consts)
    det = out.detach()
    rep = lambda v: v.reshape(1).repeat(batch_size)
    # the translation term alone never meets a float64 target in the reference (:1241-1248): its two logging values keep
    # the dtype of rigids_0 - rigids, float32 for the loader's batches
    trans_dt = torch.promote_types(batch["rigids_0"].dtype, model_out["rigids"].dtype)
    aux = {"batch_train_loss": rep(det[7]), "batch_rot_loss": rep(det[4]), "batch_trans_loss": rep(det[5]).to(trans_dt),
           "batch_torsion_loss": rep(det[6]), "total_loss": det[0], "rot_loss": det[1], "trans_loss": det[2].to(trans_dt),
           "torsion_loss": det[3]}
    return out[0], aux
