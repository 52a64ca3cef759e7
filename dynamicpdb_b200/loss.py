"""Training loss of the DFOLDv2 score network on the device (SURVEY.md §8 f3).

``score_network_loss(model_out, batch, exp_conf)`` returns what ``Experiment.loss_fn`` returns after its model call
(reference train_DFOLD_dynamics.py:1206-1400): ``(loss, aux_data)`` with the same keys and dtypes (float64: its loader hands
float64 targets, which promotes every expression they enter) and the same gradients.  Only the last trajectory
frame is trained on (:1222, :1248, :1312), so the whole loss is ONE kernel over the N residues of that frame
(csrc/loss.cu) that also emits the gradients w.r.t. ``angles``, ``rot_score`` and the translation of ``rigids``; the
backward pass only scales them.  ``t`` and ``rot_score_scaling`` are read on the device (no host synchronisation, so the
step stays CUDA-graph capturable).

The reference also builds a backbone-atom MSE and a pair-distance loss over two O((5N)^2) tensors (:1316-1365) and
leaves them out of ``final_loss`` through two commented-out lines (:1370-1371).  By default they are not computed here
either.  ``aux_losses=True`` adds them as those lines would: both terms over EVERY frame of the window, against the
ground-truth backbone ``all_atom.compute_backbone`` builds from ``rigids_0`` and psi (aatype 0 for every residue), gated
by ``t < *_t_filter`` on the device, in one more kernel pair (csrc/aux_loss.cu) that tiles the pairs and never
materialises a (5N)^2 buffer.  Their gradient enters ``model_out["atom37"]`` of every frame.
"""
import numbers
from typing import Dict, Tuple

import torch
from torch.autograd import Function

from . import feats as _feats
from . import kernels as K

AUX_KEYS = ("bb_atom_loss_weight", "bb_atom_loss_t_filter", "dist_mat_loss_weight", "dist_mat_loss_t_filter",
            "aux_loss_weight")
_AUX_TILE = 128             # atoms per row tile of csrc/aux_loss.cu: the workspace holds 5 partials per (frame, tile)


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


class _AuxLossFn(Function):
    @staticmethod
    @K._on_device
    def forward(ctx, atom37, gt_atom37, res_mask, fixed_mask, t, consts):
        """atom37 [nf,N,37,3] predicted; gt_atom37 [nf,N,37,3] fp32 ground-truth backbone; masks [nf,N] and t fp64 ->
        out [2 + 2 nf] (bb_atom_loss, dist_mat_loss normalised, then per frame), d out[0:2] / d atom37 saved."""
        K._need_cuda(atom37, gt_atom37, res_mask, fixed_mask, t)
        nf, N = res_mask.shape
        if t.numel() not in (1, nf):
            raise ValueError(f"batch['t'] has {t.numel()} values for a window of {nf} frames")
        dev = atom37.device
        pred = atom37.detach().to(torch.float32).contiguous()
        work = torch.empty(nf * -(-5 * N // _AUX_TILE) * 5, dtype=torch.float64, device=dev)
        out = torch.empty(2 + 2 * nf, dtype=torch.float64, device=dev)
        d_bb = torch.empty(nf, N, 5, 3, dtype=torch.float64, device=dev)
        d_dm = torch.empty_like(d_bb)
        K.launch("dfold_aux_loss_fwd", pred, gt_atom37, res_mask, fixed_mask, t, 0 if t.numel() == 1 else 1, nf, N,
                 *[float(c) for c in consts], work, out, d_bb, d_dm)
        ctx.save_for_backward(d_bb, d_dm)
        ctx.meta = (atom37.shape, atom37.dtype)
        return out

    @staticmethod
    @K._on_device
    def backward(ctx, g):
        d_bb, d_dm = ctx.saved_tensors
        shape, dtype = ctx.meta
        ga = torch.zeros(shape, dtype=dtype, device=d_bb.device)
        ga[:, :, :5] = (g[0] * d_bb + g[1] * d_dm).to(dtype)      # out[2:] are logging values
        return ga, None, None, None, None, None


def aux_conf(exp_conf) -> Tuple[float, ...]:
    """The five weights and filters of the auxiliary losses (config/train_DFOLDv2.yaml:151-155), in ``AUX_KEYS`` order.
    Raises ValueError when one is missing or is not a number."""
    vals = []
    for k in AUX_KEYS:
        v = exp_conf.get(k) if isinstance(exp_conf, dict) else getattr(exp_conf, k, None)
        if isinstance(v, bool) or not isinstance(v, numbers.Real):
            raise ValueError(f"experiment.{k} must be a number for the auxiliary losses, got {v!r}")
        vals.append(float(v))
    return tuple(vals)


def ground_truth_backbone(batch: Dict[str, torch.Tensor]) -> torch.Tensor:
    """``all_atom.compute_backbone(Rigid.from_tensor_7(rigids_0.float()), psi)`` (train_DFOLD_dynamics.py:1318-1320,
    all_atom.py:157-180) on the device: [nf,N,37,3] fp32 atom37 of alanine (aatype 0 for every residue) with psi for all
    seven torsions; atoms 0..4 are N, CA, C, CB, O, the reference's gt_atom37[:, :, :5]."""
    rig = batch["rigids_0"].to(torch.float32)
    nf, N = rig.shape[:2]
    dev = rig.device
    quat, trans = rig[..., :4].contiguous(), rig[..., 4:].contiguous()
    alpha = batch["torsion_angles_sin_cos"][..., 2:3, :].to(torch.float32).expand(nf, N, 7, 2).contiguous()
    aatype = torch.zeros(nf, N, dtype=torch.long, device=dev)
    a37 = torch.empty(nf, N, 37, 3, dtype=torch.float32, device=dev)
    K.launch("dfold_frames_to_atoms_fwd", quat, 0, trans, alpha, aatype,
             *[_feats.table(k, dev) for k in _feats._TABLE_NAMES], None, None, a37, nf * N)
    return a37


def score_network_loss(model_out: Dict[str, torch.Tensor], batch: Dict[str, torch.Tensor], exp_conf, diffuse_rot: bool = True,
                       aux_losses: bool = False) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """``Experiment.loss_fn`` after the model call.  `exp_conf` needs torsion_loss_weight, rot_loss_weight,
    trans_loss_weight, rot_loss_t_threshold, separate_rot_loss (config/train_DFOLDv2.yaml:145-156).

    ``aux_losses=True`` adds the backbone-atom and pair-distance losses to the objective, as uncommenting
    train_DFOLD_dynamics.py:1370-1371 does, and their four values to ``aux_data`` (:1380-1381, :1388-1389); `exp_conf`
    then also needs the five ``AUX_KEYS``."""
    res_mask = batch["res_mask"]
    aux_consts = aux_conf(exp_conf) if aux_losses else None
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
    if not aux_losses:
        aux = {"batch_train_loss": rep(det[7]), "batch_rot_loss": rep(det[4]), "batch_trans_loss": rep(det[5]).to(trans_dt),
               "batch_torsion_loss": rep(det[6]), "total_loss": det[0], "rot_loss": det[1], "trans_loss": det[2].to(trans_dt),
               "torsion_loss": det[3]}
        return out[0], aux
    w_bb, t_bb, w_dm, t_dm, w_aux = aux_consts
    extra = _AuxLossFn.apply(model_out["atom37"], ground_truth_backbone(batch), fixed[5], fixed[6], f64(batch["t"]).reshape(-1),
                             (w_bb, t_bb, w_dm, t_dm, w_aux))
    loss = out[0] + extra[0] + extra[1]
    ex = extra.detach()
    # both terms keep the dtype of atom37 * loss_mask (:1333, :1353): float32 for the loader's float32 masks
    aux_dt = torch.promote_types(torch.promote_types(model_out["atom37"].dtype, res_mask.dtype), batch["fixed_mask"].dtype)
    bb, dm = ex[2:2 + batch_size].to(aux_dt), ex[2 + batch_size:].to(aux_dt)
    rot, trans, tor = rep(det[4]), rep(det[5]).to(trans_dt), rep(det[6])
    # the reference's dict order (:1376-1390) with its two auxiliary lines of each block restored
    aux = {"batch_train_loss": rot + trans + bb + dm + tor, "batch_rot_loss": rot, "batch_trans_loss": trans,
           "batch_bb_atom_loss": bb, "batch_dist_mat_loss": dm, "batch_torsion_loss": tor, "total_loss": loss.detach(),
           "rot_loss": det[1], "trans_loss": det[2].to(trans_dt), "bb_atom_loss": ex[0].to(aux_dt),
           "dist_mat_loss": ex[1].to(aux_dt), "torsion_loss": det[3]}
    return loss, aux
