"""Trajectory metrics of the evaluator on the device (SURVEY.md §8 f6, csrc/metrics.cu).

The reference scores every sampled test window on the host (``Experiment.eval_fn``, train_DFOLD_dynamics.py:765-928, and
``compute_validation_metrics_all``, :99-154): a device-to-host copy of the trajectory, a synchronisation, then numpy /
torch-CPU / Bio arithmetic per window.  Here the same numbers come from fp64 kernels: device tensors in, device tensors out,
no ``.item()`` and no host synchronisation, so a whole evaluation loop (prefetch, sample, score) can stay on the device and
read back only the metrics.  CPU tensors raise, as everywhere in the package.

Definitions kept from the reference on purpose (each is tested):
* the translation MAE of ``rot_trans_error`` is not masked (src/toolbox/rot_trans_error.py:16);
* ``rmsd_all`` / ``rmsd_ca`` add ``1e-4`` to the mask count (:143-146);
* ``drmsd`` divides by ``n (n - 1)`` with ``n`` the minimum over frames of the mask count (validation_metrics.py:32);
* ``rmsd_ca_aligned`` superimposes all N CA positions, the masked ones zeroed (:113-150);
* ``window_metrics`` drops the last atom of the last residue of the last frame from the mask (``atom_mask[-1, -1, -1] =
  0``, :893), unless ``drop_last_atom=False``.
Where the reference computes in fp32 (the predicted quaternions are normalised in the model's fp32, a fp32 mask makes
``1 / (n (n - 1))`` fp32), the kernels compute in fp64.
"""
from typing import Dict, Optional

import torch

from . import kernels as K

_TILE = 64          # dRMSD tile edge (csrc/metrics.cu kTile)


def _src(t: torch.Tensor):
    """A contiguous fp32 / fp64 view of ``t`` (other dtypes are upcast to fp64) and the kernel's dtype flag."""
    t = t.detach()
    if t.dtype not in (torch.float32, torch.float64):
        t = t.to(torch.float64)
    return t.contiguous(), int(t.dtype == torch.float64)


def _f64(*shape, device):
    return torch.empty(*shape, dtype=torch.float64, device=device)


def rot_trans_error(pred_rigids: torch.Tensor, gt_rigids: torch.Tensor, ref_frame: int = -2):
    """``Experiment._calc_rot_trans_error`` (train_DFOLD_dynamics.py:1549-1568) of pred / gt rigids [nf, N, 7] (w,x,y,z, trans):
    (ave_rot, ave_trans, ref_ave_rot, ref_ave_trans), each [nf] fp64 -- the mean quaternion angle in degrees and the
    unmasked translation MAE of the prediction against the ground truth, and of ground-truth frame ``ref_frame`` (the
    reference's baseline, frame -2) broadcast over the window."""
    K._need_cuda(pred_rigids, gt_rigids)
    if pred_rigids.dim() != 3 or pred_rigids.shape[-1] != 7 or pred_rigids.shape != gt_rigids.shape:
        raise ValueError(f"rot_trans_error: need pred / gt rigids [nf, N, 7] of one shape, got {tuple(pred_rigids.shape)} "
                         f"and {tuple(gt_rigids.shape)}")
    nf, N = gt_rigids.shape[0], gt_rigids.shape[1]
    rf = ref_frame + nf if ref_frame < 0 else ref_frame
    if not 0 <= rf < nf:
        raise ValueError(f"rot_trans_error: ref_frame {ref_frame} outside a window of {nf} frames")
    dev = gt_rigids.device
    with torch.cuda.device(dev):
        p, p64 = _src(pred_rigids)
        g, g64 = _src(gt_rigids)
        out = _f64(4, nf, device=dev)
        K.launch("dfold_rot_trans_error", p, p64, g, g64, nf, N, rf, out)
    return out[0], out[1], out[2], out[3]


def atom_errors(atom37_pred: torch.Tensor, atom37_gt: torch.Tensor, atom37_mask: torch.Tensor,
                drop_last_atom: bool = False) -> Dict[str, torch.Tensor]:
    """Per-frame masked atom errors of pred / gt [nf, N, A, 3] under mask [nf, N, A] (CA = atom column 1), each [nf] fp64:
    ``mae`` / ``mse`` as eval_fn computes them (:892-912, mean over the xyz-expanded mask; an empty frame gives NaN),
    ``rmsd_all`` / ``rmsd_ca`` as compute_validation_metrics_all (:143-146, ``+ 1e-4`` in the denominator)."""
    K._need_cuda(atom37_pred, atom37_gt, atom37_mask)
    if atom37_pred.dim() != 4 or atom37_pred.shape[-1] != 3 or atom37_pred.shape != atom37_gt.shape \
            or tuple(atom37_mask.shape) != tuple(atom37_gt.shape[:-1]):
        raise ValueError(f"atom_errors: need pred / gt [nf, N, A, 3] and mask [nf, N, A], got {tuple(atom37_pred.shape)}, "
                         f"{tuple(atom37_gt.shape)}, {tuple(atom37_mask.shape)}")
    nf, N, A = atom37_gt.shape[:3]
    dev = atom37_gt.device
    with torch.cuda.device(dev):
        p, p64 = _src(atom37_pred)
        g, g64 = _src(atom37_gt)
        m, m64 = _src(atom37_mask)
        out = _f64(6, nf, device=dev)
        K.launch("dfold_atom_errors", p, p64, g, g64, m, m64, nf, N, A, int(bool(drop_last_atom)), out)
    return {"mae": out[0], "mse": out[1], "rmsd_all": out[2], "rmsd_ca": out[3]}


def _superimpose(ref, ref64, x, x64, offset, sstride, pstride, mask, m64, moff, msstride, mpstride, mode, B, P, dev,
                 with_coords, with_transform):
    rmsd = _f64(B, device=dev)
    coords = _f64(B, P, 3, device=dev) if with_coords else None
    rot = _f64(B, 3, 3, device=dev) if with_transform else None
    trans = _f64(B, 3, device=dev) if with_transform else None
    K.launch("dfold_superimpose", K._ptr(ref, offset), ref64, K._ptr(x, offset), x64, sstride, pstride,
             K._ptr(mask, moff), m64, msstride, mpstride, mode, B, P, rmsd, rot, trans, coords)
    return coords, rmsd, rot, trans


def superimpose(reference: torch.Tensor, coords: torch.Tensor, mask: Optional[torch.Tensor] = None,
                return_transform: bool = False):
    """``openfold.utils.superimposition.superimpose`` batched on the device: superimposes ``coords`` [*, P, 3] onto
    ``reference`` [*, P, 3] (Kabsch, fp64, proper rotations) and returns (superimposed [*, P, 3], rmsd [*]), both fp64.
    ``mask`` [*, P] (optional) weights the points -- a 0/1 mask selects them, as eval_fn's ``sup.set(pred[idx], gt[idx])``
    (:902-908) -- and every point is transformed.  An empty selection gives rmsd NaN and the coordinates unchanged.
    With ``return_transform`` also (rot [*, 3, 3], trans [*, 3]) with superimposed = coords @ rot^T + trans."""
    K._need_cuda(reference, coords, mask)
    if reference.dim() < 2 or reference.shape[-1] != 3 or reference.shape != coords.shape:
        raise ValueError(f"superimpose: need reference / coords [*, P, 3] of one shape, got {tuple(reference.shape)} and "
                         f"{tuple(coords.shape)}")
    if mask is not None and tuple(mask.shape) != tuple(reference.shape[:-1]):
        raise ValueError(f"superimpose: mask {tuple(mask.shape)} does not match points {tuple(reference.shape[:-1])}")
    batch, P = reference.shape[:-2], reference.shape[-2]
    B = 1
    for b in batch:
        B *= b
    if B == 0 or P == 0:
        raise ValueError("superimpose: empty batch or point set")
    dev = reference.device
    with torch.cuda.device(dev):
        r, r64 = _src(reference)
        x, x64 = _src(coords)
        m, m64 = _src(mask) if mask is not None else (None, 0)
        out, rmsd, rot, trans = _superimpose(r, r64, x, x64, 0, 3 * P, 3, m, m64, 0, P, 1, 0 if m is None else 1, B, P, dev,
                                             True, return_transform)
    res = (out.reshape(*batch, P, 3), rmsd.reshape(batch))
    if return_transform:
        res = res + (rot.reshape(*batch, 3, 3), trans.reshape(*batch, 3))
    return res


def _drmsd(s1, a64, s2, b64, offset, sstride, pstride, mask, m64, moff, msstride, mpstride, premul, B, N, dev):
    T = (N + _TILE - 1) // _TILE
    if B > 65535:
        raise ValueError(f"drmsd: {B} structure pairs exceed 65535")
    partial = _f64(B * T * T, device=dev)
    out = _f64(B, device=dev)
    K.launch("dfold_drmsd", K._ptr(s1, offset), a64, K._ptr(s2, offset), b64, sstride, pstride,
             K._ptr(mask, moff), m64, msstride, mpstride, int(premul), B, N, partial, out)
    return out


def drmsd(structure_1: torch.Tensor, structure_2: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``openfold.utils.validation_metrics.drmsd`` (:17-36) of [*, N, 3] structures on the device: [*] fp64.  The pair
    sum is masked by ``mask_i mask_j`` and divided by ``n (n - 1)`` with ``n`` the MINIMUM over all leading indices of
    ``mask.sum(-1)`` (N without a mask); ``n <= 1`` gives 0."""
    K._need_cuda(structure_1, structure_2, mask)
    if structure_1.dim() < 2 or structure_1.shape[-1] != 3 or structure_1.shape != structure_2.shape:
        raise ValueError(f"drmsd: need structures [*, N, 3] of one shape, got {tuple(structure_1.shape)} and "
                         f"{tuple(structure_2.shape)}")
    if mask is not None and tuple(mask.shape) != tuple(structure_1.shape[:-1]):
        raise ValueError(f"drmsd: mask {tuple(mask.shape)} does not match points {tuple(structure_1.shape[:-1])}")
    batch, N = structure_1.shape[:-2], structure_1.shape[-2]
    B = 1
    for b in batch:
        B *= b
    if B == 0 or N == 0:
        raise ValueError("drmsd: empty batch or structure")
    dev = structure_1.device
    with torch.cuda.device(dev):
        a, a64 = _src(structure_1)
        b, b64 = _src(structure_2)
        m, m64 = _src(mask) if mask is not None else (None, 0)
        out = _drmsd(a, a64, b, b64, 0, 3 * N, 3, m, m64, 0, N, 1, False, B, N, dev)
    return out.reshape(batch)


def _check_atom37(gt_pos, out_pos, gt_mask, what):
    K._need_cuda(gt_pos, out_pos, gt_mask)
    if gt_pos.dim() != 4 or gt_pos.shape[-1] != 3 or gt_pos.shape[-2] < 2 or gt_pos.shape != out_pos.shape \
            or tuple(gt_mask.shape) != tuple(gt_pos.shape[:-1]):
        raise ValueError(f"{what}: need positions [nf, N, A, 3] (A >= 2) and mask [nf, N, A], got {tuple(gt_pos.shape)}, "
                         f"{tuple(out_pos.shape)}, {tuple(gt_mask.shape)}")


def validation_metrics_all(gt_pos: torch.Tensor, out_pos: torch.Tensor, gt_mask: torch.Tensor) -> Dict[str, torch.Tensor]:
    """``compute_validation_metrics_all(gt_pos, out_pos, gt_mask, superimposition_metrics=True)`` (train_DFOLD_dynamics.py:
    99-154) of atom37 positions [nf, N, 37, 3] and mask [nf, N, 37]: {rmsd_all, rmsd_ca, drmsd_ca, rmsd_ca_aligned}, each
    [nf] fp64.  The CA columns are read in place (no copies)."""
    _check_atom37(gt_pos, out_pos, gt_mask, "validation_metrics_all")
    nf, N, A = gt_pos.shape[:3]
    dev = gt_pos.device
    with torch.cuda.device(dev):
        g, g64 = _src(gt_pos)
        p, p64 = _src(out_pos)
        m, m64 = _src(gt_mask)
        err = atom_errors(p, g, m)
        ca = 1                       # residue_constants.atom_order["CA"]
        d = _drmsd(p, p64, g, g64, 3 * ca, 3 * N * A, 3 * A, m, m64, ca, N * A, A, True, nf, N, dev)
        _, aligned, _, _ = _superimpose(g, g64, p, p64, 3 * ca, 3 * N * A, 3 * A, m, m64, ca, N * A, A, 2, nf, N, dev,
                                        False, False)
    return {"rmsd_all": err["rmsd_all"], "rmsd_ca": err["rmsd_ca"], "drmsd_ca": d, "rmsd_ca_aligned": aligned}


def window_metrics(rigid_pred: torch.Tensor, atom37_pred: torch.Tensor, rigids_0: torch.Tensor, atom37_pos: torch.Tensor,
                   atom37_mask: torch.Tensor, drop_last_atom: bool = True) -> Dict[str, torch.Tensor]:
    """eval_fn's per-window row (train_DFOLD_dynamics.py:883-912) from the sampler's final prediction ``rigid_pred``
    [nf, N, 7] and ``atom37_pred`` [nf, N, 37, 3] (``rigid_traj[0]`` / ``prot_traj[0]``, t = min_t) and the window's
    ``rigids_0``, ``atom37_pos``, ``atom37_mask``:
    ``ave_rot``, ``ave_trans``, ``all_atom_mae``, ``all_atom_mse`` -- the last frame's values, [1] fp64 (eval_fn keeps
    ``[-1:]``) -- and ``all_atom_rmsd`` [1]: the RMSD of the last frame's masked atoms after superposition.
    ``per_frame`` holds the full [nf] vectors (``ave_rot``, ``ave_trans``, ``ref_ave_rot``, ``ref_ave_trans``,
    ``all_atom_mae``, ``all_atom_mse``).  ``drop_last_atom`` applies eval_fn's ``atom_mask[-1, -1, -1] = 0.0``."""
    _check_atom37(atom37_pos, atom37_pred, atom37_mask, "window_metrics")
    rot, tr, rrot, rtr = rot_trans_error(rigid_pred, rigids_0, -2)
    err = atom_errors(atom37_pred, atom37_pos, atom37_mask, drop_last_atom=drop_last_atom)
    nf, N, A = atom37_pos.shape[:3]
    dev = atom37_pos.device
    with torch.cuda.device(dev):
        sel = atom37_mask[-1].detach().to(torch.float64).reshape(N * A).clone()
        if drop_last_atom:
            sel[-1:].fill_(0.0)          # a device fill: no host copy, so the call can be graph-captured
        # Bio's sup.set(pred[idx], gt[idx]) (:905): the ground truth is moved onto the prediction; the RMSD is symmetric
        _, rmsd = superimpose(atom37_pred[-1].reshape(N * A, 3), atom37_pos[-1].reshape(N * A, 3), sel)
    per_frame = {"ave_rot": rot, "ave_trans": tr, "ref_ave_rot": rrot, "ref_ave_trans": rtr,
                 "all_atom_mae": err["mae"], "all_atom_mse": err["mse"]}
    return {"ave_rot": rot[-1:], "ave_trans": tr[-1:], "all_atom_mae": err["mae"][-1:], "all_atom_mse": err["mse"][-1:],
            "all_atom_rmsd": rmsd.reshape(1), "per_frame": per_frame}


HORIZON_KEYS = ("ave_rot", "ave_trans", "all_atom_mae", "all_atom_mse", "all_atom_rmsd", "persist_rot", "persist_trans")


def horizon_metrics(rigid_traj: torch.Tensor, atom_traj: torch.Tensor, last_seen: torch.Tensor, rigids_0: torch.Tensor,
                    atom37_pos: torch.Tensor, atom37_mask: torch.Tensor, drop_last_atom: bool = True) -> torch.Tensor:
    """eval_fn's row (``window_metrics``) at every frame of a rollout: [L, 7] fp64 in ``HORIZON_KEYS`` order, row j scoring
    ``rigid_traj[j]`` [N, 7] / ``atom_traj[j]`` [N, 37, 3] against the MD frame it predicts (``rigids_0[j]``,
    ``atom37_pos[j]`` under ``atom37_mask[j]``, each [L, ...]).  ``drop_last_atom`` applies eval_fn's ``atom_mask[-1, -1, -1]
    = 0`` to every frame, as eval_fn applies it to the one frame it scores.  ``persist_rot`` / ``persist_trans`` are the
    errors of repeating ``last_seen`` [N, 7], the last MD frame the network was given, at every horizon: the
    ``ref_frame`` baseline of ``rot_trans_error`` with that frame prepended.  Every row is computed by the kernels as
    ``window_metrics`` computes its last frame, so row 0 of a rollout equals its row bit for bit.  Nothing is read back."""
    L, N = rigid_traj.shape[:2]
    A = atom37_pos.shape[2]
    if rigids_0.shape != rigid_traj.shape or tuple(last_seen.shape) != (N, 7) or atom_traj.shape != atom37_pos.shape \
            or tuple(atom37_mask.shape) != (L, N, A) or tuple(atom_traj.shape[:2]) != (L, N):
        raise ValueError(f"horizon_metrics: need rigids [L, N, 7], last_seen [N, 7], atoms [L, N, A, 3] and mask [L, N, A], got "
                         f"{tuple(rigid_traj.shape)}, {tuple(rigids_0.shape)}, {tuple(last_seen.shape)}, "
                         f"{tuple(atom_traj.shape)}, {tuple(atom37_pos.shape)}, {tuple(atom37_mask.shape)}")
    K._need_cuda(rigid_traj, atom_traj, last_seen, rigids_0, atom37_pos, atom37_mask)
    dev = rigids_0.device
    with torch.cuda.device(dev):
        seen = last_seen.unsqueeze(0)
        gt = torch.cat([seen.to(rigids_0.dtype), rigids_0])
        pred = torch.cat([seen.to(rigid_traj.dtype), rigid_traj])
        rot, tr, prot, ptr = rot_trans_error(pred, gt, ref_frame=0)
        mask = torch.empty(L, N, A, dtype=torch.float64, device=dev).copy_(atom37_mask)
        if drop_last_atom:
            mask[:, -1, -1].fill_(0.0)
        err = atom_errors(atom_traj, atom37_pos, mask)
        # as window_metrics: the ground truth is moved onto the prediction
        _, rmsd = superimpose(atom_traj.reshape(L, N * A, 3), atom37_pos.reshape(L, N * A, 3), mask.reshape(L, N * A))
        return torch.stack([rot[1:], tr[1:], err["mae"], err["mse"], rmsd, prot[1:], ptr[1:]], dim=1)


# the sampler inputs eval_fn builds (:826-844) besides the ones it makes itself
_EVAL_WINDOW_KEYS = ("torsion_angles_sin_cos", "torsion_angles_mask", "node_repr", "edge_repr", "aatype", "rigids_t", "rigids_0",
                     "force", "vel")


def eval_sampler_inputs(window: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The sampler inputs eval_fn (train_DFOLD_dynamics.py:826-844) and eval_extension (:954-966) build from a window:
    the window's own fields of ``_EVAL_WINDOW_KEYS`` (the same tensors, not copies) plus ``res_mask`` ones, ``fixed_mask``
    zeros, ``sc_ca_t`` zeros and ``seq_idx = arange(1, N + 1)`` (not the residue index)."""
    nf, N = window["rigids_0"].shape[:2]
    dev = window["rigids_0"].device
    init = {k: window[k] for k in _EVAL_WINDOW_KEYS}
    init.update({
        "res_mask": torch.ones(nf, N, dtype=torch.float64, device=dev),
        "fixed_mask": torch.zeros(nf, N, dtype=torch.float64, device=dev),
        "seq_idx": torch.arange(1, N + 1, device=dev).unsqueeze(0).repeat(nf, 1),
        "sc_ca_t": torch.zeros(nf, N, 3, dtype=torch.float32, device=dev),
    })
    return init


def evaluate_window(sampler, window: Dict[str, torch.Tensor], num_t: int, min_t: float, noise_scale: float = 1.0):
    """One protein of eval_fn (train_DFOLD_dynamics.py:813-912) on the device.  ``window`` is an evaluation item of
    ``WindowPrefetcher(..., training=False, diffuser=..., targets=True)`` (``rigids_t`` from ``sample_ref``, plus
    ``atom37_pos`` / ``atom37_mask``); ``sampler`` a ``DeviceReverseDiffusion``.  The sampler's inputs are built as eval_fn
    builds them (``eval_sampler_inputs``); the targets never enter the sampler's graph.  Runs ``sampler.sample_graphed`` and
    returns ``window_metrics`` of its ``rigid_pred`` / ``prot_traj[0]`` -- device tensors; nothing is read back."""
    missing = [k for k in _EVAL_WINDOW_KEYS + ("atom37_pos", "atom37_mask") if k not in window]
    if missing:
        raise ValueError(f"evaluate_window: the window lacks {missing} (WindowPrefetcher(training=False, diffuser=..., "
                         "targets=True) provides them)")
    out = sampler.sample_graphed(eval_sampler_inputs(window), num_t, min_t, noise_scale)
    return window_metrics(out["rigid_pred"], out["prot_traj"][0], window["rigids_0"], window["atom37_pos"],
                          window["atom37_mask"])
