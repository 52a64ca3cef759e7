"""fp64 torch restatement of the evaluator's trajectory metrics (what dynamicpdb_b200/metrics.py computes with
csrc/metrics.cu).  Plain functions on CPU or CUDA tensors, everything upcast to float64; each cites the reference lines it
restates (train_DFOLD_dynamics.py unless a file is named).  Pinned against the unmodified reference by
tests/golden/metrics.pt (oracle/make_metrics_golden.py); its Kabsch against scipy's Rotation.align_vectors."""
import math

import torch

CA = 1      # openfold/np/residue_constants.py atom_order["CA"]


def _d(x):
    return x.detach().to(torch.float64)


def quaternion_angles_deg(q1, q2):
    """src/toolbox/rot_trans_error.py:50-60: q / |q|, degrees(2 acos |clip(q1 . q2, -1, 1)|)."""
    q1, q2 = _d(q1), _d(q2)
    q1 = q1 / q1.norm(dim=-1, keepdim=True)
    q2 = q2 / q2.norm(dim=-1, keepdim=True)
    dot = (q1 * q2).sum(-1).clamp(-1.0, 1.0)
    return torch.rad2deg(2.0 * torch.acos(dot.abs()))


def rot_trans_error(pred, gt, ref_frame=-2):
    """Experiment._calc_rot_trans_error (:1549-1568) over rot_trans_error.py:7-73: per frame the mean angle (degrees) and
    the UNMASKED translation MAE (mean over residues and xyz, :16) of pred vs gt and of gt[ref_frame] (broadcast) vs gt."""
    pred, gt = _d(pred), _d(gt)
    ref = gt[ref_frame].unsqueeze(0).expand_as(gt)
    rot = quaternion_angles_deg(gt[..., :4], pred[..., :4]).mean(-1)
    tr = (gt[..., 4:] - pred[..., 4:]).abs().mean(dim=(-1, -2))
    rrot = quaternion_angles_deg(gt[..., :4], ref[..., :4]).mean(-1)
    rtr = (gt[..., 4:] - ref[..., 4:]).abs().mean(dim=(-1, -2))
    return rot, tr, rrot, rtr


def eval_mask(atom37_mask, drop_last_atom=True):
    """eval_fn's atom mask (:892-893): [nf, N, 37] with ``atom_mask[-1, -1, -1] = 0.0``."""
    m = _d(atom37_mask).clone()
    if drop_last_atom:
        m[-1, -1, -1] = 0.0
    return m


def atom_errors(pred, gt, mask, drop_last_atom=False):
    """Per frame: eval_fn's MAE / MSE (:895, :911; the mask expanded over xyz, so the count is 3 sum m; 0/0 = NaN) and
    compute_validation_metrics_all's rmsd_all / rmsd_ca (:113-146; (gt m - pred m)^2, denominator sum m + 1e-4)."""
    pred, gt = _d(pred), _d(gt)
    m = eval_mask(mask, drop_last_atom)
    m3 = m.unsqueeze(-1).expand_as(gt)
    mae = ((gt - pred).abs() * m3).sum(dim=(-1, -2, -3)) / m3.sum(dim=(-1, -2, -3))
    mse = ((gt - pred) ** 2 * m3).sum(dim=(-1, -2, -3)) / m3.sum(dim=(-1, -2, -3))
    diff = gt * m[..., None] - pred * m[..., None]
    rmsd_all = torch.sqrt((diff ** 2).sum(dim=(-1, -2, -3)) / (m.sum(dim=(-1, -2)) + 1e-4))
    dca = diff[..., CA, :]
    rmsd_ca = torch.sqrt((dca ** 2).sum(dim=(-1, -2)) / (m[..., CA].sum(-1) + 1e-4))
    return {"mae": mae, "mse": mse, "rmsd_all": rmsd_all, "rmsd_ca": rmsd_ca}


def kabsch(reference, coords, weights=None):
    """Weighted Kabsch of coords [*, P, 3] onto reference [*, P, 3] in fp64 (the algorithm of the reference's own
    ``rmsdalign``, :74-97, and of Bio's SVDSuperimposer): centroids, then the CENTRED covariance H = sum w (x - cx)(r - cr)^T,
    H = U S V^T, the determinant fix d = sign(det(V U^T)), R = V diag(1, 1, d) U^T; the RMSD from the applied transform.
    Returns (superimposed [*, P, 3], rmsd [*], R [*, 3, 3], t [*, 3]) with superimposed = coords R^T + t.
    An empty selection (sum w = 0) gives rmsd NaN, R = I, t = 0."""
    r, x = _d(reference), _d(coords)
    w = torch.ones(r.shape[:-1], dtype=torch.float64, device=r.device) if weights is None else _d(weights)
    W = w.sum(-1)
    cr = (w[..., None] * r).sum(-2) / W[..., None]
    cx = (w[..., None] * x).sum(-2) / W[..., None]
    rc, xc = r - cr[..., None, :], x - cx[..., None, :]
    H = torch.einsum("...p,...pi,...pj->...ij", w, xc, rc)
    empty = ~(W != 0)
    H = torch.where(empty[..., None, None], torch.zeros_like(H), H)
    U, S, Vh = torch.linalg.svd(H)
    V = Vh.mT
    d = torch.sign(torch.linalg.det(V @ U.mT))
    d = torch.where(d == 0, torch.ones_like(d), d)
    D = torch.diag_embed(torch.stack([torch.ones_like(d), torch.ones_like(d), d], -1))
    R = V @ D @ U.mT
    R = torch.where(empty[..., None, None], torch.eye(3, dtype=torch.float64, device=r.device).expand_as(R), R)
    y = xc @ R.mT
    rmsd = torch.sqrt((w * ((y - rc) ** 2).sum(-1)).sum(-1) / W)
    t = cr - (R @ cx[..., None])[..., 0]
    sup = torch.where(empty[..., None, None], x, y + cr[..., None, :])
    t = torch.where(empty[..., None], torch.zeros_like(t), t)
    return sup, rmsd, R, t


def superimpose(reference, coords, mask=None):
    """openfold/utils/superimposition.py:45-77 (one SVDSuperimposer per set) batched: (superimposed, rmsd)."""
    sup, rmsd, _, _ = kabsch(reference, coords, mask)
    return sup, rmsd


def drmsd(s1, s2, mask=None):
    """openfold/utils/validation_metrics.py:17-36: n = min over every leading index of sum(mask, -1) (N without a mask);
    sum (d1 - d2)^2 m_i m_j / (n (n - 1)) when n > 1, else 0."""
    s1, s2 = _d(s1), _d(s2)
    d1 = ((s1[..., :, None, :] - s1[..., None, :, :]) ** 2).sum(-1).sqrt()
    d2 = ((s2[..., :, None, :] - s2[..., None, :, :]) ** 2).sum(-1).sqrt()
    dd = (d1 - d2) ** 2
    if mask is not None:
        m = _d(mask)
        dd = dd * (m[..., None] * m[..., None, :])
    tot = dd.sum(dim=(-1, -2))
    n = float(s1.shape[-2]) if mask is None else float(_d(mask).sum(-1).min())
    return torch.sqrt(tot * (1.0 / (n * (n - 1.0)))) if n > 1 else torch.sqrt(tot * 0.0)


def validation_metrics_all(gt_pos, out_pos, gt_mask):
    """compute_validation_metrics_all(..., superimposition_metrics=True) (:99-154): coordinates multiplied by the mask,
    drmsd_ca of the masked CA positions with the CA mask, rmsd_all / rmsd_ca with ``+ 1e-4``, rmsd_ca_aligned over ALL N
    masked (zeroed) CA positions."""
    g, p, m = _d(gt_pos), _d(out_pos), _d(gt_mask)
    gm, pm = g * m[..., None], p * m[..., None]
    err = atom_errors(p, g, m)
    return {"rmsd_all": err["rmsd_all"], "rmsd_ca": err["rmsd_ca"],
            "drmsd_ca": drmsd(pm[..., CA, :], gm[..., CA, :], m[..., CA]),
            "rmsd_ca_aligned": superimpose(gm[..., CA, :], pm[..., CA, :])[1]}


def window_metrics(rigid_pred, atom37_pred, rigids_0, atom37_pos, atom37_mask, drop_last_atom=True):
    """eval_fn's per-window row (:883-912): last-frame ave_rot / ave_trans / all_atom_mae / all_atom_mse ([1]) and the
    last frame's all-atom RMSD after superposition of the atoms its (quirk-adjusted) mask selects."""
    rot, tr, rrot, rtr = rot_trans_error(rigid_pred, rigids_0, -2)
    err = atom_errors(atom37_pred, atom37_pos, atom37_mask, drop_last_atom)
    m = eval_mask(atom37_mask, drop_last_atom)[-1].reshape(-1)
    P = m.numel()
    _, rmsd = superimpose(_d(atom37_pred)[-1].reshape(P, 3), _d(atom37_pos)[-1].reshape(P, 3), m)
    per_frame = {"ave_rot": rot, "ave_trans": tr, "ref_ave_rot": rrot, "ref_ave_trans": rtr,
                 "all_atom_mae": err["mae"], "all_atom_mse": err["mse"]}
    return {"ave_rot": rot[-1:], "ave_trans": tr[-1:], "all_atom_mae": err["mae"][-1:], "all_atom_mse": err["mse"][-1:],
            "all_atom_rmsd": rmsd.reshape(1), "per_frame": per_frame}


def key_matrix_gap(reference, coords, weights=None):
    """Relative gap (lambda_1 - lambda_2) / (|lambda_1| + tiny) of the top two eigenvalues of Horn's 4x4 key matrix, in
    fp64: where it is small the optimal rotation is (nearly) not unique and only the RMSD is comparable.  An empty set
    (sum w = 0) has gap 0."""
    r, x = _d(reference), _d(coords)
    w = torch.ones(r.shape[:-1], dtype=torch.float64, device=r.device) if weights is None else _d(weights)
    W = w.sum(-1)
    rc = r - ((w[..., None] * r).sum(-2) / W[..., None])[..., None, :]
    xc = x - ((w[..., None] * x).sum(-2) / W[..., None])[..., None, :]
    S = torch.einsum("...p,...pi,...pj->...ij", w, xc, rc)
    xx, xy, xz, yx, yy, yz, zx, zy, zz = S.reshape(*S.shape[:-2], 9).unbind(-1)
    Kq = torch.stack([torch.stack([xx + yy + zz, yz - zy, zx - xz, xy - yx], -1),
                      torch.stack([yz - zy, xx - yy - zz, xy + yx, zx + xz], -1),
                      torch.stack([zx - xz, xy + yx, -xx + yy - zz, yz + zy], -1),
                      torch.stack([xy - yx, zx + xz, yz + zy, -xx - yy + zz], -1)], -2)
    ev = torch.linalg.eigvalsh(torch.nan_to_num(Kq, nan=0.0).cpu())
    gap = (ev[..., 3] - ev[..., 2]) / (ev[..., 3].abs() + math.ulp(1.0))
    return torch.where((W != 0).cpu(), gap, torch.zeros_like(gap)).to(r.device)
