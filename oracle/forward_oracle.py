"""Forward-diffusion oracle: the reference's SE3Diffuser.forward_marginal / sample_ref (src/data/se3_diffuser.py:47-110,
:217-280) and SO3Diffuser's IGSO(3) tables (src/data/so3_diffuser.py:132-180, :215-327; r3_diffuser.py:39-43, :81-104,
:159-177) restated in fp64 torch, with the random draws as inputs.

TEST INFRASTRUCTURE, like oracle/dfold_oracle.py (whose rigid algebra and sigma schedule it reuses): only tests/ may import
it.  It is pinned against the unmodified reference by tests/golden/forward.pt (oracle/make_forward_golden.py).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle.dfold_oracle import _sigma_of_t, quat_mul


def discrete_sigma(dc) -> np.ndarray:
    return _sigma_of_t(np.linspace(0.0, 1.0, dc.num_sigma), dc)                   # so3_diffuser.py:182-186


def discrete_omega(num_omega: int) -> torch.Tensor:
    return torch.from_numpy(np.linspace(0, np.pi, num_omega + 1)[1:])            # so3_diffuser.py:133


def sigma_idx(t: float, dc) -> int:
    return int(np.digitize(_sigma_of_t(np.float64(t), dc), discrete_sigma(dc)) - 1)   # t_to_idx :211-213


def _igso3_series(omega: torch.Tensor, sigma: torch.Tensor, L: int):
    """igso3_expansion (:9-49) and the numerator sum of score (:107-116) for omega [..., W] and sigma [..., 1] (fp64):
    (expansion, d expansion / d omega).  Terms whose weight exp(-l(l+1) sigma^2 / 2) is exactly 0 are left out."""
    s2h = float(sigma.min()) ** 2 / 2
    Lc = next((l for l in range(L) if -l * (l + 1) * s2h < -746.0), L)
    ls = torch.arange(Lc, dtype=torch.int64, device=omega.device)
    om = omega[..., None]
    decay = (2 * ls + 1) * torch.exp(-ls * (ls + 1) * sigma[..., None] ** 2 / 2)
    h = ls + 0.5
    hi, lo = torch.sin(om * h), torch.sin(om / 2)
    dhi, dlo = h * torch.cos(om * h), 0.5 * torch.cos(om / 2)
    return (decay * hi / lo).sum(-1), (decay * (lo * dhi - hi * dlo) / lo ** 2).sum(-1)


def igso3_tables(dc, rows=None, L: int = 1000, device="cpu", chunk: int = 8):
    """SO3Diffuser's tables (so3_diffuser.py:132-180) for the sigma rows ``rows`` (default: all): {cdf [R, num_omega],
    pdf, score_norms, score_scaling [R]}, fp64."""
    num_omega = getattr(dc, "num_omega", 1000)
    sig = torch.from_numpy(discrete_sigma(dc)).to(device)
    rows = torch.arange(dc.num_sigma) if rows is None else torch.as_tensor(rows)
    om = discrete_omega(num_omega).to(device)
    out = {"cdf": [], "pdf": [], "score_norms": [], "score_scaling": []}
    for r0 in range(0, len(rows), chunk):
        s = sig[rows[r0:r0 + chunk].to(device)][:, None]
        e, de = _igso3_series(om.expand(s.shape[0], -1), s, L)
        pdf = e * (1 - torch.cos(om)) / math.pi                                   # density(marginal=True) :63-65
        sn = de / (e + 1e-4)                                                     # score :117
        out["pdf"].append(pdf)
        out["cdf"].append(pdf.cumsum(-1) / num_omega * math.pi)
        out["score_norms"].append(sn)
        out["score_scaling"].append(torch.sqrt(torch.abs((sn ** 2 * pdf).sum(-1) / pdf.sum(-1))) / math.sqrt(3))
    return {k: torch.cat(v) for k, v in out.items()}


def interp(x: torch.Tensor, xp: torch.Tensor, fp: torch.Tensor) -> torch.Tensor:
    """np.interp (numpy/_core/src/multiarray/compiled_base.c arr_interp) for increasing xp: j = last index with
    xp[j] <= x, clamps to fp[0] / fp[-1] outside, fp[j] on an exact hit, slope form otherwise."""
    n = xp.numel()
    j = torch.searchsorted(xp, x, right=True) - 1
    jc = j.clamp(0, n - 2)
    slope = (fp[jc + 1] - fp[jc]) / (xp[jc + 1] - xp[jc])
    r = slope * (x - xp[jc]) + fp[jc]
    r = torch.where(xp[j.clamp(0, n - 1)] == x, fp[j.clamp(0, n - 1)], r)
    r = torch.where(j >= n - 1, fp[-1], r)
    r = torch.where(x > xp[-1], fp[-1], r)
    return torch.where(x < xp[0], fp[0], r)


def _quat_of_rotvec(axis: torch.Tensor, ang: torch.Tensor) -> torch.Tensor:
    return torch.cat([torch.cos(ang / 2)[..., None], torch.sin(ang / 2)[..., None] * axis], dim=-1)


def forward_marginal(rig7_0: torch.Tensor, t: float, draws, dc, cdf_row: torch.Tensor, score_scaling: float,
                     diffuse_mask=None, diffuse_rot: bool = True, diffuse_trans: bool = True, L: int = 1000):
    """SE3Diffuser.forward_marginal (se3_diffuser.py:47-110) with the draws given: draws = {z_axis [n,3], u [n], z_trans [n,3]}
    fp64 (numpy consumes so3 randn(n,3), so3 rand(n), then r3 normal(size=(n,3)), :323 / :230 / r3_diffuser.py:95).
    cdf_row = cdf[t_to_idx(t)] and score_scaling = _score_scaling[t_to_idx(t)].  Returns rigids_t [...,7] fp64 (quaternion
    w >= 0, translation unscaled), rot_score / trans_score [...,3] fp64 and both scalings (floats)."""
    shp = rig7_0.shape[:-1]
    n = int(np.prod(shp))
    q0 = F.normalize(rig7_0[..., :4].reshape(n, 4).double(), dim=-1)
    x0 = rig7_0[..., 4:].reshape(n, 3)                                           # fp32, as _extract_trans_rots gives it
    if diffuse_rot:
        axis = draws["z_axis"].reshape(n, 3).double()
        axis = axis / torch.linalg.norm(axis, dim=-1, keepdim=True)              # sample :246-248
        ang = interp(draws["u"].reshape(n).double(), cdf_row.double(), discrete_omega(cdf_row.numel()).to(axis.device))
        vec = axis * ang[:, None]
        omega = torch.linalg.norm(vec, dim=-1) + 1e-6                            # torch_score, fp64 :292
        sigma = torch.tensor(discrete_sigma(dc)[sigma_idx(t, dc)], dtype=torch.float64, device=vec.device)
        e, de = _igso3_series(omega, sigma.reshape(1), L)
        rs = (de / (e + 1e-4))[:, None] * vec / (omega[:, None] + 1e-6)
        q = quat_mul(q0, _quat_of_rotvec(axis, ang))                             # R_0 Exp(v), :325-326
        q = F.normalize(q, dim=-1)
        q = torch.where(q[:, :1] < 0, -q, q)
        rsc = float(score_scaling)
    else:
        q, rs, rsc = torch.where(q0[:, :1] < 0, -q0, q0), torch.zeros(n, 3, dtype=torch.float64, device=q0.device), 1.0
    if diffuse_trans:
        cs = dc.coordinate_scaling
        beta = t * dc.min_b + (1 / 2) * (t ** 2) * (dc.max_b - dc.min_b)        # marginal_b_t :42-43
        xs = (x0 * np.float32(cs)).double()                                      # float32 array * scaling stays fp32
        xt = math.exp(-1 / 2 * beta) * xs + math.sqrt(1 - math.exp(-beta)) * draws["z_trans"].reshape(n, 3).double()
        ts = -(xt - math.exp(-1 / 2 * beta) * xs) / (1 - math.exp(-beta))       # score :169-177
        xt = xt / cs
        tsc = 1 / math.sqrt(1 - math.exp(-beta))                                 # score_scaling :103-104
    else:
        xt, ts, tsc = x0.double(), torch.zeros(n, 3, dtype=torch.float64, device=x0.device), 1.0
    if diffuse_mask is not None:                                                 # _apply_mask :86-101
        m = torch.as_tensor(diffuse_mask).reshape(n, 1).double().to(q0.device)
        xt = m * xt + (1 - m) * x0.double()
        rs, ts = m * rs, m * ts
        q0s = torch.where(q0[:, :1] < 0, -q0, q0)
        q = torch.where(m > 0.5, q, q0s)
    return {"rigids_t": torch.cat([q, xt], dim=-1).reshape(shp + (7,)), "rot_score": rs.reshape(shp + (3,)),
            "trans_score": ts.reshape(shp + (3,)), "rot_score_scaling": rsc, "trans_score_scaling": tsc}


def sample_ref(n_samples: int, frame_time: int, draws, dc, cdf_last: torch.Tensor) -> torch.Tensor:
    """SE3Diffuser.sample_ref (se3_diffuser.py:217-280) in the dynamics layout: IGSO(3) rotation vectors at t = 1
    (so3_diffuser.py:250-251; cdf_last = cdf[t_to_idx(1)]) and N(0, I) translations unscaled (r3_diffuser.py:39-40, :265)
    -> [frame_time, n_samples / frame_time, 7] fp64 (quaternion w >= 0)."""
    axis = draws["z_axis"].reshape(n_samples, 3).double()
    axis = axis / torch.linalg.norm(axis, dim=-1, keepdim=True)
    ang = interp(draws["u"].reshape(n_samples).double(), cdf_last.double(), discrete_omega(cdf_last.numel()).to(axis.device))
    q = _quat_of_rotvec(axis, ang)
    x = draws["z_trans"].reshape(n_samples, 3).double() / dc.coordinate_scaling
    return torch.cat([q, x], dim=-1).reshape(frame_time, n_samples // frame_time, 7)
