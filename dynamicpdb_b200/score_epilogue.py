"""Closed-form score epilogue of the network (SURVEY.md §8 row a11) as a diffuser-shaped object.

``FullScoreNetwork(model_conf, diffuser)`` only needs two methods of the diffuser it is handed:
``calc_rot_score(rots_t, rots_0, t)`` and ``calc_trans_score(trans_t, trans_0, t, use_torch=True, scale=True)``
(reference src/data/se3_diffuser.py:115-125).  ``SE3ScoreDiffuser`` provides exactly those, with the same numerics
as the reference path  se3_diffuser.calc_rot_score -> utils.quat_to_rotvec (src/data/utils.py:589-606) ->
so3_diffuser.torch_score (:274-305, use_cached_score=False) -> igso3_expansion (:9-49) / score (:71-117), and
r3_diffuser.score (:169-177) — but the sigma(t) lookup stays on the device (the reference does
``du.move_to_np(t)``, a host synchronisation inside the model forward).  The reference's own ``SE3Diffuser`` can be
passed instead; this class exists so bench / tests run without a checkout of the reference.
"""
import numpy as np
import torch

from . import kernels as K
from . import rigid_utils as ru


class SE3ScoreDiffuser:
    def __init__(self, se3_conf):
        so3, r3 = se3_conf.so3, se3_conf.r3
        self.min_sigma, self.max_sigma, self.num_sigma = so3.min_sigma, so3.max_sigma, so3.num_sigma
        self.min_b, self.max_b, self.coordinate_scaling = r3.min_b, r3.max_b, r3.coordinate_scaling
        self.L = 1000
        self._grid_np = self._sigma_np(np.linspace(0.0, 1.0, self.num_sigma))      # discrete_sigma, so3_diffuser.py:183
        self._grid = {}

    @classmethod
    def from_reference(cls, diffuser):
        """Device-resident twin of a reference ``SE3Diffuser`` (src/data/se3_diffuser.py:31-45): same schedules, read from
        the object's own sub-diffusers.  Returns None when `diffuser` is not shaped like one, or uses the cached-score
        lookup (so3_diffuser.py:288-295), which this class does not mirror."""
        so3, r3 = getattr(diffuser, "_so3_diffuser", None), getattr(diffuser, "_r3_diffuser", None)
        try:
            if so3 is None or r3 is None or so3.use_cached_score or so3.schedule != "logarithmic":
                return None
            from types import SimpleNamespace
            conf = SimpleNamespace(
                so3=SimpleNamespace(min_sigma=so3.min_sigma, max_sigma=so3.max_sigma, num_sigma=so3.num_sigma),
                r3=SimpleNamespace(min_b=r3.min_b, max_b=r3.max_b, coordinate_scaling=r3._r3_conf.coordinate_scaling))
            return cls(conf)
        except AttributeError:
            return None

    def grid(self, device) -> torch.Tensor:
        if device not in self._grid:
            self._grid[device] = torch.from_numpy(self._grid_np).to(device)
        return self._grid[device]

    def fused_scores(self, rigids_t, rigids_pred, t, mask, ipa_coordinate_scaling: float):
        """Both masked scores of the trunk epilogue (ipa_pytorch_dynamic.py:883-897) in ONE kernel launch
        (csrc/epilogue.cu `score_fwd_kernel`, K9).  `rigids_pred` holds the translation BEFORE unscaling."""
        q_t, q_p = rigids_t.get_rots().get_quats(), rigids_pred.get_rots().get_quats()
        return K.score_epilogue(q_p, q_t, rigids_pred.get_trans(), rigids_t.get_trans(), t, self.grid(q_p.device), mask,
                                max_sigma=self.max_sigma, min_sigma=self.min_sigma, min_b=self.min_b, max_b=self.max_b,
                                r3_scale=self.coordinate_scaling, ipa_scale=ipa_coordinate_scaling, L=self.L)

    def _sigma_np(self, t):
        return np.log(t * np.exp(self.max_sigma) + (1 - t) * np.exp(self.min_sigma))   # :192-199 (logarithmic)

    def _sigma_of(self, t: torch.Tensor) -> torch.Tensor:
        """sigma(t) snapped to the reference's 1000-point grid: discrete_sigma[digitize(sigma(t)) - 1]."""
        grid = self.grid(t.device)
        t64 = t.to(torch.float64)
        s = torch.log(t64 * float(np.exp(self.max_sigma)) + (1 - t64) * float(np.exp(self.min_sigma)))
        idx = torch.bucketize(s, grid, right=True) - 1
        return grid[idx.clamp(0, grid.numel() - 1)]

    # ---- reverse-diffusion step on the device (se3_diffuser.py:160-215) ----
    def sigma(self, t: float) -> float:
        return float(self._sigma_np(np.float64(t)))

    def rot_diffusion_coef(self, t: float) -> float:
        """so3_diffuser.py:201-210."""
        s = self.sigma(t)
        return float(np.sqrt(2 * (np.exp(self.max_sigma) - np.exp(self.min_sigma)) * s / np.exp(s)))

    def b_t(self, t: float) -> float:
        """r3_diffuser.py:26-29."""
        return float(self.min_b + t * (self.max_b - self.min_b))

    def reverse(self, rigid_t, rot_score, trans_score, t: float, dt: float, diffuse_mask=None, center: bool = True,
                noise_scale: float = 1.0, device=None, z_rot=None, z_trans=None, generator=None):
        """``SE3Diffuser.reverse`` with the reference's signature, executed by ONE kernel on the tensors' device
        (csrc/epilogue.cu `reverse_step_kernel`): no scipy rotation-vector round trip, no host copies.  Scores / mask may be
        tensors or numpy arrays (the reference passes numpy).  ``z_rot`` / ``z_trans`` [..,N,3] inject the normal draws
        (default: drawn on the device from ``generator``; the reference draws from numpy's global stream, so samples agree
        in distribution, and exactly when the same draws are injected)."""
        q_t, x_t = rigid_t.get_rots().get_quats(), rigid_t.get_trans()
        dev = q_t.device
        as_t = lambda a, dt_=None: (a if torch.is_tensor(a) else torch.as_tensor(np.asarray(a))).to(dev) if a is not None else None
        rot_score, trans_score, mask = as_t(rot_score), as_t(trans_score), as_t(diffuse_mask)
        shp = x_t.shape
        if z_rot is None:
            z_rot = torch.randn(shp, device=dev, generator=generator)
        if z_trans is None:
            z_trans = torch.randn(shp, device=dev, generator=generator)
        lead = shp[:-2]
        F_ = int(np.prod(lead)) if len(lead) else 1
        N_ = shp[-2]
        v = lambda a, c: a.reshape(F_, N_, c)
        q1, x1 = K.reverse_step(v(q_t, 4), v(x_t, 3), v(rot_score, 3), v(trans_score, 3), v(as_t(z_rot), 3), v(as_t(z_trans), 3),
                                None if mask is None else mask.reshape(F_, N_).float(),
                                g_rot=self.rot_diffusion_coef(t), g_trans=float(np.sqrt(self.b_t(t))), b_t=self.b_t(t), dt=dt,
                                noise_scale=noise_scale, r3_scale=self.coordinate_scaling, center=center)
        return ru.Rigid(ru.Rotation(quats=q1.reshape(shp[:-1] + (4,)), normalize_quats=False), x1.reshape(shp))

    # ---- se3_diffuser.py:119-125 ----
    def calc_rot_score(self, rots_t, rots_0, t, eps: float = 1e-6):
        q_t, q_0 = rots_t.get_quats(), rots_0.get_quats()
        if q_t.is_cuda and eps == 1e-6:
            shp = torch.broadcast_shapes(q_t.shape, q_0.shape)
            rot, _ = K.score_epilogue(q_0.expand(shp), q_t.expand(shp), None, None, t, self.grid(q_t.device), None, max_sigma=self.max_sigma, min_sigma=self.min_sigma,
                                      min_b=self.min_b, max_b=self.max_b, r3_scale=1.0, ipa_scale=1.0, L=self.L)
            return rot
        # host-side tensors (callers outside the model: data pipeline, CPU tests): the same arithmetic in torch
        quats_0_inv = rots_0.invert().get_quats()
        quats_0t = ru.quat_multiply(quats_0_inv, rots_t.get_quats())
        vec = _quat_to_rotvec(quats_0t)
        omega = torch.linalg.norm(vec, dim=-1) + eps                      # fp32
        sigma = self._sigma_of(t)[:, None, None]                          # fp64 [1,1,1]
        ls = torch.arange(self.L, device=vec.device)[None, None]          # int64
        om = omega[..., None]
        half = ls + 1 / 2                                                 # fp32, as in the reference
        decay = (2 * ls + 1) * torch.exp(-ls * (ls + 1) * sigma ** 2 / 2) # fp64
        hi, lo = torch.sin(om * half), torch.sin(om / 2)
        series = (decay * hi / lo).sum(dim=-1)
        dhi, dlo = half * torch.cos(om * half), 0.5 * torch.cos(om / 2)
        dseries = (decay * (lo * dhi - hi * dlo) / lo ** 2).sum(dim=-1)
        norm = dseries / (series + 1e-4)
        return norm[..., None] * vec / (omega[..., None] + eps)

    # ---- se3_diffuser.py:115-117 -> r3_diffuser.py:169-177 ----
    def calc_trans_score(self, trans_t, trans_0, t, use_torch=False, scale=True):
        if scale:
            trans_t = trans_t * self.coordinate_scaling
            trans_0 = trans_0 * self.coordinate_scaling
        beta = t * self.min_b + (1 / 2) * (t ** 2) * (self.max_b - self.min_b)
        exp = torch.exp if use_torch else np.exp
        return -(trans_t - exp(-1 / 2 * beta) * trans_0) / (1 - exp(-beta))


def _quat_to_rotvec(quat, eps=1e-6):
    quat = torch.where(quat[..., :1] < 0, -quat, quat)
    angle = 2 * torch.atan2(torch.linalg.norm(quat[..., 1:], dim=-1), quat[..., 0])
    a2 = angle * angle
    small = 2 + a2 / 12 + 7 * a2 * a2 / 2880
    large = angle / torch.sin(angle / 2 + eps)
    is_small = (angle <= 1e-3).float()
    return (small * is_small + (1 - is_small) * large)[..., None] * quat[..., 1:]
