"""Shared building blocks of the host-side mirror: the AlphaFold-style ``Linear`` with named initialisers
(reference src/model/ipa_pytorch_dynamic.py:107-172 and openfold/model/primitives.py:102-167), ``LayerNorm``
(primitives.py:170-199) and the invariant-point-attention driver used by both IPA variants.
All arithmetic goes through ``kernels`` (hand-written sm_90a CUDA behind the C-ABI); no CPU fallback.
"""
import math
from typing import Callable, List, Optional

import torch
import torch.nn as nn

from . import kernels as K
from .rigid_utils import Rigid


# --------------------------------------------------------------------------------------------------
# helpers with the reference's public names (ipa_pytorch_dynamic.py:19-104)
# --------------------------------------------------------------------------------------------------
def permute_final_dims(tensor: torch.Tensor, inds: List[int]):
    zero_index = -1 * len(inds)
    first_inds = list(range(len(tensor.shape[:zero_index])))
    return tensor.permute(first_inds + [zero_index + i for i in inds])


def flatten_final_dims(t: torch.Tensor, no_dims: int):
    return t.reshape(t.shape[:-no_dims] + (-1,))


def ipa_point_weights_init_(weights):
    with torch.no_grad():
        weights.fill_(0.541324854612918)  # softplus^-1(1)


def _calculate_fan(linear_weight_shape, fan="fan_in"):
    fan_out, fan_in = linear_weight_shape
    if fan == "fan_in":
        return fan_in
    if fan == "fan_out":
        return fan_out
    if fan == "fan_avg":
        return (fan_in + fan_out) / 2
    raise ValueError("Invalid fan option")


_TRUNC_STD = 0.87962566103423978  # std of a unit normal truncated to [-2, 2]


def trunc_normal_init_(weights, scale=1.0, fan="fan_in"):
    """Variance-scaled truncated normal (ref :55-66).  Drawn with torch (the reference samples scipy's truncnorm
    on the host); the distribution is the same, the stream is not — initial weights are not part of parity."""
    f = _calculate_fan(weights.shape, fan)
    std = math.sqrt(scale / max(1, f)) / _TRUNC_STD
    with torch.no_grad():
        nn.init.trunc_normal_(weights, mean=0.0, std=std, a=-2.0 * std, b=2.0 * std)


def lecun_normal_init_(weights):
    trunc_normal_init_(weights, scale=1.0)


def he_normal_init_(weights):
    trunc_normal_init_(weights, scale=2.0)


def glorot_uniform_init_(weights):
    nn.init.xavier_uniform_(weights, gain=1)


def final_init_(weights):
    with torch.no_grad():
        weights.fill_(0.0)


def gating_init_(weights):
    with torch.no_grad():
        weights.fill_(0.0)


def normal_init_(weights):
    torch.nn.init.kaiming_normal_(weights, nonlinearity="linear")


class Linear(nn.Linear):
    """``nn.Linear`` with the AlphaFold named initialisers (ref :107-172); forward runs the split-precision
    wgmma GEMM (or the SIMT kernel for tiny shapes) through ``kernels.linear``."""

    def __init__(self, in_dim: int, out_dim: int, bias: bool = True, init: str = "default",
                 init_fn: Optional[Callable[[torch.Tensor, torch.Tensor], None]] = None):
        super().__init__(in_dim, out_dim, bias=bias)
        if bias:
            with torch.no_grad():
                self.bias.fill_(0)
        if init_fn is not None:
            init_fn(self.weight, self.bias)
        elif init == "default":
            lecun_normal_init_(self.weight)
        elif init == "relu":
            he_normal_init_(self.weight)
        elif init == "glorot":
            glorot_uniform_init_(self.weight)
        elif init == "gating":
            gating_init_(self.weight)
            if bias:
                with torch.no_grad():
                    self.bias.fill_(1.0)
        elif init == "normal":
            normal_init_(self.weight)
        elif init == "final":
            final_init_(self.weight)
        else:
            raise ValueError("Invalid init string.")

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return K.linear(x, self.weight, self.bias)


def _lin(mod: nn.Linear, x: torch.Tensor, act: Optional[str] = None) -> torch.Tensor:
    return K.linear(x, mod.weight, mod.bias, act=act)



class LayerNorm(nn.Module):
    """openfold/model/primitives.py:170-199 (same parameter names: weight, bias)."""

    def __init__(self, c_in, eps=1e-5):
        super().__init__()
        self.c_in = (c_in,)
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(c_in))
        self.bias = nn.Parameter(torch.zeros(c_in))

    def forward(self, x):
        return K.layer_norm(x, self.weight, self.bias, self.eps)


def _is_frame_broadcast(t: torch.Tensor) -> bool:
    """True when the leading (frame) axis of ``t`` is an expand() of one slice."""
    return t.dim() >= 3 and (t.shape[0] == 1 or t.stride(0) == 0)


def ipa_forward(mod, s, z, r: Rigid, mask, *, dfold: bool):
    """Shared driver for the DFOLD fork and the vanilla OpenFold IPA (structure_module.py:231-431)."""
    H, C, Pq, Pv = mod.no_heads, mod.c_hidden, mod.no_qk_points, mod.no_v_points
    batch_shape = s.shape[:-2]
    N = s.shape[-2]
    quat = r.get_rots().get_quats()
    trans = r.get_trans()
    quat = quat.expand(batch_shape + (N, 4)).reshape(-1, N, 4).contiguous()
    trans = trans.expand(batch_shape + (N, 3)).reshape(-1, N, 3).contiguous()
    Fn = quat.shape[0]
    mask2 = mask.expand(batch_shape + (N,)).reshape(Fn, N).to(torch.float32).contiguous()

    # ---- frame-shared or per-frame projections (ref :350-390) ----
    s3 = s.reshape((-1,) + s.shape[-2:]) if s.dim() > 2 else s[None]
    s_u = s3[:1] if _is_frame_broadcast(s3) else s3                 # [Fs,N,c_s]
    Fs = s_u.shape[0]
    q = _lin(mod.linear_q, s_u)                                      # [Fs,N,H*C]
    kv = _lin(mod.linear_kv, s_u)                                    # [Fs,N,H*2C]  per head [K | V]
    q_raw = _lin(mod.linear_q_points, s_u)                           # [Fs,N,3*H*Pq] coordinate-major
    kv_raw = _lin(mod.linear_kv_points, s_u)                         # [Fs,N,3*H*(Pq+Pv)]

    z3 = z if z.dim() == 3 else z.reshape((-1,) + z.shape[-3:])
    zb = z3 if z3.dim() == 4 else z3[None]                           # [Fz,N,N,c_z]
    if zb.shape[0] > 1 and zb.stride(0) == 0:
        zb = zb[:1]
    Fz = zb.shape[0]
    # pair bias b[.., i, j, h] written head-major [Fz,H,N,N]; pair values for the o_pair aggregation
    b_hm = K.linear(zb.reshape(Fz * N * N, -1), mod.linear_b.weight, mod.linear_b.bias) \
        .reshape(Fz, N, N, H).permute(0, 3, 1, 2)
    if dfold:
        pair = _lin(mod.down_z, zb.reshape(Fz * N * N, -1)).reshape(Fz, N, N, -1)    # ref :498
    else:
        pair = zb.to(torch.float32)

    # scalar logits  q.k / sqrt(3C) + b / sqrt(3)   (ref :402-407)  -> [Fl,H,N,N]
    logit0 = K.qk_logits(q.reshape(Fs, N, H, C), kv.reshape(Fs, N, H, 2 * C), b_hm,
                         math.sqrt(1.0 / (3 * C)), math.sqrt(1.0 / 3))

    # global-frame points (ref :363-390)
    q_pts = K.ipa_points(q_raw, quat, trans, H)                      # [F,N,H,Pq,3]
    kv_pts = K.ipa_points(kv_raw, quat, trans, H)                    # [F,N,H,Pq+Pv,3]

    gamma = torch.nn.functional.softplus(mod.head_weights) * math.sqrt(1.0 / (3 * (Pq * 9.0 / 2)))   # ref :415-420
    cat = K.ipa_attention(logit0, kv.reshape(Fs, N, H, 2 * C), q_pts, kv_pts, pair, quat, trans, mask2, gamma,
                          Pq=Pq, Pv=Pv, dfold=dfold, inf=mod.inf, eps=mod.eps)       # [F,N,D]
    out = _lin(mod.linear_out, cat.to(z.dtype))                      # ref :510-514
    return out.reshape(batch_shape + (N, -1))


