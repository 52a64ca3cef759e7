"""Structure epilogue of the score network (SURVEY.md §8 row a13): torsion angles -> 8 rigid groups per residue ->
idealised atom14 -> atom37.  Mirrors ``openfold/utils/feats.py:165-228`` (``torsion_angles_to_frames``),
``src/data/all_atom.py:114-154`` (``frames_to_atom14_pos``) and ``src/model/Dfold_network_dynamic.py:574-594``
(``atom14_to_atom37``).

Unlike the reference, the residue tables live on the compute device (cached per device), so the forward has no
host round trip (the reference moves ``aatype`` to the CPU-resident ``GROUP_IDX``, all_atom.py:129-136).
"""
import os
from typing import Dict, Tuple

import numpy as np
import torch

from . import kernels as K
from .rigid_utils import Rigid, Rotation

_NPZ = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "residue_tables.npz")
_HOST: Dict[str, torch.Tensor] = {}
_DEV: Dict[Tuple[str, str, torch.dtype], torch.Tensor] = {}


def table(name: str, device, dtype=None) -> torch.Tensor:
    """default_frames [21,8,4,4] | atom14_group [21,14] | atom14_mask [21,14] | atom14_pos [21,14,3] |
    atom37_to_atom14 [21,37] | atom37_mask [21,37]  (dumped from the reference by oracle/make_constants.py)."""
    if not _HOST:
        d = np.load(_NPZ)
        for k in d.files:
            _HOST[k] = torch.from_numpy(d[k])
    t = _HOST[name]
    dtype = dtype if (dtype is not None and t.dtype.is_floating_point) else t.dtype
    key = (name, str(device), dtype)
    if key not in _DEV:
        _DEV[key] = t.to(device=device, dtype=dtype)
    return _DEV[key]


def torsion_angles_to_frames(r: Rigid, alpha: torch.Tensor, aatype: torch.Tensor, rrgdf: torch.Tensor) -> Rigid:
    """r Rigid[*,N], alpha [*,N,7,2] (sin,cos), aatype [*,N], rrgdf [21,8,4,4] -> Rigid[*,N,8] (to global)."""
    default_r = Rigid.from_tensor_4x4(rrgdf[aatype, ...])                   # [*,N,8]
    bb = alpha.new_zeros(alpha.shape[:-2] + (1, 2))
    bb[..., 1] = 1
    al = torch.cat([bb, alpha], dim=-2)                                     # [*,N,8,2]; group 0 = identity
    sin, cos = al[..., 0], al[..., 1]
    one, zero = torch.ones_like(sin), torch.zeros_like(sin)
    # rotation about x:  [[1,0,0],[0,cos,-sin],[0,sin,cos]]
    rots = torch.stack([torch.stack([one, zero, zero], dim=-1),
                        torch.stack([zero, cos, -sin], dim=-1),
                        torch.stack([zero, sin, cos], dim=-1)], dim=-2)
    all_frames = default_r.compose(Rigid(Rotation(rot_mats=rots), None))
    chi1_to_bb = all_frames[..., 4]
    chi2_to_bb = chi1_to_bb.compose(all_frames[..., 5])
    chi3_to_bb = chi2_to_bb.compose(all_frames[..., 6])
    chi4_to_bb = chi3_to_bb.compose(all_frames[..., 7])
    to_bb = Rigid.cat([all_frames[..., :5], chi2_to_bb.unsqueeze(-1), chi3_to_bb.unsqueeze(-1),
                       chi4_to_bb.unsqueeze(-1)], dim=-1)
    return r[..., None].compose(to_bb)


def frames_to_atom14_pos(r: Rigid, aatype: torch.Tensor) -> torch.Tensor:
    """r Rigid[*,N,8] -> [*,N,14,3] idealised atom positions (masked)."""
    dev = r.device
    grp = table("atom14_group", dev)[aatype, ...]                           # [*,N,14]
    rot = r.get_rots().get_rot_mats()                                       # [*,N,8,3,3]
    trn = r.get_trans()                                                     # [*,N,8,3]
    rot14 = torch.gather(rot, -3, grp[..., None, None].expand(grp.shape + (3, 3)))
    trn14 = torch.gather(trn, -2, grp[..., None].expand(grp.shape + (3,)))
    pos = table("atom14_pos", dev, trn.dtype)[aatype, ...]                  # [*,N,14,3]
    out = Rigid(Rotation(rot_mats=rot14), trn14).apply(pos)
    return out * table("atom14_mask", dev, trn.dtype)[aatype, ...].unsqueeze(-1)


def atom14_to_atom37(atom14_data: torch.Tensor, aatype: torch.Tensor):
    """(*, N, 14, ...) -> (*, N, 37, ...), mask (*, N, 37)."""
    idx = table("atom37_to_atom14", aatype.device)[aatype]
    mask = table("atom37_mask", aatype.device)[aatype]
    nb = aatype.dim() - 1
    if atom14_data.dim() == nb + 2:
        return torch.gather(atom14_data, -1, idx) * mask, mask
    if atom14_data.dim() == nb + 3:
        out = torch.gather(atom14_data, -2, idx[..., None].expand(idx.shape + (atom14_data.shape[-1],)))
        return out * mask[..., None].to(out.dtype), mask
    raise ValueError("Incorrectly shaped data")


_TABLE_NAMES = ("default_frames", "atom14_group", "atom14_mask", "atom14_pos", "atom37_to_atom14", "atom37_mask")


def _take(src: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """src [*, G, ...], idx [*, A] -> [*, A, ...]: torch.gather along the G axis as a sum of one-hot selections.  Exact for
    finite src, and its backward sums in a fixed order, where gather's backward (a scatter_add with atomics) does not."""
    nb = idx.dim() - 1
    rest = (1,) * (src.dim() - idx.dim())
    out = None
    for g in range(src.shape[nb]):
        term = (idx == g).to(src.dtype).reshape(idx.shape + rest) * src.select(nb, g).unsqueeze(nb)
        out = term if out is None else out + term
    return out


def _frames_to_atom14_pos_ordered(r: Rigid, aatype: torch.Tensor) -> torch.Tensor:
    """frames_to_atom14_pos with _take for its gathers."""
    dev = r.device
    grp = table("atom14_group", dev)[aatype, ...]
    rot14 = _take(r.get_rots().get_rot_mats(), grp)
    trn14 = _take(r.get_trans(), grp)
    pos = table("atom14_pos", dev, trn14.dtype)[aatype, ...]
    out = Rigid(Rotation(rot_mats=rot14), trn14).apply(pos)
    return out * table("atom14_mask", dev, trn14.dtype)[aatype, ...].unsqueeze(-1)


def _eager_chain(rot_is_matrix: bool):
    """The differentiable statement of the fused kernel (used by its backward): the three reference-shaped functions above,
    with their gathers as fixed-order sums (_take), so that the gradient of atom14 / atom37 is the same from run to run."""
    def run(rot, trans, alpha, aatype, want_frames):
        rots = Rotation(rot_mats=rot) if rot_is_matrix else Rotation(quats=rot, normalize_quats=False)
        frames = torsion_angles_to_frames(Rigid(rots, trans), alpha, aatype, table("default_frames", alpha.device, alpha.dtype))
        a14 = _frames_to_atom14_pos_ordered(frames, aatype)
        a37 = _take(a14, table("atom37_to_atom14", aatype.device)[aatype]) * table("atom37_mask", aatype.device, a14.dtype)[aatype][..., None]
        return (a14, a37, frames.to_tensor_4x4()) if want_frames else (a14, a37)
    return run


def frames_to_atoms(r: Rigid, alpha: torch.Tensor, aatype: torch.Tensor, want_frames: bool = False):
    """``torsion_angles_to_frames`` -> ``frames_to_atom14_pos`` -> ``atom14_to_atom37`` as ONE kernel (csrc/epilogue.cu
    `frames_to_atoms_kernel`, K10): r Rigid[*,N], alpha [*,N,7,2], aatype [*,N] -> (atom14 [*,N,14,3], atom37 [*,N,37,3]
    [, frames [*,N,8,4,4]]).  fp32 out whatever alpha's dtype, as the reference (Rotation forces fp32)."""
    rots = r.get_rots()
    is_mat = rots._quats is None
    rot = rots.get_rot_mats() if is_mat else rots.get_quats()
    tables = {k: table(k, alpha.device) for k in _TABLE_NAMES}
    return K.frames_to_atoms(rot, r.get_trans(), alpha, aatype, tables, _eager_chain(is_mat), want_frames, is_mat)
