"""Plain-torch restatement of the trajectory rollout (Experiment.eval_extension, train_DFOLD_dynamics.py:931-1000), over the
network oracle ``dfold_oracle.full_forward``.  TEST INFRASTRUCTURE: the tests hold the device rollout
(dynamicpdb_b200/rollout.py) and the reference's loop (tests/golden/rollout.pt) against it.

Per step the network runs on the current inputs, the last frame of its prediction is kept (``rigid_pred[-1:]``,
``atom_pred[-1:]``, :993-994) and the inputs advance by ``rigids_0 <- cat(rigid_pred[1:], rigid_pred[-1:])`` (:996).  Every
other input keeps the starting window's value.  The trunk reads neither ``t`` nor ``rigids_t`` (DESIGN §5.5), so the
prediction at t = min_t of the reference's ``num_t``-step sampler is this one forward at t = min_t.
"""
from typing import Dict

import torch

from oracle import dfold_oracle as O

# the window fields the sampler inputs take over unchanged (eval_fn :826-844, eval_extension :954-966 + its repair)
WINDOW_KEYS = ("torsion_angles_sin_cos", "torsion_angles_mask", "node_repr", "edge_repr", "aatype", "rigids_t", "rigids_0",
               "force", "vel")


def eval_inputs(window: Dict[str, torch.Tensor], min_t: float = 0.01) -> Dict[str, torch.Tensor]:
    """The sampler inputs of eval_fn / eval_extension: the window's fields, ``res_mask`` ones, ``fixed_mask`` zeros,
    ``seq_idx = arange(1, N + 1)``, ``sc_ca_t`` zeros and ``t = min_t``.  ``rigids_0`` is a copy (the rollout advances it)."""
    nf, N = window["rigids_0"].shape[:2]
    dev = window["rigids_0"].device
    feats = {k: window[k] for k in WINDOW_KEYS}
    feats.update({
        "rigids_0": window["rigids_0"].clone(),
        "res_mask": torch.ones(nf, N, dtype=torch.float64, device=dev),
        "fixed_mask": torch.zeros(nf, N, dtype=torch.float64, device=dev),
        "seq_idx": torch.arange(1, N + 1, device=dev).unsqueeze(0).repeat(nf, 1),
        "sc_ca_t": torch.zeros(nf, N, 3, dtype=torch.float32, device=dev),
        "t": torch.full((1,), float(min_t), dtype=torch.float32, device=dev),
    })
    return feats


def step(p: Dict[str, torch.Tensor], feats: Dict[str, torch.Tensor], conf, dc):
    """One network evaluation: (rigid_pred [nf, N, 7], atom37 [nf, N, 37, 3])."""
    out = O.full_forward(p, feats, conf, dc)
    return out["rigids"], out["atom37"]


def advance(rigids_0: torch.Tensor, rigid_pred: torch.Tensor) -> torch.Tensor:
    """:996 -- ``cat(rigid_pred[1:], rigid_pred[-1:])`` in the dtype of the current ``rigids_0``.  The prediction is
    unscaled (ipa_pytorch_dynamic.py:890) while the network reads ``rigids_0`` as it is, so with ``coordinate_scaling`` c
    != 1 every step multiplies the history's translations by 1 / c; the reference does the same."""
    return torch.cat([rigid_pred[1:], rigid_pred[-1:]], dim=0).to(rigids_0.dtype)


def rollout(p: Dict[str, torch.Tensor], window: Dict[str, torch.Tensor], length: int, conf, dc, min_t: float = 0.01,
            feats=None):
    """``length`` steps from ``window`` (or from prepared ``feats``): {"rigid_traj": [L, N, 7], "atom_traj": [L, N, 37, 3]}."""
    feats = dict(feats) if feats is not None else eval_inputs(window, min_t)
    rig, atoms = [], []
    for _ in range(length):
        rp, a37 = step(p, feats, conf, dc)
        rig.append(rp[-1])
        atoms.append(a37[-1])
        feats["rigids_0"] = advance(feats["rigids_0"], rp)
    return {"rigid_traj": torch.stack(rig), "atom_traj": torch.stack(atoms)}
