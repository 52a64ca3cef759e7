"""Generate tests/golden/aux_loss.pt from the UNMODIFIED reference (a checkout of it at $DFOLD_REFERENCE_ROOT):

    python oracle/make_aux_loss_golden.py

The reference's objective with its backbone-atom and pair-distance terms in final_loss, as uncommenting
train_DFOLD_dynamics.py:1370-1371 makes it.  The unmodified Experiment.loss_fn runs over the reference FullScoreNetwork
(tiny preset, synthetic.random_state weights) on the batches of CASES, as oracle/make_objective_golden.py runs it.  Its
locals bb_atom_loss, dist_mat_loss, rot_loss, trans_loss, torsion_loss, batch_loss_mask, gt_atom37 and atom37_mask are
captured when it returns (sys.setprofile), so no reference file is edited.  From them the uncommented final_loss and
its normalised value are formed and backpropagated.  Stored: the loss, aux_data with the four restored keys in the
reference's order, the ground-truth backbone and its mask, every gradient norm and the small gradients whole.  Inputs and
weights are not stored: the tests rebuild them with case_batch() / case_weights().
Importing this module does not need the reference; running it does.
"""
import os
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from dynamicpdb_b200 import synthetic as syn  # noqa: E402
from oracle import make_objective_golden as _obj  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "aux_loss.pt")

# t on both sides of the 0.25 filters (0.25 itself is gated off: the gate is a strict <), coordinate_scaling 0.1 and 1,
# and a 20-frame window, where the product runs its dead-frame pyramid and the aux terms reach every frame's output.
# case_batch() holds a fixed residue and two masked ones.
CASES = {
    "t_low": dict(nf=3, N=12, seed=41, t=0.1, coordinate_scaling=1.0, separate_rot_loss=False),
    "t_at_filter": dict(nf=3, N=12, seed=46, t=0.25, coordinate_scaling=1.0, separate_rot_loss=False),
    "t_high": dict(nf=3, N=12, seed=43, t=0.6, coordinate_scaling=1.0, separate_rot_loss=False),
    "scaled_separate": dict(nf=3, N=12, seed=44, t=0.2, coordinate_scaling=0.1, separate_rot_loss=True),
    "pyramid_nf20": dict(nf=20, N=16, seed=45, t=0.1, coordinate_scaling=1.0, separate_rot_loss=False),
}
EXP_CONF = _obj.EXP_CONF
AUX_ORDER = ("batch_train_loss", "batch_rot_loss", "batch_trans_loss", "batch_bb_atom_loss", "batch_dist_mat_loss",
             "batch_torsion_loss", "total_loss", "rot_loss", "trans_loss", "bb_atom_loss", "dist_mat_loss", "torsion_loss")
CAPTURED = ("bb_atom_loss", "dist_mat_loss", "rot_loss", "trans_loss", "torsion_loss", "batch_loss_mask", "gt_atom37",
            "atom37_mask")

case_batch = _obj.case_batch
case_weights = _obj.case_weights


def exp_conf(c):
    from oracle import dfold_oracle as O
    return O.default_exp_conf(separate_rot_loss=c["separate_rot_loss"], **EXP_CONF)


def loss_fn_locals(exp, batch):
    """Run exp.loss_fn(batch) and return its locals CAPTURED at its return."""
    got = {}

    def prof(frame, event, arg):
        if event == "return" and frame.f_code.co_name == "loss_fn" and "dist_mat_loss" in frame.f_locals:
            got.update({k: frame.f_locals[k] for k in CAPTURED})

    sys.setprofile(prof)
    try:
        exp.loss_fn(batch)
    finally:
        sys.setprofile(None)
    if set(got) != set(CAPTURED):
        raise RuntimeError("Experiment.loss_fn returned without the expected locals")
    return got


def main():
    from oracle import ref_shims
    ref_shims.install_trainer_stubs()
    from src.model import Dfold_network_dynamic as RefNet
    from src.data import se3_diffuser
    res = {}
    for name, c in CASES.items():
        cs = c["coordinate_scaling"]
        diffuser = se3_diffuser.SE3Diffuser(syn.diffuser_conf(cs))
        net = RefNet.FullScoreNetwork(syn.model_conf(c["nf"], coordinate_scaling=cs, **syn.PRESET_TINY), diffuser)
        net.load_state_dict(case_weights(c, {k: v.shape for k, v in net.state_dict().items()}))
        model_conf = SimpleNamespace(cfg_drop_in_train=True, cfg_drop_rate=0.0, embed=SimpleNamespace(embed_self_conditioning=False))
        exp = ref_shims.reference_experiment(net, diffuser, model_conf, exp_conf(c), SimpleNamespace(diffuse_rot=True))
        v = loss_fn_locals(exp, case_batch(c))
        # :1367-1373 with :1370-1371 uncommented, then normalize_loss (:1374-1375)
        final = v["rot_loss"] + v["trans_loss"] + v["bb_atom_loss"] + v["dist_mat_loss"] + v["torsion_loss"]
        norm = lambda x: x.sum() / (v["batch_loss_mask"].sum() + 1e-10)
        loss = norm(final)
        loss.backward()
        vals = {"batch_train_loss": final, "batch_rot_loss": v["rot_loss"], "batch_trans_loss": v["trans_loss"],
                "batch_bb_atom_loss": v["bb_atom_loss"], "batch_dist_mat_loss": v["dist_mat_loss"],
                "batch_torsion_loss": v["torsion_loss"], "total_loss": loss, "rot_loss": norm(v["rot_loss"]),
                "trans_loss": norm(v["trans_loss"]), "bb_atom_loss": norm(v["bb_atom_loss"]),
                "dist_mat_loss": norm(v["dist_mat_loss"]), "torsion_loss": norm(v["torsion_loss"])}
        grads = {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}
        small = {k: g for k, g in grads.items() if g.numel() <= 512}
        # the small gradients as views of one flat tensor, so the file stores one record for them, not one per tensor
        flat = torch.cat([g.reshape(-1) for g in small.values()])
        offs = torch.tensor([0] + [g.numel() for g in small.values()]).cumsum(0).tolist()
        small = {k: flat[o:o + g.numel()].view(g.shape) for (k, g), o in zip(small.items(), offs)}
        res[name] = {"case": c, "loss": loss.detach(), "aux": {k: vals[k].detach() for k in AUX_ORDER},
                     "gt_atom37": v["gt_atom37"].detach().clone(), "atom37_mask": v["atom37_mask"].detach().clone(),
                     "grads": small,                                      # small gradients whole, norms of all
                     "grad_norms": {k: float(g.norm()) for k, g in grads.items()}}
        print(f"[golden] aux_loss/{name}: loss {float(loss.detach()):.6f}, bb {float(vals['bb_atom_loss'].detach()):.6f}, "
              f"dist {float(vals['dist_mat_loss'].detach()):.6f}, {len(grads)} gradients")
    torch.save(res, OUT)


if __name__ == "__main__":
    main()
