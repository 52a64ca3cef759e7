"""Generate tests/golden/objective.pt from the UNMODIFIED reference (a checkout of it at $DFOLD_REFERENCE_ROOT):

    python oracle/make_objective_golden.py

One training step of the reference's objective, as tests/golden/boundary.pt holds it for the default settings: the
unmodified Experiment.loss_fn (train_DFOLD_dynamics.py:1181) driving the reference FullScoreNetwork (tiny preset,
synthetic.random_state weights) on the batches of CASES, storing loss, aux_data, every gradient norm and the small
gradient tensors whole.  Inputs and weights are not stored: the tests rebuild them with case_batch() / case_weights().
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

OUT = os.path.join(ROOT, "tests", "golden", "objective.pt")

# what boundary.pt does not reach: the shipped coordinate_scaling with the axis / angle rotation loss, the rotation term
# gated off by t, and a window long enough (nf > 17) for the product to run its dead-frame pyramid where the reference
# runs the full ConvNet
CASES = {
    "scaled_separate": dict(nf=3, N=12, seed=31, t=0.5, coordinate_scaling=0.1, separate_rot_loss=True),
    "t_low": dict(nf=3, N=12, seed=32, t=0.1, coordinate_scaling=1.0, separate_rot_loss=False),
    "pyramid_nf20": dict(nf=20, N=16, seed=33, t=0.5, coordinate_scaling=1.0, separate_rot_loss=False),
}
EXP_CONF = dict(bb_atom_loss_weight=1.0, bb_atom_loss_t_filter=0.25, dist_mat_loss_weight=1.0,
                dist_mat_loss_t_filter=0.25, aux_loss_weight=0.25)


def target_in_output_units(feats, coordinate_scaling: float):
    """The trunk never scales the frames it is given but divides its prediction by coordinate_scaling
    (ipa_pytorch_dynamic.py:890), and the loss compares that with rigids_0[-1] as it stands
    (train_DFOLD_dynamics.py:1241).  The last frame of rigids_0 is read by the loss only (the trunk's last input frame is
    its predecessor, :819), so it is put where the prediction lands, keeping its offset from the previous frame: the
    translation term then stays under the loss's `< 100` gate at every chain length."""
    if coordinate_scaling != 1.0:
        x = feats["rigids_0"][..., 4:]
        feats["rigids_0"][-1, :, 4:] = x[-2] / coordinate_scaling + (x[-1] - x[-2])
    return feats


def case_batch(c):
    """Loader-dtype batch of one case: two masked residues and one fixed residue."""
    cs = c["coordinate_scaling"]
    feats = syn.make_feats(c["nf"], c["N"], seed=c["seed"], t=c["t"], coordinate_scaling=cs, loader_dtypes=True)
    feats = syn.add_loss_targets(feats, seed=c["seed"])
    feats["fixed_mask"][:, 2] = 1
    feats["res_mask"][:, -2:] = 0
    return target_in_output_units(feats, cs)


def case_weights(c, shapes):
    return syn.random_state(shapes, seed=c["seed"] + 100)


def exp_conf(c):
    from oracle import dfold_oracle as O
    return O.default_exp_conf(separate_rot_loss=c["separate_rot_loss"], **EXP_CONF)


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
        exp._conf = SimpleNamespace(model=SimpleNamespace(cfg_drop_rate=0.0, cfg_gamma=1.0))
        exp._data_conf = SimpleNamespace(num_t=4, min_t=0.01)
        loss, aux = exp.loss_fn(case_batch(c))
        loss.backward()
        grads = {k: p.grad.detach().clone() for k, p in net.named_parameters() if p.grad is not None}
        res[name] = {"case": c, "loss": loss.detach(),
                     "aux": {k: v.detach() if torch.is_tensor(v) else v for k, v in aux.items()},
                     "grads": {k: g for k, g in grads.items() if g.numel() <= 4096},      # small gradients whole, norms of all
                     "grad_norms": {k: float(g.norm()) for k, g in grads.items()}}
        print(f"[golden] objective/{name}: loss {float(loss.detach()):.6f}, {len(grads)} gradients")
    torch.save(res, OUT)


if __name__ == "__main__":
    main()
