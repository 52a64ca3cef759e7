"""The drop-in boundary against the REFERENCE'S OWN CALLER (VERDICT r1 item 8).  What is compared: the loss, aux_data and
parameter gradients that the unmodified ``Experiment.loss_fn`` (train_DFOLD_dynamics.py:1181) produced over the
reference's FullScoreNetwork on a synthetic batch (stored by oracle/make_golden.py in tests/golden/boundary.pt), against
the oracle's restatement of that loss (oracle/dfold_oracle.py loss_fn) over this package's FullScoreNetwork with the same
weights (operators routed to the oracle so the host logic runs on CPU).  The reference's caller itself does not run here."""
import os

import torch

from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from oracle import dfold_oracle as O
from tests.test_cpu_oracle import close

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "boundary.pt")
# oracle/make_golden.py BOUNDARY_EXP_CONF
EXP_CONF = dict(bb_atom_loss_weight=1.0, bb_atom_loss_t_filter=0.25, dist_mat_loss_weight=1.0,
                dist_mat_loss_t_filter=0.25, aux_loss_weight=0.25)


def _batch():
    """oracle/make_golden.py boundary_batch (kept in sync by the golden itself)."""
    feats = syn.add_loss_targets(syn.make_feats(3, 12, seed=21, loader_dtypes=True), seed=21)
    feats["fixed_mask"][:, 2] = 1
    return feats


def test_overlay_model_matches_reference_loss_fn_golden(oracle_ops):
    """Same loss, aux_data and parameter gradients as Experiment.loss_fn over the reference network."""
    g = torch.load(GOLDEN)
    ours = FullScoreNetwork(syn.model_conf(3, **syn.PRESET_TINY), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    ours.load_state_dict(syn.random_state({k: v.shape for k, v in ours.state_dict().items()}, seed=131), strict=True)
    batch = _batch()
    loss, aux = O.loss_fn(ours(dict(batch)), batch, O.default_exp_conf(**EXP_CONF))
    loss.backward()
    assert loss.dtype == g["loss"].dtype and close(loss.detach(), g["loss"], 1e-5)
    assert set(aux) == set(g["aux"]), (sorted(aux), sorted(g["aux"]))
    for k in g["aux"]:
        assert close(torch.as_tensor(aux[k]).detach(), torch.as_tensor(g["aux"][k]), 1e-5), k
    grads = {k: p.grad for k, p in ours.named_parameters() if p.grad is not None}
    assert set(grads) == set(g["grad_norms"]) and len(grads) > 50
    for k, ref in g["grads"].items():
        assert close(grads[k], ref, 2e-4), k
    for k, n in g["grad_norms"].items():
        assert abs(float(grads[k].norm()) - n) <= 2e-4 * max(1.0, n), k           # the scale of close()
