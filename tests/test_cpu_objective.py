"""The oracle's training objective against the reference's own caller at the settings tests/golden/boundary.pt does not
reach (tests/golden/objective.pt, oracle/make_objective_golden.py): coordinate_scaling 0.1 with the axis / angle rotation
loss, t below the rotation threshold, and a 20-frame window.  As tests/test_cpu_boundary.py: this package's
FullScoreNetwork with every operator routed to the oracle, and the oracle's loss_fn.  tests/test_gpu_training_objective.py
compares the CUDA kernels with the same file."""
import os

import pytest
import torch

from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from oracle import dfold_oracle as O
from oracle import make_objective_golden as G
from tests.test_cpu_oracle import close

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "objective.pt")


def test_fixture_holds_the_cases_the_generator_defines():
    g = torch.load(GOLDEN)
    assert {k: v["case"] for k, v in g.items()} == G.CASES


@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_objective_matches_reference_loss_fn_golden(name, oracle_ops):
    g = torch.load(GOLDEN)[name]
    c = G.CASES[name]
    cs = c["coordinate_scaling"]
    ours = FullScoreNetwork(syn.model_conf(c["nf"], coordinate_scaling=cs, **syn.PRESET_TINY), SE3ScoreDiffuser(syn.diffuser_conf(cs)))
    ours.load_state_dict(G.case_weights(c, {k: v.shape for k, v in ours.state_dict().items()}), strict=True)
    batch = G.case_batch(c)
    loss, aux = O.loss_fn(ours(dict(batch)), batch, G.exp_conf(c))
    loss.backward()
    # not vacuous: the `< 100` gate is open, the torsion term counts, the rotation term is on exactly when t > 0.2
    assert 0 < float(g["aux"]["trans_loss"]) < 100 and float(g["aux"]["torsion_loss"]) > 0
    assert (float(g["aux"]["rot_loss"]) > 0) == (c["t"] > 0.2)
    assert loss.dtype == g["loss"].dtype and close(loss.detach(), g["loss"], 1e-5)
    assert set(aux) == set(g["aux"]), (sorted(aux), sorted(g["aux"]))
    for k in g["aux"]:
        assert close(torch.as_tensor(aux[k]).detach(), torch.as_tensor(g["aux"][k]), 1e-5), k
    grads = {k: p.grad for k, p in ours.named_parameters() if p.grad is not None}
    assert set(grads) == set(g["grad_norms"]) and len(grads) > 50
    for k, ref in g["grads"].items():
        assert close(grads[k], ref, 2e-4), k
    for k, n in g["grad_norms"].items():
        assert abs(float(grads[k].norm()) - n) <= 2e-4 * max(1.0, n), k
