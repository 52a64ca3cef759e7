"""The host side of the auxiliary structure losses (``score_network_loss(aux_losses=True)``,
``Trainer(aux_losses=True)``) and the oracle's restatement of them against the unmodified reference.

tests/golden/aux_loss.pt (oracle/make_aux_loss_golden.py) holds the reference's Experiment.loss_fn with its backbone-atom
and pair-distance terms in final_loss.  Here this package's FullScoreNetwork with every operator routed to the oracle,
and oracle.aux_loss_oracle.loss_fn_aux, must reproduce it, as tests/test_cpu_objective.py does for the default objective.
tests/test_gpu_aux_loss.py compares the CUDA kernels with the same file."""
import logging
import os

import pytest
import torch

from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.loss import AUX_KEYS, score_network_loss
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from dynamicpdb_b200.trainer import LOGGED_AUX, Trainer
from oracle import aux_loss_oracle as A
from oracle import dfold_oracle as O
from oracle import make_aux_loss_golden as G
from tests.test_cpu_oracle import close
from tests.test_cpu_trainer import _conf, _csv

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "aux_loss.pt")


def test_fixture_holds_the_cases_the_generator_defines():
    g = torch.load(GOLDEN)
    assert {k: v["case"] for k, v in g.items()} == G.CASES
    assert all(list(v["aux"]) == list(G.AUX_ORDER) for v in g.values())
    # not vacuous: the terms count below the filters and are gated off at and above them
    for k, v in g.items():
        assert (float(v["aux"]["bb_atom_loss"]) > 0) == (v["case"]["t"] < 0.25), k
        assert (float(v["aux"]["dist_mat_loss"]) > 0) == (v["case"]["t"] < 0.25), k


@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_ground_truth_backbone_matches_reference(name):
    g = torch.load(GOLDEN)[name]
    batch = G.case_batch(G.CASES[name])
    gt = A.compute_backbone(batch["rigids_0"].to(torch.float64), batch["torsion_angles_sin_cos"][..., 2, :])
    assert close(gt, g["gt_atom37"], 1e-5)
    assert torch.equal(torch.any(gt != 0, dim=-1), g["atom37_mask"])


@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_aux_objective_matches_reference_golden(name, oracle_ops):
    g = torch.load(GOLDEN)[name]
    c = G.CASES[name]
    cs = c["coordinate_scaling"]
    ours = FullScoreNetwork(syn.model_conf(c["nf"], coordinate_scaling=cs, **syn.PRESET_TINY), SE3ScoreDiffuser(syn.diffuser_conf(cs)))
    ours.load_state_dict(G.case_weights(c, {k: v.shape for k, v in ours.state_dict().items()}), strict=True)
    batch = G.case_batch(c)
    loss, aux = A.loss_fn_aux(ours(dict(batch)), batch, G.exp_conf(c))
    loss.backward()
    # the oracle's trunk is fp32; at t = 0.25 these random weights give a rotation term of ~20, whose fp32 rounding reaches
    # 1e-5 of the loss and 3e-4 of the largest gradients
    big = float(g["aux"]["rot_loss"]) > 10
    gtol = 1e-3 if big else 2e-4
    assert loss.dtype == g["loss"].dtype and close(loss.detach(), g["loss"], 1e-4)
    assert list(aux) == list(g["aux"])
    for k, ref in g["aux"].items():
        assert aux[k].dtype == ref.dtype and close(aux[k].detach(), ref, 1e-4), k
    grads = {k: p.grad for k, p in ours.named_parameters() if p.grad is not None}
    assert set(grads) == set(g["grad_norms"]) and len(grads) > 50
    for k, ref in g["grads"].items():
        assert close(grads[k], ref, gtol), k
    for k, n in g["grad_norms"].items():
        assert abs(float(grads[k].norm()) - n) <= gtol * max(1.0, n), k


@pytest.mark.parametrize("bad", [None, "0.25", True])
def test_loss_checks_the_aux_keys_before_device_work(bad):
    """A missing or non-numeric key raises ValueError, before the loss notices the batch is on the host."""
    c = G.CASES["t_low"]
    conf = vars(G.exp_conf(c)).copy()
    if bad is None:
        del conf["dist_mat_loss_t_filter"]
    else:
        conf["dist_mat_loss_t_filter"] = bad
    batch = G.case_batch(c)
    with pytest.raises(ValueError, match="dist_mat_loss_t_filter"):
        score_network_loss({}, batch, O.default_exp_conf(**conf), aux_losses=True)


@pytest.mark.parametrize("key", AUX_KEYS)
@pytest.mark.parametrize("bad", ["missing", "text"])
def test_trainer_checks_the_aux_keys_before_device_work(tmp_path, key, bad):
    conf = _conf(_csv(tmp_path / "train.csv", [12]))
    conf["experiment"].update(G.EXP_CONF)
    if bad == "missing":
        del conf["experiment"][key]
    else:
        conf["experiment"][key] = "0.25"
    with pytest.raises(ValueError, match=key):
        Trainer(conf, None, None, aux_losses=True)
    # the same config trains the default objective, which reads none of them (it fails later, on the missing network)
    with pytest.raises(AttributeError):
        Trainer(conf, None, None)


class _HostAuxTrainer(Trainer):
    """The Trainer's loop with the device side replaced by a host fake, on the aux objective."""

    def __init__(self, conf, aux):
        self._configure(conf, 1, 0, 1, aux_losses=True)
        self.aux = list(aux)

    def _prefetch(self, steps):
        yield from steps

    def _update(self, slots):
        self.current = self.aux.pop(0)

    def _keep_logged(self):
        self.kept = [float(self.current[k]) for k in self.logged_keys]

    def _read_logged(self):
        return self.kept

    def _save(self, path):
        pass


def test_trainer_logs_the_six_values_in_reference_order(tmp_path, caplog):
    conf = _conf(_csv(tmp_path / "train.csv", [12, 12]), num_epoch=1)
    conf["experiment"].update(G.EXP_CONF)
    vals = [{k: float(i + 1) + j / 8 for j, k in enumerate(LOGGED_AUX)} for i in range(2)]
    tr = _HostAuxTrainer(conf, vals)
    with caplog.at_level(logging.INFO, logger="dynamicpdb_b200.trainer"):
        tr.train()
    lines = [r.getMessage() for r in caplog.records if "trained_steps" in r.getMessage()]
    assert len(lines) == 2
    assert ("total_loss=1.0000 rot_loss=1.1250 trans_loss=1.2500 bb_atom_loss=1.3750 dist_mat_loss=1.5000 "
            "torsion_loss=1.6250, steps/sec=") in lines[0]
    assert LOGGED_AUX == ("total_loss", "rot_loss", "trans_loss", "bb_atom_loss", "dist_mat_loss", "torsion_loss")
