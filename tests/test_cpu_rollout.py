"""The trajectory rollout's oracle (oracle/rollout_oracle.py) against the unmodified reference's eval_extension loop
(tests/golden/rollout.pt), the coordinate-scaling quirk, and the argument checks of TrajectoryRollout and of the C-ABI
entry point dfold_rollout_advance.

Bars.  A single step is held to the network bar: per-residue L2 error of the rigids below NET_TOL = 1e-4.  Free-running,
rounding differences compound through 200 fed-back predictions.  Measured on the CPU (fp32, torch 2.11), the oracle's
largest per-residue error against the reference is 3.7e-6 over the first 10 steps and 2.4e-3 over all 200 (step 199, case
5 x 16): the loop amplifies a one-step difference about 640-fold.  The first FREE_STEPS = 10 steps keep the network bar;
all 200 are held to DRIFT_TOL = that amplification times the network bar, 0.064 (about 1e-3 of the trajectory's
coordinates, up to 91 A), which covers a rollout whose every step is only within the network bar."""
import ctypes
import os

import pytest
import torch

from dynamicpdb_b200 import kernels as K
from dynamicpdb_b200 import synthetic as syn
from oracle import dfold_oracle as O
from oracle import rollout_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NET_TOL = 1e-4
FREE_STEPS = 10
ATOM_TOL = 2e-3        # per-residue L2 over the 37 x 3 atom coordinates, the bar tests/test_gpu_goldens.py holds atom37 to
MEASURED_STEP_ERR, MEASURED_DRIFT = 3.7e-6, 2.4e-3
DRIFT_TOL = MEASURED_DRIFT / MEASURED_STEP_ERR * NET_TOL
CASES = ("nf2_N12", "nf5_N16")


def rollout_fixture():
    return torch.load(os.path.join(ROOT, "tests", "golden", "rollout.pt"), weights_only=False)


def case_shapes(c):
    """Parameter names and shapes of the case's network (the reference's state_dict has the same)."""
    from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
    from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
    net = FullScoreNetwork(syn.model_conf(c["nf"], **syn.PRESET_TINY, coordinate_scaling=c["cs"]),
                           SE3ScoreDiffuser(syn.diffuser_conf(c["cs"])))
    return {k: tuple(v.shape) for k, v in net.state_dict().items()}


def case_setup(c):
    """(weights, starting window, oracle model conf, oracle diffuser conf) of a fixture case, rebuilt from its seeds."""
    p = syn.random_state(case_shapes(c), seed=c["wseed"])
    w = syn.make_feats(c["nf"], c["N"], seed=c["seed"], loader_dtypes=True)
    return p, w, O.default_conf(**syn.PRESET_TINY, coordinate_scaling=c["cs"]), O.default_diffuser_conf(c["cs"])


def res_l2(a, b):
    """Largest L2 norm of the difference along the last axis: per residue for rigids [..., N, 7], per atom for [..., 3]."""
    return float((a.double() - b.double()).norm(dim=-1).max())


def atom_l2(a, b):
    """Largest per-residue L2 norm of the difference of atom37 frames [..., N, 37, 3]."""
    return float((a.double() - b.double()).flatten(-2).norm(dim=-1).max())


@pytest.mark.parametrize("name", CASES)
def test_oracle_single_steps_match_reference(name):
    """Teacher-forced: each stored input window of the reference gives its next frame, its shifted next input and, where
    stored, its kept atom frame."""
    g = rollout_fixture()["cases"][name]
    p, w, conf, dc = case_setup(g["case"])
    steps = g["steps"]
    feats = RO.eval_inputs(w)
    assert torch.equal(g["rigids_0"][0], w["rigids_0"])          # step 0 reads the window itself
    for i, j in enumerate(steps):
        feats["rigids_0"] = g["rigids_0"][i].clone()
        rp, a37 = RO.step(p, feats, conf, dc)
        assert res_l2(rp[-1], g["rigid_traj"][j]) < NET_TOL, (name, j)
        if i + 1 < len(steps) and steps[i + 1] == j + 1:
            assert res_l2(RO.advance(feats["rigids_0"], rp), g["rigids_0"][i + 1]) < NET_TOL, (name, j)
        if j in g["atom_steps"]:
            k = g["atom_steps"].index(j)
            assert atom_l2(a37[-1], g["atom_traj"][k]) < ATOM_TOL, (name, j)


def free_running_errors(name):
    g = rollout_fixture()["cases"][name]
    p, w, conf, dc = case_setup(g["case"])
    out = RO.rollout(p, w, 200, conf, dc)
    err = (out["rigid_traj"].double() - g["rigid_traj"].double()).norm(dim=-1).amax(dim=-1)      # [200]
    return out, g, err


@pytest.mark.parametrize("name", CASES)
def test_oracle_free_running_matches_reference(name):
    out, g, err = free_running_errors(name)
    assert out["rigid_traj"].shape == (200, g["case"]["N"], 7) and out["atom_traj"].shape == (200, g["case"]["N"], 37, 3)
    assert float(err[:FREE_STEPS].max()) < NET_TOL, err[:FREE_STEPS]
    assert float(err.max()) < DRIFT_TOL, float(err.max())


def test_coordinate_scaling_quirk():
    """coordinate_scaling = 0.1: the unscaled prediction is fed back as it is (:996), so the history's translations grow by
    1 / 0.1 per step.  Three steps of the reference's loop against the oracle's, relative to the growing magnitude."""
    g = rollout_fixture()["cases"]["scaled_nf2_N12"]
    c = g["case"]
    assert c["cs"] == 0.1 and g["rigid_pred"].shape[0] == 3
    p, w, conf, dc = case_setup(c)
    feats = RO.eval_inputs(w)
    for j in range(3):
        assert torch.equal(feats["rigids_0"].float(), g["rigids_0"][j]) if j == 0 else \
            res_l2(feats["rigids_0"], g["rigids_0"][j]) < NET_TOL * float(g["rigids_0"][j].abs().max())
        rp, _ = RO.step(p, feats, conf, dc)
        ref = g["rigid_pred"][j]
        assert res_l2(rp, ref) < NET_TOL * max(1.0, float(ref.abs().max())), j
        feats["rigids_0"] = RO.advance(feats["rigids_0"], rp)
    t = g["rigid_pred"][:, -1, :, 4:].norm(dim=-1).mean(dim=-1)                       # mean |translation| per step
    assert float(t[1] / t[0]) > 5.0 and float(t[2] / t[1]) > 5.0, t


# ------------------------------------------------------------------------------------------------------------------
# argument checks (no GPU needed)
# ------------------------------------------------------------------------------------------------------------------
def _cpu_rollout():
    from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
    from dynamicpdb_b200.rollout import TrajectoryRollout
    from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
    net = FullScoreNetwork(syn.model_conf(2, **syn.PRESET_TINY), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    return TrajectoryRollout(net)


def test_rollout_refuses_cpu_tensors_and_bad_arguments():
    r = _cpu_rollout()
    w = syn.make_feats(2, 6, seed=1, loader_dtypes=True)
    before = {k: v.clone() for k, v in w.items()}
    with pytest.raises(RuntimeError, match="CUDA"):
        r.rollout(w, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        r.rollout(w, 3, literal=True, num_t=2)
    for kw, msg in ((dict(length=0), "length"), (dict(length=2.0), "length"), (dict(length=True), "length"),
                    (dict(length=2, min_t=0.0), "min_t"), (dict(length=2, min_t=1.5), "min_t"),
                    (dict(length=2, literal=True), "num_t"), (dict(length=2, literal=True, num_t=0), "num_t")):
        with pytest.raises(ValueError, match=msg):
            r.rollout(w, **kw)
    with pytest.raises(ValueError, match="lacks"):
        r.rollout({k: v for k, v in w.items() if k != "force"}, 2)
    for bad in (w["rigids_0"][:1], w["rigids_0"].double(), w["rigids_0"][..., :6]):
        with pytest.raises(ValueError, match="rigids_0"):
            r.rollout(dict(w, rigids_0=bad), 2)
    for k in before:
        assert torch.equal(before[k], w[k]), k


def test_rollout_advance_binding_refuses_cpu_tensors():
    z = torch.zeros
    with pytest.raises(RuntimeError, match="CUDA"):
        K.rollout_advance(z(2, 3, 7), z(2, 3, 37, 3), z(2, 3, 7), z(4, 3, 7), z(4, 3, 37, 3), z(1, dtype=torch.int64))


def test_rollout_advance_entry_point_validates_arguments():
    """Rejected before anything touches a device (fake non-null pointers are never dereferenced)."""
    L = K.lib()
    P, Q = ctypes.c_void_p(1 << 20), ctypes.c_void_p(2 << 20)
    cases = [
        (lambda: L.dfold_rollout_advance(None, P, Q, P, P, P, 2, 4, 37, 8, None), "null pointer"),
        (lambda: L.dfold_rollout_advance(P, P, Q, P, P, None, 2, 4, 37, 8, None), "null pointer"),
        (lambda: L.dfold_rollout_advance(P, P, Q, P, P, P, 1, 4, 37, 8, None), "nf >= 2"),
        (lambda: L.dfold_rollout_advance(P, P, Q, P, P, P, 2, 0, 37, 8, None), "N >= 1"),
        (lambda: L.dfold_rollout_advance(P, P, Q, P, P, P, 2, 4, 0, 8, None), "A >= 1"),
        (lambda: L.dfold_rollout_advance(P, P, Q, P, P, P, 2, 4, 37, 0, None), "L >= 1"),
        (lambda: L.dfold_rollout_advance(P, P, P, P, P, P, 2, 4, 37, 8, None), "aliases"),
        (lambda: L.dfold_rollout_advance(P, P, ctypes.c_void_p((1 << 20) + 4 * 7 * 4 * 2 - 4), P, P, P, 2, 4, 37, 8, None),
         "aliases"),
    ]
    for call, msg in cases:
        assert call() == 1
        assert msg in L.dfold_last_error().decode() or pytest.fail(f"{msg!r} not in {L.dfold_last_error().decode()!r}")
