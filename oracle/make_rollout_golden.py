"""Generate tests/golden/rollout.pt from the UNMODIFIED reference (a checkout of it at $DFOLD_REFERENCE_ROOT):

    python oracle/make_rollout_golden.py

Runs ``Experiment.eval_extension`` (train_DFOLD_dynamics.py:931-1000) through ``ref_shims.reference_experiment`` on the
reference network (tiny preset, ``synthetic.random_state`` weights) for one window of ``synthetic.make_feats`` per case, with
its hard-coded ``length = 200`` (:933), and reads its ``extension.npz`` back.  The weights and the window are rebuilt by the
tests from the seeds (the parameter shapes from the package's own FullScoreNetwork, whose state_dict matches).

The single repair.  eval_extension's ``init_feats`` (:954-966) lack ``force``, ``vel`` and ``torsion_angles_mask``, and its
``torsion_angles_sin_cos`` is ``[1, N, 7, 2]`` (so ``[N, 7, 2]`` after the flatten), so the network stops with a KeyError
(ipa_pytorch_dynamic.py:821).  ``exp.inference_fn`` is wrapped to complete its ``data_init`` with the window's flattened
``force``, ``vel``, ``torsion_angles_sin_cos`` and ``torsion_angles_mask`` before calling the reference's own inference_fn.
Nothing else is changed.  The wrapper also records each step's ``rigids_0`` (the input the tests feed to a single step).

The coordinate-scaling case (c = 0.1) runs the same loop and is stopped by the wrapper after 3 steps: the unscaled
prediction fed back (:996) multiplies the translations by 1 / c per step and overflows fp32 long before step 200.
"""
import os
import sys
import tempfile
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402

ref_shims.install_trainer_stubs()
from src.data import se3_diffuser  # noqa: E402
from src.model import Dfold_network_dynamic as RefNet  # noqa: E402
from dynamicpdb_b200 import synthetic as syn  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
STEPS = list(range(10)) + [50, 100, 199]       # steps whose input rigids_0 is stored
ATOM_STEPS = [0, 199]                          # steps whose kept atom37 frame is stored
CASES = {
    "nf2_N12": dict(nf=2, N=12, seed=61, wseed=161, num_t=2, cs=1.0, stop=None),
    "nf5_N16": dict(nf=5, N=16, seed=62, wseed=162, num_t=3, cs=1.0, stop=None),
    "scaled_nf2_N12": dict(nf=2, N=12, seed=63, wseed=163, num_t=2, cs=0.1, stop=3),
}
REPAIR_KEYS = ("force", "vel", "torsion_angles_sin_cos", "torsion_angles_mask")


class _Stop(Exception):
    pass


def window(c):
    """The starting window of a case (also rebuilt by the tests)."""
    return syn.make_feats(c["nf"], c["N"], seed=c["seed"], loader_dtypes=True)


def run_case(c):
    nf, N, cs = c["nf"], c["N"], c["cs"]
    dconf = syn.diffuser_conf(cs)
    dconf.dynamics, dconf.frame_time = True, nf
    diffuser = se3_diffuser.SE3Diffuser(dconf)
    net = RefNet.FullScoreNetwork(syn.model_conf(nf, **syn.PRESET_TINY, coordinate_scaling=cs), diffuser)
    shapes = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    net.load_state_dict(syn.random_state(shapes, seed=c["wseed"]))
    model_conf = SimpleNamespace(embed=SimpleNamespace(embed_self_conditioning=True))     # config/train_DFOLDv2.yaml:83
    exp = ref_shims.reference_experiment(net, diffuser, model_conf, None, SimpleNamespace(diffuse_rot=True))
    exp._conf = SimpleNamespace(model=SimpleNamespace(cfg_drop_rate=0.0, cfg_gamma=1.0))
    exp._data_conf = SimpleNamespace(num_t=c["num_t"], min_t=0.01)

    w = window(c)
    valid_feats = {k: w[k][None].clone() for k in ("aatype", "rigids_0", "force", "vel", "torsion_angles_sin_cos",
                                                   "torsion_angles_mask")}
    valid_feats["node_repr"], valid_feats["edge_repr"] = w["node_repr"][None].clone(), w["edge_repr"][None].clone()
    inputs, preds = [], []
    inference_fn = exp.inference_fn

    def repaired(data_init, **kw):
        for k in REPAIR_KEYS:
            data_init[k] = valid_feats[k].flatten(0, 1)
        inputs.append(data_init["rigids_0"].clone())
        out = inference_fn(data_init, **kw)
        preds.append(torch.as_tensor(np.array(out["rigid_traj"][0])))
        if c["stop"] is not None and len(preds) == c["stop"]:
            raise _Stop
        return out

    exp.inference_fn = repaired
    np.random.seed(c["seed"])
    torch.manual_seed(c["seed"])
    with tempfile.TemporaryDirectory() as tmp:
        try:
            exp.eval_extension(tmp, [(valid_feats, ["window.pdb"])], "cpu", min_t=0.01, num_t=c["num_t"])
        except _Stop:
            pass
        ext = dict(np.load(os.path.join(tmp, "extension.npz"))) if c["stop"] is None else None
    res = {"case": dict(c)}
    if ext is None:
        res["rigids_0"] = torch.stack(inputs).float()                          # [stop, nf, N, 7]
        res["rigid_pred"] = torch.stack(preds).float()                         # [stop, nf, N, 7]
        return res
    rigid_traj, atom_traj = torch.as_tensor(ext["rigid_traj"]), torch.as_tensor(ext["atom_traj"])
    assert rigid_traj.shape == (200, N, 7) and atom_traj.shape == (200, N, 37, 3), (rigid_traj.shape, atom_traj.shape)
    assert torch.equal(rigid_traj, torch.stack([p[-1] for p in preds]).to(rigid_traj.dtype))
    res.update({"steps": STEPS, "rigids_0": torch.stack([inputs[j] for j in STEPS]).float(), "rigid_traj": rigid_traj.float(),
                "atom_steps": ATOM_STEPS, "atom_traj": atom_traj[ATOM_STEPS].float()})
    return res


def main():
    res = {"repair": "exp.inference_fn wrapped to complete data_init with the window's flattened " + ", ".join(REPAIR_KEYS),
           "length": 200, "min_t": 0.01, "cases": {}}
    for name, c in CASES.items():
        res["cases"][name] = run_case(c)
        print(f"[golden] rollout/{name} done")
    path = os.path.join(OUT, "rollout.pt")
    torch.save(res, path)
    print(f"[golden] {path}: {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
