"""Generate tests/golden/metrics.pt from the UNMODIFIED reference (a checkout of it at $DFOLD_REFERENCE_ROOT):

    python oracle/make_metrics_golden.py

Runs, on the inputs of oracle/metrics_cases.py (rebuilt by the tests from numpy seeds; the fixture keeps a checksum):
- src/toolbox/rot_trans_error.py average_quaternion_distances / average_translation_distances and
  Experiment._calc_rot_trans_error (train_DFOLD_dynamics.py:1549-1568);
- openfold/utils/validation_metrics.py drmsd;
- rmsdalign (train_DFOLD_dynamics.py:74-97, the reference's own torch Kabsch);
- compute_validation_metrics_all(..., superimposition_metrics=True) (:99-154);
- Experiment.eval_fn (:765-928) on one frame_time = 5, N = 256 window, with inference_fn replaced by an injected
  sample_out and sample_ref by a fixed draw.
Predictions are run as fp32 (what the model returns) and upcast to fp64.

Bio is not installed here and oracle/ref_shims.py stubs it inertly, so where the reference calls Bio's SVDSuperimposer
(eval_fn :904-908 and openfold/utils/superimposition.py:20-35) this generator substitutes a superimposer built on the
reference's own rmsdalign.  Both minimise the same RMSD over proper rotations; the fixture records the substitution.
"""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import metrics_cases as C  # noqa: E402
from oracle import ref_shims  # noqa: E402

ref_shims.install_trainer_stubs()
import train_DFOLD_dynamics as T  # noqa: E402
from openfold.utils import superimposition as RefSup  # noqa: E402
from openfold.utils import validation_metrics as RefVM  # noqa: E402
from src.toolbox import rot_trans_error as RefRTE  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


class RmsdalignSuperimposer:
    """Bio.SVDSuperimposer's interface (set / run / get_transformed / get_rms) over the reference's rmsdalign, fp64."""

    def set(self, reference, coords):
        self.ref = np.asarray(reference, dtype=np.float64)
        self.x = np.asarray(coords, dtype=np.float64)

    def run(self):
        self.y = T.rmsdalign(torch.from_numpy(self.ref), torch.from_numpy(self.x)).numpy()

    def get_transformed(self):
        return self.y

    def get_rms(self):
        return float(np.sqrt(((self.y - self.ref) ** 2).sum(-1).mean()))


T.SVDSuperimposer = RmsdalignSuperimposer
RefSup.SVDSuperimposer = RmsdalignSuperimposer


def _np(x):
    return torch.as_tensor(np.asarray(x)).clone()


def rigid_cases():
    res = {}
    exp = object.__new__(T.Experiment)
    for name, (nf, N, seed) in C.RIGID_CASES.items():
        gt, pred = C.rigids(nf, N, seed)
        c = {"check": C.checksum(gt, pred)}
        for prec, p in (("fp32", pred), ("fp64", pred.double())):
            g, pn = gt.numpy(), p.numpy()
            c[prec] = {
                "quat": _np(RefRTE.average_quaternion_distances(g[..., :4], pn[..., :4])),
                "trans": _np(RefRTE.average_translation_distances(g[..., 4:], pn[..., 4:], measurement="MAE")),
                "calc": [_np(v) for v in exp._calc_rot_trans_error(pn, gt_rigids=g)],
            }
        res[name] = c
    return res


def atom_cases():
    res = {}
    for name, (nf, N, seed, kind) in C.ATOM_CASES.items():
        gt, pred, mask = C.atoms(nf, N, seed, kind)
        c = {"check": C.checksum(gt, pred, mask)}
        for prec, p in (("fp32", pred), ("fp64", pred.double())):
            vm = T.compute_validation_metrics_all(gt.clone(), p.numpy().copy(), mask.clone(), superimposition_metrics=True)
            pm, gm = p.double() * mask[..., None], gt * mask[..., None]
            c[prec] = {"validation": {k: v.clone() for k, v in vm.items()},
                       "drmsd_ca": RefVM.drmsd(pm[..., 1, :], gm[..., 1, :], mask=mask[..., 1]).clone(),
                       "drmsd_ca_nomask": RefVM.drmsd(p[..., 1, :].double(), gt[..., 1, :]).clone()}
        res[name] = c
    return res


def kabsch_cases():
    res = {}
    for name, seed in C.KABSCH_CASES.items():
        ref, x = C.point_sets(name, seed)
        y = T.rmsdalign(ref, x)
        res[name] = {"check": C.checksum(ref, x), "superimposed": y.clone(),
                     "rmsd": torch.sqrt(((y - ref) ** 2).sum(-1).mean()).clone()}
    return res


class _FixedRef:
    def __init__(self, rigids_t):
        self.rigids_t = rigids_t

    def sample_ref(self, n_samples, as_tensor_7=True, **kw):
        assert n_samples == self.rigids_t.shape[0] * self.rigids_t.shape[1]
        return {"rigids_t": self.rigids_t.clone()}


def eval_window_case():
    w = C.eval_window()
    nf, N = w["rigids_0"].shape[:2]
    res = {"check": C.checksum(*w.values())}
    for prec, cast in (("fp32", lambda t: t), ("fp64", lambda t: t.double())):
        exp = object.__new__(T.Experiment)
        exp._diffuser = _FixedRef(torch.zeros(nf, N, 7))
        rigid_traj = np.stack([cast(w["rigid_pred"]).numpy(), np.zeros((nf, N, 7), np.float32)])
        prot_traj = np.stack([cast(w["atom37_pred"]).numpy(), np.zeros((nf, N, 37, 3), np.float32)])
        exp.inference_fn = lambda init_feats, **kw: {"rigid_traj": rigid_traj, "prot_traj": prot_traj}
        feats = {
            "aatype": torch.zeros(1, nf, N, dtype=torch.long), "torsion_angles_sin_cos": torch.zeros(1, nf, N, 7, 2),
            "torsion_angles_mask": torch.zeros(1, nf, N, 7), "node_repr": torch.zeros(1, N, 4), "edge_repr": torch.zeros(1, N, N, 2),
            "rigids_0": w["rigids_0"][None].clone(), "atom37_pos": w["atom37_pos"][None].clone(),
            "atom37_mask": w["atom37_mask"][None].clone(), "force": torch.zeros(1, nf, N, 3), "vel": torch.zeros(1, nf, N, 3),
        }
        with tempfile.TemporaryDirectory() as tmp:
            d = exp.eval_fn(tmp, [(feats, ["window.pdb"])], "cpu", min_t=0.01, num_t=2)
        vm = T.compute_validation_metrics_all(w["atom37_pos"].clone(), cast(w["atom37_pred"]).numpy().copy(),
                                              w["atom37_mask"].clone(), superimposition_metrics=True)
        res[prec] = {"eval_fn": {k: _np(np.concatenate(d[k]) if isinstance(d[k], list) else d[k])
                                 for k in ("ave_rot", "ave_trans", "all_atom_mae", "all_atom_mse", "all_atom_rmsd")},
                     "validation": {k: v.clone() for k, v in vm.items()}}
    return res


def main():
    res = {"superimposer": "Bio.SVDSuperimposer replaced by a superimposer over the reference's rmsdalign "
                           "(train_DFOLD_dynamics.py:74-97)",
           "rigid": rigid_cases(), "atoms": atom_cases(), "kabsch": kabsch_cases(), "eval_window": eval_window_case()}
    path = os.path.join(OUT, "metrics.pt")
    torch.save(res, path)
    print(f"[golden] {path}: {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
