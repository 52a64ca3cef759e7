"""Generate tests/golden/evaluator.pt from the UNMODIFIED reference (a checkout of it at $DFOLD_REFERENCE_ROOT):

    python oracle/make_evaluator_golden.py

Drives ``Experiment.eval_fn`` (train_DFOLD_dynamics.py:765-928) through ``ref_shims.reference_experiment`` over the
unmodified ``PdbDataset(is_training=False, is_testing=True)`` in a batch-1 ``DataLoader``, as
``Evaluator.start_evaluation`` (eval_DFOLD_dynamics.py:152-204) builds it, on a synthetic test csv (oracle/synth_traj.py):
proteins of 17, 23 and 40 residues, a row above ``filtering.max_len`` that the loader drops, ``frame_time`` 3 every 2nd
frame from frame 3.  ``inference_fn`` is replaced by a seeded injection of ``rigid_traj`` / ``prot_traj`` (fp64, so that
every metric eval_fn computes is fp64); the translations of the 23-residue protein are pushed by 2e4 so that its
``ave_trans >= 10000`` and the printed means divide by fewer rows than they sum.  Bio's SVDSuperimposer is replaced as
oracle/make_metrics_golden.py replaces it.

The fixture holds the case, the csv text, per protein the loader's window fields and the injected predictions, eval_fn's
returned dict and the lines it printed, and ``ave_rot`` / ``ave_trans`` recomputed with the loader's fp32 ``rigids_0``
upcast to fp64 (``gt64``: the spread of the reference's own fp32 arithmetic).
"""
import contextlib
import io
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402
from oracle import synth_traj  # noqa: E402
from oracle.make_metrics_golden import T  # noqa: E402  (the reference trainer, Bio's superimposer replaced)

OUT = os.path.join(ROOT, "tests", "golden")
# csv rows in order: (name, residues, seed); None: a row above max_len whose files do not exist
PROTEINS = [("prot40.A", 40, 33), ("long.B", None, None), ("prot17", 17, 31), ("prot23.pdb", 23, 32)]
CASE = dict(T=10, frame_time=3, frame_sample_step=2, fix_sample_start=3, max_len=48, long_len=64, noise_scale=0.1,
            num_t=4, min_t=0.01, pushed="prot23", push=2e4, seed=11)
WINDOW_KEYS = ("aatype", "seq_idx", "rigids_0", "atom37_pos", "atom37_mask", "torsion_angles_sin_cos",
               "torsion_angles_mask", "force", "vel")


class _ZeroRef:
    """The diffuser of the loader and of eval_fn: only ``sample_ref`` is called, whose draw the injected sample ignores."""

    def sample_ref(self, n_samples, impute=None, diffuse_mask=None, as_tensor_7=True):
        return {"rigids_t": torch.zeros(n_samples, 7)}


def write_split(root):
    """The synthetic trajectories and the test csv under ``root``; -> (csv path, csv text)."""
    lines = ["name,seq_len,atlas_npz,force_path,vel_path,embed_path,pdb_path"]
    for name, N, seed in PROTEINS:
        stem = name.split(".")[0]
        if N is None:
            lines.append(f"{name},{CASE['long_len']},{stem}.npz,{stem}_F.pkl,{stem}_V.pkl,{stem}_emb.npz,{stem}.pdb")
            continue
        row = synth_traj.write_files(synth_traj.make_trajectory(T=CASE["T"], N=N, seed=seed), root, name=stem)
        lines.append(f"{name},{N}," + ",".join(row) + f",{stem}.pdb")
    text = "\n".join(lines) + "\n"
    path = os.path.join(root, "test.csv")
    with open(path, "w") as f:
        f.write(text)
    return path, text


def main():
    if not ref_shims.reference_available():
        raise SystemExit("set DFOLD_REFERENCE_ROOT to a checkout of the reference")
    from src.data import Dfold_data_loader_dynamic as L
    rng = np.random.default_rng(CASE["seed"])
    windows, predictions = [], []

    def inject(init_feats, **kw):
        """rigid_traj / prot_traj of inference_fn: the ground truth moved by seeded noise, at t = min_t first."""
        rig0 = init_feats["rigids_0"].double().numpy()
        nf, N = rig0.shape[:2]
        q = rig0[..., :4] + 0.2 * rng.standard_normal((nf, N, 4))
        rigid = np.concatenate([q / np.linalg.norm(q, axis=-1, keepdims=True),
                                rig0[..., 4:] + 0.7 * rng.standard_normal((nf, N, 3))], axis=-1)
        atom = init_feats["atom37_pos"].double().numpy() + 0.5 * rng.standard_normal((nf, N, 37, 3))
        predictions.append({"rigid_pred": torch.from_numpy(rigid), "atom37_pred": torch.from_numpy(atom)})
        return {"rigid_traj": np.stack([rigid, np.zeros_like(rigid)]), "prot_traj": np.stack([atom, np.zeros_like(atom)])}

    with tempfile.TemporaryDirectory() as d:
        csv_path, csv_text = write_split(d)
        data_conf = types.SimpleNamespace(
            test_csv_path=csv_path, filtering=types.SimpleNamespace(max_len=CASE["max_len"]), frame_time=CASE["frame_time"],
            frame_sample_step=CASE["frame_sample_step"], fix_sample_start=CASE["fix_sample_start"], dynamics=True,
            num_t=CASE["num_t"], min_t=CASE["min_t"], keep_first=None)
        dataset = L.PdbDataset(data_conf=data_conf, diffuser=_ZeroRef(), is_training=False, is_testing=True)
        loader = torch.utils.data.DataLoader(dataset, batch_size=1, shuffle=False, num_workers=0, drop_last=False)
        names = []

        def recorded():
            for feats, pdb_names in loader:
                windows.append({k: feats[k][0].clone() for k in WINDOW_KEYS})
                names.append(pdb_names[0])
                yield feats, pdb_names

        exp = ref_shims.reference_experiment(None, _ZeroRef(), None, None, None)
        exp._data_conf = data_conf

        def inference_fn(init_feats, **kw):
            out = inject(init_feats)
            if names[-1].split(".")[0] == CASE["pushed"]:
                out["rigid_traj"][0][..., 4:] += CASE["push"]
                predictions[-1]["rigid_pred"][..., 4:] += CASE["push"]
            return out

        exp.inference_fn = inference_fn
        out = io.StringIO()
        with contextlib.redirect_stdout(out):
            result = exp.eval_fn(os.path.join(d, "eval"), recorded(), "cpu", noise_scale=CASE["noise_scale"],
                                 is_training=False)
    # the loader's rigids_0 is fp32, and eval_fn normalises its quaternions in fp32: the same rows with it upcast first
    # give the spread the fp64 kernels may differ by
    gt64 = [exp._calc_rot_trans_error(p["rigid_pred"].numpy(), gt_rigids=w["rigids_0"].double().numpy())
            for w, p in zip(windows, predictions)]
    res = {"case": dict(CASE), "proteins": PROTEINS, "csv": csv_text, "loader_names": names, "windows": windows,
           "predictions": predictions, "result": result, "stdout": out.getvalue().splitlines(),
           "gt64": {"ave_rot": np.concatenate([g[0][-1:] for g in gt64]), "ave_trans": np.concatenate([g[1][-1:] for g in gt64])}}
    path = os.path.join(OUT, "evaluator.pt")
    torch.save(res, path)
    print(f"[golden] {path}: {os.path.getsize(path)} bytes, names {result['name']}, printed {res['stdout']}")


if __name__ == "__main__":
    main()
