"""Input pipeline (SURVEY.md §8 f4) on the host: the oracle restatement of the loader's featurisation and the window
arithmetic of TrajectoryStore against tests/golden/loader.pt (generated from the unmodified PdbDataset._process_csv_row)."""
import numpy as np
import pytest
import torch

from dynamicpdb_b200.input_pipeline import TrajectoryStore
from oracle import dfold_oracle as O
from oracle import synth_traj
from tests.test_cpu_oracle import close, load

CONF = dict(frame_time=3, frame_sample_step=2, keep_first=8)


def _window(tmp_path):
    traj = synth_traj.make_trajectory()
    row = synth_traj.write_files(traj, str(tmp_path))
    store = TrajectoryStore(pin=False, **CONF)
    ent = store.protein(*row)
    np.random.seed(5)                                   # the golden's numpy stream
    sl = store.window_index(ent["atom37"].shape[0], training=True)
    return store, ent, sl, row


def test_window_selection_follows_the_reference_stream(tmp_path):
    gold = load("loader")
    store, ent, sl, row = _window(tmp_path)
    assert close(ent["force"][sl], gold["force"], 0) and close(ent["vel"][sl], gold["vel"], 0)
    assert ent["force"][sl].dtype == gold["force"].dtype
    assert torch.equal(ent["aatype"][None].expand(3, -1), gold["aatype"])
    assert torch.equal(ent["residue_index"][None].expand(3, -1), gold["seq_idx"])
    assert store.protein(*row) is ent                   # cached: the archive is decoded once
    assert store.window_index(8, training=False) == slice(0, 6, 2)


def test_oracle_featurisation_matches_reference_loader(tmp_path):
    gold = load("loader")
    _, ent, sl, _ = _window(tmp_path)
    R0, t0, sc, alt, mask = O.featurize_window(ent["atom37"][sl], ent["atom_mask"], ent["aatype"])
    assert close(R0, gold["rot_0"].double(), 2e-6) and close(t0, gold["rigids_0"][..., 4:].double(), 1e-6)
    assert close(sc, gold["torsion_angles_sin_cos"], 1e-6)      # the reference runs this transform on fp64 copies of fp32 data
    assert close(alt, gold["alt_torsion_angles_sin_cos"], 1e-6)
    assert torch.equal(mask, gold["torsion_angles_mask"])
    assert close(ent["atom_mask"][:, 1].double()[None].expand(3, -1), gold["res_mask"].double(), 0)
    # rigids_0: the reference's quaternion (eigen-decomposition, arbitrary sign) encodes the same rotation
    q = gold["rigids_0"][..., :4].double()
    assert close(O.quat_to_rot(q / q.norm(dim=-1, keepdim=True)), R0, 2e-6)


def _eval_store(tmp_path, fix_sample_start=None):
    gold = load("loader_eval")
    c = gold["case"]
    row = synth_traj.write_files(synth_traj.make_trajectory(T=c["T"]), str(tmp_path))
    fix = c["fix_sample_start"] if fix_sample_start is None else fix_sample_start
    store = TrajectoryStore(frame_time=c["frame_time"], frame_sample_step=c["frame_sample_step"], keep_first=c["keep_first"],
                            fix_sample_start=fix, pin=False)
    return gold, store, store.protein(*row)


def test_evaluation_window_ignores_keep_first_as_the_reference_loader(tmp_path):
    """tests/golden/loader_eval.pt: evaluation reads the whole trajectory from fix_sample_start, past keep_first."""
    gold, store, ent = _eval_store(tmp_path)
    sl = store.window_index(ent["atom37"].shape[0], training=False)
    assert sl == slice(4, 10, 2)
    assert torch.equal(ent["force"][sl], gold["force"]) and torch.equal(ent["vel"][sl], gold["vel"])
    assert torch.equal(ent["atom_mask"].double().expand(3, -1, -1), gold["atom37_mask"])
    # the loader zeroes the coordinates of atoms outside the mask; the store keeps the archive's
    assert torch.equal(ent["atom37"][sl].double() * gold["atom37_mask"][..., None], gold["atom37_pos"])
    R0, t0, sc, alt, mask = O.featurize_window(ent["atom37"][sl], ent["atom_mask"], ent["aatype"])
    assert close(R0, gold["rot_0"].double(), 2e-6) and close(t0, gold["rigids_0"][..., 4:].double(), 1e-6)
    assert close(sc, gold["torsion_angles_sin_cos"], 1e-6) and torch.equal(mask, gold["torsion_angles_mask"])


def test_training_windows_stay_within_keep_first(tmp_path):
    """The store keeps frames past keep_first for the evaluation window; training windows never draw from them."""
    gold, store, ent = _eval_store(tmp_path)
    assert ent["atom37"].shape[0] > gold["case"]["keep_first"]
    np.random.seed(0)
    stops = {store.window_index(ent["atom37"].shape[0], training=True).stop for _ in range(200)}
    assert stops == set(range(6, gold["case"]["keep_first"] + 1))


def test_evaluation_window_past_the_trajectory_raises_as_the_reference_loader(tmp_path):
    """fix_sample_start=10 of 12 frames leaves fewer than frame_time: the reference's select_first_samples raises."""
    gold, store, ent = _eval_store(tmp_path, fix_sample_start=load("loader_eval")["case"]["fix_sample_start_error"])
    with pytest.raises(ValueError, match=gold["error"]):
        store.window_index(ent["atom37"].shape[0], training=False)
    short = TrajectoryStore(frame_time=3, frame_sample_step=4, fix_sample_start=4, pin=False)    # 3 <= 8 frames, but 4, 8, 12
    with pytest.raises(ValueError, match="reaches past"):
        short.window_index(12, training=False)
