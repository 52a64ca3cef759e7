"""-m gpu: Evaluator.extend, the reference's eval_extension over a test split scored against the MD frames that follow each
window, on splits written in the reference loader's formats (oracle/synth_traj.py), tiny preset.

  * every score row equals bit for bit a loop written by hand from the public pieces (windows built one at a time,
    TrajectoryRollout.rollout(graph=False), the continuation featurised on its own, rot_trans_error, atom_errors and
    superimpose frame by frame), run after run;
  * horizon 1 equals Evaluator.evaluate()'s row bit for bit: both score the trunk's prediction at min_t;
  * on one short case the trajectory matches the network oracle's rollout and the scores the fp64 metric oracle;
  * the extension.npz of a one-protein split equals TrajectoryRollout.rollout on its window;
  * over lengths 17, 40, 23, 40, 17 no CUDA graph is made, the peak allocation stays within 10 % of the largest protein's
    extension (five 40-residue proteins, so the prefetch ring is as full of its windows), the allocation returns to where
    it was, and nothing is read back to the host before the end (sync debug mode "error").
"""
import gc
import os

import numpy as np
import pytest
import torch

from dynamicpdb_b200 import metrics as M
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.evaluator import Evaluator, eval_seeds
from dynamicpdb_b200.input_pipeline import TrajectoryStore, featurize_window
from dynamicpdb_b200.metrics import HORIZON_KEYS
from dynamicpdb_b200.rollout import TrajectoryRollout
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from oracle import dfold_oracle as O
from oracle import metrics_oracle as MO
from oracle import rollout_oracle as RO
from oracle import synth_traj
from tests.test_cpu_metrics import SUM_TOL, angle_ratio, ratio
from tests.test_cpu_rollout import ATOM_TOL, NET_TOL, atom_l2, res_l2
from tests.test_gpu_evaluator import CONF, MIN_T, NF, SEEDS, _conf, _net, _weights, rows_of
from tests.test_gpu_input_pipeline import _reference

pytestmark = pytest.mark.gpu
DEV = "cuda"
L = 6
T_FRAMES = CONF["fix_sample_start"] + (NF + L - 1) * CONF["frame_sample_step"] + 1     # one frame to spare


@pytest.fixture(autouse=True)
def _collect_garbage():
    """Evaluators and networks hold reference cycles: free them when each test ends, not at a moment of the collector's
    choosing inside a later test that measures the allocation."""
    yield
    gc.collect()


def _split(root, lengths, name="test.csv"):
    """The csv of one protein per entry of ``lengths``, trajectories of T_FRAMES frames -> (path, rows)."""
    files = {}
    for n in sorted(set(lengths)):
        files[n] = synth_traj.write_files(synth_traj.make_trajectory(T=T_FRAMES, N=n, seed=SEEDS[n]), str(root),
                                          name=f"n{n}")
    path = os.path.join(str(root), name)
    with open(path, "w") as f:
        f.write("name,seq_len,atlas_npz,force_path,vel_path,embed_path,pdb_path\n")
        for i, n in enumerate(lengths):
            f.write(f"p{i}.n{n},{n}," + ",".join(files[n]) + ",x.pdb\n")
    return path, [files[n] for n in lengths]


def scores_of(d):
    return np.stack([d[k] for k in HORIZON_KEYS], axis=-1)


def _targets(row):
    """The MD frames rollout frames 0 .. L-1 predict, featurised on their own: (rigids [L, N, 7], atoms fp64, mask)."""
    ent = TrajectoryStore(frame_time=NF, pin=False).protein(*row)
    k, s = CONF["frame_sample_step"], CONF["fix_sample_start"]
    md = ent["atom37"][[s + (NF - 1 + j) * k for j in range(L)]].to(DEV)
    mask = ent["atom_mask"].to(DEV)
    gt = featurize_window(md, mask, ent["aatype"].to(DEV))
    m = mask.double().unsqueeze(0).repeat(L, 1, 1)
    m[:, -1, -1] = 0.0                                   # eval_fn's atom_mask[-1, -1, -1] = 0, at every horizon
    return gt["rigids_0"], md.double(), m


def _hand_loop(rows, net, diffuser, seed):
    window_seed, _ = eval_seeds(seed)
    windows = _reference(CONF, rows, False, diffuser, window_seed, 0, True)
    roller = TrajectoryRollout(net)
    out = []
    for row, w in zip(rows, windows):
        traj = roller.rollout(w, L, min_t=MIN_T, graph=False)
        rig, atoms, mask = _targets(row)
        N = rig.shape[1]
        rot, tr, _, _ = M.rot_trans_error(traj["rigid_traj"], rig, ref_frame=0)
        prot, ptr, _, _ = M.rot_trans_error(w["rigids_0"][NF - 2].unsqueeze(0).repeat(L, 1, 1), rig, ref_frame=0)
        err = M.atom_errors(traj["atom_traj"], atoms, mask)
        rmsd = torch.cat([M.superimpose(traj["atom_traj"][j].reshape(N * 37, 3), atoms[j].reshape(N * 37, 3),
                                        mask[j].reshape(N * 37))[1].reshape(1) for j in range(L)])
        out.append(torch.stack([rot, tr, err["mae"], err["mse"], rmsd, prot, ptr], dim=1))
    return torch.stack(out).cpu().numpy()


@pytest.mark.timeout(600)
def test_scores_equal_a_hand_written_loop_and_horizon_one_equals_evaluate(tmp_path, capsys):
    csv_path, rows = _split(tmp_path, [17, 23, 40])
    conf = _conf(csv_path, _weights(_net(), str(tmp_path / "w.pth")))
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    torch.manual_seed(123)
    global_state = torch.cuda.get_rng_state()
    ev = Evaluator(conf, _net(seed=1), diffuser, seed=5)
    first = ev.extend(L)
    assert torch.equal(torch.cuda.get_rng_state(), global_state)            # the global generator is not touched
    got = scores_of(first)
    second = scores_of(ev.extend(L))
    printed = capsys.readouterr().out.splitlines()
    assert len(printed) == 2 * len(HORIZON_KEYS) and printed[0].startswith("ave_rot: h1 ") and f" h{L} " in printed[0]
    want = _hand_loop(rows, ev.net, diffuser, 5)
    assert want.shape == (3, L, 7) and np.isfinite(want).all()
    assert np.array_equal(got, want), np.abs(got - want).max()
    assert np.array_equal(second, want)
    assert first["name"] == ["p0", "p1", "p2"]
    # the rollout moves away from the data and the persistence baseline is not the rollout's error
    assert (got[:, -1, 4] > 0).all() and not np.array_equal(got[..., 0], got[..., 5])
    # horizon 1: the same prediction eval_fn scores, the trunk's at min_t (neither t nor the noised frames enter it)
    rows_eval = rows_of(ev.evaluate())
    capsys.readouterr()
    assert np.array_equal(got[:, 0, :5], rows_eval), np.abs(got[:, 0, :5] - rows_eval).max()
    assert not ev.roller._graphs


@pytest.mark.timeout(600)
def test_one_short_case_against_the_float64_oracles(tmp_path, capsys):
    """The trajectory against rollout_oracle within the network bars, the scores against metrics_oracle on the same
    trajectory within tests/test_cpu_metrics.py's bounds, persist_* against the oracle's error of the repeated frame."""
    csv_path, rows = _split(tmp_path, [17])
    net = _net(seed=2)
    conf = _conf(csv_path, _weights(net, str(tmp_path / "w.pth")))
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    ev = Evaluator(conf, net, diffuser, seed=0)
    got = scores_of(ev.extend(L, out_dir=tmp_path / "out"))[0]
    capsys.readouterr()
    with np.load(tmp_path / "out" / "p0" / "extension.npz") as f:
        rigid_traj, atom_traj = torch.from_numpy(f["rigid_traj"]), torch.from_numpy(f["atom_traj"])
    w = {k: v.cpu() for k, v in _reference(CONF, rows, False, diffuser, eval_seeds(0)[0], 0, True)[0].items()}
    p = {k: v.detach().cpu() for k, v in net.state_dict().items()}
    ref = RO.rollout(p, w, L, O.default_conf(**syn.PRESET_TINY), O.default_diffuser_conf(1.0), MIN_T)
    assert res_l2(rigid_traj, ref["rigid_traj"]) < NET_TOL
    assert atom_l2(atom_traj, ref["atom_traj"]) < ATOM_TOL
    rig, atoms, mask = (t.cpu() for t in _targets(rows[0]))
    rot, tr, _, _ = MO.rot_trans_error(rigid_traj, rig, ref_frame=0)
    err = MO.atom_errors(atom_traj, atoms, mask)
    _, rmsd = MO.superimpose(atom_traj.reshape(L, -1, 3), atoms.reshape(L, -1, 3), mask.reshape(L, -1))
    prot, ptr, _, _ = MO.rot_trans_error(w["rigids_0"][NF - 2].unsqueeze(0).repeat(L, 1, 1), rig, ref_frame=0)
    want = {"ave_rot": rot, "ave_trans": tr, "all_atom_mae": err["mae"], "all_atom_mse": err["mse"], "all_atom_rmsd": rmsd,
            "persist_rot": prot, "persist_trans": ptr}
    for j, k in enumerate(HORIZON_KEYS):
        g = torch.from_numpy(got[:, j].copy())
        bound = angle_ratio(g, want[k]) if k.endswith("rot") else ratio(g, want[k], SUM_TOL)
        assert bound <= 1.0, (k, bound)


@pytest.mark.timeout(600)
def test_extension_file_equals_the_rollout_of_the_window(tmp_path, capsys):
    csv_path, rows = _split(tmp_path, [23])
    net = _net(seed=3)
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    ev = Evaluator(_conf(csv_path, _weights(net, str(tmp_path / "w.pth"))), net, diffuser, seed=4)
    ev.extend(L, out_dir=str(tmp_path / "out"))
    capsys.readouterr()
    w = _reference(CONF, rows, False, diffuser, eval_seeds(4)[0], 0, True)[0]
    want = TrajectoryRollout(net).rollout(w, L, min_t=MIN_T)
    with np.load(os.path.join(str(tmp_path), "out", "p0", "extension.npz")) as f:
        got = dict(f)
    assert sorted(got) == ["aatype", "atom_traj", "rigid_traj"]
    for k in ("rigid_traj", "atom_traj"):
        assert got[k].dtype == np.float32 and np.array_equal(got[k], want[k].cpu().numpy()), k
    assert got["aatype"].dtype == np.int64 and np.array_equal(got["aatype"], w["aatype"][None].cpu().numpy())


class _Reads(Evaluator):
    """Counts the device-to-host reads of the loop's one read-back; sync debug mode is lifted for it alone."""

    def _read(self, rows):
        self.reads = getattr(self, "reads", 0) + 1
        torch.cuda.set_sync_debug_mode(0)
        return super()._read(rows)


@pytest.mark.timeout(600)
def test_memory_is_bounded_and_nothing_is_read_back_per_protein(tmp_path, monkeypatch, capsys):
    weights = _weights(_net(), str(tmp_path / "w.pth"))
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    net = _net(seed=1)
    lengths = [17, 40, 23, 40, 17]
    mixed = _Reads(_conf(_split(tmp_path, lengths)[0], weights), net, diffuser)
    # the 40-residue protein alone, with the prefetcher's ring as full as it is over the mixed split: as many windows,
    # every one of them of 40 residues.  While the loop holds one window, the queue holds depth more and the worker one
    # made for a full queue, and the windows carry their horizons' targets, so fewer than len(lengths) would not fill it.
    single = _Reads(_conf(_split(tmp_path, [40] * len(lengths), name="one.csv")[0], weights), net, diffuser)

    def no_graph(*a, **k):
        raise AssertionError("the extension loop made a CUDA graph")
    monkeypatch.setattr(torch.cuda, "CUDAGraph", no_graph)
    single.extend(L)                                   # warm-up: diffuser tables, weight planes, allocator
    gc.collect()                                       # what earlier tests left must not be freed inside the window
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    single.extend(L)
    torch.cuda.synchronize()
    one = torch.cuda.max_memory_allocated() - base
    assert torch.cuda.memory_allocated() == base
    torch.cuda.reset_peak_memory_stats()
    torch.cuda.set_sync_debug_mode("error")
    try:
        mixed.extend(L)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    with capsys.disabled():
        print(f"\n[extension memory] base {base} B, 40 x {len(lengths)} {one} B, {lengths} {peak} B")
    assert mixed.reads == 1
    assert peak <= 1.10 * one, (peak, one)
    assert torch.cuda.memory_allocated() == base
    assert not mixed.roller._graphs and not single.roller._graphs
    capsys.readouterr()
