"""-m gpu: dynamicpdb_b200.evaluator on test splits of several residue counts written in the reference loader's formats
(oracle/synth_traj.py), tiny preset.

  * with the fixture's predictions injected for the sampler, every window equals the unmodified loader's window
    (tests/golden/evaluator.pt) and every row eval_fn's, within the metric bounds of tests/test_cpu_metrics.py;
  * with the real sampler, every row equals bit for bit a loop written by hand from the public pieces (windows built one
    at a time, DeviceReverseDiffusion.sample, window_metrics) with the same two seeded generators, run after run, and
    with the prefetcher's side stream stalled behind one window (the rows score the trunk's prediction, which reads
    neither t nor the noised frames, so another seed gives the same rows too);
  * over lengths 17, 40, 23, 40, 17 no CUDA graph is made, the peak allocation stays within 10 % of the largest
    protein's evaluation (with the prefetch ring full of its windows) and the allocation returns to where it was;
  * the loop reads nothing back to the host before the end (sync debug mode "error");
  * a save_checkpoint file and a module.-prefixed reference-style dict give the same rows; a mismatched one raises and
    leaves the weights.
"""
import os

import numpy as np
import pytest
import torch

from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.checkpoint import save_checkpoint
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.evaluator import ROW_KEYS, Evaluator, eval_seeds
from dynamicpdb_b200.inference import DeviceReverseDiffusion
from dynamicpdb_b200.input_pipeline import TrajectoryStore, WindowPrefetcher
from dynamicpdb_b200.loss import score_network_loss
from dynamicpdb_b200.metrics import eval_sampler_inputs, window_metrics
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from dynamicpdb_b200.train_step import TrainStep
from oracle import dfold_oracle as O
from oracle import metrics_oracle as MO
from oracle import synth_traj
from tests.test_cpu_evaluator import fixture, row_bounds
from tests.test_cpu_metrics import SUM_TOL, angle_ratio, ratio
from tests.test_gpu_input_pipeline import _reference, _sleep_cycles, _StalledPrefetcher

pytestmark = pytest.mark.gpu
DEV = "cuda"
NF, T_FRAMES = 3, 10
SEEDS = {17: 31, 23: 32, 40: 33}
CONF = dict(frame_time=NF, frame_sample_step=2, fix_sample_start=3)
NUM_T, MIN_T, NOISE = 5, 0.01, 0.1


def _net(seed=7):
    net = FullScoreNetwork(syn.model_conf(NF, **syn.PRESET_TINY), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    state = syn.random_state({k: v.shape for k, v in net.state_dict().items()}, seed=seed)
    net.load_state_dict(state, strict=True)
    return net.to(DEV)


def _weights(net, path, prefix=""):
    torch.save({"model": {prefix + k: v.detach().cpu() for k, v in net.state_dict().items()}, "conf": None}, path)
    return path


def _split(root, lengths, name="test.csv"):
    """The csv of one protein per entry of ``lengths`` (files written once per length) -> (path, rows)."""
    files = {}
    for n in sorted(set(lengths)):
        files[n] = synth_traj.write_files(synth_traj.make_trajectory(T=T_FRAMES, N=n, seed=SEEDS[n]), str(root), name=f"n{n}")
    path = os.path.join(str(root), name)
    with open(path, "w") as f:
        f.write("name,seq_len,atlas_npz,force_path,vel_path,embed_path,pdb_path\n")
        for i, n in enumerate(lengths):
            f.write(f"p{i}.n{n},{n}," + ",".join(files[n]) + ",x.pdb\n")
    return path, [files[n] for n in lengths]


def _conf(csv_path, weights, frame_time=NF, num_t=NUM_T, **data):
    conf = {"eval": {"weights_path": weights, "eval_batch_size": 1}, "experiment": {"noise_scale": NOISE},
            "data": {"test_csv_path": csv_path, "filtering": {"max_len": 256}, "frame_time": frame_time,
                     "frame_sample_step": CONF["frame_sample_step"], "fix_sample_start": CONF["fix_sample_start"],
                     "num_t": num_t, "min_t": MIN_T}}
    conf["data"].update(data)
    return conf


def rows_of(d):
    return np.stack([d["ave_rot"], d["ave_trans"], d["all_atom_mae"], np.concatenate(d["all_atom_mse"]), d["all_atom_rmsd"]],
                    axis=1)


class _Injected(Evaluator):
    """The fixture's predictions in place of the sampler; every window it is handed kept."""

    def _sample(self, index, window, generator):
        self.seen.append({k: v.clone() for k, v in window.items()})
        p = fixture()["predictions"][index]
        return p["rigid_pred"].to(DEV), p["atom37_pred"].to(DEV)


@pytest.mark.timeout(300)
def test_windows_and_rows_match_eval_fn_with_injected_predictions(tmp_path, capsys):
    g = fixture()
    c = g["case"]
    lines = ["name,seq_len,atlas_npz,force_path,vel_path,embed_path,pdb_path"]
    for name, n, seed in g["proteins"]:
        stem = name.split(".")[0]
        if n is None:
            lines.append(f"{name},{c['long_len']},{stem}.npz,{stem}_F.pkl,{stem}_V.pkl,{stem}_emb.npz,{stem}.pdb")
        else:
            row = synth_traj.write_files(synth_traj.make_trajectory(T=c["T"], N=n, seed=seed), str(tmp_path), name=stem)
            lines.append(f"{name},{n}," + ",".join(row) + f",{stem}.pdb")
    csv_path = tmp_path / "test.csv"
    csv_path.write_text("\n".join(lines) + "\n")
    conf = _conf(str(csv_path), _weights(_net(), str(tmp_path / "w.pth")), frame_time=c["frame_time"], num_t=c["num_t"],
                 frame_sample_step=c["frame_sample_step"], fix_sample_start=c["fix_sample_start"],
                 filtering={"max_len": c["max_len"]})
    ev = _Injected(conf, _net(), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    ev.seen = []
    d = ev.evaluate()
    printed = capsys.readouterr().out.splitlines()
    assert d["name"] == g["result"]["name"] and len(printed) == 4
    assert len(ev.seen) == len(g["windows"])
    got_rows = rows_of(d)
    for i, (w, gold, p) in enumerate(zip(ev.seen, g["windows"], g["predictions"])):
        # the window: the loader's fields; coordinates of the atoms inside the mask (the loader zeroes the others)
        for k in ("aatype", "seq_idx", "force", "vel", "atom37_mask", "torsion_angles_mask"):
            assert w[k].dtype == gold[k].dtype and torch.equal(w[k].cpu(), gold[k]), (i, k)
        assert torch.equal((w["atom37_pos"] * w["atom37_mask"][..., None]).cpu(), gold["atom37_pos"]), i
        # the kernel's fp32 dihedrals against the reference's fp64 ones of the same fp32 coordinates: a few fp32 ulps,
        # times the conditioning of the dihedral (the metrics do not read these; the sampler does)
        assert float((w["torsion_angles_sin_cos"].cpu() - gold["torsion_angles_sin_cos"]).abs().max()) < 1e-5
        assert torch.equal(w["rigids_0"][..., 4:].cpu(), gold["rigids_0"][..., 4:]), i      # translations: the CA atoms
        q, qg = w["rigids_0"][..., :4].double().cpu(), gold["rigids_0"][..., :4].double()
        rot_err = (O.quat_to_rot(q) - O.quat_to_rot(qg / qg.norm(dim=-1, keepdim=True))).abs().max()
        assert float(rot_err) < 2e-6, (i, float(rot_err))     # the same rotation (the reference's sign is arbitrary)
        # the device row against the oracle on the same window, within the metric bounds
        want = MO.window_metrics(p["rigid_pred"], p["atom37_pred"], w["rigids_0"].cpu(), w["atom37_pos"].cpu(),
                                 w["atom37_mask"].cpu())
        for j, k in enumerate(ROW_KEYS):
            got = torch.from_numpy(got_rows[i, j:j + 1].copy())
            tol = angle_ratio(got, want[k]) if k == "ave_rot" else ratio(got, want[k], SUM_TOL)
            assert tol <= 1.0, (i, k, tol)
        # and against eval_fn's row: the same bounds; the rotation error moves with the featurisation's rotation (2e-6
        # per matrix entry above: 2e-4 degrees at most)
        got = {k: torch.from_numpy(got_rows[i, j:j + 1].copy()) for j, k in enumerate(ROW_KEYS)}
        worst = row_bounds(got, i)
        worst["ave_rot"] = angle_ratio(got["ave_rot"], torch.from_numpy(g["result"]["ave_rot"][i:i + 1].copy()),
                                       torch.full((1,), 2e-4, dtype=torch.float64))
        assert all(v <= 1.0 for v in worst.values()), (i, worst)
    assert [ln.split()[0] for ln in printed] == [ln.split()[0] for ln in g["stdout"]]


def _hand_loop(rows, net, diffuser, seed):
    """Windows built one at a time on the current stream, sampled and scored with the public pieces."""
    window_seed, reverse_seed = eval_seeds(seed)
    windows = _reference(CONF, rows, False, diffuser, window_seed, 0, True)
    gen = torch.Generator(DEV).manual_seed(reverse_seed)
    sampler = DeviceReverseDiffusion(net)
    out = []
    for w in windows:
        s = sampler.sample(eval_sampler_inputs(w), NUM_T, MIN_T, NOISE, generator=gen)
        sampler.memo.reset()
        m = window_metrics(s["rigid_pred"], s["prot_traj"][0], w["rigids_0"], w["atom37_pos"], w["atom37_mask"])
        out.append(torch.cat([m[k] for k in ROW_KEYS]))
    return torch.stack(out).cpu().numpy()


class _Stalled(Evaluator):
    """The prefetcher's side stream sleeps ~100 ms before window 1 while the worker thread makes the next ones."""

    def _prefetcher(self, generator):
        pf = super()._prefetcher(generator)
        return _StalledPrefetcher(pf.store, pf.rows, pf.device, training=False, depth=pf.depth, diffuser=pf.diffuser,
                                  min_t=pf.min_t, generator=generator, targets=True, stall_at=1, cycles=_sleep_cycles(100))


@pytest.mark.timeout(600)
def test_rows_equal_a_hand_written_loop_bit_for_bit(tmp_path, capsys):
    csv_path, rows = _split(tmp_path, [17, 23, 40])
    conf = _conf(csv_path, _weights(_net(), str(tmp_path / "w.pth")))
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    torch.manual_seed(123)
    global_state = torch.cuda.get_rng_state()
    ev = Evaluator(conf, _net(seed=1), diffuser, seed=5)
    first = rows_of(ev.evaluate())
    assert torch.equal(torch.cuda.get_rng_state(), global_state)            # the global generator is not touched
    second = rows_of(ev.evaluate())
    stalled = rows_of(_Stalled(conf, _net(seed=1), diffuser, seed=5).evaluate())
    want = _hand_loop(rows, ev.net, diffuser, 5)
    assert np.isfinite(want).all() and want.shape == (3, 5)
    assert np.array_equal(first, want), np.abs(first - want).max()
    assert np.array_equal(second, want) and np.array_equal(stalled, want)
    # the rows score the prediction at t = min_t, which the trunk makes without reading t or the noised frames: another
    # seed draws other frames and the same rows
    other = rows_of(Evaluator(conf, _net(seed=1), diffuser, seed=6).evaluate())
    assert np.array_equal(other, want)
    capsys.readouterr()


class _Reads(Evaluator):
    """Counts the device-to-host reads of the loop's one read-back; sync debug mode is lifted for it alone."""

    def _read(self, rows):
        self.reads = getattr(self, "reads", 0) + 1
        torch.cuda.set_sync_debug_mode(0)
        return super()._read(rows)


@pytest.mark.timeout(600)
def test_memory_is_bounded_and_nothing_is_read_back_per_window(tmp_path, monkeypatch, capsys):
    weights = _weights(_net(), str(tmp_path / "w.pth"))
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    net = _net(seed=1)
    mixed = _Reads(_conf(_split(tmp_path, [17, 40, 23, 40, 17])[0], weights), net, diffuser)
    # the 40-residue protein alone, with the prefetcher's ring as full as it ever is (depth + 1 windows of it)
    single = _Reads(_conf(_split(tmp_path, [40] * (mixed.depth + 1), name="one.csv")[0], weights), net, diffuser)

    def no_graph(*a, **k):
        raise AssertionError("the evaluator made a CUDA graph")
    monkeypatch.setattr(torch.cuda, "CUDAGraph", no_graph)
    single.evaluate()                                  # warm-up: diffuser tables, weight planes, allocator
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    single.evaluate()
    torch.cuda.synchronize()
    one = torch.cuda.max_memory_allocated() - base
    assert torch.cuda.memory_allocated() == base
    torch.cuda.reset_peak_memory_stats()
    torch.cuda.set_sync_debug_mode("error")
    try:
        mixed.evaluate()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print(f"[evaluator memory] base {base} B, one protein of 40 {one} B, 17 40 23 40 17 {peak} B")
    assert mixed.reads == 1
    assert peak <= 1.10 * one, (peak, one)
    assert torch.cuda.memory_allocated() == base
    assert not mixed.sampler._graphs and not single.sampler._graphs
    capsys.readouterr()


class _Exp:
    torsion_loss_weight, rot_loss_weight, trans_loss_weight = 1.0, 0.5, 1.0
    rot_loss_t_threshold, separate_rot_loss = 0.2, False


@pytest.mark.timeout(600)
def test_checkpoint_formats_load_alike_and_a_mismatch_changes_nothing(tmp_path, capsys):
    csv_path, rows = _split(tmp_path, [17, 23])
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    trained = _net(seed=3)
    example, = list(WindowPrefetcher(TrajectoryStore(frame_time=NF), rows[:1], DEV, diffuser=diffuser))
    step = TrainStep(trained, lambda out, w: score_network_loss(out, w, _Exp), example, lr=1e-3, graph=False,
                     loss_reads_window=True)
    ours = str(tmp_path / "step_1.pth")
    save_checkpoint(ours, step, {"model": "conf"}, 0, 1)
    ref_style = _weights(trained, str(tmp_path / "ref.pth"), prefix="module.")
    a = rows_of(Evaluator(_conf(csv_path, ours), _net(seed=1), diffuser).evaluate())
    b = rows_of(Evaluator(_conf(csv_path, ref_style), _net(seed=2), diffuser).evaluate())
    assert np.array_equal(a, b)
    sd = {k: v.detach().cpu() for k, v in trained.state_dict().items()}
    k0 = next(k for k, v in sd.items() if v.dim() >= 1)
    bad = str(tmp_path / "bad.pth")
    torch.save({"model": {**sd, k0: torch.zeros(*sd[k0].shape[:-1], sd[k0].shape[-1] + 1)}}, bad)
    net = _net(seed=4)
    before = {k: v.clone() for k, v in net.state_dict().items()}
    with pytest.raises(ValueError, match=f"'{k0}' has shape"):
        Evaluator(_conf(csv_path, bad), net, diffuser)
    assert all(torch.equal(v, before[k]) for k, v in net.state_dict().items())
    capsys.readouterr()
