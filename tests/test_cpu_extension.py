"""The host side of Evaluator.extend (the reference's eval_extension over a test split, scored per horizon).

Arguments the loop refuses raise before any device work; the evaluation store's extended entry is the trajectory's frames
on the window's grid, its first frame_time frames the store's entry without horizons; a trajectory one frame short raises
naming its archive; the returned dict and printed lines equal a numpy restatement of injected scores; and the
extension.npz writer gives eval_extension's keys, shapes and dtypes."""
import copy
import re

import numpy as np
import pytest
import torch

from dynamicpdb_b200.evaluator import Evaluator, write_extension
from dynamicpdb_b200.input_pipeline import EvaluationStore
from dynamicpdb_b200.metrics import HORIZON_KEYS
from oracle import synth_traj
from tests.test_cpu_evaluator import _conf, _csv


class _HostExtension(Evaluator):
    """The Evaluator with no network and its device side replaced by given scores."""

    def __init__(self, conf, scores=None):
        self._configure(conf)
        self.fake = scores

    def _run_extension(self, length, out_dir):
        if self.fake is None:
            raise AssertionError("the extension loop started")
        return torch.from_numpy(self.fake)


def test_bad_arguments_raise_before_device_work(tmp_path):
    csv_path = _csv(tmp_path / "test.csv", [("a", 17)])
    conf = copy.deepcopy(_conf(csv_path))
    conf["data"]["frame_time"] = 1
    # the weights file does not exist: the config is refused before it is read
    with pytest.raises(ValueError, match=re.escape("data.frame_time must be an integer >= 2")):
        Evaluator(conf, None, None)
    ev = _HostExtension(_conf(csv_path))
    for length in (0, -1, True, 2.0, "200", None):
        with pytest.raises(ValueError, match="length must be an int >= 1"):
            ev.extend(length)
    for out_dir in (3, ["a"], 1.5):
        with pytest.raises(ValueError, match="out_dir must be a path or None"):
            ev.extend(5, out_dir)
    with pytest.raises(ValueError, match="min_t"):
        _HostExtension(_conf(csv_path, min_t=0.0)).extend(5)
    with pytest.raises(AssertionError, match="loop started"):
        ev.extend(5, tmp_path)                                   # a valid call reaches the loop


def _protein(tmp_path, T, N=17, seed=41):
    traj = synth_traj.make_trajectory(T=T, N=N, seed=seed)
    return traj, synth_traj.write_files(traj, str(tmp_path), name="p")


@pytest.mark.parametrize("nf,k,fix,L", [(2, 1, 0, 1), (2, 1, 0, 7), (3, 2, 3, 4), (3, 3, 2, 2), (5, 1, 1, 3)])
def test_extended_entry_is_the_window_and_its_continuation(tmp_path, nf, k, fix, L):
    need = fix + (nf + L - 2) * k + 1                            # the last frame read, plus one
    traj, row = _protein(tmp_path, need + 2)
    store = EvaluationStore(frame_time=nf, frame_sample_step=k, fix_sample_start=fix, pin=False, horizons=L)
    got = store.protein(*row)
    sl = slice(fix, fix + (nf + L - 1) * k, k)
    assert got["atom37"].shape[0] == nf + L - 1 and not store._cache
    for key, raw in (("atom37", "all_atom_positions"), ("force", "force"), ("vel", "vel")):
        assert torch.equal(got[key], torch.from_numpy(np.ascontiguousarray(traj[raw][sl])).to(got[key].dtype)), key
    assert store.window_index(got["atom37"].shape[0], training=False) == slice(0, nf, 1)
    plain = EvaluationStore(frame_time=nf, frame_sample_step=k, fix_sample_start=fix, pin=False).protein(*row)
    for key in ("atom37", "force", "vel"):
        assert torch.equal(got[key][:nf], plain[key]), key
    for key in ("atom_mask", "aatype", "residue_index", "node_repr", "edge_repr"):
        assert torch.equal(got[key], plain[key]), key
    with pytest.raises(ValueError, match=f"holds {nf + L - 1} frames"):
        store.window_index(nf + L, training=False)


@pytest.mark.parametrize("nf,k,fix,L", [(2, 1, 0, 5), (3, 2, 3, 4)])
def test_a_trajectory_one_frame_short_names_its_archive(tmp_path, nf, k, fix, L):
    need = fix + (nf + L - 2) * k + 1
    _, row = _protein(tmp_path, need)
    EvaluationStore(frame_time=nf, frame_sample_step=k, fix_sample_start=fix, pin=False, horizons=L).protein(*row)
    _, short = _protein(tmp_path / "short", need - 1)
    with pytest.raises(ValueError, match=re.escape(short[0]) + f": {L} horizons after the evaluation window .* reach past"):
        EvaluationStore(frame_time=nf, frame_sample_step=k, fix_sample_start=fix, pin=False, horizons=L).protein(*short)


def test_horizons_must_be_a_count():
    for h in (-1, True, 1.0):
        with pytest.raises(ValueError, match="horizons must be an int >= 0"):
            EvaluationStore(frame_time=2, horizons=h)


@pytest.mark.parametrize("L", [1, 7, 10, 150, 200])
def test_returned_dict_and_printed_lines_equal_a_numpy_restatement(tmp_path, capsys, L):
    names = [("a", 17), ("b.x", 23), ("c", 40)]
    scores = np.random.default_rng(L).standard_normal((len(names), L, len(HORIZON_KEYS))) * 10.0
    scores[1, 0, 2] = np.nan                                     # an empty frame's MAE is NaN; its mean is NaN too
    d = _HostExtension(_conf(_csv(tmp_path / "test.csv", names)), scores).extend(L)
    printed = capsys.readouterr().out.splitlines()
    assert list(d) == ["name", *HORIZON_KEYS] and d["name"] == ["a", "b", "c"]
    horizons = [h for h in (1, 10, 100) if h < L] + [L]
    assert len(printed) == len(HORIZON_KEYS)
    for j, k in enumerate(HORIZON_KEYS):
        assert type(d[k]) is np.ndarray and d[k].dtype == np.float64 and d[k].shape == (len(names), L), k
        assert np.array_equal(d[k], scores[:, :, j], equal_nan=True), k
        label, *fields = printed[j].split()
        assert label == f"{k}:" and fields[0::2] == [f"h{h}" for h in horizons], printed[j]
        want = [sum(scores[i, h - 1, j] for i in range(len(names))) / len(names) for h in horizons]
        got = [float(v) for v in fields[1::2]]
        assert np.allclose(got, want, rtol=1e-15, atol=0, equal_nan=True), (k, got, want)


def test_extension_file_has_eval_extensions_keys_shapes_and_dtypes(tmp_path):
    """eval_extension (train_DFOLD_dynamics.py:997-1000) saves the concatenated fp32 predictions and the loader's aatype
    batch of one, [1, nf, N] int64."""
    L, nf, N = 6, 3, 11
    g = torch.Generator().manual_seed(0)
    rigid, atoms = torch.randn(L, N, 7, generator=g), torch.randn(L, N, 37, 3, generator=g)
    aatype = torch.randint(0, 20, (N,), generator=g).unsqueeze(0).expand(nf, -1)
    path = tmp_path / "p0" / "extension.npz"
    write_extension(str(path), rigid.numpy(), atoms.numpy(), aatype.numpy())
    with np.load(path) as f:
        got = dict(f)
    assert sorted(got) == ["aatype", "atom_traj", "rigid_traj"]
    assert got["atom_traj"].dtype == np.float32 and got["atom_traj"].shape == (L, N, 37, 3)
    assert got["rigid_traj"].dtype == np.float32 and got["rigid_traj"].shape == (L, N, 7)
    assert got["aatype"].dtype == np.int64 and got["aatype"].shape == (1, nf, N)
    assert np.array_equal(got["atom_traj"], atoms.numpy()) and np.array_equal(got["rigid_traj"], rigid.numpy())
    assert np.array_equal(got["aatype"][0], aatype.numpy())
