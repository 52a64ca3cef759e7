"""The host side of dynamicpdb_b200.evaluator against the reference evaluator's own loop.

tests/golden/evaluator.pt (oracle/make_evaluator_golden.py) holds what the unmodified ``Experiment.eval_fn`` returned and
printed over the unmodified test loader of a synthetic split, with seeded predictions injected for ``inference_fn``.
Here the Evaluator's loop runs with its device side replaced by the fixture's per-window rows and must give the same
dict and the same lines; the rows themselves are pinned to the fp64 oracle.  Configurations the evaluator refuses raise
before any device work (the network passed is None), and the evaluation store is checked against an ordinary one."""
import copy
import os
import re

import numpy as np
import pytest
import torch

from dynamicpdb_b200.evaluator import ROW_KEYS, Evaluator, eval_seeds, load_weights, split_rows
from dynamicpdb_b200.input_pipeline import EvaluationStore, TrajectoryStore
from oracle import metrics_oracle as MO
from oracle import synth_traj
from tests.test_cpu_metrics import SUM_TOL, angle_ratio, ratio

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "evaluator.pt")
_FIX = []


def fixture():
    if not _FIX:
        _FIX.append(torch.load(GOLDEN, weights_only=False))
    return _FIX[0]


def fixture_rows():
    """eval_fn's per-window rows [n, 5] (ROW_KEYS) out of its returned dict."""
    r = fixture()["result"]
    return np.stack([r["ave_rot"], r["ave_trans"], r["all_atom_mae"], np.concatenate(r["all_atom_mse"]), r["all_atom_rmsd"]],
                    axis=1)


def _csv(path, rows):
    with open(path, "w") as f:
        f.write("name,seq_len,atlas_npz,force_path,vel_path,embed_path,pdb_path\n")
        for name, n in rows:
            f.write(f"{name},{n},{name}.npz,{name}_F.pkl,{name}_V.pkl,{name}_emb.npz,{name}.pdb\n")
    return str(path)


def _conf(csv_path, **data):
    c = fixture()["case"]
    conf = {"eval": {"weights_path": "weights.pth", "eval_batch_size": 1},
            "experiment": {"noise_scale": c["noise_scale"]},
            "data": {"test_csv_path": csv_path, "filtering": {"max_len": c["max_len"]}, "frame_time": c["frame_time"],
                     "frame_sample_step": c["frame_sample_step"], "fix_sample_start": c["fix_sample_start"],
                     "num_t": c["num_t"], "min_t": c["min_t"], "is_extrapolation": False}}
    conf["data"].update(data)
    return conf


class _HostEvaluator(Evaluator):
    """The Evaluator with its device side replaced by given rows."""

    def __init__(self, conf, rows):
        self._configure(conf)
        self.fake = rows

    def _run(self):
        return torch.from_numpy(self.fake)


def _set(conf, path, value):
    d = conf
    *head, last = path.split(".")
    for k in head:
        d = d[k]
    if value is KeyError:
        del d[last]
    else:
        d[last] = value


@pytest.mark.parametrize("path,value", [
    ("eval.weights_path", KeyError), ("eval.weights_path", 3), ("eval.eval_batch_size", 0), ("eval.eval_batch_size", "1"),
    ("data.frame_time", 1), ("data.frame_sample_step", 0), ("data.fix_sample_start", -1), ("data.fix_sample_start", 2.0),
    ("data.num_t", 0), ("data.num_t", True), ("data.min_t", 1.5), ("data.min_t", KeyError), ("data.filtering.max_len", "48"),
    ("data.test_csv_path", KeyError), ("experiment.noise_scale", -0.1), ("experiment.noise_scale", KeyError)])
def test_malformed_config_raises_before_device_work(path, value, tmp_path):
    conf = copy.deepcopy(_conf(_csv(tmp_path / "test.csv", [("a", 17)])))
    _set(conf, path, value)
    with pytest.raises(ValueError, match=re.escape(path)):
        Evaluator(conf, None, None)


def test_refused_splits_raise_before_device_work(tmp_path):
    csv_path = _csv(tmp_path / "test.csv", [("a", 17), ("b", 23)])
    conf = _conf(csv_path)
    conf["eval"]["eval_batch_size"] = 2
    with pytest.raises(ValueError, match="eval_batch_size=2"):
        Evaluator(conf, None, None)
    with pytest.raises(ValueError, match="is_extrapolation"):
        Evaluator(_conf(csv_path, is_extrapolation=True), None, None)
    with pytest.raises(ValueError, match="no row with seq_len <= 10"):
        Evaluator(_conf(csv_path, filtering={"max_len": 10}), None, None)
    no_name = tmp_path / "no_name.csv"
    no_name.write_text("seq_len,atlas_npz,force_path,vel_path,embed_path\n17,a,b,c,d\n")
    with pytest.raises(ValueError, match=r"no column \['name'\]"):
        Evaluator(_conf(str(no_name)), None, None)
    # the default of an absent key: not an extrapolation, fix_sample_start None is 0
    conf = _conf(csv_path, fix_sample_start=None)
    del conf["data"]["is_extrapolation"]
    ev = _HostEvaluator(conf, None)
    assert ev.fix_start == 0 and ev.names == ["a", "b"]


def test_rows_in_csv_order_with_any_mix_of_lengths(tmp_path):
    """PdbDataset's test split: seq_len <= max_len in csv order, lengths mixed; names are name.split('.')[0]."""
    g = fixture()
    path = tmp_path / "test.csv"
    path.write_text(g["csv"])
    rows = split_rows(str(path), g["case"]["max_len"])
    assert [n for n, _ in rows] == g["result"]["name"] == [n.split(".")[0] for n in g["loader_names"]]
    kept = [ln.split(",") for ln in g["csv"].splitlines()[1:] if float(ln.split(",")[1]) <= g["case"]["max_len"]]
    assert len(kept) == len(g["proteins"]) - 1
    assert [r for _, r in rows] == [tuple(k[2:6]) for k in kept]
    ev = _HostEvaluator(_conf(str(path)), None)
    assert ev.rows == rows
    # the training csv's single-length check is the Trainer's alone
    assert len({int(k[1]) for k in kept}) == 3


def test_returned_dict_and_printed_lines_equal_eval_fn(tmp_path, capsys):
    g = fixture()
    path = tmp_path / "test.csv"
    path.write_text(g["csv"])
    d = _HostEvaluator(_conf(str(path)), fixture_rows()).evaluate()
    assert capsys.readouterr().out.splitlines() == g["stdout"]
    want = g["result"]
    assert list(d) == list(want)
    assert d["name"] == want["name"]
    for k in ("ave_rot", "ave_trans", "all_atom_mae", "all_atom_rmsd"):
        assert type(d[k]) is np.ndarray and d[k].dtype == want[k].dtype and d[k].shape == want[k].shape, k
        assert np.array_equal(d[k], want[k]), k
    assert type(d["all_atom_mse"]) is list and len(d["all_atom_mse"]) == len(want["all_atom_mse"])
    for a, b in zip(d["all_atom_mse"], want["all_atom_mse"]):
        assert type(a) is np.ndarray and a.dtype == b.dtype and a.shape == b.shape == (1,) and np.array_equal(a, b)
    # the quirk: one row is past the bound, so each mean divides the sum over all rows by one row fewer
    mask = want["ave_trans"] < 10000.0
    assert mask.sum() == len(mask) - 1
    assert float(g["stdout"][1].split()[1]) == want["ave_trans"].sum() / mask.sum()


def row_bounds(got_row, i):
    """max over ROW_KEYS of |got - eval_fn's row i| / bound, with test_cpu_metrics' bounds (fp64 sums 1e-12 (1 + |ref|),
    angles 1e-5 degrees) plus, for the rigid errors, the spread of eval_fn's fp32 arithmetic on the loader's fp32
    rigids_0 (its quaternions are normalised in fp32; the kernels and the oracle upcast them first)."""
    g = fixture()
    ref = fixture_rows()[i]
    out = {}
    for j, k in enumerate(ROW_KEYS):
        r = torch.from_numpy(ref[j:j + 1].copy())
        spread = torch.from_numpy(ref[j:j + 1] - g["gt64"][k][i:i + 1]) if k in g["gt64"] else None
        out[k] = angle_ratio(got_row[k], r, spread) if k == "ave_rot" else ratio(got_row[k], r, SUM_TOL, spread)
    return out


def test_fixture_rows_match_the_oracle():
    """eval_fn's rows against metrics_oracle.window_metrics on the same windows and injected predictions."""
    g = fixture()
    for i, (w, p) in enumerate(zip(g["windows"], g["predictions"])):
        got = MO.window_metrics(p["rigid_pred"], p["atom37_pred"], w["rigids_0"], w["atom37_pos"], w["atom37_mask"])
        worst = row_bounds(got, i)
        assert all(v <= 1.0 for v in worst.values()), (i, worst)
    assert float(np.abs(fixture_rows()[:, 0] - g["gt64"]["ave_rot"]).max()) > 1e-6      # the spread is not nothing


def _protein(tmp_path, N=17, T=12, seed=31, name="p"):
    return synth_traj.write_files(synth_traj.make_trajectory(T=T, N=N, seed=seed), str(tmp_path), name=name)


@pytest.mark.parametrize("k,fix", [(1, 0), (2, 3), (3, 2)])
def test_evaluation_store_holds_only_the_window(tmp_path, k, fix):
    """The entry holds frame_time frames, equal to the ordinary store's window; nothing is cached."""
    row = _protein(tmp_path)
    plain = TrajectoryStore(frame_time=3, frame_sample_step=k, fix_sample_start=fix, pin=False)
    ent = plain.protein(*row)
    sl = plain.window_index(ent["atom37"].shape[0], training=False)
    store = EvaluationStore(frame_time=3, frame_sample_step=k, fix_sample_start=fix, pin=False)
    got = store.protein(*row)
    assert not store._cache
    win = store.window_index(got["atom37"].shape[0], training=False)
    assert got["atom37"].shape[0] == got["force"].shape[0] == got["vel"].shape[0] == 3 and win == slice(0, 3, 1)
    for key in ("atom37", "force", "vel"):
        assert got[key].dtype == ent[key].dtype and torch.equal(got[key][win], ent[key][sl]), key
    for key in ("atom_mask", "aatype", "residue_index", "node_repr", "edge_repr"):
        assert torch.equal(got[key], ent[key]), key
    with pytest.raises(ValueError, match="evaluation windows only"):
        store.window_index(3, training=True)


def test_evaluation_store_names_the_row_of_a_short_trajectory(tmp_path):
    """The reference loader's errors, prefixed with the row's archive."""
    row = _protein(tmp_path, T=8)
    with pytest.raises(ValueError, match=re.escape(row[0]) + ": t cannot be greater than the number of samples"):
        EvaluationStore(frame_time=3, fix_sample_start=6, pin=False).protein(*row)
    with pytest.raises(ValueError, match=re.escape(row[0]) + ": the evaluation window .* reaches past"):
        EvaluationStore(frame_time=3, frame_sample_step=3, fix_sample_start=2, pin=False).protein(*row)


def test_seeds_are_two_streams_of_the_seed():
    a, b = eval_seeds(0)
    assert a != b and eval_seeds(0) == (a, b) and eval_seeds(1) != (a, b)
    assert all(0 <= s < 2 ** 64 for s in (a, b))


class _Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.a = torch.nn.Linear(3, 4)
        self.b = torch.nn.Linear(4, 2)


def test_weights_load_strictly_and_a_mismatch_leaves_them(tmp_path):
    """A module.-prefixed reference-style dict loads; unknown, missing or reshaped keys raise naming them and change
    nothing."""
    torch.manual_seed(0)
    src, dst = _Net(), _Net()
    path = str(tmp_path / "ref.pth")
    torch.save({"model": {"module." + k: v for k, v in src.state_dict().items()}, "conf": None}, path)
    load_weights(dst, path)
    assert all(torch.equal(a, b) for a, b in zip(src.state_dict().values(), dst.state_dict().values()))
    before = {k: v.clone() for k, v in _Net().state_dict().items()}
    for model, msg in [({**src.state_dict(), "c.weight": torch.zeros(1)}, r"unknown keys \[c.weight\]"),
                       ({k: v for k, v in src.state_dict().items() if k != "b.bias"}, r"missing keys \[b.bias\]"),
                       ({**src.state_dict(), "b.weight": torch.zeros(2, 5)}, r"'b.weight' has shape \(2, 5\)")]:
        net = _Net()
        net.load_state_dict(before)
        torch.save({"model": model}, path)
        with pytest.raises(ValueError, match=msg):
            load_weights(net, path)
        assert all(torch.equal(v, before[k]) for k, v in net.state_dict().items())
    torch.save({"state": {}}, path)
    with pytest.raises(ValueError, match="no 'model' state_dict"):
        load_weights(_Net(), path)
