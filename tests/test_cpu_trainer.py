"""The host side of dynamicpdb_b200.trainer against the reference trainer's own loop.

tests/golden/trainer_log.pt (oracle/make_trainer_golden.py) holds what the unmodified ``Experiment.start_training`` /
``train_epoch`` did over a stub loader of known indices and an ``update_fn`` returning seeded ``aux_data``: the indices
each rank received, the log lines and the checkpoints.  Here the Trainer's loop runs with its device side replaced by a
host fake that hands out the same ``aux_data`` step by step, and must reproduce all of it.  Configurations the trainer
does not train raise before any device work (the network passed is None)."""
import copy
import logging
import os
import re

import pytest
import torch
from torch.utils.data.distributed import DistributedSampler

from dynamicpdb_b200.trainer import LOGGED, Trainer, epoch_order

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "trainer_log.pt")
SPEED = re.compile(r", steps/sec=\d+\.\d{5}$")


def _csv(path, lengths):
    with open(path, "w") as f:
        f.write("name,seq_len,atlas_npz,force_path,vel_path,embed_path,pdb_path\n")
        for i, n in enumerate(lengths):
            f.write(f"p{i},{n},p{i}.npz,p{i}_F.pkl,p{i}_V.pkl,p{i}_emb.npz,p{i}.pdb\n")
    return str(path)


def _conf(csv_path, batch_size=1, num_epoch=2, log_freq=1, ckpt_freq=1, ckpt_dir=None, max_len=256):
    return {"experiment": {"batch_size": batch_size, "num_epoch": num_epoch, "log_freq": log_freq, "ckpt_freq": ckpt_freq,
                           "ckpt_dir": ckpt_dir, "learning_rate": 1e-4, "torsion_loss_weight": 1.0, "rot_loss_weight": 7.0,
                           "trans_loss_weight": 100.0, "rot_loss_t_threshold": 0.0, "separate_rot_loss": False},
            "data": {"csv_path": csv_path, "filtering": {"max_len": max_len}, "frame_time": 2, "frame_sample_step": 1,
                     "keep_first": 100000, "min_t": 0.01}}


class _HostTrainer(Trainer):
    """The Trainer's loop with the device side replaced: a step's windows are their dataset indices, and its aux_data
    comes from the fixture in order."""

    def __init__(self, conf, world_size, rank, aux, accumulate=1):
        self._configure(conf, world_size, rank, accumulate)
        self.aux, self.seen, self.saved = list(aux), [], []

    def _prefetch(self, steps):
        yield from steps

    def _update(self, slots):
        self.seen.append((self.trained_epochs, list(slots)))
        self.current = self.aux.pop(0)

    def _keep_logged(self):
        self.kept = [float(self.current[k]) for k in LOGGED]

    def _read_logged(self):
        return self.kept

    def _save(self, path):
        self.saved.append((os.path.basename(path), self.trained_epochs, self.trained_steps))


def _cases():
    return torch.load(GOLDEN)["cases"]


@pytest.mark.parametrize("world", [1, 2, 3, 4])
@pytest.mark.parametrize("n", [1, 4, 5, 7, 10])
def test_order_is_the_distributed_samplers(world, n, tmp_path):
    """Every rank's slots at every step over three epochs: rank r of `world` ranks, and slot r of one rank accumulating
    `world` windows, both get DistributedSampler(num_replicas=world, rank=r) after set_epoch(epoch), padding included."""
    conf = _conf(_csv(tmp_path / "train.csv", [12] * n), batch_size=world)
    acc = _HostTrainer(conf, 1, 0, [], accumulate=world)
    for epoch in range(3):
        want = []
        for r in range(world):
            s = DistributedSampler(list(range(n)), num_replicas=world, rank=r)
            s.set_epoch(epoch)
            want.append(list(s))
        assert epoch_order(n, world, epoch) == want
        assert len({len(w) for w in want}) == 1 and len(want[0]) * world >= n
        for r in range(world):
            assert [step[0] for step in _HostTrainer(conf, world, r, []).windows(epoch)] == want[r]
        assert acc.windows(epoch) == [list(step) for step in zip(*want)]


@pytest.mark.parametrize("name", list(_cases()))
def test_loop_matches_reference_train_epoch_golden(name, tmp_path, caplog):
    """Indices per update, log lines (all but the measured steps/sec), checkpoint names, epochs and steps, and the final
    counters of Experiment.start_training, rank by rank; the same run with accumulate=world on one rank logs and saves as
    the reference's rank 0."""
    c = _cases()[name]
    conf = _conf(_csv(tmp_path / "train.csv", [64] * c["n"]), batch_size=c["world"], num_epoch=c["num_epoch"],
                 log_freq=c["log_freq"], ckpt_freq=c["ckpt_freq"], ckpt_dir=str(tmp_path / "ckpt"))
    runs = [(r, _HostTrainer(conf, c["world"], r, ref["aux"])) for r, ref in enumerate(c["ranks"])]
    # one rank accumulating the whole world: its slot 0 is the reference's rank 0, and only rank 0's values are logged
    acc = _HostTrainer(conf, 1, 0, c["ranks"][0]["aux"], accumulate=c["world"])
    for r, tr in runs + [(0, acc)]:
        ref = c["ranks"][r]
        tr.trained_epochs, tr.trained_steps = c["trained_epochs"], c["trained_steps"]
        caplog.clear()
        with caplog.at_level(logging.INFO, logger="dynamicpdb_b200.trainer"):
            tr.train()
        got = [m for m in caplog.messages if m.startswith("Epoch[")]
        want = [m for m in ref["log"] if m.startswith("Epoch[")]
        assert len(got) == len(want) and want, (name, r)
        for g, w in zip(got, want):
            assert SPEED.search(g) and SPEED.search(w), (g, w)
            assert SPEED.sub("", g) == SPEED.sub("", w), (name, r, g, w)
        assert [(e, slots[0]) for e, slots in tr.seen] == ref["updates"], (name, r)
        assert (tr.trained_epochs, tr.trained_steps) == (ref["trained_epochs"], ref["trained_steps"])
        want_ckpt = [(os.path.basename(k["path"]), k["epoch"], k["step"]) for k in ref["ckpts"]] if r == 0 else []
        assert tr.saved == want_ckpt, (name, r)             # the reference writes from every rank, the trainer from rank 0
        assert not tr.aux
    for step, (e, slots) in enumerate(acc.seen):
        assert slots == [ref["updates"][step][1] for ref in c["ranks"]] and e == c["ranks"][0]["updates"][step][0]


def test_logged_values_are_those_of_the_first_step_after_the_previous_line(tmp_path, caplog):
    """The quirk the fixture pins, on its own: with log_freq 3 the line at step 3 shows step 2's values (step 1 had its
    own line), the one at step 6 step 4's, and an epoch boundary drops the steps not yet logged."""
    conf = _conf(_csv(tmp_path / "train.csv", [64] * 4), num_epoch=2, log_freq=3)
    aux = [{k: float(10 * s + i) for i, k in enumerate(LOGGED)} for s in range(1, 9)]
    tr = _HostTrainer(conf, 1, 0, aux)
    with caplog.at_level(logging.INFO, logger="dynamicpdb_b200.trainer"):
        tr.train()
    shown = [int(float(re.search(r"total_loss=([\d.]+)", m).group(1))) // 10 for m in caplog.messages]
    assert shown == [1, 2, 5], caplog.messages          # steps 1, 3 (epoch 0) and 6 (epoch 1: from its first step, 5)


def test_mixed_lengths_raise_before_device_work(tmp_path):
    conf = _conf(_csv(tmp_path / "train.csv", [64, 64, 80, 300, 96]))
    with pytest.raises(ValueError, match=r"3 residue counts \(64, 80, 96\)"):
        Trainer(conf, None, None)
    # rows above filtering.max_len are dropped first, as PdbDataset._init_metadata drops them
    tr = _HostTrainer(_conf(_csv(tmp_path / "one.csv", [64, 300, 64]), max_len=256), 1, 0, [])
    assert tr.num_res == 64 and len(tr.rows) == 2 and tr.rows[1] == ("p2.npz", "p2_F.pkl", "p2_V.pkl", "p2_emb.npz")
    with pytest.raises(ValueError, match="no row with seq_len <= 50"):
        Trainer(_conf(_csv(tmp_path / "short.csv", [64]), max_len=50), None, None)


@pytest.mark.parametrize("batch_size,world,accumulate", [(2, 1, 1), (8, 2, 2), (5, 2, 1), (1, 2, 1), (2, 1, 4)])
def test_a_per_rank_batch_other_than_one_window_raises(batch_size, world, accumulate, tmp_path):
    conf = _conf(_csv(tmp_path / "train.csv", [64] * 4), batch_size=batch_size)
    with pytest.raises(ValueError, match="one window per rank"):
        Trainer(conf, None, None, world_size=world, accumulate=accumulate)


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
    ("experiment.log_freq", 0), ("experiment.log_freq", 2.5), ("experiment.ckpt_freq", 0), ("experiment.num_epoch", -1),
    ("experiment.num_epoch", True), ("experiment.batch_size", "1"), ("experiment.learning_rate", -1e-4),
    ("experiment.learning_rate", KeyError), ("experiment.rot_loss_weight", KeyError), ("experiment.ckpt_dir", 3),
    ("data.frame_time", 0), ("data.frame_sample_step", None), ("data.keep_first", 0), ("data.min_t", 1.5),
    ("data.filtering.max_len", "256"), ("data.csv_path", KeyError)])
def test_malformed_config_raises_before_device_work(path, value, tmp_path):
    conf = copy.deepcopy(_conf(_csv(tmp_path / "train.csv", [64] * 3)))
    _set(conf, path, value)
    with pytest.raises(ValueError, match=re.escape(path)):
        Trainer(conf, None, None)


@pytest.mark.parametrize("kw", [dict(world_size=0), dict(rank=2, world_size=2), dict(rank=-1), dict(accumulate=0),
                                dict(accumulate=1.0)])
def test_malformed_world_raises(kw, tmp_path):
    with pytest.raises(ValueError):
        Trainer(_conf(_csv(tmp_path / "train.csv", [64] * 3)), None, None, **kw)
