"""The reference trainer's epoch loop (train_DFOLD_dynamics.py ``start_training`` / ``train_epoch`` / ``update_fn``,
:591-763) on the captured training step.

``Trainer`` reads the training csv as ``PdbDataset._init_metadata`` does, orders it per epoch with the reference's
``DistributedSampler``, builds the noised windows on the device (``input_pipeline.WindowPrefetcher``) and trains each
optimizer step with one ``train_step.TrainStep`` replay on ``loss.score_network_loss``, the objective of
``Experiment.loss_fn``.  Its counters, log line, checkpoint cadence and file names are the reference's, so a run can be
followed and resumed as one of the reference trainer.  Nothing is read back to the host per step: the step's
``aux_data`` stays on the device and is read once per log line.

Scope: proteins of one residue count (the released recipe trains on a split in time of the same trajectories), one
window per rank and optimizer step.  Not reproduced: evaluation during training (the reference runs it under
``if False``), tensorboard / wandb, and the random streams of forked loader workers (see ``Trainer``).
"""
import csv
import logging
import numbers
import os
import time
import types
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch.utils.data.distributed import DistributedSampler

from . import checkpoint as _ckpt
from .input_pipeline import TrajectoryStore, WindowPrefetcher
from .loss import AUX_KEYS, aux_conf, score_network_loss
from .train_step import TrainStep, check_ema_decay

ROW_FIELDS = ("atlas_npz", "force_path", "vel_path", "embed_path")
LOGGED = ("total_loss", "rot_loss", "trans_loss", "torsion_loss")     # score_network_loss's aux_data keys without 'batch'
# with aux_losses=True, in the reference's aux_data order (train_DFOLD_dynamics.py:1384-1390)
LOGGED_AUX = ("total_loss", "rot_loss", "trans_loss", "bb_atom_loss", "dist_mat_loss", "torsion_loss")

_log = logging.getLogger(__name__)


def _get(conf, path: str, default=KeyError):
    """``conf.a.b`` or ``conf['a']['b']`` (a namespace, a dict or an OmegaConf config)."""
    v = conf
    for k in path.split("."):
        if isinstance(v, dict) and k in v:
            v = v[k]
        elif not isinstance(v, dict) and hasattr(v, k):
            v = getattr(v, k)
        elif default is KeyError:
            raise ValueError(f"config has no '{path}'")
        else:
            return default
    return v


def _int(conf, path: str, low: int, default=KeyError) -> int:
    v = _get(conf, path, default)
    if isinstance(v, bool) or not isinstance(v, numbers.Integral) or v < low:
        raise ValueError(f"{path} must be an integer >= {low}, got {v!r}")
    return int(v)


def kept_rows(csv_path: str, max_len, columns: Sequence[str] = ("seq_len",) + ROW_FIELDS) -> List[Dict[str, str]]:
    """The rows of a split's csv that ``PdbDataset._init_metadata`` keeps (``seq_len <= filtering.max_len``), in csv
    order, as dicts.  Raises ValueError when one of ``columns`` is absent or when no row is left."""
    with open(csv_path, newline="") as f:
        reader = csv.DictReader(f)
        missing = [k for k in columns if k not in (reader.fieldnames or ())]
        if missing:
            raise ValueError(f"{csv_path}: no column {missing}")
        kept = [r for r in reader if float(r["seq_len"]) <= max_len]
    if not kept:
        raise ValueError(f"{csv_path}: no row with seq_len <= {max_len}")
    return kept


def read_rows(csv_path: str, max_len) -> Tuple[List[Tuple[str, str, str, str]], int]:
    """The rows of the training csv that ``PdbDataset._init_metadata`` keeps (``seq_len <= filtering.max_len``), as
    ``TrajectoryStore.protein`` arguments, and their residue count.  Raises ValueError when none is left or when they
    have more than one residue count: one captured step trains one shape."""
    kept = kept_rows(csv_path, max_len)
    lengths = sorted({float(r["seq_len"]) for r in kept})
    if len(lengths) > 1:
        raise ValueError(f"{csv_path}: the rows with seq_len <= {max_len} have {len(lengths)} residue counts "
                         f"({', '.join(f'{n:g}' for n in lengths)}); the trainer trains proteins of one length")
    return [tuple(r[k] for k in ROW_FIELDS) for r in kept], int(lengths[0])


def epoch_order(n: int, world: int, epoch: int) -> List[List[int]]:
    """The dataset indices each of `world` ranks trains on in `epoch`, in order: ``DistributedSampler(num_replicas=world,
    rank=r)`` with its defaults (shuffle, seed 0, padded to a multiple of world, nothing dropped) after
    ``set_epoch(epoch)``, as the reference's loader draws them (train_DFOLD_dynamics.py:548, :645)."""
    order = []
    for r in range(world):
        s = DistributedSampler(range(n), num_replicas=world, rank=r)
        s.set_epoch(epoch)
        order.append(list(s))
    return order


class Trainer:
    """``Experiment.start_training`` on the captured step, for a network of the reference config's shapes.

    ``conf`` holds the reference's keys (a namespace, dict or OmegaConf config): ``experiment.batch_size``, ``num_epoch``,
    ``log_freq``, ``ckpt_freq``, ``ckpt_dir`` (None: no checkpoints), ``learning_rate`` and the loss weights
    ``torsion_loss_weight``, ``rot_loss_weight``, ``trans_loss_weight``, ``rot_loss_t_threshold``, ``separate_rot_loss``;
    ``data.csv_path``, ``filtering.max_len``, ``frame_time``, ``frame_sample_step``, ``keep_first``, ``min_t``; and
    ``diffuser.diffuse_rot`` if present (default True).  Everything is checked, and the csv read, before any device work.

    Rank ``rank`` of ``world_size`` trains one window per optimizer step, as the reference's loader with ``batch_size //
    world_size == 1`` (:551); any other batch size raises.  ``accumulate=k`` stands in for ``world_size * k`` ranks:
    slot s of rank r trains the window rank ``r * k + s`` of that world would, and the step averages the gradient over all
    of them (``batch_size // (world_size * k)`` must then be 1).  Slot 0 of each rank is what that rank logs.

    Random streams: the constructor seeds ``np.random`` and ``torch`` with the rank, as the reference does (:416-424).
    Window starts are drawn from numpy's global stream and t and the noise from the device's default generator, in window
    order.  That is the reference's stream with ``num_loader_workers=0``; its forked loader workers each draw from a copy of
    it, which is not reproduced, and neither is the per-rank stream of the ranks ``accumulate`` stands in for.

    ``graph=False`` runs eager steps (a gloo process group cannot be captured); ``max_grad_norm`` and ``lr_schedule`` are
    ``TrainStep``'s.

    ``aux_losses=True`` trains on the objective with the backbone-atom and pair-distance losses added
    (``score_network_loss(aux_losses=True)``); ``experiment.bb_atom_loss_weight``, ``bb_atom_loss_t_filter``,
    ``dist_mat_loss_weight``, ``dist_mat_loss_t_filter`` and ``aux_loss_weight`` must then be numbers, and the log line
    carries ``bb_atom_loss`` and ``dist_mat_loss`` too, in the reference's order.

    ``batched=True`` trains each step's ``accumulate`` windows through one batched forward and backward
    (``TrainStep(batched=True)``): the same windows in the same order, the same log line and checkpoints as
    ``accumulate`` alone, with the gradient summed in another fp32 order.

    ``ema_decay=d`` keeps OpenFold's moving average of the weights (``TrainStep(ema_decay=d)``); the checkpoints then
    carry it as ``ema`` and ``resume`` restores it."""

    def __init__(self, conf, net: torch.nn.Module, diffuser, *, world_size: int = 1, rank: int = 0, accumulate: int = 1,
                 graph: bool = True, warmup: int = 3, max_grad_norm: Optional[float] = None, lr_schedule=None,
                 aux_losses: bool = False, batched: bool = False, ema_decay: Optional[float] = None):
        if not isinstance(batched, bool):
            raise ValueError(f"batched must be True or False, got {batched!r}")
        check_ema_decay(ema_decay)
        self._configure(conf, world_size, rank, accumulate, aux_losses=aux_losses)
        self._build(net, diffuser, graph=graph, warmup=warmup, max_grad_norm=max_grad_norm, lr_schedule=lr_schedule,
                    batched=batched, ema_decay=ema_decay)
        np.random.seed(rank)
        torch.manual_seed(rank)

    def _configure(self, conf, world_size: int, rank: int, accumulate: int, aux_losses: bool = False):
        """Everything that needs no device: the config checked, the csv read."""
        self.conf = conf
        for name, v, low in (("world_size", world_size, 1), ("accumulate", accumulate, 1), ("rank", rank, 0)):
            if isinstance(v, bool) or not isinstance(v, numbers.Integral) or v < low:
                raise ValueError(f"{name} must be an integer >= {low}, got {v!r}")
        if rank >= world_size:
            raise ValueError(f"rank {rank} out of range for world_size {world_size}")
        self.world, self.rank, self.accumulate = int(world_size), int(rank), int(accumulate)
        self.ranks = self.world * self.accumulate                   # the world of the reference run this one trains as
        batch_size = _int(conf, "experiment.batch_size", 1)
        if batch_size // self.ranks != 1:
            raise ValueError(f"experiment.batch_size={batch_size} gives {batch_size // self.ranks} windows per rank over "
                             f"{self.ranks} ranks (world_size {self.world} x accumulate {self.accumulate}); the trainer "
                             "trains one window per rank and step, not the reference's flattened batch of several")
        self.num_epoch = _int(conf, "experiment.num_epoch", 0)
        self.log_freq = _int(conf, "experiment.log_freq", 1)
        self.ckpt_freq = _int(conf, "experiment.ckpt_freq", 1)
        self.ckpt_dir = _get(conf, "experiment.ckpt_dir", None)
        if self.ckpt_dir is not None and not isinstance(self.ckpt_dir, (str, os.PathLike)):
            raise ValueError(f"experiment.ckpt_dir must be a path or None, got {self.ckpt_dir!r}")
        self.lr = _get(conf, "experiment.learning_rate")
        if isinstance(self.lr, bool) or not isinstance(self.lr, numbers.Real) or not self.lr >= 0:
            raise ValueError(f"experiment.learning_rate must be a non-negative number, got {self.lr!r}")
        self.exp_conf = types.SimpleNamespace(**{k: _get(conf, "experiment." + k) for k in (
            "torsion_loss_weight", "rot_loss_weight", "trans_loss_weight", "rot_loss_t_threshold", "separate_rot_loss")})
        self.aux_losses = bool(aux_losses)
        self.logged_keys = LOGGED_AUX if self.aux_losses else LOGGED
        if self.aux_losses:
            for k in AUX_KEYS:
                setattr(self.exp_conf, k, _get(conf, "experiment." + k))
            aux_conf(self.exp_conf)
        self.diffuse_rot = bool(_get(conf, "diffuser.diffuse_rot", True))
        self.frame_time = _int(conf, "data.frame_time", 1)
        self.frame_step = _int(conf, "data.frame_sample_step", 1)
        keep_first = _get(conf, "data.keep_first", None)
        self.keep_first = None if keep_first is None else _int(conf, "data.keep_first", 1)
        self.min_t = _get(conf, "data.min_t")
        if isinstance(self.min_t, bool) or not isinstance(self.min_t, numbers.Real) or not 0.0 <= self.min_t <= 1.0:
            raise ValueError(f"data.min_t must be a number in [0, 1], got {self.min_t!r}")
        max_len = _get(conf, "data.filtering.max_len")
        if isinstance(max_len, bool) or not isinstance(max_len, numbers.Real):
            raise ValueError(f"data.filtering.max_len must be a number, got {max_len!r}")
        self.rows, self.num_res = read_rows(_get(conf, "data.csv_path"), max_len)
        self.trained_epochs = 0
        self.trained_steps = 0

    def _build(self, net, diffuser, **step_kw):
        self.net, self.diffuser = net, diffuser
        self.device = next(net.parameters()).device
        self.store = TrajectoryStore(self.frame_time, self.frame_step, keep_first=self.keep_first)
        # the first window of the first epoch shapes the static input slots; the step overwrites them before it trains
        example, = list(WindowPrefetcher(self.store, self.rows[:1], self.device, diffuser=diffuser, min_t=self.min_t))
        self.step = TrainStep(net, self._loss, example, lr=float(self.lr), world_size=self.world, accumulate=self.accumulate,
                              loss_reads_window=True, **step_kw)
        self.logged = torch.zeros(len(self.logged_keys), dtype=torch.float64, device=self.device)

    def _loss(self, out, window):
        return score_network_loss(out, window, self.exp_conf, self.diffuse_rot, aux_losses=self.aux_losses)

    def windows(self, epoch: int) -> List[List[int]]:
        """The dataset indices of this rank's slots at every step of `epoch`: ``[step][slot]``."""
        order = epoch_order(len(self.rows), self.ranks, epoch)
        mine = order[self.rank * self.accumulate:(self.rank + 1) * self.accumulate]
        return [list(step) for step in zip(*mine)]

    # the device side of one step, replaced by a host fake in the loop's CPU test
    def _update(self, slots: Sequence[Dict[str, torch.Tensor]]):
        for s, w in enumerate(slots):
            self.step.load(w, slot=s)
        self.step()

    def _keep_logged(self):
        """The values this step logs: one device-to-device copy of TrainStep.aux, read at the next log line."""
        self.logged.copy_(torch.stack([self.step.aux[k].to(torch.float64) for k in self.logged_keys]))

    def _read_logged(self) -> List[float]:
        return self.logged.tolist()

    def _save(self, path: str):
        os.makedirs(self.ckpt_dir, exist_ok=True)
        _log.info(f"Serializing experiment state to {path}")
        _ckpt.save_checkpoint(path, self.step, self.conf, self.trained_epochs, self.trained_steps)

    def _prefetch(self, steps: List[List[int]]):
        """This epoch's windows, grouped per step."""
        rows = [self.rows[i] for step in steps for i in step]
        it = iter(WindowPrefetcher(self.store, rows, self.device, diffuser=self.diffuser, min_t=self.min_t))
        for _ in steps:
            yield [next(it) for _ in range(self.accumulate)]

    def train(self):
        """``start_training``: the epochs ``trained_epochs ... num_epoch - 1``."""
        for epoch in range(self.trained_epochs, self.num_epoch):
            self.train_epoch(epoch)

    def train_epoch(self, epoch: int):
        """``train_epoch`` of the reference: one optimizer step per entry of this rank's sampler; the log line every
        ``log_freq`` steps with the values of the first step after the previous line (the reference's
        ``tree.map_structure(np.mean, ...)`` averages each step on its own and ``v[0]`` picks the first); at the end a
        checkpoint ``step_{trained_steps}.pth`` from rank 0 when ``trained_epochs`` is a non-zero multiple of
        ``ckpt_freq``."""
        self.trained_epochs = epoch
        steps = self.windows(epoch)
        keep = True                    # the reference's log_lossses is empty: this step's values are the next line's
        log_time = time.time()
        for slots in self._prefetch(steps):
            self._update(slots)
            if keep:
                self._keep_logged()
                keep = False
            self.trained_steps += 1
            if self.trained_steps == 1 or self.trained_steps % self.log_freq == 0:
                values = self._read_logged()
                elapsed = time.time() - log_time
                log_time = time.time()
                losses = " ".join(f"{k}={v:.4f}" for k, v in zip(self.logged_keys, values))
                _log.info(f"Epoch[{self.trained_epochs}/{self.num_epoch}] trained_steps: [{self.trained_steps}]: "
                          f"{losses}, steps/sec={self.log_freq / elapsed:.5f}")
                keep = True
        if (self.ckpt_dir is not None and self.trained_epochs != 0 and self.trained_epochs % self.ckpt_freq == 0
                and self.rank == 0):
            self._save(os.path.join(self.ckpt_dir, f"step_{self.trained_steps}.pth"))

    def resume(self, path: str):
        """Loads a checkpoint of this trainer or of the reference trainer (``checkpoint.load_checkpoint``) and continues
        after it: the checkpoint is written at the end of epoch ``epoch``, so training resumes with epoch ``epoch + 1``
        and step ``step``.  Every rank loads the same file."""
        epoch, step = _ckpt.load_checkpoint(path, self.step)
        self.trained_epochs, self.trained_steps = int(epoch) + 1, int(step)
