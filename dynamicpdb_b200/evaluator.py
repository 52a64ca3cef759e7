"""The reference evaluator (eval_DFOLD_dynamics.py ``Evaluator.start_evaluation`` -> train_DFOLD_dynamics.py
``Experiment.eval_fn``, :765-928) on the device.

``Evaluator`` reads the test csv as ``PdbDataset._init_metadata`` does in test mode (every row with ``seq_len <=
filtering.max_len``, in csv order, of any mix of lengths), loads a checkpoint into the caller's network as
``Evaluator._load_ckpt`` does, and scores one window per protein: the window is built on a side stream
(``input_pipeline.WindowPrefetcher`` over an ``EvaluationStore``, ``rigids_t`` from ``sample_ref``), sampled with the
memoised reverse diffusion (``inference.DeviceReverseDiffusion.sample``: one trunk pass and ``num_t`` pairs of small
kernels) and scored by the fp64 metric kernels (``metrics.window_metrics``).  The rows stay on the device and are read
back once, after the last protein; the returned dict and the four printed lines are then eval_fn's, built with numpy in
its order.

The sampler runs eagerly rather than from one CUDA graph per residue count (``sample_graphed``): a test split has about
one window per length, so each captured graph would be replayed once, after a warm-up and a capture that cost more than
the eager run, and its private memory pool would stay allocated for the rest of the process.

``Evaluator.extend`` is the evaluator's other driver, ``Experiment.eval_extension`` (train_DFOLD_dynamics.py:931-1000),
made to work over a split: each protein's evaluation window is rolled forward frame by frame
(``rollout.TrajectoryRollout``, eagerly for the reasons above) and every rollout frame is scored with eval_fn's metrics
against the MD frame it predicts, which the same ``EvaluationStore`` decode supplies (``horizons``): error against
horizon.  Rollout frame j predicts MD frame ``fix_sample_start + (frame_time - 1 + j) * frame_sample_step``, because the
network replaces the window's last frame by the one before it (ipa_pytorch_dynamic.py:819) and the rollout appends each
prediction as the new last frame (:996).

Not reproduced: the directories, ``eval_conf.yaml``, plots and PDB files eval_fn writes, and the reference's random
streams (see ``Evaluator``).
"""
import numbers
import os
from typing import Dict, List, Tuple

import numpy as np
import torch

from . import checkpoint as _ckpt
from .inference import DeviceReverseDiffusion
from .input_pipeline import EvaluationStore, WindowPrefetcher
from .metrics import HORIZON_KEYS, eval_sampler_inputs, horizon_metrics, window_metrics
from .rollout import TrajectoryRollout
from .trainer import ROW_FIELDS, _get, _int, kept_rows

ROW_KEYS = ("ave_rot", "ave_trans", "all_atom_mae", "all_atom_mse", "all_atom_rmsd")   # one device row per window
PRINTED = (("ave_rot", "ave_rot"), ("ave_trans", "ave_trans"), ("ave_atom_mae", "all_atom_mae"),
           ("ave_atom_rmsd", "all_atom_rmsd"))                                        # eval_fn's summary lines (:925-928)
MASK_BOUND = 10000.0                                                                  # eval_fn's ``ave_trans < 10000``
PRINTED_HORIZONS = (1, 10, 100)                        # with the rollout's length: the horizons ``extend`` prints


def split_rows(csv_path: str, max_len) -> List[Tuple[str, Tuple[str, str, str, str]]]:
    """The rows ``PdbDataset(is_training=False, is_testing=True)`` iterates: ``seq_len <= max_len``, in csv order, as
    (name, ``TrajectoryStore.protein`` arguments).  The name is eval_fn's ``save_name``, ``name.split('.')[0]`` (:873)."""
    kept = kept_rows(csv_path, max_len, ("seq_len", "name") + ROW_FIELDS)
    return [(r["name"].split(".")[0], tuple(r[k] for k in ROW_FIELDS)) for r in kept]


def eval_seeds(seed: int) -> Tuple[int, int]:
    """The seeds of the evaluator's two CUDA generators: (windows' ``sample_ref``, reverse steps), two independent
    streams spawned from ``seed``."""
    return tuple(int(s.generate_state(1, np.uint64)[0]) for s in np.random.SeedSequence(seed).spawn(2))


def load_weights(net: torch.nn.Module, path: str, ema: bool = False) -> None:
    """Loads ``path``'s ``model`` state_dict into ``net`` strictly, ``module.`` prefixes stripped, as the reference
    evaluator's ``_load_ckpt`` does (eval_DFOLD_dynamics.py:131-136): a checkpoint of ``checkpoint.save_checkpoint`` or of
    the reference trainer.  ``ema=True`` loads the moving average of the weights instead, ``ema['params']`` of a checkpoint
    written with ``TrainStep(ema_decay=...)`` (OpenFold's layout), and raises ValueError naming the file when it has none.
    Every key and shape is checked first (``checkpoint.check_model`` / ``check_ema``), so a mismatch raises ValueError and
    leaves ``net`` as it was.  Checkpoints are trusted input: ``conf`` is an arbitrary pickled object, so the file is read
    with ``weights_only=False`` as the reference does; never load one from an untrusted source."""
    ckpt = torch.load(path, map_location="cpu", weights_only=False)
    shapes = {k: v.shape for k, v in net.state_dict().items()}
    if ema:
        model = _ckpt.check_ema(ckpt, shapes)
        if model is None:
            raise ValueError(f"{path}: the checkpoint has no 'ema' (moving average of the weights) to evaluate")
    else:
        model = _ckpt.check_model(ckpt, shapes)
    net.load_state_dict(model, strict=True)


def write_extension(path: str, rigid_traj, atom_traj, aatype) -> None:
    """eval_extension's ``extension.npz`` (:997-1000) from host arrays: ``atom_traj`` [L, N, 37, 3] and ``rigid_traj``
    [L, N, 7] float32, and ``aatype``, the window's [nf, N], as the loader's batch of one, [1, nf, N] int64.  The file's
    directory is made if it does not exist."""
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    np.savez_compressed(path, atom_traj=np.asarray(atom_traj, dtype=np.float32),
                        rigid_traj=np.asarray(rigid_traj, dtype=np.float32), aatype=np.asarray(aatype, dtype=np.int64)[None])


class Evaluator:
    """``Evaluator.start_evaluation`` / ``Experiment.eval_fn`` for a network of the reference config's shapes:
    ``Evaluator(conf, net, diffuser, seed=0).evaluate()``.

    ``conf`` holds the reference's keys (a namespace, dict or OmegaConf config): ``eval.weights_path`` and
    ``eval.eval_batch_size`` (1: eval_fn reads only item 0 of a batch); ``data.test_csv_path``, ``filtering.max_len``,
    ``frame_time`` (>= 2: the rotation error's baseline is frame -2), ``frame_sample_step``, ``fix_sample_start`` (None
    is 0), ``num_t``, ``min_t`` and ``is_extrapolation`` (True raises: the reference names a dataset class it does not
    define); ``experiment.noise_scale``.  Everything is checked, and the csv read, before the checkpoint is read and before
    any device work.  ``net`` is built by the caller (from the checkpoint's ``conf.model`` where it has one) with a
    ``score_epilogue.SE3ScoreDiffuser``; ``diffuser`` is the one the windows' ``sample_ref`` draws from.  The weights are
    loaded into ``net`` in the constructor and ``net`` is put in eval mode; ``ema=True`` loads the checkpoint's moving
    average of the weights (``load_weights``), so ``evaluate`` and ``extend`` run on it.

    Random streams: two CUDA generators seeded from ``seed`` (``eval_seeds``), one for the windows' ``sample_ref`` (drawn by
    the prefetcher's worker thread), one for the reverse steps (drawn by the calling thread), so a run is reproducible bit
    for bit whatever the threads' timing.  The global generators are not touched.  The reference draws both from numpy's
    global stream on the host; those numbers are not reproduced."""

    def __init__(self, conf, net: torch.nn.Module, diffuser, *, seed: int = 0, depth: int = 2, ema: bool = False):
        if not isinstance(ema, bool):
            raise ValueError(f"ema must be True or False, got {ema!r}")
        self._configure(conf)
        load_weights(net, self.weights_path, ema=ema)
        net.eval()
        self.net, self.diffuser, self.seed, self.depth = net, diffuser, int(seed), depth
        self.device = next(net.parameters()).device
        self.sampler = DeviceReverseDiffusion(net)
        self.roller = TrajectoryRollout(net)

    def _configure(self, conf):
        """Everything that needs no device: the config checked, the csv read."""
        self.conf = conf
        self.weights_path = _get(conf, "eval.weights_path")
        if not isinstance(self.weights_path, (str, bytes)) and not hasattr(self.weights_path, "__fspath__"):
            raise ValueError(f"eval.weights_path must be a path, got {self.weights_path!r}")
        batch_size = _int(conf, "eval.eval_batch_size", 1)
        if batch_size != 1:
            raise ValueError(f"eval.eval_batch_size={batch_size}: eval_fn scores item 0 of each batch only; the evaluator "
                             "scores one window per protein (eval.eval_batch_size=1)")
        if bool(_get(conf, "data.is_extrapolation", False)):
            raise ValueError("data.is_extrapolation=True: the reference evaluator's PdbDatasetExtrapolation is not "
                             "defined; only the test windows of PdbDataset are evaluated")
        self.frame_time = _int(conf, "data.frame_time", 2)
        self.frame_step = _int(conf, "data.frame_sample_step", 1)
        fix = _get(conf, "data.fix_sample_start", None)
        self.fix_start = 0 if fix is None else _int(conf, "data.fix_sample_start", 0)
        self.num_t = _int(conf, "data.num_t", 1)
        self.min_t = _get(conf, "data.min_t")
        if isinstance(self.min_t, bool) or not isinstance(self.min_t, numbers.Real) or not 0.0 <= self.min_t <= 1.0:
            raise ValueError(f"data.min_t must be a number in [0, 1], got {self.min_t!r}")
        self.noise_scale = _get(conf, "experiment.noise_scale")
        if isinstance(self.noise_scale, bool) or not isinstance(self.noise_scale, numbers.Real) or not self.noise_scale >= 0:
            raise ValueError(f"experiment.noise_scale must be a non-negative number, got {self.noise_scale!r}")
        max_len = _get(conf, "data.filtering.max_len")
        if isinstance(max_len, bool) or not isinstance(max_len, numbers.Real):
            raise ValueError(f"data.filtering.max_len must be a number, got {max_len!r}")
        test_csv = _get(conf, "data.test_csv_path")
        self.rows = split_rows(test_csv, max_len)
        self.names = [name for name, _ in self.rows]

    def generators(self) -> Tuple[torch.Generator, torch.Generator]:
        """Fresh (windows, reverse steps) generators on the network's device, seeded from ``seed``."""
        return tuple(torch.Generator(self.device).manual_seed(s) for s in eval_seeds(self.seed))

    def _prefetcher(self, generator: torch.Generator, horizons: int = 0):
        store = EvaluationStore(self.frame_time, self.frame_step, fix_sample_start=self.fix_start, horizons=horizons)
        return WindowPrefetcher(store, [row for _, row in self.rows], self.device, training=False, depth=self.depth,
                                diffuser=self.diffuser, min_t=self.min_t, generator=generator, targets=True)

    # the device sampler, replaced by injected predictions in the fixture's GPU test
    def _sample(self, index: int, window: Dict[str, torch.Tensor], generator: torch.Generator):
        """(``rigid_traj[0]``, ``prot_traj[0]``) of eval_fn's ``inference_fn`` call (:857-863): the sample at t = min_t."""
        out = self.sampler.sample(eval_sampler_inputs(window), self.num_t, float(self.min_t), float(self.noise_scale),
                                  generator=generator)
        self.sampler.memo.reset()                 # the trunk outputs of this window go with it
        return out["rigid_pred"], out["prot_traj"][0]

    # the device side of the loop, replaced by the fixture's rows in the CPU test
    def _run(self) -> torch.Tensor:
        """Every protein's row ``ROW_KEYS`` as one [n, 5] fp64 device tensor; nothing is read back to the host."""
        window_gen, reverse_gen = self.generators()
        rows = torch.empty(len(self.rows), len(ROW_KEYS), dtype=torch.float64, device=self.device)
        for i, window in enumerate(self._prefetcher(window_gen)):
            rigid_pred, atom37_pred = self._sample(i, window, reverse_gen)
            m = window_metrics(rigid_pred, atom37_pred, window["rigids_0"], window["atom37_pos"], window["atom37_mask"])
            rows[i].copy_(torch.cat([m[k] for k in ROW_KEYS]))
        return rows

    def _read(self, rows: torch.Tensor) -> np.ndarray:
        """The one device-to-host read of an evaluation."""
        return rows.cpu().numpy()

    def evaluate(self) -> Dict[str, object]:
        """eval_fn's return value over the test split, and its four summary lines printed (:915-928), quirks kept:
        ``all_atom_mse`` stays a list of [1] arrays while the other metrics are concatenated, and each printed mean is the
        sum over ALL rows divided by the number of rows with ``ave_trans < 10000``."""
        return self.summarise(self._read(self._run()))

    def summarise(self, rows: np.ndarray) -> Dict[str, object]:
        """eval_fn's dict and printed lines from the host rows [n, 5] (``ROW_KEYS``), in eval_fn's order of operations."""
        d = {"name": list(self.names), **{k: [rows[i, j:j + 1].copy() for i in range(len(rows))]
                                          for j, k in enumerate(ROW_KEYS)}}
        for k in ("ave_rot", "ave_trans", "all_atom_mae", "all_atom_rmsd"):
            d[k] = np.concatenate(d[k], axis=0)
        mask = d["ave_trans"] < MASK_BOUND
        for label, k in PRINTED:
            print(f"{label}:", d[k].sum() / mask.sum())
        return d

    def extend(self, length: int = 200, out_dir=None) -> Dict[str, object]:
        """``eval_extension`` over the test split, scored against the MD frames that follow each window.

        For each protein, in csv order: the evaluation window of ``evaluate`` (the same frames, from the same seeded window
        generator), rolled forward ``length`` frames by ``TrajectoryRollout.rollout(..., graph=False)`` at ``min_t``
        (200 is eval_extension's hard-coded length, :933); then rollout frame j (horizon j + 1) is scored against MD
        frame ``fix_sample_start + (frame_time - 1 + j) * frame_sample_step`` with ``metrics.horizon_metrics``: eval_fn's
        ``ave_rot``, ``ave_trans``, ``all_atom_mae``, ``all_atom_mse`` and ``all_atom_rmsd`` (its ``atom_mask[-1, -1, -1]
        = 0`` applied to every frame), and ``persist_rot`` / ``persist_trans``, the error of repeating the last MD frame
        the network was given (window frame ``frame_time - 2``).  Horizon 1 scores the same prediction as ``evaluate``'s
        row.  A trajectory too short for ``length`` horizons stops the loop; the store's ValueError, naming its archive,
        is the cause of the prefetcher's error.

        The scores stay in one [n, length, 7] fp64 device tensor read back once, after the last protein.  With ``out_dir``
        each protein's rollout is also written to ``<out_dir>/<name>/extension.npz`` (``write_extension``, eval_extension's
        keys, shapes and dtypes), which reads that trajectory back to the host: the only per-protein read.

        Returns {"name": [n names], key: [n, length] fp64 for each of ``HORIZON_KEYS``} and prints, per key, the mean over
        proteins at horizons 1, 10, 100 and ``length`` (those <= ``length``).  ``length`` and ``out_dir`` are checked
        before any device work, as the config (``frame_time`` >= 2, which the rollout and ``persist_*`` need) was."""
        if isinstance(length, bool) or not isinstance(length, int) or length < 1:
            raise ValueError(f"extend: length must be an int >= 1, got {length!r}")
        if out_dir is not None and not isinstance(out_dir, (str, bytes)) and not hasattr(out_dir, "__fspath__"):
            raise ValueError(f"extend: out_dir must be a path or None, got {out_dir!r}")
        if not self.min_t > 0.0:
            raise ValueError(f"extend: the rollout runs at data.min_t, which must be > 0, got {self.min_t!r}")
        return self.summarise_extension(self._read(self._run_extension(length, out_dir)))

    # the device side of the extension loop, replaced by the fixture's scores in the CPU test
    def _run_extension(self, length: int, out_dir) -> torch.Tensor:
        """Every protein's ``horizon_metrics`` as one [n, length, 7] fp64 device tensor."""
        window_gen, _ = self.generators()
        nf = self.frame_time
        scores = torch.empty(len(self.rows), length, len(HORIZON_KEYS), dtype=torch.float64, device=self.device)
        for i, window in enumerate(self._prefetcher(window_gen, horizons=length)):
            traj = self.roller.rollout(window, length, min_t=float(self.min_t), graph=False)
            scores[i].copy_(horizon_metrics(traj["rigid_traj"], traj["atom_traj"], window["rigids_0"][nf - 2],
                                            window["horizon_rigids_0"], window["horizon_atom37_pos"],
                                            window["horizon_atom37_mask"]))
            if out_dir is not None:
                write_extension(os.path.join(os.fsdecode(out_dir), self.names[i], "extension.npz"),
                                *self._read_trajectory(traj, window))
        return scores

    def _read_trajectory(self, traj: Dict[str, torch.Tensor], window: Dict[str, torch.Tensor]):
        """The per-protein device-to-host read of ``extend(out_dir=...)``: (rigid_traj, atom_traj, aatype) as numpy."""
        return traj["rigid_traj"].cpu().numpy(), traj["atom_traj"].cpu().numpy(), window["aatype"].cpu().numpy()

    def summarise_extension(self, scores: np.ndarray) -> Dict[str, object]:
        """``extend``'s dict and printed lines from the host scores [n, length, 7] (``HORIZON_KEYS``).  Each printed value
        is the mean over proteins at one horizon."""
        d = {"name": list(self.names), **{k: scores[:, :, j].copy() for j, k in enumerate(HORIZON_KEYS)}}
        length = scores.shape[1]
        horizons = sorted({h for h in PRINTED_HORIZONS + (length,) if h <= length})
        for k in HORIZON_KEYS:
            means = d[k][:, [h - 1 for h in horizons]].mean(axis=0)
            print(f"{k}:", " ".join(f"h{h} {m}" for h, m in zip(horizons, means)))
        return d
