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

Not reproduced: the directories, ``eval_conf.yaml``, plots and PDB files eval_fn writes, and the reference's random
streams (see ``Evaluator``).
"""
import numbers
from typing import Dict, List, Tuple

import numpy as np
import torch

from . import checkpoint as _ckpt
from .inference import DeviceReverseDiffusion
from .input_pipeline import EvaluationStore, WindowPrefetcher
from .metrics import eval_sampler_inputs, window_metrics
from .trainer import ROW_FIELDS, _get, _int, kept_rows

ROW_KEYS = ("ave_rot", "ave_trans", "all_atom_mae", "all_atom_mse", "all_atom_rmsd")   # one device row per window
PRINTED = (("ave_rot", "ave_rot"), ("ave_trans", "ave_trans"), ("ave_atom_mae", "all_atom_mae"),
           ("ave_atom_rmsd", "all_atom_rmsd"))                                        # eval_fn's summary lines (:925-928)
MASK_BOUND = 10000.0                                                                  # eval_fn's ``ave_trans < 10000``


def split_rows(csv_path: str, max_len) -> List[Tuple[str, Tuple[str, str, str, str]]]:
    """The rows ``PdbDataset(is_training=False, is_testing=True)`` iterates: ``seq_len <= max_len``, in csv order, as
    (name, ``TrajectoryStore.protein`` arguments).  The name is eval_fn's ``save_name``, ``name.split('.')[0]`` (:873)."""
    kept = kept_rows(csv_path, max_len, ("seq_len", "name") + ROW_FIELDS)
    return [(r["name"].split(".")[0], tuple(r[k] for k in ROW_FIELDS)) for r in kept]


def eval_seeds(seed: int) -> Tuple[int, int]:
    """The seeds of the evaluator's two CUDA generators: (windows' ``sample_ref``, reverse steps), two independent
    streams spawned from ``seed``."""
    return tuple(int(s.generate_state(1, np.uint64)[0]) for s in np.random.SeedSequence(seed).spawn(2))


def load_weights(net: torch.nn.Module, path: str) -> None:
    """Loads ``path``'s ``model`` state_dict into ``net`` strictly, ``module.`` prefixes stripped, as the reference
    evaluator's ``_load_ckpt`` does (eval_DFOLD_dynamics.py:131-136): a checkpoint of ``checkpoint.save_checkpoint`` or of
    the reference trainer.  Every key and shape is checked first (``checkpoint.check_model``), so a mismatch raises
    ValueError and leaves ``net`` as it was.  Checkpoints are trusted input: ``conf`` is an arbitrary pickled object, so the
    file is read with ``weights_only=False`` as the reference does; never load one from an untrusted source."""
    ckpt = torch.load(path, map_location="cpu", weights_only=False)
    model = _ckpt.check_model(ckpt, {k: v.shape for k, v in net.state_dict().items()})
    net.load_state_dict(model, strict=True)


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
    loaded into ``net`` in the constructor and ``net`` is put in eval mode.

    Random streams: two CUDA generators seeded from ``seed`` (``eval_seeds``), one for the windows' ``sample_ref`` (drawn by
    the prefetcher's worker thread), one for the reverse steps (drawn by the calling thread), so a run is reproducible bit
    for bit whatever the threads' timing.  The global generators are not touched.  The reference draws both from numpy's
    global stream on the host; those numbers are not reproduced."""

    def __init__(self, conf, net: torch.nn.Module, diffuser, *, seed: int = 0, depth: int = 2):
        self._configure(conf)
        load_weights(net, self.weights_path)
        net.eval()
        self.net, self.diffuser, self.seed, self.depth = net, diffuser, int(seed), depth
        self.device = next(net.parameters()).device
        self.sampler = DeviceReverseDiffusion(net)

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

    def _prefetcher(self, generator: torch.Generator):
        store = EvaluationStore(self.frame_time, self.frame_step, fix_sample_start=self.fix_start)
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
