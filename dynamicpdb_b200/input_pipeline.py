"""Input pipeline of the DFOLDv2 trainer on the device (SURVEY.md §8 f4).

The reference builds every training sample on the host, inside ``PdbDataset.__getitem__`` (src/data/
Dfold_data_loader_dynamic.py:192-259, :312-360): it re-opens and decompresses the WHOLE trajectory archive of the protein
(``dict(np.load(...))``), unpickles the whole force / velocity trajectories, slices ``frame_time`` frames out of them, and
runs the OpenFold feature transforms (``atom37_to_frames``, ``atom37_to_torsion_angles``) plus a CPU eigen-decomposition
(``rot_to_quat``) on the slice.  At the throughput of this package (hundreds of frames per second per GPU) that loader
cannot keep one GPU fed, let alone eight.  Here:

* ``TrajectoryStore`` keeps each protein's trajectory decoded ONCE, in pinned host memory (atom37 coordinates as fp32:
  that is what the archive holds), and hands out frame windows with the reference's own index arithmetic and random
  stream (``select_random_samples`` / ``select_first_samples``, :164-190);
* ``EvaluationStore`` is the store of an evaluation over a test split: it pins only each window's frames and keeps
  nothing once the window is built;
* ``featurize_window`` computes ``rigids_0`` and the torsion features of a window with one kernel on the device
  (csrc/featurize.cu), from the fp32 coordinates of the ``frame_time`` selected frames only;
* ``WindowPrefetcher`` overlaps the next window's host->device copy (side stream, straight from the store's pinned
  memory) with the current training step;
* given a diffuser (``score_epilogue.SE3ScoreDiffuser``), the same side stream also noises the window (:332-349):
  in training ``t ~ U(min_t, 1)`` is drawn on the device and ``forward_marginal`` (csrc/diffuse.cu) adds ``t``,
  ``rigids_t``, both scores and both score scalings; in evaluation ``t = 1`` and ``sample_ref`` gives ``rigids_t``.
  No value goes back to the host, so a window is a complete training batch without per-window host work.

With ``targets=True`` each item also carries the evaluation targets ``atom37_pos`` / ``atom37_mask`` (fp64, as the
loader returns them) for ``metrics.evaluate_window``.  The other evaluation-only fields (``atom14_pos``,
``rigidgroups_0``, ``residx_atom14_to_atom37``) are not produced.
"""
import pickle
import threading
from typing import Dict, Iterator, Optional, Sequence, Tuple

import numpy as np
import torch

from . import kernels as K
from .feats import table


def featurize_window(atom37: torch.Tensor, atom_mask: torch.Tensor, aatype: torch.Tensor) -> Dict[str, torch.Tensor]:
    """atom37 [nf,N,37,3] fp32 (device), atom_mask [N,37], aatype [N] int64 ->
    {rigids_0 [nf,N,7] fp32, torsion_angles_sin_cos / alt_torsion_angles_sin_cos [nf,N,7,2] fp64, torsion_angles_mask
    [nf,N,7] fp64, res_mask [nf,N]} as ``_process_csv_row`` + ``__getitem__`` (rigids_0 up to the quaternion sign, which the
    reference's eigen-decomposition leaves arbitrary)."""
    K._need_cuda(atom37, atom_mask, aatype)
    nf, N = atom37.shape[0], atom37.shape[1]
    dev = atom37.device
    pos = atom37.to(torch.float32).contiguous()
    am = atom_mask.to(torch.float32).contiguous()
    aa = aatype.to(torch.int64).contiguous()
    rig = torch.empty(nf, N, 7, dtype=torch.float32, device=dev)
    tor = torch.empty(nf, N, 7, 2, dtype=torch.float64, device=dev)
    alt = torch.empty_like(tor)
    tm = torch.empty(nf, N, 7, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        K.launch("dfold_featurize_window", pos, am, aa, table("chi_atom_indices", dev), table("chi_angles_mask", dev),
                 table("chi_pi_periodic", dev), nf, N, rig, tor, alt, tm)
    return {"rigids_0": rig, "torsion_angles_sin_cos": tor, "alt_torsion_angles_sin_cos": alt, "torsion_angles_mask": tm,
            "res_mask": am[:, 1].to(torch.float64).unsqueeze(0).expand(nf, -1)}


class TrajectoryStore:
    """Decoded trajectories of the proteins of a split, pinned in host memory, keyed by the csv row fields the reference
    reads (``atlas_npz``, ``force_path``, ``vel_path``, ``embed_path``; README "Data Preparation")."""

    def __init__(self, frame_time: int, frame_sample_step: int = 1, keep_first: Optional[int] = None, fix_sample_start: int = 0,
                 pin: bool = True):
        self.frame_time, self.step, self.keep_first, self.fix_start = frame_time, frame_sample_step, keep_first, fix_sample_start
        self.pin = pin and torch.cuda.is_available()
        self._cache: Dict[str, Dict[str, torch.Tensor]] = {}

    def _pin(self, a: np.ndarray, dtype) -> torch.Tensor:
        t = torch.from_numpy(np.ascontiguousarray(a)).to(dtype)
        return t.pin_memory() if self.pin else t

    def protein(self, atlas_npz: str, force_path: str, vel_path: str, embed_path: str) -> Dict[str, torch.Tensor]:
        """Load (once) and cache one protein: the file naming follows Dfold_data_loader_dynamic.py:194-198.  The frames
        kept are the first ``keep_first`` (training windows) and the ones up to the end of the evaluation window, which
        starts at ``fix_sample_start`` whatever ``keep_first`` is (:214-218)."""
        if atlas_npz in self._cache:
            return self._cache[atlas_npz]
        kf = self.keep_first
        if kf is not None:
            kf = max(kf, self.fix_start + self.frame_time * self.step)
        ent = self._entry(_decode(atlas_npz, force_path, vel_path, embed_path), slice(None, kf))
        self._cache[atlas_npz] = ent
        return ent

    def _entry(self, raw: Dict[str, np.ndarray], frames: slice) -> Dict[str, torch.Tensor]:
        """A decoded protein with the frames ``frames`` of its trajectories, in pinned memory."""
        return {
            "atom37": self._pin(raw["all_atom_positions"][frames], torch.float32),           # [T,N,37,3]
            "force": self._pin(np.asarray(raw["force"])[frames], torch.float64),             # [T,N,3] (the loader's dtype)
            "vel": self._pin(np.asarray(raw["vel"])[frames], torch.float64),
            "atom_mask": self._pin(raw["all_atom_mask"], torch.float32),                     # [N,37]
            "aatype": torch.from_numpy(np.argmax(raw["aatype"], axis=-1)).long(),            # [N]
            "residue_index": torch.from_numpy(np.asarray(raw["residue_index"])).long(),
            "node_repr": self._pin(raw["node_repr"], torch.float32),
            "edge_repr": self._pin(raw["edge_repr"], torch.float32),
        }

    def window_index(self, n_frames: int, training: bool) -> slice:
        """The reference's window arithmetic (:164-190, :214-218), drawing from numpy's global stream exactly as it does.
        ``n_frames`` is the number of frames ``protein`` kept.  Training windows lie in the first ``keep_first`` frames;
        evaluation windows start at ``fix_sample_start`` and may reach past them.  An evaluation window shorter than
        ``frame_time`` raises (the reference raises when fewer than ``frame_time`` frames follow the start)."""
        t, k = self.frame_time, self.step
        if training:
            n = n_frames if self.keep_first is None else min(n_frames, self.keep_first)
            if t > n:
                raise ValueError("t cannot be greater than the number of samples")
            start = np.random.randint(0, n - t * k + 1)
        else:
            start = self.fix_start
            n = n_frames - start
            if t > n:
                raise ValueError("t cannot be greater than the number of samples")
            if (t - 1) * k >= n:
                raise ValueError(f"the evaluation window ({t} frames every {k} from frame {start}) reaches past the "
                                 f"{n_frames} frames of the trajectory")
        return slice(start, start + t * k, k)


def _decode(atlas_npz: str, force_path: str, vel_path: str, embed_path: str) -> Dict[str, np.ndarray]:
    """The arrays of one protein's files, named as the loader names them (Dfold_data_loader_dynamic.py:194-198)."""
    with np.load(atlas_npz, allow_pickle=True) as zf:
        raw = {k: zf[k] for k in ("all_atom_positions", "all_atom_mask", "aatype", "residue_index")}
    with open(force_path.replace(".pkl", "_Ca.pkl"), "rb") as f:
        raw["force"] = pickle.load(f)
    with open(vel_path.replace(".pkl", "_ca.pkl"), "rb") as f:
        raw["vel"] = pickle.load(f)
    with np.load(embed_path) as ef:
        raw.update({k: ef[k] for k in ("node_repr", "edge_repr")})
    return raw


class EvaluationStore(TrajectoryStore):
    """The store an evaluation over a test split reads: each protein is decoded when its window is made, only the
    ``frame_time`` frames of that window (every ``frame_sample_step``-th from ``fix_sample_start``) are pinned, and
    nothing is kept once the window is built.  A split of many proteins then holds in pinned memory only the windows a
    ``WindowPrefetcher`` has in flight (at most depth + 1), whatever the length of the trajectories; a ``TrajectoryStore``
    would keep every trajectory from frame 0 to the end of its window for the life of the store.

    ``protein`` returns an entry whose frame 0 is the window's first frame, and ``window_index`` the whole of it.  A
    trajectory too short for the window raises the reference loader's ValueError, prefixed with the row's archive.

    ``horizons=L`` (>= 1) also keeps the MD frames a rollout of ``L`` frames from the window predicts: the entry holds
    ``frame_time + L - 1`` frames on the same grid (frame ``frame_time - 1 + j`` is the target of rollout frame ``j``),
    ``window_index`` still names the window's ``frame_time``, and a ``WindowPrefetcher`` adds the targets to each item.  A
    trajectory too short for ``L`` horizons raises ValueError, prefixed with the row's archive.  0 (the default) keeps the
    window alone."""

    def __init__(self, frame_time: int, frame_sample_step: int = 1, fix_sample_start: int = 0, pin: bool = True,
                 horizons: int = 0):
        super().__init__(frame_time, frame_sample_step, keep_first=None, fix_sample_start=fix_sample_start, pin=pin)
        if isinstance(horizons, bool) or not isinstance(horizons, int) or horizons < 0:
            raise ValueError(f"horizons must be an int >= 0, got {horizons!r}")
        self.horizons = horizons
        self.n_frames = frame_time + max(horizons - 1, 0)

    def protein(self, atlas_npz: str, force_path: str, vel_path: str, embed_path: str) -> Dict[str, torch.Tensor]:
        raw = _decode(atlas_npz, force_path, vel_path, embed_path)
        T = raw["all_atom_positions"].shape[0]
        try:
            frames = TrajectoryStore.window_index(self, T, training=False)
            frames = slice(frames.start, frames.start + self.n_frames * self.step, self.step)
            if frames.start + (self.n_frames - 1) * self.step >= T:
                raise ValueError(f"{self.horizons} horizons after the evaluation window ({self.n_frames} frames every "
                                 f"{self.step} from frame {frames.start}) reach past the {T} frames of the trajectory")
        except ValueError as e:
            raise ValueError(f"{atlas_npz}: {e}") from e
        return self._entry(raw, frames)

    def window_index(self, n_frames: int, training: bool) -> slice:
        if training:
            raise ValueError("an EvaluationStore holds evaluation windows only")
        if n_frames != self.n_frames:
            raise ValueError(f"an EvaluationStore entry holds {self.n_frames} frames, not {n_frames}")
        return slice(0, self.frame_time, 1)


class WindowPrefetcher:
    """Iterates device-resident feature dicts, one protein window per item: while the consumer trains on window i, a worker
    thread has a side stream copy window i+1 to the device and featurise it.

    Each item's tensors are recorded on the stream that is current when the item is handed out, so their memory is not
    reused before the work queued there on them has run, even when the consumer drops the item long before.  A consumer
    that reads them on yet another stream must ``record_stream`` that stream itself.  Leaving the loop early (``break``)
    stops the worker thread."""

    def __init__(self, store: TrajectoryStore, rows: Sequence[Tuple[str, str, str, str]], device, training: bool = True, depth: int = 2,
                 diffuser=None, min_t: float = 0.01, generator: Optional[torch.Generator] = None, targets: bool = False):
        """``diffuser`` (an ``SE3ScoreDiffuser``, optional) makes every item a noised training batch (see the module
        docstring); ``min_t`` is the loader's ``data_conf.min_t``; ``generator`` (a CUDA generator on ``device``) feeds t
        and the diffusion draws, default: the device's default generator.  ``targets`` adds the evaluation targets
        ``atom37_pos`` [nf, N, 37, 3] and ``atom37_mask`` [nf, N, 37], fp64 as ``_process_csv_row`` returns them (:249-250),
        which ``metrics.evaluate_window`` scores the sample against (atoms outside the mask keep the archive's coordinates,
        which the loader zeroes; every metric masks them).

        An ``EvaluationStore(horizons=L)`` with L >= 1 makes each item also carry the targets of a rollout of ``L`` frames
        from the window, the entry's frames ``frame_time - 1 ..``: ``horizon_rigids_0`` [L, N, 7] fp32,
        ``horizon_atom37_pos`` [L, N, 37, 3] and ``horizon_atom37_mask`` [L, N, 37], fp64.  The window and its targets come
        from one copy and one ``featurize_window`` launch over all ``frame_time + L - 1`` frames; the window's fields are
        its first ``frame_time`` frames and equal, bit for bit, the item made without horizons."""
        dev = torch.device(device)
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.store, self.rows, self.device, self.training, self.depth = store, list(rows), dev, training, depth
        self.horizons = getattr(store, "horizons", 0)
        self.diffuser, self.min_t, self.generator, self.targets = diffuser, float(min_t), generator, bool(targets)
        if not 0.0 <= self.min_t <= 1.0:
            raise ValueError(f"min_t={min_t} outside [0, 1]")
        self.stream = torch.cuda.Stream(device=self.device)
        if diffuser is not None:
            diffuser.tables(self.device)                    # built once, before the side stream reads them
            self.stream.wait_stream(torch.cuda.current_stream(self.device))
        self._thread: Optional[threading.Thread] = None

    def _make(self, row) -> Tuple[Dict[str, torch.Tensor], torch.cuda.Event]:
        ent = self.store.protein(*row)
        sl = self.store.window_index(ent["atom37"].shape[0], self.training)
        nf = self.store.frame_time
        with torch.cuda.stream(self.stream):
            cp = lambda t: t.to(self.device, non_blocking=True)
            # the contiguous frame range straight from the store, whose pinned memory nothing writes; every step-th frame
            # is then taken on the device
            frames = lambda t: cp(t[sl.start:sl.stop])[::sl.step].contiguous()
            atom_mask = cp(ent["atom_mask"])
            if self.horizons:
                # the window and the frames that follow it, featurised together; the window is their first nf
                whole = cp(ent["atom37"])
                feats = featurize_window(whole, atom_mask, cp(ent["aatype"]))
                horizon = {"horizon_rigids_0": feats["rigids_0"][nf - 1:],
                           "horizon_atom37_pos": whole[nf - 1:].to(torch.float64),
                           "horizon_atom37_mask": atom_mask.to(torch.float64).unsqueeze(0).expand(self.horizons, -1, -1)}
                feats = {k: v[:nf] for k, v in feats.items()}
                feats.update(horizon)
                atom37 = whole[:nf]
            else:
                atom37 = frames(ent["atom37"])
                feats = featurize_window(atom37, atom_mask, cp(ent["aatype"]))
            if self.targets:
                feats["atom37_pos"] = atom37.to(torch.float64)
                feats["atom37_mask"] = atom_mask.to(torch.float64).unsqueeze(0).expand(nf, -1, -1)
            feats.update({
                "aatype": cp(ent["aatype"]).unsqueeze(0).expand(nf, -1),
                "seq_idx": cp(ent["residue_index"]).unsqueeze(0).expand(nf, -1),
                "residue_index": cp(ent["residue_index"]).unsqueeze(0).expand(nf, -1),
                "force": frames(ent["force"]), "vel": frames(ent["vel"]),
                "node_repr": cp(ent["node_repr"]), "edge_repr": cp(ent["edge_repr"]),
                "fixed_mask": torch.zeros(nf, atom37.shape[1], dtype=torch.float64, device=self.device),
                "sc_ca_t": torch.zeros(nf, atom37.shape[1], 3, dtype=torch.float32, device=self.device),
            })
            if self.diffuser is not None:
                feats.update(self._noise(feats["rigids_0"]))
            ev = torch.cuda.Event()
            ev.record(self.stream)
        return feats, ev

    def _noise(self, rigids_0: torch.Tensor) -> Dict[str, torch.Tensor]:
        """Dfold_data_loader_dynamic.py:332-357 on the device: training t = rng.uniform(min_t, 1) and forward_marginal; eval
        t = 1 and sample_ref of nf * N frames.  ``t`` is a [1] fp64 tensor (the loader's t, batched)."""
        nf, N = rigids_0.shape[0], rigids_0.shape[1]
        if self.training:
            u = torch.rand(1, dtype=torch.float64, device=self.device, generator=self.generator)
            t = self.min_t + (1.0 - self.min_t) * u
            out = self.diffuser.forward_marginal(rigids_0, t, diffuse_mask=None, generator=self.generator)
        else:
            t = torch.ones(1, dtype=torch.float64, device=self.device)
            out = self.diffuser.sample_ref(nf * N, frame_time=nf, generator=self.generator, device=self.device)
        out["t"] = t
        return out

    def __iter__(self) -> Iterator[Dict[str, torch.Tensor]]:
        import queue
        q: "queue.Queue" = queue.Queue(maxsize=self.depth)
        stop = threading.Event()

        def put(item) -> bool:
            """Queue ``item`` unless the consumer has left; False once it has."""
            while not stop.is_set():
                try:
                    q.put(item, timeout=0.05)
                    return True
                except queue.Full:
                    pass
            return False

        def work():
            try:
                torch.cuda.set_device(self.device)
                for row in self.rows:
                    if not put(self._make(row)):
                        return
                put(None)
            except BaseException as e:       # noqa: BLE001  (hand the failure to the consumer instead of blocking it forever)
                put(e)
        self._thread = threading.Thread(target=work, daemon=True)
        self._thread.start()
        try:
            while True:
                item = q.get(timeout=600)
                if item is None:
                    break
                if isinstance(item, BaseException):
                    raise RuntimeError("WindowPrefetcher worker failed") from item
                feats, ev = item
                consumer = torch.cuda.current_stream(self.device)
                consumer.wait_event(ev)
                for v in feats.values():
                    v.record_stream(consumer)
                yield feats
        finally:
            stop.set()
