"""Trajectory rollout on the device (DESIGN §1 f7, csrc/rollout.cu): a trajectory longer than one window, predicted frame by
frame with the predictions fed back, as ``Experiment.eval_extension`` (train_DFOLD_dynamics.py:931-1000) defines it.

From one evaluation window the sampler inputs are built as eval_fn builds them (``metrics.eval_sampler_inputs``); then for
``j = 0 .. length - 1``:

1. the network runs on the current inputs;
2. ``rigid_pred[-1]`` becomes ``rigid_traj[j]`` and ``atom37[-1]`` becomes ``atom_traj[j]`` (:993-994);
3. ``rigids_0 <- cat(rigid_pred[1:], rigid_pred[-1:])`` (:996).

Every other input -- ``force``, ``vel``, torsions and masks, ``node_repr`` / ``edge_repr``, ``aatype``, ``seq_idx`` -- keeps
the starting window's value.  (The reference's own loop omits ``force``, ``vel`` and ``torsion_angles_mask`` from its inputs
and cannot run; this is the reading in which it does.)

The reference keeps the prediction at t = min_t of a full ``num_t``-step reverse diffusion per frame.  The trunk reads
neither ``t`` nor the noised frames (DESIGN §5.5), so that prediction is ONE forward at t = min_t: the default path is one
network forward plus one ``dfold_rollout_advance`` launch per frame, captured once as a CUDA graph and replayed ``length``
times with no host work between frames.  ``literal=True`` runs the reference's schedule instead (fresh ``sample_ref``
draws, ``num_t`` full forwards per frame) and gives the same bits; it exists to show that.

Warning -- coordinate scaling.  The network returns unscaled frames (ipa_pytorch_dynamic.py:890) but reads ``rigids_0``
as it is, so with ``coordinate_scaling`` c != 1 every step multiplies the history's translations by 1 / c.  The reference
does the same and it is reproduced here; the released configuration (``run_train.sh`` / ``run_eval.sh``) uses c = 1.
"""
from typing import Dict

import torch

from . import kernels as K
from . import metrics as M

_ATOMS = 37


class TrajectoryRollout:
    """``TrajectoryRollout(net).rollout(window, length)`` for a ``FullScoreNetwork`` ``net`` on a CUDA device.  One CUDA
    graph is kept per (length, input shapes and dtypes); weights are read by the graph from the parameters themselves, so
    in-place weight updates between rollouts take effect."""

    def __init__(self, net):
        from .inference import DeviceReverseDiffusion
        self.net = net
        self.sampler = DeviceReverseDiffusion(net)        # the literal route; checks the diffuser
        self._graphs: Dict = {}

    def _step(self, feats, rigid_traj, atom_traj, step):
        out = self.net(feats)
        K.rollout_advance(out["rigids"], out["atom37"], feats["rigids_0"], rigid_traj, atom_traj, step)

    @staticmethod
    def _buffers(length, N, dev):
        return (torch.zeros(length, N, 7, dtype=torch.float32, device=dev),
                torch.zeros(length, N, _ATOMS, 3, dtype=torch.float32, device=dev),
                torch.zeros(1, dtype=torch.int64, device=dev))

    @torch.no_grad()
    def rollout(self, window: Dict[str, torch.Tensor], length: int, *, min_t: float = 0.01, literal: bool = False,
                num_t=None, noise_scale: float = 1.0, graph: bool = True) -> Dict[str, torch.Tensor]:
        """Roll ``window`` forward ``length`` frames: {"rigid_traj": [L, N, 7], "atom_traj": [L, N, 37, 3]}, fp32 device
        tensors.  ``window`` holds the fields of an evaluation item of ``WindowPrefetcher(training=False, diffuser=...)``
        (``rigids_0`` [nf, N, 7] fp32 with nf >= 2, ``rigids_t``, torsions and mask, ``force``, ``vel``, ``node_repr``,
        ``edge_repr``, ``aatype``) on one CUDA device; it is not modified.
        ``literal=True`` runs ``DeviceReverseDiffusion.sample(..., literal=True)`` with ``num_t`` steps (required) and
        fresh ``sample_ref`` draws per frame, as eval_extension does; ``noise_scale`` applies to it only.  ``graph=False``
        runs the default path's step eagerly.  Nothing is read back to the host."""
        if isinstance(length, bool) or not isinstance(length, int) or length < 1:
            raise ValueError(f"rollout: length must be an int >= 1, got {length!r}")
        if not 0.0 < float(min_t) <= 1.0:
            raise ValueError(f"rollout: min_t must lie in (0, 1], got {min_t}")
        if literal and (num_t is None or isinstance(num_t, bool) or not isinstance(num_t, int) or num_t < 1):
            raise ValueError(f"rollout: literal=True needs num_t >= 1 reverse steps, got {num_t!r}")
        missing = [k for k in M._EVAL_WINDOW_KEYS if k not in window]
        if missing:
            raise ValueError(f"rollout: the window lacks {missing} (WindowPrefetcher(training=False, diffuser=...) provides them)")
        rig = window["rigids_0"]
        if rig.dim() != 3 or rig.shape[-1] != 7 or rig.shape[0] < 2 or rig.dtype != torch.float32:
            raise ValueError(f"rollout: need rigids_0 [nf >= 2, N, 7] fp32, got {tuple(rig.shape)} {rig.dtype}")
        K._need_cuda(*[window[k] for k in M._EVAL_WINDOW_KEYS])
        init = M.eval_sampler_inputs(window)
        with torch.cuda.device(rig.device):
            if literal:
                return self._literal(init, length, float(min_t), num_t, noise_scale)
            if not graph:
                return self._eager(init, length, float(min_t))
            return self._graphed(init, length, float(min_t))

    def _eager(self, init, length, min_t):
        nf, N = init["rigids_0"].shape[:2]
        dev = init["rigids_0"].device
        feats = dict(init)
        feats["rigids_0"] = init["rigids_0"].clone()
        feats["t"] = torch.full((1,), min_t, dtype=torch.float32, device=dev)
        rigid_traj, atom_traj, step = self._buffers(length, N, dev)
        for _ in range(length):
            self._step(feats, rigid_traj, atom_traj, step)
        return {"rigid_traj": rigid_traj, "atom_traj": atom_traj}

    def _literal(self, init, length, min_t, num_t, noise_scale):
        nf, N = init["rigids_0"].shape[:2]
        dev = init["rigids_0"].device
        feats = dict(init)
        feats["rigids_0"] = init["rigids_0"].clone()
        rigid_traj, atom_traj, step = self._buffers(length, N, dev)
        for _ in range(length):
            feats["rigids_t"] = self.sampler.diffuser.sample_ref(nf * N, frame_time=nf, device=dev)["rigids_t"]
            out = self.sampler.sample(feats, num_t, min_t, noise_scale, literal=True)
            K.rollout_advance(out["rigid_pred"], out["prot_traj"][0], feats["rigids_0"], rigid_traj, atom_traj, step)
        return {"rigid_traj": rigid_traj, "atom_traj": atom_traj}

    def _graphed(self, init, length, min_t):
        key = (length, tuple((k, tuple(v.shape), v.dtype) for k, v in sorted(init.items())))
        ent = self._graphs.get(key)
        if ent is None:
            N, dev = init["rigids_0"].shape[1], init["rigids_0"].device
            static = {k: v.clone() for k, v in init.items()}
            static["t"] = torch.full((1,), min_t, dtype=torch.float32, device=dev)
            bufs = self._buffers(length, N, dev)
            cur = torch.cuda.current_stream()
            side = torch.cuda.Stream()
            side.wait_stream(cur)
            with torch.cuda.stream(side):                     # warm-up: allocator pools, library load, plane caches
                self._step(static, *bufs)
            cur.wait_stream(side)
            torch.cuda.synchronize()
            K.invalidate_weight_cache()                       # the weight planes must be built inside the graph
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._step(static, *bufs)
            K.invalidate_weight_cache()                       # eager callers must not reuse planes in the graph's pool
            ent = (g, static, bufs)
            self._graphs[key] = ent
        g, static, (rigid_traj, atom_traj, step) = ent
        for k, v in init.items():
            static[k].copy_(v)
        static["t"].fill_(min_t)
        step.zero_()
        for _ in range(length):
            g.replay()
        return {"rigid_traj": rigid_traj.clone(), "atom_traj": atom_traj.clone()}
