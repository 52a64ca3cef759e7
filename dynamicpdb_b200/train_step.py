"""One data-parallel training step of the score network, captured in a CUDA graph.

The reference trainer wraps the model in ``DistributedDataParallel(find_unused_parameters=True)`` and calls
``loss.backward(); optimizer.step()`` from Python (train_DFOLD_dynamics.py:612-616, 660-668); that keeps working on top
of this package (tests/test_cpu_ddp.py).  At these kernel speeds the ~700 kernel launches of a step would cost host time
comparable to the device time, so the step is:

    static input buffers  ->  [ forward + loss + backward + ONE flat NCCL all-reduce of the gradients + Adam ]  (one graph)

* gradients live in a single flat fp32 buffer (each ``param.grad`` is a view), so data parallelism is one
  ``all_reduce`` of 737.7 MB over NVLink per step and parameters without gradient (the dead-output embedder,
  ``linear_rbf``) simply contribute zeros — the reason the reference needs ``find_unused_parameters=True``;
* ``torch.cuda.graph`` captures the whole step (the C-ABI kernels are plain stream launches; TMA descriptors are
  by-value kernel arguments), replays have no Python / launch overhead;
* if capture is not possible the same step runs eagerly (``graph=False`` or on capture failure);
* ``max_grad_norm`` clips the data-parallel mean gradient by its global norm inside the same graph, as
  ``torch.nn.utils.clip_grad_norm_`` between ``loss.backward()`` and ``optimizer.step()`` would (the option the reference
  trainer keeps commented out, train_DFOLD_dynamics.py:665); ``grad_norm`` holds the norm before clipping;
* ``lr_schedule=AlphaFoldSchedule(...)`` moves the learning rate along AlphaFold's schedule, the scheduler the reference
  trainer imports (train_DFOLD_dynamics.py:56, its ``step()`` commented out at :652): a one-thread kernel inside the graph
  computes the step's lr from the device step counter, and Adam reads it from device memory (``current_lr``);
* ``accumulate=k`` averages the gradient over k windows per rank before the update (k input slots, filled with
  ``load(feats, slot=i)``): one optimizer step then sees the mean over world_size * k windows, as DDP over that many ranks;
* ``state_dict()`` / ``load_state_dict()`` save and resume the weights and the Adam(amsgrad) state in the reference
  trainer's checkpoint format, loading in place so the captured graph keeps running (checkpoint.py).
"""
import dataclasses
import math
import copy
import numbers
import os
import sys
import time
from typing import Callable, Dict, Optional

import torch
import torch.distributed as dist

from . import checkpoint as _ckpt
from . import kernels as _kernels


@dataclasses.dataclass(frozen=True)
class AlphaFoldSchedule:
    """The learning-rate schedule of AlphaFold 2 (AlphaFoldLRScheduler, openfold/utils/lr_schedulers.py; the defaults are
    AlphaFold's): a linear warmup from base_lr, a plateau at max_lr, then a decay by decay_factor every decay_every_n_steps
    steps after start_decay_after_n_steps.  Settings on which that scheduler fails or means nothing raise ValueError."""
    base_lr: float = 0.0
    max_lr: float = 0.001
    warmup_no_steps: int = 1000
    start_decay_after_n_steps: int = 50000
    decay_every_n_steps: int = 50000
    decay_factor: float = 0.95

    def __post_init__(self):
        for k in ("base_lr", "max_lr", "decay_factor"):
            v = getattr(self, k)
            if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(v):
                raise ValueError(f"AlphaFoldSchedule: {k} must be a finite number, got {v!r}")
            object.__setattr__(self, k, float(v))
        for k in ("warmup_no_steps", "start_decay_after_n_steps", "decay_every_n_steps"):
            v = getattr(self, k)
            if isinstance(v, bool) or not isinstance(v, numbers.Integral) or v < 0:
                raise ValueError(f"AlphaFoldSchedule: {k} must be a non-negative integer, got {v!r}")
            object.__setattr__(self, k, int(v))
        if not self.max_lr > 0:
            raise ValueError(f"AlphaFoldSchedule: max_lr must be positive, got {self.max_lr!r}")
        if self.warmup_no_steps == 0:
            raise ValueError("AlphaFoldSchedule: warmup_no_steps must be positive (the schedule divides by it)")
        if self.decay_every_n_steps == 0:
            raise ValueError("AlphaFoldSchedule: decay_every_n_steps must be positive (the schedule divides by it)")
        if self.warmup_no_steps > self.start_decay_after_n_steps:
            raise ValueError(f"AlphaFoldSchedule: warmup_no_steps ({self.warmup_no_steps}) must not exceed "
                             f"start_decay_after_n_steps ({self.start_decay_after_n_steps})")

    def lr(self, step: int) -> float:
        """AlphaFoldLRScheduler.get_lr() at last_epoch = step, in float64 as it is evaluated there: the lr of optimizer step
        step + 1 (the scheduler steps once when it is constructed), and the lr a checkpoint at step `step` resumes with."""
        if step <= self.warmup_no_steps:
            return self.base_lr + (step / self.warmup_no_steps) * self.max_lr
        if step > self.start_decay_after_n_steps:
            return self.max_lr * (self.decay_factor ** ((step - self.start_decay_after_n_steps) // self.decay_every_n_steps + 1))
        return self.max_lr


class TrainStep:
    def __init__(self, net: torch.nn.Module, loss_fn: Callable[[Dict[str, torch.Tensor]], torch.Tensor],
                 example_feats: Dict[str, torch.Tensor], *, lr: float = 1e-4, world_size: int = 1, graph: bool = True,
                 warmup: int = 3, max_grad_norm: Optional[float] = None, lr_schedule: Optional[AlphaFoldSchedule] = None,
                 accumulate: int = 1):
        self.max_grad_norm = _check_max_grad_norm(max_grad_norm)
        if lr_schedule is not None and not isinstance(lr_schedule, AlphaFoldSchedule):
            raise ValueError(f"lr_schedule must be None or an AlphaFoldSchedule, got {type(lr_schedule).__name__}")
        self.schedule = lr_schedule
        if isinstance(accumulate, bool) or not isinstance(accumulate, numbers.Integral) or accumulate < 1:
            raise ValueError(f"accumulate must be a positive integer (windows per rank and optimizer step), got {accumulate!r}")
        self.accumulate = int(accumulate)
        self.fused_adam = os.environ.get("DFOLD_TORCH_ADAM", "0") != "1"
        self.chunks = max(1, int(os.environ.get("DFOLD_ALLREDUCE_CHUNKS", "1")))
        if self.max_grad_norm is not None and self.fused_adam and world_size > 1 and self.chunks > 1:
            raise ValueError("max_grad_norm needs the whole all-reduced gradient before the first update, but "
                             f"DFOLD_ALLREDUCE_CHUNKS={self.chunks} updates each piece as soon as it is reduced: "
                             "unset it to clip")
        self.net, self.loss_fn, self.world = net, loss_fn, world_size
        # the summed gradient of world_size ranks x accumulate windows becomes their mean
        self.grad_scale = 1.0 / (world_size * self.accumulate)
        self.params = [p for p in net.parameters() if p.requires_grad]
        self.layout = _ckpt.flat_layout(net)             # where each trained parameter sits in the flat buffers
        dev = self.params[0].device
        padded = self.layout.numel                         # padded to a multiple of 4: the fused optimizer runs float4-wide
        self.flat_grad = torch.zeros(padded, dtype=torch.float32, device=dev)
        # Adam(amsgrad) as the reference trainer (train_DFOLD_dynamics.py:412).  Default: ONE fused kernel over flat
        # parameter / gradient / moment buffers (csrc/simt.cu adam_amsgrad_kernel, step counter on the device); with
        # DFOLD_TORCH_ADAM=1: torch.optim.Adam(capturable, foreach) on the same gradient views.  With a schedule the lr is a
        # device scalar that dfold_lr_schedule rewrites before every update; `lr` is then only the optimizer's initial_lr.
        self.lr = lr
        self.current_lr: Optional[torch.Tensor] = None
        if self.schedule is not None:
            self.current_lr = torch.full((), self.schedule.lr(0), dtype=torch.float32, device=dev)
        if self.fused_adam:
            self.flat_param = torch.zeros(padded, dtype=torch.float32, device=dev)
        off = 0
        with torch.no_grad():
            for p in self.params:
                n = p.numel()
                if self.fused_adam:
                    self.flat_param[off:off + n].copy_(p.reshape(-1))
                    p.data = self.flat_param[off:off + n].view_as(p)       # the module's parameters become views of the flat buffer
                p.grad = self.flat_grad[off:off + n].view_as(p)
                off += n
        if self.fused_adam:
            self.exp_avg = torch.zeros_like(self.flat_param)
            self.exp_avg_sq = torch.zeros_like(self.flat_param)
            self.max_exp_avg_sq = torch.zeros_like(self.flat_param)
            self.step_count = torch.zeros((), dtype=torch.float32, device=dev)
            self.opt = None
            _kernels.invalidate_weight_cache()
        else:
            self.opt = torch.optim.Adam(self.params, lr=lr if self.current_lr is None else self.current_lr, amsgrad=True,
                                        capturable=True, foreach=True)
            if self.current_lr is not None:
                self.current_lr = self.opt.param_groups[0]["lr"]           # the tensor the optimizer reads
                self._step0 = torch.zeros((), dtype=torch.float32, device=dev)    # the step count before Adam has state
        # one set of static input buffers per accumulated window
        self.slots = [{k: v.clone() for k, v in example_feats.items()} for _ in range(self.accumulate)]
        self.static = self.slots[0]
        self.loss = torch.zeros((), dtype=torch.float32, device=dev)
        # the global norm of the mean gradient before clipping, overwritten by every step (None: no clipping, no norm)
        self.grad_norm: Optional[torch.Tensor] = None
        if self.max_grad_norm is not None:
            self.grad_norm = torch.zeros((), dtype=torch.float32, device=dev)
            if self.fused_adam:
                self.clip_coef = torch.ones((), dtype=torch.float32, device=dev)
                self.norm_partial = torch.zeros(1024, dtype=torch.float64, device=dev)      # dfold_grad_norm's workspace
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.graph_error: Optional[str] = None
        verbose = os.environ.get("DFOLD_BENCH_VERBOSE", "0") == "1"
        # The warm-up steps below are REAL steps (they must be: they size the allocator pools and initialise NCCL and the
        # capturable Adam state before capture).  Training must nevertheless start from the weights and optimizer state
        # the caller handed in, so both are snapshotted here and restored after capture.
        with torch.no_grad():
            saved_params = [p.detach().clone() for p in self.params]
        saved_opt = copy.deepcopy(self.opt.state_dict()) if self.opt is not None else None
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for it in range(max(1, warmup)):
                self._eager()
                if verbose:
                    torch.cuda.synchronize()
                    print(f"[train_step t={time.perf_counter():.1f}] eager warm-up step {it} done", file=sys.stderr, flush=True)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        if graph:
            try:
                _kernels.invalidate_weight_cache()
                g = torch.cuda.CUDAGraph()
                # captured at a higher priority than the side stream of the convolution weight gradients (kernels.py): the
                # block scheduler then serves the backward's critical path first, and the weight gradients fill the SMs
                # it leaves idle instead of holding them while it waits
                with torch.cuda.graph(g, stream=torch.cuda.Stream(device=dev, priority=-1)):
                    self._eager()
                self.graph = g
            except Exception as e:                       # noqa: BLE001  (report and fall back to eager launches)
                self.graph_error = f"{type(e).__name__}: {str(e)[:200]}"
                self.graph = None
                torch.cuda.synchronize()
        self._restore(saved_params, saved_opt)

    def _restore(self, saved_params, saved_opt):
        """Undo the warm-up / capture steps: parameters back to their values at construction; Adam moments zeroed and the
        step counter reset IN PLACE (the captured graph holds pointers to these very state tensors)."""
        with torch.no_grad():
            for p, v in zip(self.params, saved_params):
                p.copy_(v)
            if self.opt is None:
                for t in (self.exp_avg, self.exp_avg_sq, self.max_exp_avg_sq, self.step_count):
                    t.zero_()
            else:
                fresh = not saved_opt["state"]
                for i, p in enumerate(self.params):
                    st = self.opt.state.get(p)
                    if not st:
                        continue
                    old = None if fresh else saved_opt["state"].get(i)
                    for k, v in st.items():
                        if torch.is_tensor(v):
                            if old is not None and k in old:
                                v.copy_(old[k].to(v.device))
                            else:
                                v.zero_()
            self.flat_grad.zero_()
            if self.grad_norm is not None:
                self.grad_norm.zero_()
            if self.current_lr is not None:
                self.current_lr.fill_(self.schedule.lr(0))
        _kernels.invalidate_weight_cache()
        torch.cuda.synchronize()

    def _eager(self):
        self.flat_grad.zero_()
        for i, feats in enumerate(self.slots):
            out = self.net(dict(feats))
            loss = self.loss_fn(out)
            del out                                  # with the backward below, frees the window's activations before the next
            prev, _kernels.GRAD_ACCUMULATE_INPLACE = _kernels.GRAD_ACCUMULATE_INPLACE, True     # wgrad kernels add into the flat buffer
            try:
                loss.backward()                      # AccumulateGrad adds into the param.grad views of the flat buffer
            finally:
                _kernels.GRAD_ACCUMULATE_INPLACE = prev
                # the convolution weight gradients added on the side stream are complete before anything reads the buffer;
                # joining once per window also frees the activation planes they read before the next window's forward
                _kernels.join_side_stream()
            if i == 0:
                self.loss.copy_(loss.detach().float())
            else:
                self.loss.add_(loss.detach().float())
            del loss
        if self.accumulate > 1:
            self.loss.div_(self.accumulate)
        if self.world > 1 and self.opt is None and self.chunks > 1:
            # optional (DFOLD_ALLREDUCE_CHUNKS > 1): the gradient exchange in pieces, the Adam update of piece c running while
            # piece c + 1 is on the wire.  Smaller NCCL operations can lose more than the hidden Adam update gains, and
            # the single 738 MB all-reduce is the default.
            n = self.flat_grad.numel()
            per = (n // self.chunks + 3) // 4 * 4
            bounds = [(a, min(n, a + per)) for a in range(0, n, per)]
            works = [dist.all_reduce(self.flat_grad[a:b], async_op=True) for a, b in bounds]
            for c, ((a, b), w) in enumerate(zip(bounds, works)):
                w.wait()
                self._adam(a, b, tick=(c == 0))
            _kernels.invalidate_weight_cache()
        else:
            if self.world > 1:
                dist.all_reduce(self.flat_grad)
            if self.opt is not None and self.grad_scale != 1.0:
                self.flat_grad.mul_(self.grad_scale)        # (the fused optimizer scales the summed gradient on the fly)
            self.optimizer_step()

    def _schedule_lr(self, step: torch.Tensor):
        """current_lr = the schedule's lr at `step` optimizer steps taken (device counter, read before this step's tick)."""
        s = self.schedule
        _kernels.launch("dfold_lr_schedule", step, s.base_lr, s.max_lr, s.warmup_no_steps, s.start_decay_after_n_steps,
                        s.decay_every_n_steps, s.decay_factor, self.current_lr)

    def _adam(self, a: int, b: int, tick: bool):
        coef = None if self.max_grad_norm is None else self.clip_coef
        if self.schedule is not None:
            if tick:
                self._schedule_lr(self.step_count)
            _kernels.launch("dfold_adam_amsgrad_dlr", self.flat_param[a:b], self.flat_grad[a:b], self.exp_avg[a:b],
                            self.exp_avg_sq[a:b], self.max_exp_avg_sq[a:b], b - a, self.step_count, 1 if tick else 0,
                            self.current_lr, 0.9, 0.999, 1e-8, self.grad_scale, coef)
            return
        args = (self.flat_param[a:b], self.flat_grad[a:b], self.exp_avg[a:b], self.exp_avg_sq[a:b], self.max_exp_avg_sq[a:b],
                b - a, self.step_count, 1 if tick else 0, self.lr, 0.9, 0.999, 1e-8, self.grad_scale)
        if coef is None:
            _kernels.launch("dfold_adam_amsgrad", *args)
        else:
            _kernels.launch("dfold_adam_amsgrad_clip", *args, coef)

    def optimizer_step(self):
        if self.opt is not None:
            if self.max_grad_norm is not None:
                # no host synchronisation with error_if_nonfinite=False, so this stays inside the captured graph
                self.grad_norm.copy_(torch.nn.utils.clip_grad_norm_(self.params, self.max_grad_norm, foreach=True))
            if self.schedule is not None:
                st = self.opt.state.get(self.params[0])          # Adam creates its state on its first step
                self._schedule_lr(st["step"] if st else self._step0)
            self.opt.step()
            return
        n = self.flat_param.numel()
        if self.max_grad_norm is not None:
            _kernels.launch("dfold_grad_norm", self.flat_grad, n, self.grad_scale, self.max_grad_norm, self.norm_partial,
                            self.grad_norm, self.clip_coef)
        self._adam(0, n, tick=True)
        _kernels.invalidate_weight_cache()                # the weights moved without touching their version counters

    def load(self, feats: Dict[str, torch.Tensor], slot: int = 0):
        """Copy a new window into the static input buffers of `slot` (0 ... accumulate - 1; H2D when `feats` is pinned host
        memory).  A step uses the windows of all its slots."""
        if isinstance(slot, bool) or not isinstance(slot, numbers.Integral) or not 0 <= slot < self.accumulate:
            raise IndexError(f"slot {slot!r} out of range: the step has {self.accumulate} input slot(s)")
        for k, v in feats.items():
            self.slots[slot][k].copy_(v, non_blocking=True)

    def __call__(self) -> torch.Tensor:
        if self.graph is not None:
            self.graph.replay()
            _kernels.invalidate_weight_cache()      # the replay moved the weights without touching their version counters
        else:
            self._eager()
        return self.loss

    def _host_flat(self, tensors) -> torch.Tensor:
        """Per-parameter device tensors (in self.params order) gathered into one host buffer of the flat layout."""
        flat = torch.zeros(self.layout.numel, dtype=torch.float32)
        with torch.no_grad():
            for t, v in zip(tensors, (v for v in _ckpt.views(self.layout, flat) if v is not None)):
                v.copy_(t)
        return flat

    def state_dict(self) -> Dict[str, object]:
        """``{'model': net.state_dict() on the host, 'optimizer': torch.optim.Adam(net.parameters(), lr,
        amsgrad=True).state_dict()}`` (checkpoint.py).  Each flat buffer is copied to the host once; the per-parameter
        tensors are views of those copies."""
        if self.opt is None:
            flat = [t.cpu() for t in (self.flat_param, self.exp_avg, self.exp_avg_sq, self.max_exp_avg_sq)]
            step = float(self.step_count)
        else:
            flat = [self._host_flat(self.params)] + [self._host_flat(self.opt.state[p][k] for p in self.params)
                                                     for k in _ckpt.MOMENTS]
            step = float(self.opt.state[self.params[0]]["step"])     # foreach Adam advances every parameter's step together
        trained = {n: v for n, v in zip(self.layout.names, _ckpt.views(self.layout, flat[0])) if v is not None}
        model = {k: trained[k] if k in trained else v.detach().cpu() for k, v in self.net.state_dict().items()}
        if self.schedule is None:
            opt = _ckpt.optimizer_state_dict(self.layout, *flat[1:], step, self.lr)
        else:       # the lr the next step uses, and the optimizer's lr from before the scheduler, as LRScheduler leaves them
            opt = _ckpt.optimizer_state_dict(self.layout, *flat[1:], step, self.schedule.lr(int(step)), initial_lr=self.lr)
        return {"model": model, "optimizer": opt}

    def load_state_dict(self, sd: Dict[str, object]) -> None:
        """Loads ``state_dict()``'s dict or a checkpoint of the reference trainer (``module.`` prefixes, a non-capturable
        optimizer's CPU ``step``) IN PLACE: the captured graph holds pointers to the parameter, moment and step buffers,
        and keeps replaying them.  No ``optimizer`` (or None) is a weights-only warm start with zero moments and step.
        Everything is validated before the first write (checkpoint.check_state): a refused load raises ValueError and
        leaves the step as it was.  Every data-parallel rank loads the same file, so no collective is needed.  With a
        schedule, the checkpoint's lr must be the schedule's lr at its step: a run saved under another schedule is refused."""
        model, entries, step = _ckpt.check_state(sd, self.layout, {k: v.shape for k, v in self.net.state_dict().items()},
                                                 self.lr, self.schedule)
        moments = _ckpt.optimizer_to_flat(self.layout, entries)
        trained = {n for n, o in zip(self.layout.names, self.layout.offsets) if o is not None}
        with torch.no_grad():
            if self.opt is None:
                self.flat_param.copy_(_ckpt.model_to_flat(self.layout, model))
                for buf, m in zip((self.exp_avg, self.exp_avg_sq, self.max_exp_avg_sq), moments):
                    buf.copy_(m)
                self.step_count.fill_(step)
            else:
                per = [[v for v in _ckpt.views(self.layout, m) if v is not None] for m in moments]
                for j, p in enumerate(self.params):
                    st = self.opt.state[p]
                    for k, src in zip(_ckpt.MOMENTS, per):
                        st[k].copy_(src[j])
                    st["step"].fill_(step)
            for k, v in self.net.state_dict().items():
                if self.opt is not None or k not in trained:
                    v.copy_(model[k])
            if self.current_lr is not None:
                self.current_lr.fill_(self.schedule.lr(int(step)))
        _kernels.invalidate_weight_cache()          # no bf16 weight plane from before the load may be reused
        torch.cuda.synchronize()


def _check_max_grad_norm(v) -> Optional[float]:
    """None, or a positive number (``math.inf`` reports the norm without clipping, torch's idiom)."""
    if v is None:
        return None
    if isinstance(v, bool) or not isinstance(v, numbers.Real) or not float(v) > 0:      # (NaN fails the comparison)
        raise ValueError(f"max_grad_norm must be None or a positive number (math.inf: report the norm only), got {v!r}")
    return float(v)
