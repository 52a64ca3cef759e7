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
* ``state_dict()`` / ``load_state_dict()`` save and resume the weights and the Adam(amsgrad) state in the reference
  trainer's checkpoint format, loading in place so the captured graph keeps running (checkpoint.py).
"""
import copy
import os
import sys
import time
from typing import Callable, Dict, Optional

import torch
import torch.distributed as dist

from . import checkpoint as _ckpt
from . import kernels as _kernels


class TrainStep:
    def __init__(self, net: torch.nn.Module, loss_fn: Callable[[Dict[str, torch.Tensor]], torch.Tensor],
                 example_feats: Dict[str, torch.Tensor], *, lr: float = 1e-4, world_size: int = 1, graph: bool = True,
                 warmup: int = 3):
        self.net, self.loss_fn, self.world = net, loss_fn, world_size
        self.params = [p for p in net.parameters() if p.requires_grad]
        self.layout = _ckpt.flat_layout(net)             # where each trained parameter sits in the flat buffers
        dev = self.params[0].device
        padded = self.layout.numel                         # padded to a multiple of 4: the fused optimizer runs float4-wide
        self.flat_grad = torch.zeros(padded, dtype=torch.float32, device=dev)
        # Adam(amsgrad) as the reference trainer (train_DFOLD_dynamics.py:412).  Default: ONE fused kernel over flat
        # parameter / gradient / moment buffers (csrc/simt.cu adam_amsgrad_kernel, step counter on the device); with
        # DFOLD_TORCH_ADAM=1: torch.optim.Adam(capturable, foreach) on the same gradient views.
        self.fused_adam = os.environ.get("DFOLD_TORCH_ADAM", "0") != "1"
        self.lr = lr
        self.chunks = max(1, int(os.environ.get("DFOLD_ALLREDUCE_CHUNKS", "1")))
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
            self.opt = torch.optim.Adam(self.params, lr=lr, amsgrad=True, capturable=True, foreach=True)
        self.static = {k: v.clone() for k, v in example_feats.items()}
        self.loss = torch.zeros((), dtype=torch.float32, device=dev)
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
                with torch.cuda.graph(g):
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
        _kernels.invalidate_weight_cache()
        torch.cuda.synchronize()

    def _eager(self):
        self.flat_grad.zero_()
        out = self.net(dict(self.static))
        loss = self.loss_fn(out)
        prev, _kernels.GRAD_ACCUMULATE_INPLACE = _kernels.GRAD_ACCUMULATE_INPLACE, True     # wgrad kernels add into the flat buffer
        try:
            loss.backward()
        finally:
            _kernels.GRAD_ACCUMULATE_INPLACE = prev
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
                if self.opt is not None:
                    self.flat_grad.mul_(1.0 / self.world)   # (the fused optimizer scales the summed gradient on the fly)
            self.optimizer_step()
        self.loss.copy_(loss.detach().float())

    def _adam(self, a: int, b: int, tick: bool):
        K = _kernels
        K._check(K.lib().dfold_adam_amsgrad(K._ptr(self.flat_param, a), K._ptr(self.flat_grad, a), K._ptr(self.exp_avg, a),
                                            K._ptr(self.exp_avg_sq, a), K._ptr(self.max_exp_avg_sq, a), b - a,
                                            K._ptr(self.step_count), 1 if tick else 0, self.lr, 0.9, 0.999, 1e-8,
                                            1.0 / self.world, K._stream()), "dfold_adam_amsgrad")

    def optimizer_step(self):
        if self.opt is not None:
            self.opt.step()
            return
        self._adam(0, self.flat_param.numel(), tick=True)
        _kernels.invalidate_weight_cache()                # the weights moved without touching their version counters

    def load(self, feats: Dict[str, torch.Tensor]):
        """Copy a new window into the static input buffers (H2D when `feats` is pinned host memory)."""
        for k, v in feats.items():
            self.static[k].copy_(v, non_blocking=True)

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
        return {"model": model, "optimizer": _ckpt.optimizer_state_dict(self.layout, *flat[1:], step, self.lr)}

    def load_state_dict(self, sd: Dict[str, object]) -> None:
        """Loads ``state_dict()``'s dict or a checkpoint of the reference trainer (``module.`` prefixes, a non-capturable
        optimizer's CPU ``step``) IN PLACE: the captured graph holds pointers to the parameter, moment and step buffers,
        and keeps replaying them.  No ``optimizer`` (or None) is a weights-only warm start with zero moments and step.
        Everything is validated before the first write (checkpoint.check_state): a refused load raises ValueError and
        leaves the step as it was.  Every data-parallel rank loads the same file, so no collective is needed."""
        model, entries, step = _ckpt.check_state(sd, self.layout, {k: v.shape for k, v in self.net.state_dict().items()},
                                                 self.lr)
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
        _kernels.invalidate_weight_cache()          # no bf16 weight plane from before the load may be reused
        torch.cuda.synchronize()
