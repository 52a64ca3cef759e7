"""-m gpu: the training-recipe options of the captured training step, TrainStep(lr_schedule=..., accumulate=...).

* dfold_lr_schedule gives fp32 of the reference AlphaFoldLRScheduler's lr (tests/golden/lr_schedule.pt) bit for bit, with
  the device step counter written directly; dfold_adam_amsgrad_dlr with a device lr of fp32(x) gives the bits of
  dfold_adam_amsgrad / dfold_adam_amsgrad_clip called with lr = x.
* Under a schedule (tiny preset, warmup 4, start 7, every 2, 12 steps) every captured step equals dfold_adam_amsgrad called
  directly with the host-computed lr on the step's own gradient, and the eagerly launched step, bit for bit (with and
  without max_grad_norm); DFOLD_TORCH_ADAM=1 is within the per-element Adam bound of tests/test_gpu_simt.py.
* accumulate=k (2, 4; tiny preset and preset A at 8 x 64): the flat gradient is the sum of the k single-window gradients
  of an accumulate=1 step up to k u sum |g_i| per element (plus (k + 1) B u times the summed magnitude of the in-place adds
  of the shared convolution weights, B per window), the loss is the mean of the k losses, replays repeat their
  bits, every param.grad stays a view of the flat buffer, and the peak memory grows only by the extra input slots.
* Checkpoints under a schedule resume bit for bit, a different schedule is refused without a write, and a checkpoint of
  torch.optim.Adam + an LRScheduler (initial_lr in its param group) loads.
"""
import copy
import gc
import math
import os

import pytest
import torch

from dynamicpdb_b200 import checkpoint as C
from dynamicpdb_b200 import kernels as K
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.train_step import AlphaFoldSchedule, TrainStep
from tests.test_gpu_checkpoint import PRESETS, _assert_same, _net, _snapshot
from tests.test_gpu_grad_clip import _assert_bits, _state
from tests.test_gpu_simt import DEV, U, _adam_ref, _ok, _within

pytestmark = pytest.mark.gpu
GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lr_schedule.pt"))
LR = 1e-4
RECIPE = AlphaFoldSchedule(**GOLD["settings"]["recipe"]["kwargs"])        # warmup 4, start 7, every 2
N_STEPS = 12


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _windows(preset, n, seed=40):
    _, nf, N = PRESETS[preset]
    return [{k: v.cuda() for k, v in syn.make_feats(nf, N, seed=seed + i).items()} for i in range(n)]


# --------------------------------------------------------------------------------------------------
# kernels
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setting", sorted(GOLD["settings"]))
def test_schedule_kernel_matches_reference(setting):
    g = GOLD["settings"][setting]
    s = AlphaFoldSchedule(**g["kwargs"])
    steps = torch.tensor(g["steps"], dtype=torch.float32, device=DEV)
    assert steps.cpu().long().tolist() == g["steps"]                       # exact as fp32 counters
    out = torch.full((len(g["steps"]),), float("nan"), device=DEV)
    for i in range(len(g["steps"])):
        K.launch("dfold_lr_schedule", K._ptr(steps, i), s.base_lr, s.max_lr, s.warmup_no_steps, s.start_decay_after_n_steps,
                 s.decay_every_n_steps, s.decay_factor, K._ptr(out, i))
    torch.cuda.synchronize()
    want = torch.tensor(g["lr"], dtype=torch.float64).float()
    bad = [(st, float(o), float(w)) for st, o, w in zip(g["steps"], out.cpu(), want)
           if torch.tensor(float(o)).view(torch.int32) != torch.tensor(float(w)).view(torch.int32)]
    assert not bad and torch.equal(out.cpu().view(torch.int32), want.view(torch.int32)), bad[:5]


def test_schedule_kernel_refuses_bad_settings():
    L = K.lib()
    step, out = torch.zeros((), device=DEV), torch.full((), float("nan"), device=DEV)
    for args in ((0.0, 1e-3, 0, 5, 1, 0.9), (0.0, 1e-3, 4, 5, 0, 0.9), (0.0, 1e-3, 6, 5, 1, 0.9), (0.0, 0.0, 4, 5, 1, 0.9),
                 (0.0, math.inf, 4, 5, 1, 0.9), (0.0, math.nan, 4, 5, 1, 0.9)):
        assert L.dfold_lr_schedule(K._ptr(step), *args, K._ptr(out), K._stream()) != 0, args
    assert L.dfold_lr_schedule(None, 0.0, 1e-3, 4, 5, 1, 0.9, K._ptr(out), K._stream()) != 0
    g = torch.zeros(8, device=DEV)
    assert L.dfold_adam_amsgrad_dlr(*(K._ptr(g),) * 5, 8, K._ptr(step), 1, None, 0.9, 0.999, 1e-8, 1.0, None, K._stream()) != 0
    assert "null learning rate" in L.dfold_last_error().decode()
    torch.cuda.synchronize()
    assert torch.isnan(out) and float(step) == 0.0


@pytest.mark.parametrize("clip", [False, True])
def test_device_lr_adam_equals_by_value_lr(clip):
    n = 4096 + 8
    gen = torch.Generator(device=DEV).manual_seed(3)
    ref = [torch.randn(n, generator=gen, device=DEV)] + [torch.zeros(n, device=DEV) for _ in range(3)]
    dev = [b.clone() for b in ref]
    s_ref, s_dev = torch.zeros((), device=DEV), torch.zeros((), device=DEV)
    coef = torch.tensor(0.37, device=DEV) if clip else None
    lr_dev = torch.empty((), device=DEV)
    for it, lr in enumerate((3e-4, 1e-3 / 3, 0.95 ** 7 * 1e-3, 2.5e-5)):
        grad = torch.randn(n, generator=gen, device=DEV) * 10.0 ** (it - 2)
        lr_dev.fill_(lr)
        if clip:
            K.launch("dfold_adam_amsgrad_clip", ref[0], grad, *ref[1:], n, s_ref, 1, lr, 0.9, 0.999, 1e-8, 0.5, coef)
        else:
            K.launch("dfold_adam_amsgrad", ref[0], grad, *ref[1:], n, s_ref, 1, lr, 0.9, 0.999, 1e-8, 0.5)
        K.launch("dfold_adam_amsgrad_dlr", dev[0], grad, *dev[1:], n, s_dev, 1, lr_dev, 0.9, 0.999, 1e-8, 0.5, coef)
        torch.cuda.synchronize()
        assert float(s_ref) == float(s_dev) == it + 1
        _assert_bits(ref, dev, f"device lr against by-value lr, step {it + 1}")


# --------------------------------------------------------------------------------------------------
# TrainStep(lr_schedule=...)
# --------------------------------------------------------------------------------------------------
def _make(preset, seed=0, windows=None, **kw):
    windows = windows or _windows(preset, 1)
    kw.setdefault("graph", True)
    ts = TrainStep(_net(preset, seed), syn.surrogate_loss, windows[0], lr=kw.pop("lr", LR), warmup=2, **kw)
    assert (ts.graph is not None) == kw["graph"], ts.graph_error
    return ts


@pytest.mark.parametrize("max_grad_norm", [None, 1e-3])
def test_scheduled_step_against_by_value_adam_and_eager(max_grad_norm):
    windows = _windows("tiny", N_STEPS)
    runs = []
    for graph in (True, False):
        ts = _make("tiny", windows=windows, graph=graph, lr_schedule=RECIPE, max_grad_norm=max_grad_norm)
        assert float(ts.current_lr) == _f32(RECIPE.lr(0))
        losses = []
        for k, w in enumerate(windows, 1):
            ts.load(w)
            before = [t.clone() for t in (ts.flat_param, ts.exp_avg, ts.exp_avg_sq, ts.max_exp_avg_sq, ts.step_count)]
            losses.append(ts().clone())
            torch.cuda.synchronize()
            assert float(ts.step_count) == k
            assert float(ts.current_lr) == _f32(RECIPE.lr(k - 1)), k
            if graph:                   # the same update from the by-value entry point, on the step's own gradient
                args = (before[0], ts.flat_grad, *before[1:4], ts.flat_grad.numel(), before[4], 1, RECIPE.lr(k - 1), 0.9,
                        0.999, 1e-8, 1.0)
                if max_grad_norm is None:
                    K.launch("dfold_adam_amsgrad", *args)
                else:
                    K.launch("dfold_adam_amsgrad_clip", *args, ts.clip_coef)
                torch.cuda.synchronize()
                _assert_bits(before[:4], [ts.flat_param, ts.exp_avg, ts.exp_avg_sq, ts.max_exp_avg_sq],
                             f"step {k} against dfold_adam_amsgrad(lr={RECIPE.lr(k - 1)!r})")
        if max_grad_norm is not None:
            assert float(ts.clip_coef) < 1.0                               # clipping is active
        runs.append((torch.stack(losses), _state(ts)))
        del ts
        torch.cuda.empty_cache()
    assert torch.equal(runs[0][0].view(torch.int32), runs[1][0].view(torch.int32))
    _assert_bits(runs[0][1], runs[1][1], "graph replay against eager scheduled steps")


def test_scheduled_torch_adam_within_the_adam_bound(monkeypatch):
    monkeypatch.setenv("DFOLD_TORCH_ADAM", "1")
    windows = _windows("tiny", N_STEPS)
    ts = _make("tiny", windows=windows, lr_schedule=RECIPE)
    assert ts.opt.param_groups[0]["lr"] is ts.current_lr and ts.current_lr.is_cuda
    worst = 0.0
    for k, w in enumerate(windows, 1):
        ts.load(w)
        before = [b.double() for b in _state(ts)]
        ts()
        torch.cuda.synchronize()
        assert float(ts.current_lr) == _f32(RECIPE.lr(k - 1)), k
        refs, errs = _adam_ref(before[0], ts.flat_grad.double(), *before[1:], k, _f32(RECIPE.lr(k - 1)), 0.9, 0.999, 1e-8,
                               1.0)
        for name, f, r, e in zip(("p", "m", "v", "vmax"), _state(ts), refs, errs):
            worst = max(worst, _within(f"torch Adam step {k} {name}", (f.double() - r).abs(), e, "adam"))
    assert worst > 0


# --------------------------------------------------------------------------------------------------
# TrainStep(accumulate=k)
# --------------------------------------------------------------------------------------------------
def _peak(make):
    """(object, peak bytes allocated on top of what was live before, while it was built and stepped once)."""
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    obj = make()
    torch.cuda.synchronize()
    return obj, torch.cuda.max_memory_allocated() - base


def _grads_are_views(ts):
    lo = ts.flat_grad.data_ptr()
    hi = lo + ts.flat_grad.numel() * 4
    for p in ts.params:
        assert lo <= p.grad.data_ptr() and p.grad.data_ptr() + p.grad.numel() * 4 <= hi


def _spy_on_inplace_wgrad(monkeypatch):
    """The convolution's weight gradients are added into the flat buffer in place, one add per use of the shared weight
    (GRAD_ACCUMULATE_INPLACE), so even one window's gradient there is a rounded sum of several contributions, and its
    rounding is bounded by their magnitudes, not by the window's sum.  This spy adds |each contribution| into a buffer of
    the flat layout (installed before the step is built, the adds are part of the captured graph) and counts the adds."""
    real, seen = K.launch, {"adds": {}}

    def spy(name, *args):
        real(name, *args)
        if name == "dfold_taps_to_param" and args[-1] == 1:
            taps, Co, Ci, T, acc = args[:5]
            part = torch.empty_like(acc)
            real(name, taps, Co, Ci, T, part, 0)
            base = acc._base                                    # the step's flat gradient buffer
            if "abs" not in seen:
                seen["abs"] = torch.zeros_like(base)            # first called by an eager warm-up step, before capture
            off = (acc.data_ptr() - base.data_ptr()) // 4
            seen["abs"][off:off + acc.numel()].add_(part.reshape(-1).abs())
            seen["adds"][off] = seen["adds"].get(off, 0) + 1

    monkeypatch.setattr(K, "launch", spy)
    return seen


@pytest.mark.parametrize("preset,k", [("tiny", 2), ("tiny", 4), ("A", 2), ("A", 4)])
def test_accumulated_gradient_is_the_window_mean(preset, k, monkeypatch):
    """lr = 0 keeps the parameters where they are (Adam moves them by 0 x its update), so the single-window step sees
    every window at the same weights as the accumulated step.  An element autograd accumulates gets one add per window:
    |sum - sum_i g_i| <= (k - 1) u sum_i |g_i|.  An element of a convolution weight gets B in-place adds per window, in
    window order: the accumulated sum of k B terms and each window's sum of B terms together round by at most
    (k B + B) u sum |c| over all contributions c (first order; the bound below has k u, and (k + 1) B u)."""
    windows = _windows(preset, k)
    ts = _make(preset, windows=windows, lr=0.0)
    grads, losses = [], []
    for w in windows:
        ts.load(w)
        losses.append(ts().clone())
        grads.append(ts.flat_grad.clone())
    del ts
    gsum = torch.zeros_like(grads[0], dtype=torch.float64)
    gabs = torch.zeros_like(gsum)
    for g in grads:
        gsum += g.double()
        gabs += g.double().abs()
    del grads

    seen = _spy_on_inplace_wgrad(monkeypatch)
    ts = _make(preset, windows=windows, lr=0.0, accumulate=k)
    calls = set(seen["adds"].values())
    assert len(calls) == 1 and next(iter(calls)) % (3 * k) == 0, calls        # 2 warm-up steps + the capture
    B = next(iter(calls)) // (3 * k)
    for i, w in enumerate(windows):
        ts.load(w, slot=i)
    with pytest.raises(IndexError):
        ts.load(windows[0], slot=k)
    seen["abs"].zero_()
    ts()
    torch.cuda.synchronize()
    first = ts.flat_grad.clone()
    bound = k * U * gabs + (k + 1) * B * U * seen["abs"].double()
    _within(f"accumulate={k} {preset} gradient", (first.double() - gsum).abs(), bound, "accumulate")
    mean_loss = losses[0]
    for l in losses[1:]:
        mean_loss = mean_loss + l
    assert torch.equal((mean_loss / k).view(torch.int32), ts.loss.view(torch.int32)), (float(ts.loss), float(mean_loss / k))
    ts()                                                        # same weights, same windows: the same bits again
    torch.cuda.synchronize()
    assert torch.equal(first.view(torch.int32), ts.flat_grad.view(torch.int32))
    _grads_are_views(ts)


@pytest.mark.parametrize("preset", ["tiny", "A"])
def test_accumulate_memory(preset):
    """The peak while building the step and running it once: accumulate=4 needs no more than accumulate=1 plus the three
    extra input slots, plus 10 %."""
    windows = _windows(preset, 4)

    def build_and_step(**kw):
        ts = _make(preset, windows=windows, **kw)
        ts()
        return ts

    ts, peak1 = _peak(build_and_step)
    del ts
    slot_bytes = sum(v.numel() * v.element_size() for v in windows[0].values())
    ts, peak4 = _peak(lambda: build_and_step(accumulate=4))
    assert peak4 <= 1.1 * (peak1 + 3 * slot_bytes), (peak1, peak4, slot_bytes)


def test_accumulate_one_is_the_default_step():
    windows = _windows("tiny", 3)
    runs = []
    for kw in ({}, {"accumulate": 1}):
        ts = _make("tiny", windows=windows, **kw)
        losses = []
        for w in windows:
            ts.load(w)
            losses.append(ts().clone())
        torch.cuda.synchronize()
        runs.append((torch.stack(losses), ts.flat_grad.clone(), _state(ts)))
        del ts
    assert torch.equal(runs[0][0].view(torch.int32), runs[1][0].view(torch.int32))
    _assert_bits([runs[0][1]] + runs[0][2], [runs[1][1]] + runs[1][2], "accumulate=1 against the default")


# --------------------------------------------------------------------------------------------------
# checkpoints under a schedule
# --------------------------------------------------------------------------------------------------
def _run(ts, windows):
    out = []
    for w in windows:
        ts.load(w)
        out.append(ts().clone())
    torch.cuda.synchronize()
    return torch.stack(out).cpu()


def test_scheduled_resume_is_bit_exact(tmp_path):
    windows = _windows("tiny", 7)
    ts = _make("tiny", windows=windows, lr_schedule=RECIPE)                # uninterrupted: 2 + 5 steps
    _run(ts, windows[:2])
    losses_a = _run(ts, windows[2:])
    state_a = _snapshot(ts) + [ts.current_lr.cpu()]
    del ts
    ts = _make("tiny", windows=windows, lr_schedule=RECIPE)
    _run(ts, windows[:2])                                                  # step 2: mid-warmup
    sd = ts.state_dict()
    assert sd["optimizer"]["param_groups"][0]["lr"] == RECIPE.lr(2) and sd["optimizer"]["param_groups"][0]["initial_lr"] == LR
    path = str(tmp_path / "step_2.pth")
    C.save_checkpoint(path, ts, None, 0, 2)
    del ts
    ts = _make("tiny", seed=5, windows=windows, lr_schedule=RECIPE)
    captured = ts.graph
    assert C.load_checkpoint(path, ts) == (0, 2)
    assert float(ts.current_lr) == _f32(RECIPE.lr(2))
    losses_b = _run(ts, windows[2:])
    assert ts.graph is captured
    assert torch.equal(losses_a, losses_b), (losses_a, losses_b)
    _assert_same(state_a, _snapshot(ts) + [ts.current_lr.cpu()], "state after resuming under the schedule")


@pytest.mark.parametrize("torch_adam", ["0", "1"])
def test_other_schedule_is_refused_without_a_write(torch_adam, monkeypatch):
    monkeypatch.setenv("DFOLD_TORCH_ADAM", torch_adam)
    windows = _windows("tiny", 3)
    ts = _make("tiny", windows=windows, lr_schedule=RECIPE)
    _run(ts, windows[:2])
    sd = ts.state_dict()
    _run(ts, windows[2:])
    before = _snapshot(ts) + [ts.current_lr.cpu()]
    other = copy.deepcopy(sd)
    other["optimizer"]["param_groups"][0]["lr"] = AlphaFoldSchedule(max_lr=2e-3, warmup_no_steps=4,
                                                                     start_decay_after_n_steps=7).lr(2)
    for bad in (other, {"model": sd["model"], "optimizer": dict(sd["optimizer"], param_groups=[
            dict(sd["optimizer"]["param_groups"][0], lr=LR)])}):
        with pytest.raises(ValueError, match="different schedule"):
            ts.load_state_dict(bad)
        _assert_same(before, _snapshot(ts) + [ts.current_lr.cpu()], "after a refused load")
    ts.load_state_dict(sd)
    assert float(ts.current_lr) == _f32(RECIPE.lr(2))


class _TorchAlphaFold(torch.optim.lr_scheduler.LRScheduler):
    """A torch LRScheduler with AlphaFold's schedule: what a trainer stepping the reference's scheduler leaves in the
    optimizer (initial_lr in the param group, lr = f(steps taken))."""

    def __init__(self, optimizer, schedule):
        self.schedule = schedule
        super().__init__(optimizer)

    def get_lr(self):
        return [self.schedule.lr(self.last_epoch) for _ in self.optimizer.param_groups]


def test_reference_style_checkpoint_loads(tmp_path):
    windows = _windows("tiny", 4)
    ref = _net("tiny", 0)
    opt = torch.optim.Adam(ref.parameters(), lr=LR, amsgrad=True)
    sched = _TorchAlphaFold(opt, RECIPE)
    for w in windows[:3]:
        opt.zero_grad()
        syn.surrogate_loss(ref(dict(w))).backward()
        opt.step()
        sched.step()
    g = opt.state_dict()["param_groups"][0]
    assert g["initial_lr"] == LR and g["lr"] == RECIPE.lr(3)
    path = str(tmp_path / "ref.pth")
    torch.save({"model": {"module." + k: v for k, v in ref.state_dict().items()}, "conf": None,
                "optimizer": opt.state_dict(), "epoch": 1, "step": 3}, path)
    ts = _make("tiny", seed=5, windows=windows, lr_schedule=RECIPE)
    assert C.load_checkpoint(path, ts) == (1, 3)
    assert float(ts.step_count) == 3 and float(ts.current_lr) == _f32(RECIPE.lr(3))
    _run(ts, windows[3:])
    assert float(ts.step_count) == 4 and float(ts.current_lr) == _f32(RECIPE.lr(3))
