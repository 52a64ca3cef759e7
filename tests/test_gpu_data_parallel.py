"""-m gpu: the data-parallel training step, TrainStep(world_size > 1), across real ranks.

Every rank's flat gradient before the exchange is the world-1 gradient of its own window(s) (fixed-order kernels), and at
world 2 the all-reduced sum is one correctly rounded fp32 add, the same bits whichever backend or algorithm adds the two
buffers.  So the expected state after every step is built in this process: a world-1 TrainStep(lr=0.0) at the current
weights gives each rank's gradient g_r (lr = 0 leaves the weights in place), g = fl(g_0 + g_1), and the C-ABI update the
step should run (dfold_adam_amsgrad, dfold_grad_norm + dfold_adam_amsgrad_clip, dfold_lr_schedule +
dfold_adam_amsgrad_dlr) moves this process's own copy of the parameters and moments with grad_scale = 1 / (world k).
Every rank must equal it bit for bit after every step: parameters, the three moments, the summed gradient, step, lr, norm
and clipping coefficient, and its loss the world-1 loss of its window.  Cases (tiny preset unless noted, a different
window per rank and step): the fused Adam; max_grad_norm 1e-3 (clipping active) and inf; the golden's recipe schedule over
its warmup; accumulate=2 (grad_scale 1/4); DFOLD_ALLREDUCE_CHUNKS 2, 3, 7 with and without the schedule (also the bits of
the unchunked run); preset A at 8 x 64, plain and in 3 pieces; a resume on both ranks from rank 0's state_dict.
DFOLD_TORCH_ADAM=1 leaves fl(g_0 + g_1) / 2 in the gradient buffer bit for bit, and its update lies within the float64
Adam bound of tests/test_gpu_simt.py.  At world 3 the reduction order is unspecified: the sum is held to
2u sum_r |g_r| of the float64 sum, the update to the Adam bound, and the ranks to each other's bits.

Two arms.  gloo on one GPU: every rank on cuda:0, eager steps (gloo's all-reduce takes CUDA tensors, the chunked path's
async_op=True slices included; a graph cannot capture it).  NCCL with two or more GPUs: one rank per device, captured
steps (the plain, scheduled and chunked cases, and captured against eager steps, bit for bit); skipped with fewer GPUs.

The ranks are spawned processes that meet through a FileStore (no port) and write their per-step state to disk: the fp32
scalars' bits, a digest of each flat buffer (_digest; one step of preset A is 3.7 GB of them), and host copies where a
bound is checked.  They are joined by a deadline, after which survivors are killed and the test fails.
"""
import datetime
import math
import os
import time
import traceback

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from dynamicpdb_b200 import kernels as K
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.train_step import TrainStep
from tests.test_gpu_checkpoint import PRESETS, _net
from tests.test_gpu_grad_clip import _state
from tests.test_gpu_simt import U, _adam_ref, _within
from tests.test_gpu_train_recipe import RECIPE

pytestmark = pytest.mark.gpu
LR = 1e-4
STEPS = 4
SCHED_STEPS = 6                     # RECIPE warms up over 4 steps: the lr at steps 1..6 is 0, 1/4, 1/2, 3/4, 1, 1 x max_lr
JOIN_S = 900                        # every worker of one launch must have finished by then
PG_TIMEOUT = datetime.timedelta(seconds=300)
NAMES = ("p", "m", "v", "x", "g")   # parameters, exp_avg, exp_avg_sq, max_exp_avg_sq, the flat gradient after the step


def _seed(rank, step, slot):
    """The window of `rank` in optimizer step `step` (1-based), accumulation slot `slot`: all different."""
    return 40 + 64 * step + 8 * rank + slot


def _window(preset, rank, step, slot=0):
    _, nf, N = PRESETS[preset]
    return {k: v.cuda() for k, v in syn.make_feats(nf, N, seed=_seed(rank, step, slot)).items()}


def _digest(t):
    """sum_i bits_i r_i mod 2^64 over the int32 bit patterns of fp32 `t`, with fixed odd pseudo-random int64 r_i: two
    tensors that differ in one element always differ here (r_i odd, |bits difference| < 2^32), and in several elements
    collide with probability at most 2^-32.  The same in every process (a seeded generator; integer sums are exact mod
    2^64, whatever their order)."""
    g = torch.Generator(device=t.device).manual_seed(20260401)
    r = torch.randint(-2 ** 62, 2 ** 62, (t.numel(),), generator=g, dtype=torch.int64, device=t.device) * 2 + 1
    return int((t.reshape(-1).view(torch.int32).long() * r).sum())


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _bits(t):
    return None if t is None else int(t.reshape(()).cpu().view(torch.int32))


# --------------------------------------------------------------------------------------------------
# the ranks
# --------------------------------------------------------------------------------------------------
def _record(ts, full):
    """One step's state: scalars as fp32 bit patterns, digests of the five buffers, host copies when `full`."""
    if ts.opt is None:
        bufs = [ts.flat_param, ts.exp_avg, ts.exp_avg_sq, ts.max_exp_avg_sq]
        step = float(ts.step_count)
    else:
        bufs = _state(ts)
        st = ts.opt.state.get(ts.params[0])
        step = float(st["step"]) if st else 0.0
    bufs = dict(zip(NAMES, bufs + [ts.flat_grad]))
    return {"loss": _bits(ts.loss), "step": step, "lr": _bits(ts.current_lr), "norm": _bits(ts.grad_norm),
            "coef": _bits(getattr(ts, "clip_coef", None)), "digest": {k: _digest(v) for k, v in bufs.items()},
            "full": {k: v.cpu() for k, v in bufs.items()} if full else None}


def _build(run, world, rank, seed=0):
    os.environ["DFOLD_ALLREDUCE_CHUNKS"] = str(run.get("chunks", 1))
    os.environ["DFOLD_TORCH_ADAM"] = "1" if run.get("torch_adam") else "0"
    ts = TrainStep(_net(run["preset"], seed), syn.surrogate_loss, _window(run["preset"], rank, 1), lr=LR, world_size=world,
                   graph=run["graph"], warmup=2 if run["graph"] else 1, max_grad_norm=run.get("max_grad_norm"),
                   lr_schedule=RECIPE if run.get("schedule") else None, accumulate=run.get("accumulate", 1))
    if run["graph"] and ts.graph is None:
        raise RuntimeError(f"{run['name']}: the step was not captured: {ts.graph_error}")
    return ts


def _steps(ts, run, rank, first, last, out, save=None):
    for k in range(first, last + 1):
        for s in range(ts.accumulate):
            ts.load(_window(run["preset"], rank, k, s), slot=s)
        ts()
        torch.cuda.synchronize()
        out.append(_record(ts, run.get("full", False) and rank == 0))
        if save is not None and k == save[0]:
            if rank == 0:
                torch.save(ts.state_dict(), save[1])
            dist.barrier()


def _worker(rank, world, backend, store_path, out_dir, runs):
    """Runs every entry of `runs` in turn at this rank; writes {name: [state after step 0, 1, ...]} to rank{rank}.pt, or
    the traceback to rank{rank}.err."""
    try:
        dev = rank if backend == "nccl" else 0
        torch.cuda.set_device(dev)
        if backend == "nccl":
            os.environ["TORCH_NCCL_ASYNC_ERROR_HANDLING"] = "0"            # capturing NCCL in a CUDA graph needs it
        store = dist.FileStore(store_path, world)
        dist.init_process_group(backend, store=store, rank=rank, world_size=world, timeout=PG_TIMEOUT,
                                **({"device_id": torch.device("cuda", dev)} if backend == "nccl" else {}))
        results = {}
        for run in runs:
            ts = _build(run, world, rank)
            out = [_record(ts, run.get("full", False) and rank == 0)]
            ckpt = os.path.join(out_dir, f"{run['name']}_state.pt") if run.get("save_at") else None
            _steps(ts, run, rank, 1, run["steps"], out, save=(run["save_at"], ckpt) if ckpt else None)
            results[run["name"]] = out
            del ts
            torch.cuda.empty_cache()
            if ckpt:                # a fresh step from other weights resumes from rank 0's state and runs the rest
                ts = _build(run, world, rank, seed=5)
                ts.load_state_dict(torch.load(ckpt))
                out = [_record(ts, False)]
                _steps(ts, run, rank, run["save_at"] + 1, run["steps"], out)
                results[run["name"] + "_resumed"] = out
                del ts
                torch.cuda.empty_cache()
        torch.save(results, os.path.join(out_dir, f"rank{rank}.pt"))
    except BaseException:                                                  # noqa: BLE001  (reported by the parent)
        with open(os.path.join(out_dir, f"rank{rank}.err"), "w") as f:
            f.write(traceback.format_exc())
        os._exit(1)
    if backend == "nccl":
        os._exit(0)                 # destroy_process_group blocks on a communicator a graph has captured (DESIGN.md §7)
    dist.destroy_process_group()


def _launch(out_dir, world, backend, runs):
    """Spawns the ranks and joins them by a deadline; survivors are terminated, then killed, and fail the test."""
    ctx = mp.get_context("spawn")
    store = os.path.join(out_dir, "store")
    procs = [ctx.Process(target=_worker, args=(r, world, backend, store, out_dir, runs)) for r in range(world)]
    for p in procs:
        p.start()
    deadline = time.monotonic() + JOIN_S
    try:
        for p in procs:
            p.join(max(0.0, deadline - time.monotonic()))
    finally:
        late = [r for r, p in enumerate(procs) if p.is_alive()]
        for p in procs:
            if p.is_alive():
                p.terminate()
        for p in procs:
            p.join(10)
            if p.is_alive():
                p.kill()
                p.join()
    errors = {r: open(os.path.join(out_dir, f"rank{r}.err")).read() for r in range(world)
              if os.path.exists(os.path.join(out_dir, f"rank{r}.err"))}
    assert not errors, "\n".join(f"rank {r}:\n{e}" for r, e in errors.items())
    assert not late, f"ranks {late} still running after {JOIN_S} s: terminated"
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    assert not ctx.active_children()
    return [torch.load(os.path.join(out_dir, f"rank{r}.pt")) for r in range(world)]


# --------------------------------------------------------------------------------------------------
# the expected state, built in this process
# --------------------------------------------------------------------------------------------------
class _Local:
    """World-1 TrainStep(lr=0.0) giving each rank's summed gradient and loss at given weights."""

    def __init__(self, preset, accumulate):
        self.preset = preset
        saved = os.environ.pop("DFOLD_TORCH_ADAM", None)         # the fused optimizer: flat_param is the weights
        try:
            self.ts = TrainStep(_net(preset, 0), syn.surrogate_loss, _window(preset, 0, 1), lr=0.0, graph=False,
                                warmup=1, accumulate=accumulate)
        finally:
            if saved is not None:
                os.environ["DFOLD_TORCH_ADAM"] = saved

    def grads(self, p, step, world):
        out = []
        for r in range(world):
            self.ts.flat_param.copy_(p)
            K.invalidate_weight_cache()
            for s in range(self.ts.accumulate):
                self.ts.load(_window(self.preset, r, step, s), slot=s)
            self.ts()
            out.append((self.ts.flat_grad.clone(), self.ts.loss.clone()))
        assert torch.equal(self.ts.flat_param, p)                      # lr = 0: the weights stayed where they were
        return out


_EMU = {}


def _emulate(preset, steps, world=2, accumulate=1, max_grad_norm=None, schedule=False):
    """[{"loss": [per rank], "step", "lr", "norm", "coef", "digest"}] after step 0, 1, ..., steps of the data-parallel run."""
    key = (preset, steps, world, accumulate, max_grad_norm, schedule)
    if key in _EMU:
        return _EMU[key]
    loc = _Local(preset, accumulate)
    p = loc.ts.flat_param.clone()
    n = p.numel()
    m, v, x = (torch.zeros_like(p) for _ in range(3))
    step = torch.zeros((), device=p.device)
    lr = torch.full((), RECIPE.lr(0), device=p.device) if schedule else None
    scale = 1.0 / (world * accumulate)
    norm = coef = None
    if max_grad_norm is not None:
        norm, coef = torch.zeros((), device=p.device), torch.ones((), device=p.device)
        work = torch.zeros(1024, dtype=torch.float64, device=p.device)
    g = torch.zeros_like(p)
    rec = lambda losses: {"loss": losses, "step": float(step), "lr": _bits(lr), "norm": _bits(norm), "coef": _bits(coef),
                          "digest": {k: _digest(t) for k, t in zip(NAMES, (p, m, v, x, g))}}
    out = [rec([None] * world)]
    for k in range(1, steps + 1):
        local = loc.grads(p, k, world)
        g = local[0][0]
        for g_r, _ in local[1:]:
            g = g + g_r
        if max_grad_norm is not None:
            K.launch("dfold_grad_norm", g, n, scale, max_grad_norm, work, norm, coef)
        if schedule:
            K.launch("dfold_lr_schedule", step, RECIPE.base_lr, RECIPE.max_lr, RECIPE.warmup_no_steps,
                     RECIPE.start_decay_after_n_steps, RECIPE.decay_every_n_steps, RECIPE.decay_factor, lr)
            K.launch("dfold_adam_amsgrad_dlr", p, g, m, v, x, n, step, 1, lr, 0.9, 0.999, 1e-8, scale, coef)
        elif max_grad_norm is not None:
            K.launch("dfold_adam_amsgrad_clip", p, g, m, v, x, n, step, 1, LR, 0.9, 0.999, 1e-8, scale, coef)
        else:
            K.launch("dfold_adam_amsgrad", p, g, m, v, x, n, step, 1, LR, 0.9, 0.999, 1e-8, scale)
        torch.cuda.synchronize()
        out.append(rec([_bits(l) for _, l in local]))
    del loc
    torch.cuda.empty_cache()
    _EMU[key] = out
    return out


def _assert_same_run(a, b, what, scalars=("loss", "step", "lr", "norm", "coef")):
    """Two runs' records (one rank's, or two ranks') with the same bits after every step."""
    assert len(a) == len(b), what
    for k, (x, y) in enumerate(zip(a, b)):
        bad = [f for f in scalars if x[f] != y[f]] + [f for f in NAMES if x["digest"][f] != y["digest"][f]]
        assert not bad, f"{what}, after step {k}: {bad} differ"


def _assert_matches(ranks, name, want, first=0):
    """Every rank's state after every step equals the emulation's bit for bit, and its loss the world-1 loss of its
    window(s).  `first`: the run starts after step `first` (a resumed run; its record 0 is the state it loaded)."""
    for r, recs in enumerate(ranks[1:], 1):
        _assert_same_run(ranks[0][name], recs[name], f"{name}: rank {r} against rank 0", scalars=("step", "lr", "norm", "coef"))
    for r, recs in enumerate(ranks):
        got = recs[name]
        assert len(got) == len(want) - first
        for k, (a, b) in enumerate(zip(got, want[first:]), first):
            what = f"{name}, rank {r}, after step {k}"
            assert a["step"] == b["step"] == k, (what, a["step"], b["step"])
            assert a["lr"] == b["lr"], f"{what}: lr differs from the emulation"
            if k > first:           # (record `first` holds what the construction or the load left: no step has run)
                assert a["loss"] == b["loss"][r], f"{what}: the loss differs from the world-1 loss of its window"
                for f in ("norm", "coef"):
                    assert a[f] == b[f], f"{what}: {f} differs from the emulation"
            bad = [f for f in NAMES if a["digest"][f] != b["digest"][f] and (k > first or f != "g")]
            assert not bad, f"{what}: {bad} differ from the emulation"


# --------------------------------------------------------------------------------------------------
# gloo, every rank on cuda:0, eager steps
# --------------------------------------------------------------------------------------------------
def _run(name, preset="tiny", steps=STEPS, **kw):
    return dict(name=name, preset=preset, steps=steps, graph=False, **kw)


GLOO_RUNS = [
    _run("plain", save_at=2),
    _run("clip_1e-3", max_grad_norm=1e-3),
    _run("clip_inf", max_grad_norm=math.inf),
    _run("schedule", steps=SCHED_STEPS, schedule=True),
    _run("accumulate_2", accumulate=2),
    *[_run(f"chunks_{c}", chunks=c) for c in (2, 3, 7)],
    *[_run(f"chunks_{c}_schedule", steps=SCHED_STEPS, chunks=c, schedule=True) for c in (2, 3, 7)],
    _run("torch_adam", torch_adam=True, full=True),
    _run("A", preset="A"),
    _run("A_chunks_3", preset="A", chunks=3),
]


@pytest.fixture(scope="module")
def gloo2(tmp_path_factory):
    return _launch(str(tmp_path_factory.mktemp("gloo2")), 2, "gloo", GLOO_RUNS)


@pytest.fixture(scope="module")
def gloo3(tmp_path_factory):
    return _launch(str(tmp_path_factory.mktemp("gloo3")), 3, "gloo", [_run("world3", full=True)])


def test_fused_adam(gloo2):
    _assert_matches(gloo2, "plain", _emulate("tiny", STEPS))


@pytest.mark.parametrize("max_grad_norm", [1e-3, math.inf])
def test_clipped(gloo2, max_grad_norm):
    name = "clip_1e-3" if max_grad_norm == 1e-3 else "clip_inf"
    want = _emulate("tiny", STEPS, max_grad_norm=max_grad_norm)
    _assert_matches(gloo2, name, want)
    coef = [torch.tensor(r["coef"], dtype=torch.int32).view(torch.float32).item() for r in gloo2[0][name][1:]]
    if max_grad_norm == math.inf:
        assert coef == [1.0] * STEPS
        _assert_same_run(gloo2[0][name], gloo2[0]["plain"], "max_grad_norm=inf against None", scalars=("loss", "step"))
    else:
        assert max(coef) < 1.0, coef                                                      # clipping is active


def test_scheduled(gloo2):
    want = _emulate("tiny", SCHED_STEPS, schedule=True)
    _assert_matches(gloo2, "schedule", want)
    lrs = [torch.tensor(r["lr"], dtype=torch.int32).view(torch.float32).item() for r in want[1:]]
    f32 = [torch.tensor(RECIPE.lr(k), dtype=torch.float32).item() for k in range(SCHED_STEPS)]
    assert lrs == f32                                                   # step k runs at the lr of k - 1 steps taken
    assert lrs[0] < lrs[1] < lrs[2] < lrs[3] < lrs[4] == lrs[5]         # through the warmup onto the plateau


def test_accumulated(gloo2):
    _assert_matches(gloo2, "accumulate_2", _emulate("tiny", STEPS, accumulate=2))


@pytest.mark.parametrize("schedule", [False, True])
@pytest.mark.parametrize("chunks", [2, 3, 7])
def test_chunked_exchange(gloo2, chunks, schedule):
    """Each piece all-reduced asynchronously and updated after its wait(): the bits of the whole-buffer exchange."""
    steps = SCHED_STEPS if schedule else STEPS
    name, whole = (f"chunks_{chunks}_schedule", "schedule") if schedule else (f"chunks_{chunks}", "plain")
    _assert_matches(gloo2, name, _emulate("tiny", steps, schedule=schedule))
    _assert_same_run(gloo2[0][name], gloo2[0][whole], f"{name} against the whole-buffer exchange")


def test_resume(gloo2):
    """Rank 0's state_dict after step 2, loaded by both ranks of a fresh world-2 step: steps 3-4 as the run that never
    stopped, bit for bit."""
    want = _emulate("tiny", STEPS)
    _assert_matches(gloo2, "plain_resumed", want, first=2)


def test_torch_adam(gloo2):
    """DFOLD_TORCH_ADAM=1: the buffer holds fl(g_0 + g_1) * 0.5 after the step, bit for bit, and torch.optim.Adam's
    update from the rank's own previous state lies within the per-element float64 Adam bound."""
    ranks = gloo2
    _assert_same_run(ranks[0]["torch_adam"], ranks[1]["torch_adam"], "torch_adam: rank 1 against rank 0",
                     scalars=("step", "lr"))
    recs = ranks[0]["torch_adam"]
    loc = _Local("tiny", 1)
    worst = 0.0
    for k in range(1, STEPS + 1):
        before = {f: t.cuda() for f, t in recs[k - 1]["full"].items()}
        after = {f: t.cuda() for f, t in recs[k]["full"].items()}
        local = loc.grads(before["p"], k, 2)
        for r in range(2):
            assert ranks[r]["torch_adam"][k]["loss"] == _bits(local[r][1]), f"step {k}, rank {r}: loss"
        want_g = (local[0][0] + local[1][0]) * 0.5
        assert torch.equal(after["g"].view(torch.int32), want_g.view(torch.int32)), f"step {k}: gradient buffer"
        assert recs[k]["step"] == k
        refs, errs = _adam_ref(before["p"].double(), want_g.double(), *(before[f].double() for f in ("m", "v", "x")), k,
                               _f32(LR), 0.9, 0.999, 1e-8, 1.0)
        for f, r, e in zip(("p", "m", "v", "x"), refs, errs):
            worst = max(worst, _within(f"torch Adam world 2 step {k} {f}", (after[f].double() - r).abs(), e, "adam"))
    assert worst > 0


@pytest.mark.parametrize("chunks", [1, 3])
def test_preset_a(gloo2, chunks):
    """Preset A at 8 x 64: the small-grid convolutions and their weight gradients on the side stream."""
    _assert_matches(gloo2, "A" if chunks == 1 else "A_chunks_3", _emulate("A", STEPS))


def test_world_three(gloo3):
    """Three ranks: the sum within 2u sum_r |g_r| of float64, the update within the Adam bound, the ranks equal."""
    for r in (1, 2):
        _assert_same_run(gloo3[0]["world3"], gloo3[r]["world3"], f"world3: rank {r} against rank 0", scalars=("step",))
    recs = gloo3[0]["world3"]
    loc = _Local("tiny", 1)
    gs = torch.tensor(1.0 / 3.0, dtype=torch.float32).cuda()
    for k in range(1, STEPS + 1):
        before = {f: t.cuda() for f, t in recs[k - 1]["full"].items()}
        after = {f: t.cuda() for f, t in recs[k]["full"].items()}
        local = loc.grads(before["p"], k, 3)
        for r in range(3):
            assert gloo3[r]["world3"][k]["loss"] == _bits(local[r][1]), f"step {k}, rank {r}: loss"
        exact = sum(g.double() for g, _ in local)
        mag = sum(g.double().abs() for g, _ in local)
        _within(f"world 3 step {k} summed gradient", (after["g"].double() - exact).abs(), 2 * U / (1 - 2 * U) * mag,
                "allreduce")
        g_eff = after["g"] * gs                                         # the kernel's fp32 product g * (1 / world)
        refs, errs = _adam_ref(before["p"].double(), g_eff.double(), *(before[f].double() for f in ("m", "v", "x")), k,
                               *(_f32(c) for c in (LR, 0.9, 0.999, 1e-8)), 1.0)     # the fused kernel's fp32 constants
        for f, r, e in zip(("p", "m", "v", "x"), refs, errs):
            _within(f"world 3 step {k} {f}", (after[f].double() - r).abs(), e, "adam")
        assert recs[k]["step"] == k


# --------------------------------------------------------------------------------------------------
# NCCL, one rank per GPU, captured steps
# --------------------------------------------------------------------------------------------------
def test_nccl_captured(tmp_path):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip(f"the NCCL arm needs two or more GPUs, {n} visible")
    cap = lambda name, **kw: dict(_run(name, **kw), graph=True)
    runs = [cap("plain"), _run("eager"), cap("schedule", steps=SCHED_STEPS, schedule=True),
            *[cap(f"chunks_{c}", chunks=c) for c in (2, 3, 7)],
            cap("chunks_3_schedule", steps=SCHED_STEPS, chunks=3, schedule=True)]
    ranks = _launch(str(tmp_path), 2, "nccl", runs)
    plain, sched = _emulate("tiny", STEPS), _emulate("tiny", SCHED_STEPS, schedule=True)
    for name, want in (("plain", plain), ("eager", plain), ("schedule", sched), ("chunks_2", plain),
                       ("chunks_3", plain), ("chunks_7", plain), ("chunks_3_schedule", sched)):
        _assert_matches(ranks, name, want)
    _assert_same_run(ranks[0]["plain"], ranks[0]["eager"], "captured against eager world-2 steps")
