"""-m gpu: global-norm gradient clipping, torch.nn.utils.clip_grad_norm_(params, max_norm) with norm_type 2 (the option the
reference trainer keeps commented out, train_DFOLD_dynamics.py:665), in csrc/simt.cu and in the captured training step.

* dfold_grad_norm against float64, through the C ABI: within one fp32 rounding of ||s g|| plus the fp64 summation term
  of the kernel's order; the same bits from two launches; the coefficient bit for bit as torch evaluates it from that
  total; injected inf / NaN give torch's total, coefficient and clipped gradients.
* dfold_adam_amsgrad_clip per element against float64 (the bound of tests/test_gpu_simt.py::test_adam_amsgrad), and
  bit for bit dfold_adam_amsgrad when the coefficient is 1.
* TrainStep(max_grad_norm=...): one clipped step recomputed in float64 from the step's own gradient buffer (which the
  fused optimizer leaves as it is), math.inf moves the parameters bit for bit like None, graph replay and eager steps
  agree bit for bit, and DFOLD_TORCH_ADAM=1 equals clip_grad_norm_ + torch.optim.Adam(amsgrad=True) on the same buffer.
"""
import copy
import math

import pytest
import torch

from dynamicpdb_b200 import checkpoint as C
from dynamicpdb_b200 import kernels as K
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from dynamicpdb_b200.train_step import TrainStep
from tests.test_gpu_checkpoint import PRESETS, _net, _windows
from tests.test_gpu_simt import DEV, U, UD, _adam_ref, _gen, _ok, _RefPeak, _wide, _within, cdiv

pytestmark = pytest.mark.gpu
LR = 1e-4
ROW = 4096                         # the float64 reference sums rows of this many squares, then the row sums exactly


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _preset_a_numel():
    with torch.device("meta"):
        net = FullScoreNetwork(syn.model_conf(64, **syn.PRESET_A), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    return C.flat_layout(net).numel


def _ref_norm(g, s):
    """float64 ||s g|| with an error of at most (ROW + 1) UD relative: the squares are exact in float64, each row of ROW
    of them is summed by torch (any order: <= (ROW - 1) UD relative, all terms >= 0), the row sums exactly by math.fsum."""
    with _RefPeak("reference norm"):
        q = g.double() ** 2
        q = torch.cat([q, q.new_zeros(cdiv(q.numel(), ROW) * ROW - q.numel())]).view(-1, ROW).sum(1)
        return abs(s) * math.sqrt(math.fsum(q.cpu().tolist()))


def _norm_bound(n, ref):
    """|total - ref| for total = fp32(s sqrt(S^)).  The kernel's fp64 sum S^ of n non-negative exact squares adds each
    term through at most d = 4 ceil(n4 / (256 B)) (one thread's float4s in turn) + 5 (lane butterfly) + 8 (warps in
    order) + ceil(B / 256) + 5 + 8 (the same over the B <= 1024 partials) roundings: |S^ - S| <= d UD S (1 + d UD).  The
    square root halves that, it and the product with s add UD each, the reference adds (ROW + 1) UD, and the final
    rounding to fp32 adds U |total|."""
    n4 = n // 4
    B = min(cdiv(n4, 256), 1024)
    d = 4 * cdiv(n4, 256 * B) + cdiv(B, 256) + 26
    return ref * (U * (1 + 1e-6) + (d + ROW + 8) * UD)


def _grad_norm(g, s, max_norm):
    ws = torch.full((1024,), float("nan"), dtype=torch.float64, device=DEV)
    total, coef = torch.full((), float("nan"), device=DEV), torch.full((), float("nan"), device=DEV)
    _ok(K.lib().dfold_grad_norm(K._ptr(g), g.numel(), s, max_norm, K._ptr(ws), K._ptr(total), K._ptr(coef), K._stream()))
    torch.cuda.synchronize()
    return total, coef


def _torch_coef(total, max_norm):
    """clip_grad_norm_'s coefficient from an fp32 device total, as torch evaluates it."""
    return torch.clamp(max_norm / (total + 1e-6), max=1.0)


def _same(a, b):
    """Equal bits, +0 == -0 and NaN == NaN."""
    a, b = a.reshape(-1), b.reshape(-1)
    return bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


# --------------------------------------------------------------------------------------------------
# dfold_grad_norm
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [4, 8, 1028, 4096 + 8, "preset_A"])
def test_grad_norm_against_float64(n):
    """All zeros, one non-zero entry and magnitudes 2^-40 ... 2^40; grad_scale 1 and 1/8 (1 / world of an 8-rank
    all-reduce).  n = 4096 + 8 is one float4 past 1024 threads' worth; the preset-A flat buffer (184.4 M elements,
    padding included) runs 1024 CTAs of 176 float4s per thread."""
    n = _preset_a_numel() if n == "preset_A" else n
    single = torch.zeros(n, device=DEV)
    single[n // 3] = -3.25 * 2.0 ** 37
    inputs = {"zeros": torch.zeros(n, device=DEV), "single": single, "spread": _wide(n, n, lo_exp=-40, hi_exp=40, zeros=0.01)}
    for kind, g in inputs.items():
        for s in (1.0, 0.125):
            what = f"n{n} {kind} s{s}"
            ref = _ref_norm(g, s)
            total, coef = _grad_norm(g, s, 1.0)
            again, _ = _grad_norm(g, s, 1.0)
            assert torch.equal(total.view(torch.int32), again.view(torch.int32)), f"{what}: two launches differ"
            _within(what, torch.tensor([abs(float(total) - ref)], dtype=torch.float64),
                    torch.tensor([_norm_bound(n, ref)], dtype=torch.float64), "grad_norm")
            if kind == "single":
                assert float(total) == _f32(3.25 * 2.0 ** 37 * s), what           # sqrt(x^2) is exact
            for max_norm in (1.0, _f32(0.1 * ref) or 1.0, math.inf):
                total, coef = _grad_norm(g, s, max_norm)
                assert _same(coef, _torch_coef(total, max_norm)), f"{what} max_norm {max_norm}: {float(coef)}"
            assert float(coef) == 1.0, what                                           # inf: never clips a finite norm


@pytest.mark.parametrize("n", [1028, 4096 + 8])
def test_grad_norm_non_finite_like_torch(n):
    """An inf makes the total inf and the coefficient 0: the inf entries become NaN and every other entry 0.  A NaN makes
    everything NaN.  Gradients are checked through dfold_adam_amsgrad_clip from zero moments, which leaves a parameter
    exactly in place for a zero gradient and makes it NaN for a NaN one."""
    cases = {"+inf": [(5, math.inf)], "-inf": [(n - 1, -math.inf)], "nan": [(7, math.nan)],
             "inf and nan": [(3, math.inf), (n // 2, math.nan)]}
    for case, entries in cases.items():
        for s in (1.0, 0.125):
            what = f"n{n} {case} s{s}"
            g = torch.randn(n, generator=_gen(n), device=DEV)
            for i, v in entries:
                g[i] = v
            total, coef = _grad_norm(g, s, 1.0)
            p = torch.nn.Parameter(torch.zeros(n, device=DEV))
            p.grad = g * s
            t_total = torch.nn.utils.clip_grad_norm_([p], 1.0, foreach=True)
            assert _same(total, t_total), f"{what}: total {float(total)} vs torch {float(t_total)}"
            assert _same(coef, _torch_coef(t_total, 1.0)), f"{what}: coefficient {float(coef)}"
            assert bool((torch.isnan(p.grad) | (p.grad == 0)).all()), what
            p0 = torch.randn(n, generator=_gen(n + 1), device=DEV)
            bufs = [p0.clone()] + [torch.zeros(n, device=DEV) for _ in range(3)]
            step = torch.zeros((), device=DEV)
            _ok(K.lib().dfold_adam_amsgrad_clip(K._ptr(bufs[0]), K._ptr(g), *(K._ptr(b) for b in bufs[1:]), n, K._ptr(step), 1,
                                                1e-3, 0.9, 0.999, 1e-8, s, K._ptr(coef), K._stream()))
            torch.cuda.synchronize()
            nan = torch.isnan(p.grad)
            assert torch.equal(torch.isnan(bufs[0]), nan), f"{what}: NaN positions differ from torch's clipped gradient"
            assert torch.equal(bufs[0][~nan], p0[~nan]), f"{what}: a zero clipped gradient moved its parameter"


# --------------------------------------------------------------------------------------------------
# dfold_adam_amsgrad_clip
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [4, 4096 + 8, 2162688 + 4])
def test_adam_clip_against_float64(n):
    """Steps with coefficients below 1 (grad_scale 0.5, gradient magnitudes 1e-8 ... 1e3): the kernel's gradient is
    fp32((fp32(g 0.5)) coef), two fp32 products emulated exactly here, and the update from it is held to _adam_ref's
    bound.  Then one step with coef = 1 from the same state gives the bits of dfold_adam_amsgrad."""
    lr, b1, b2, eps, gs = _f32(1e-3), _f32(0.9), _f32(0.999), _f32(1e-8), 0.5
    g = _gen(n)
    L = K.lib()
    nan = torch.full((16,), float("nan"), device=DEV)
    bufs = [torch.cat([torch.randn(n, generator=g, device=DEV), nan])] + [torch.cat([torch.zeros(n, device=DEV), nan]) for _ in range(3)]
    step = torch.zeros(1, device=DEV)
    coef = torch.empty((), device=DEV)
    dev = DEV if n > 65536 else "cpu"
    for it, c in enumerate((0.37, 2.0 ** -3, 1e-3, 0.999, 5e-6)):
        coef.fill_(c)
        grad = torch.randn(n, generator=g, device=DEV) * torch.pow(10.0, torch.empty(n, device=DEV).uniform_(-8, 3, generator=g))
        before = [b[:n].clone() for b in bufs]
        _ok(L.dfold_adam_amsgrad_clip(K._ptr(bufs[0]), K._ptr(grad), *(K._ptr(b) for b in bufs[1:]), n, K._ptr(step), 1,
                                      lr, b1, b2, eps, gs, K._ptr(coef), K._stream()))
        torch.cuda.synchronize()
        assert step.item() == it + 1
        for b in bufs:
            assert torch.isnan(b[n:]).all(), "written past n"
        g_eff = (grad * gs) * coef
        what = f"adam_clip n{n} step{it + 1} coef{c}"
        with _RefPeak(what):
            ref, err = _adam_ref(*(t.to(dev, torch.float64) for t in (before[0], g_eff, before[1], before[2], before[3])),
                                 it + 1, lr, b1, b2, eps, 1.0)
            for k, (name, r, e) in enumerate(zip(("p", "m", "v", "vmax"), ref, err)):
                _within(f"{what} {name}", (bufs[k][:n].to(dev, torch.float64) - r).abs(), e, "adam")

    grad = torch.randn(n, generator=g, device=DEV)
    coef.fill_(1.0)
    plain, clip = [b.clone() for b in bufs], [b.clone() for b in bufs]
    s_plain, s_clip = step.clone(), step.clone()
    _ok(L.dfold_adam_amsgrad(K._ptr(plain[0]), K._ptr(grad), *(K._ptr(b) for b in plain[1:]), n, K._ptr(s_plain), 1,
                             lr, b1, b2, eps, gs, K._stream()))
    _ok(L.dfold_adam_amsgrad_clip(K._ptr(clip[0]), K._ptr(grad), *(K._ptr(b) for b in clip[1:]), n, K._ptr(s_clip), 1,
                                  lr, b1, b2, eps, gs, K._ptr(coef), K._stream()))
    torch.cuda.synchronize()
    assert s_plain.item() == s_clip.item()
    for a, b in zip(plain, clip):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "coef = 1 differs from dfold_adam_amsgrad"


def test_rejected_arguments():
    L = K.lib()
    g = torch.zeros(64, device=DEV)
    ws = torch.zeros(1024, dtype=torch.float64, device=DEV)
    out = torch.full((2,), float("nan"), device=DEV)
    for n, max_norm, needle in ((6, 1.0, "multiple of 4"), (0, 1.0, "multiple of 4"), (64, 0.0, "positive"),
                                (64, -1.0, "positive"), (64, math.nan, "positive")):
        rc = L.dfold_grad_norm(K._ptr(g), n, 1.0, max_norm, K._ptr(ws), K._ptr(out), K._ptr(out, 1), K._stream())
        assert rc != 0 and needle in L.dfold_last_error().decode(), (n, max_norm)
    st = torch.zeros(1, device=DEV)
    rc = L.dfold_adam_amsgrad_clip(K._ptr(g), K._ptr(g), K._ptr(g), K._ptr(g), K._ptr(g), 64, K._ptr(st), 1, 1e-3, 0.9, 0.999,
                                   1e-8, 1.0, None, K._stream())
    assert rc != 0 and "null coefficient" in L.dfold_last_error().decode()
    torch.cuda.synchronize()
    assert torch.isnan(out).all() and st.item() == 0.0, "a rejected call wrote its output"


# --------------------------------------------------------------------------------------------------
# TrainStep(max_grad_norm=...)
# --------------------------------------------------------------------------------------------------
ROUTES = {"graph": (True, "0"), "eager": (False, "0"), "torch_adam": (True, "1")}       # graph, DFOLD_TORCH_ADAM
CASES = [(p, r) for p in PRESETS for r in ROUTES]


def _flat(ts, tensors):
    """Per-parameter device tensors (self.params order) in one fp32 buffer of the flat layout."""
    flat = torch.zeros(ts.layout.numel, dtype=torch.float32, device=DEV)
    torch.cat([t.reshape(-1) for t in tensors], out=flat[:sum(t.numel() for t in tensors)])
    return flat


def _state(ts):
    """Parameters and the three moments as flat fp32 device copies."""
    if ts.opt is None:
        return [t.clone() for t in (ts.flat_param, ts.exp_avg, ts.exp_avg_sq, ts.max_exp_avg_sq)]
    return [_flat(ts, [p.detach() for p in ts.params])] + [_flat(ts, [ts.opt.state[p][k] for p in ts.params])
                                                           for k in C.MOMENTS]


def _assert_bits(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), f"{what}: tensor {i} differs"


def _make(preset, graph, max_grad_norm, windows):
    ts = TrainStep(_net(preset, 0), syn.surrogate_loss, windows[0], lr=LR, graph=graph, warmup=2, max_grad_norm=max_grad_norm)
    assert (ts.graph is not None) == graph, ts.graph_error
    return ts


def _spy_on_clip(monkeypatch):
    """DFOLD_TORCH_ADAM=1 clips in place: keep a copy of the flat gradient as clip_grad_norm_ receives it.  Installed
    before the step is built, the copy is part of the captured graph."""
    real, seen = torch.nn.utils.clip_grad_norm_, {}

    def spy(params, *args, **kw):
        base = params[0].grad._base                     # the step's flat gradient buffer
        if "pre" not in seen:
            seen["pre"] = torch.empty_like(base)        # first called by an eager warm-up step, before capture
        seen["pre"].copy_(base)
        return real(params, *args, **kw)

    monkeypatch.setattr(torch.nn.utils, "clip_grad_norm_", spy)
    return seen


def _torch_clip(ts, flat, max_norm):
    """clip_grad_norm_(max_norm, foreach=True) over per-parameter views of a copy of `flat`: (total, clipped flat)."""
    g = flat.clone()
    params = []
    for p, v in zip(ts.params, (v for v in C.views(ts.layout, g) if v is not None)):
        q = torch.nn.Parameter(torch.empty_like(p))
        q.grad = v
        params.append(q)
    total = torch.nn.utils.clip_grad_norm_(params, max_norm, foreach=True)
    return total, g


def _check_fused_update(ts, before, t, max_norm):
    """The step's norm, coefficient and Adam update, recomputed in float64 from its own flat gradient in slices."""
    g = ts.flat_grad
    ref = _ref_norm(g, 1.0)
    _within("TrainStep grad_norm", torch.tensor([abs(float(ts.grad_norm) - ref)], dtype=torch.float64),
            torch.tensor([_norm_bound(g.numel(), ref)], dtype=torch.float64), "grad_norm")
    coef = _torch_coef(ts.grad_norm, max_norm)
    assert _same(ts.clip_coef, coef), (float(ts.clip_coef), float(coef))
    after = (ts.flat_param, ts.exp_avg, ts.exp_avg_sq, ts.max_exp_avg_sq)
    n, step = g.numel(), 1 << 24
    for a in range(0, n, step):
        b = min(n, a + step)
        g_eff = (g[a:b] * 1.0) * coef
        with _RefPeak(f"TrainStep update [{a}, {b})"):
            refs, errs = _adam_ref(before[0][a:b].double(), g_eff.double(), *(x[a:b].double() for x in before[1:]), t,
                                   _f32(LR), _f32(0.9), _f32(0.999), _f32(1e-8), 1.0)
            for name, f, r, e in zip(("p", "m", "v", "vmax"), after, refs, errs):
                _within(f"TrainStep {name} [{a}, {b})", (f[a:b].double() - r).abs(), e, "adam")
    return float(coef)


@pytest.mark.parametrize("preset,route", CASES)
def test_clipped_step(preset, route, monkeypatch):
    """max_grad_norm = 0.1 x the unclipped norm: the second step of a clipped run, from a snapshot of its state, against
    float64 (fused optimizer) or against clip_grad_norm_ + torch.optim.Adam(amsgrad=True, capturable, foreach) on the same
    gradient buffer (DFOLD_TORCH_ADAM=1, bit for bit)."""
    graph, torch_adam = ROUTES[route]
    monkeypatch.setenv("DFOLD_TORCH_ADAM", torch_adam)
    seen = _spy_on_clip(monkeypatch) if torch_adam == "1" else None
    windows = _windows(preset)[:2]
    probe = _make(preset, graph, math.inf, windows)
    probe()
    max_norm = 0.1 * float(probe.grad_norm)
    del probe
    torch.cuda.empty_cache()
    ts = _make(preset, graph, max_norm, windows)
    ts()
    ts.load(windows[1])
    before = _state(ts)
    if ts.opt is not None:
        opt_before = copy.deepcopy(ts.opt.state_dict())
    ts()
    torch.cuda.synchronize()
    assert float(ts.grad_norm) > max_norm                   # clipping is active
    if ts.opt is None:
        assert _check_fused_update(ts, before, 2, max_norm) < 1.0
        return
    total, clipped = _torch_clip(ts, seen["pre"], max_norm)
    assert _same(ts.grad_norm, total), (float(ts.grad_norm), float(total))
    assert torch.equal(ts.flat_grad.view(torch.int32), clipped.view(torch.int32)), "clipped gradient differs from torch's"
    ref_params = [torch.nn.Parameter(v.clone()) for v in C.views(ts.layout, before[0]) if v is not None]
    opt = torch.optim.Adam(ref_params, lr=LR, amsgrad=True, capturable=True, foreach=True)
    opt.load_state_dict(opt_before)
    for q, v in zip(ref_params, (v for v in C.views(ts.layout, clipped) if v is not None)):
        q.grad = v.clone()
    opt.step()
    want = [_flat(ts, [q.detach() for q in ref_params])] + [_flat(ts, [opt.state[q][k] for q in ref_params]) for k in C.MOMENTS]
    _assert_bits(_state(ts), want, "clipped step against clip_grad_norm_ + torch.optim.Adam")


@pytest.mark.parametrize("preset,route", CASES)
def test_inf_reports_the_norm_and_moves_like_none(preset, route, monkeypatch):
    """max_grad_norm=math.inf: two steps move every parameter and moment bit for bit like None, and grad_norm is the norm
    of the step's gradient (fused: within the float64 bound; DFOLD_TORCH_ADAM=1: clip_grad_norm_'s own value)."""
    graph, torch_adam = ROUTES[route]
    monkeypatch.setenv("DFOLD_TORCH_ADAM", torch_adam)
    windows = _windows(preset)[:2]
    states = []
    for max_norm in (None, math.inf):
        ts = _make(preset, graph, max_norm, windows)
        for w in windows:
            ts.load(w)
            ts()
            torch.cuda.synchronize()
            if max_norm is None:
                assert ts.grad_norm is None
            elif ts.opt is None:
                ref = _ref_norm(ts.flat_grad, 1.0)
                _within("grad_norm at inf", torch.tensor([abs(float(ts.grad_norm) - ref)], dtype=torch.float64),
                        torch.tensor([_norm_bound(ts.flat_grad.numel(), ref)], dtype=torch.float64), "grad_norm")
            else:
                total, clipped = _torch_clip(ts, ts.flat_grad, math.inf)         # coefficient 1: the buffer is unchanged
                assert _same(ts.grad_norm, total) and torch.equal(clipped, ts.flat_grad)
        states.append(_state(ts))
        del ts
        torch.cuda.empty_cache()
    _assert_bits(states[0], states[1], "max_grad_norm=inf against None")


@pytest.mark.parametrize("preset", list(PRESETS))
def test_graph_replay_equals_eager_clipped_steps(preset):
    """The captured clipped step and the same step launched eagerly give the same gradients, norms and state bits."""
    windows = _windows(preset)[:3]
    max_norm = 1e-3
    runs = []
    for graph in (True, False):
        ts = _make(preset, graph, max_norm, windows)
        norms, grads = [], []
        for w in windows:
            ts.load(w)
            ts()
            norms.append(ts.grad_norm.clone())
            grads.append(ts.flat_grad.clone())
        torch.cuda.synchronize()
        runs.append((torch.stack(norms), grads, _state(ts)))
        del ts
        torch.cuda.empty_cache()
    (n_g, g_g, s_g), (n_e, g_e, s_e) = runs
    for i, (a, b) in enumerate(zip(g_g, g_e)):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"step {i}: gradients differ between graph and eager"
    assert torch.equal(n_g.view(torch.int32), n_e.view(torch.int32)), (n_g, n_e)
    assert bool((n_g > max_norm).all())
    _assert_bits(s_g, s_e, "graph replay against eager steps")
