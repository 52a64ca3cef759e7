"""-m gpu: several same-length windows through one batched pass.

* dfold_gemm_bf16x3_windows (forward and data gradient of the 5x5 convolution over W stacked windows, full and cropped)
  equals W separate dfold_gemm_bf16x3_bn calls bit for bit: each output element is the same one-CTA k loop, and the
  window's frame halo is the 4-D map's zero fill.  W in {1, 2, 5}, F in {2, 5, 20} (20: the cropped layers of the
  dead-frame pyramid), N in {64, 130, 256} (130: a partial row tile).
* dfold_gemm_wgrad_bf16x3_windows against the sum of the W per-window weight gradients and against float64.
* dfold_global_layernorm_seg_fwd / _bwd equal one call per segment bit for bit, and agree with float64.
* FullScoreNetwork.forward_windows: each window's outputs equal net(window) bit for bit, at the tiny preset and preset A,
  k in {2, 4} windows of distinct proteins with different t; one case against the oracle at the 1e-4 bar.
* TrainStep(accumulate=k, batched=True) against accumulate=k at lr = 0, and Trainer(batched=True) against
  Trainer(accumulate=k).
"""
import math
import os

import pytest
import torch

from dynamicpdb_b200 import kernels as K
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from dynamicpdb_b200.train_step import TrainStep
from tests.test_gpu_simt import U, _within

pytestmark = pytest.mark.gpu
DEV = "cuda"
TAPS = 25


def _planes(x2):
    (hi, lo), _ = K._split2d(x2.contiguous())
    return hi, lo


def _bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# --------------------------------------------------------------------------------------------------
# windowed convolution GEMMs
# --------------------------------------------------------------------------------------------------
def _conv_case(W, F, N, ci=64, co=96, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(W * F * N, ci, device=DEV, generator=g)
    w = torch.randn(co, ci, 5, 5, device=DEV, generator=g) / math.sqrt(TAPS * ci)
    b = torch.randn(co, device=DEV, generator=g) * 0.1
    return x, w, b


@pytest.mark.parametrize("W", [1, 2, 5])
@pytest.mark.parametrize("F", [2, 5, 20])
@pytest.mark.parametrize("N", [64, 130, 256])
def test_windowed_conv_forward_and_data_gradient_equal_separate_calls(W, F, N):
    ci, co = 64, 96
    x, w, b = _conv_case(W, F, N, ci, co, seed=W * 100 + F * 10 + N)
    crops = [0, 2] if F > 17 else [0]
    f_hi, f_lo, d_hi, d_lo = K._conv_planes(w)
    x_hi, x_lo = _planes(x)
    for crop in crops:
        Fo = F - crop
        res = torch.randn(W * Fo * N, co, device=DEV)
        for bn in (64, 128):
            # forward, with bias, ReLU and residual
            got = torch.full((W * Fo * N, co), float("nan"), device=DEV)
            K._gemm(x_hi, x_lo, F, N, ci, ci, f_hi, f_lo, co, f_hi.shape[2], 5, 5, got, co, b, res, co, 1.0, 1.0, 1,
                    F_out=Fo, f_start=crop, bn=bn, windows=W)
            want = torch.full_like(got, float("nan"))
            for i in range(W):
                K._gemm(x_hi[i * F * N:(i + 1) * F * N], x_lo[i * F * N:(i + 1) * F * N], F, N, ci, ci, f_hi, f_lo, co,
                        f_hi.shape[2], 5, 5, want[i * Fo * N:(i + 1) * Fo * N], co, b, res[i * Fo * N:(i + 1) * Fo * N], co,
                        1.0, 1.0, 1, F_out=Fo, f_start=crop, bn=bn)
            torch.cuda.synchronize()
            assert _bits(got, want), (W, F, N, crop, bn, "fwd")
            # data gradient: the cropped layer's transpose, f_start = -crop
            gy = torch.randn(W * Fo * N, co, device=DEV)
            g_hi, g_lo = _planes(gy)
            got = torch.full((W * F * N, ci), float("nan"), device=DEV)
            K._gemm(g_hi, g_lo, Fo, N, co, co, d_hi, d_lo, ci, d_hi.shape[2], 5, 5, got, ci, None, None, 0, 1.0, 0.0, 0,
                    F_out=F, f_start=-crop, bn=bn, windows=W)
            want = torch.full_like(got, float("nan"))
            for i in range(W):
                K._gemm(g_hi[i * Fo * N:(i + 1) * Fo * N], g_lo[i * Fo * N:(i + 1) * Fo * N], Fo, N, co, co, d_hi, d_lo, ci,
                        d_hi.shape[2], 5, 5, want[i * F * N:(i + 1) * F * N], ci, None, None, 0, 1.0, 0.0, 0,
                        F_out=F, f_start=-crop, bn=bn)
            torch.cuda.synchronize()
            assert _bits(got, want), (W, F, N, crop, bn, "dgrad")


@pytest.mark.parametrize("W,F,N,crop", [(2, 5, 130, 0), (5, 2, 64, 0), (3, 20, 64, 2)])
def test_windowed_conv_weight_gradient(W, F, N, crop):
    """out[t][m][n] = sum over the pixels of every window of g * x(shifted by tap t).  Each output element is a sum of
    S = W * Fo * N split-bf16 products c = g_hi x_hi + g_hi x_lo + g_lo x_hi; the kernel folds them in k-blocks of 64 pixels,
    4 k-blocks per tensor-core chunk, and the chunks into an fp32 accumulator.  Against the per-window sum (W launches,
    then W - 1 fp32 adds): both are fp32 sums of the same products in different orders, each within S * 2u * sum|c| of
    the exact sum of the products (2u: the tensor core's accumulation truncates), so their difference is within
    2 * S * 2u * sum|c| + (W - 1) u sum|c|.  Against float64 of the fp32 operands, the dropped lo * lo terms and the
    bf16 rounding of the lo planes add 2^-16 * sum|g x| per element (each operand is hi + lo to 2^-16 relative)."""
    ci, co = 64, 96
    Fo = F - crop
    g = torch.Generator(device=DEV).manual_seed(7)
    x = torch.randn(W * F * N, ci, device=DEV, generator=g)
    gy = torch.randn(W * Fo * N, co, device=DEV, generator=g)
    x_hi, x_lo = _planes(x)
    g_hi, g_lo = _planes(gy)
    got = torch.zeros(co, ci, 5, 5, device=DEV)
    K._conv_wgrad(g_hi, g_lo, x_hi, x_lo, co, ci, 5, 5, F, Fo, N, crop, got, 0, windows=W)
    per = torch.zeros_like(got)
    for i in range(W):
        part = torch.zeros_like(got)
        K._conv_wgrad(g_hi[i * Fo * N:(i + 1) * Fo * N], g_lo[i * Fo * N:(i + 1) * Fo * N],
                      x_hi[i * F * N:(i + 1) * F * N], x_lo[i * F * N:(i + 1) * F * N], co, ci, 5, 5, F, Fo, N, crop, part, 0)
        per += part
    torch.cuda.synchronize()
    # float64 reference and sum |g x| per element, window by window (zero frame halo at each window's edge)
    xd = x.double().reshape(W, F, N, ci)
    gd = gy.double().reshape(W, Fo, N, co)
    ref = torch.zeros(co, ci, 5, 5, dtype=torch.float64, device=DEV)
    mag = torch.zeros_like(ref)
    xp = torch.nn.functional.pad(xd, (0, 0, 2, 2, 2, 2))          # [W, F + 4, N + 4, ci]
    for tf in range(5):
        for tn in range(5):
            xs = xp[:, crop + tf:crop + tf + Fo, tn:tn + N]              # input frame f + crop + tf - 2, residue n + tn - 2
            ref[:, :, tf, tn] = torch.einsum("wfnm,wfnc->mc", gd, xs)
            mag[:, :, tf, tn] = torch.einsum("wfnm,wfnc->mc", gd.abs(), xs.abs())
    S = W * Fo * N
    _within(f"wgrad windows vs per-window W{W} F{F} N{N} crop{crop}", (got.double() - per.double()).abs(),
            (2 * S * 2 * U + (W - 1) * U) * mag, "wgrad_windows")
    _within(f"wgrad windows vs float64 W{W} F{F} N{N} crop{crop}", (got.double() - ref).abs(),
            (S * 2 * U + 2.0 ** -16) * mag, "wgrad_windows")


# --------------------------------------------------------------------------------------------------
# segmented layer norm
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,shape", [(1, (3, 24, 32)), (2, (8, 64, 256)), (4, (2, 256, 256)), (5, (1, 7, 3))])
@pytest.mark.parametrize("silu", [False, True])
def test_segmented_layer_norm_equals_one_call_per_segment(S, shape, silu):
    """Bit for bit against the single-tensor entry points; against float64 within 64 u of the output scale (the fp32
    mean, rstd and the element-wise fp32 arithmetic; the reductions themselves run in double)."""
    g = torch.Generator(device=DEV).manual_seed(S)
    x = (torch.randn((S * shape[0],) + shape[1:], device=DEV, generator=g) * 3 + 1).requires_grad_(True)
    dy = torch.randn(x.shape, device=DEV, generator=g)
    y = K.global_layernorm(x, 1e-4, silu=silu, segments=S)
    (dx,) = torch.autograd.grad(y, x, dy)
    parts = x.detach().chunk(S)
    for i, (xi, gi) in enumerate(zip(parts, dy.chunk(S))):
        xi = xi.clone().requires_grad_(True)
        yi = K.global_layernorm(xi, 1e-4, silu=silu)
        (dxi,) = torch.autograd.grad(yi, xi, gi)
        assert _bits(y.detach().chunk(S)[i], yi.detach()), (S, shape, i, "fwd")
        assert _bits(dx.chunk(S)[i], dxi), (S, shape, i, "bwd")
        # float64
        xd = xi.detach().double().requires_grad_(True)
        h = (xd - xd.mean()) / torch.sqrt(xd.var() + 1e-4)
        yd = torch.nn.functional.silu(h) if silu else h
        (dxd,) = torch.autograd.grad(yd, xd, gi.double())
        _within(f"seg ln fwd S{S}", (yi.detach().double() - yd.detach()).abs(), 64 * U * (1 + h.detach().abs()), "seg_ln")
        _within(f"seg ln bwd S{S}", (dxi.double() - dxd).abs(), 64 * U * (dxd.abs() + dxd.abs().max() + 1e-30), "seg_ln")


# --------------------------------------------------------------------------------------------------
# forward_windows
# --------------------------------------------------------------------------------------------------
# Residue and frame counts at which no linear layer changes between the SIMT and tensor-core kernels when its rows grow
# k-fold (kernels._use_tensor_cores): the tensor-core layers have >= 32 rows per window, the others have K < 64 or
# N < 16 at every row count, so each window's outputs are produced by the same kernels as net(window).
SHAPES = {"tiny": (syn.PRESET_TINY, 3, 40), "tiny_nf20": (syn.PRESET_TINY, 20, 40), "A": (syn.PRESET_A, 4, 64)}


def _net(preset, nf, seed=0):
    torch.manual_seed(seed)
    net = FullScoreNetwork(syn.model_conf(nf, **preset), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd, seed=seed + 1)
    net.load_state_dict(sd)
    return net.cuda()


def _windows(nf, N, k, seed=50):
    return [{kk: v.cuda() for kk, v in syn.make_feats(nf, N, seed=seed + i, t=0.2 + 0.15 * i).items()} for i in range(k)]


def test_row_counts_keep_every_linear_on_one_kernel():
    """The premise of SHAPES: the kernel choice of every linear layer of the network is the same at 1x and 4x its rows."""
    for name, (preset, nf, N) in SHAPES.items():
        c = preset["c_s"]
        for rows, kin, nout in ((nf * N, 3, c), (nf * N, c, c), (N, 1, c), (N, c, c), (nf * N, 14, c), (nf * N, 7, c),
                                (N, 256, c), (N * N, 128, preset["c_z"]), (nf * N, 5 * c, 5 * c), (nf * N, 5 * c, 14),
                                (nf * N, 5 * c, 6), (N, 5 * c, 6)):
            assert K._use_tensor_cores(rows, nout, kin) == K._use_tensor_cores(4 * rows, nout, kin), (name, rows, kin, nout)


@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("k", [2, 4])
def test_forward_windows_equals_forward(shape, k):
    preset, nf, N = SHAPES[shape]
    net = _net(preset, nf)
    windows = _windows(nf, N, k)
    with torch.no_grad():
        outs = net.forward_windows([dict(w) for w in windows])
        for i, w in enumerate(windows):
            ref = net(dict(w))
            assert set(outs[i]) == set(ref)
            for key in ref:
                assert outs[i][key].shape == ref[key].shape and outs[i][key].dtype == ref[key].dtype, key
                assert _bits(outs[i][key].float(), ref[key].float()), (shape, k, i, key)


def test_forward_windows_matches_the_oracle():
    from oracle import dfold_oracle as O
    preset, nf, N = SHAPES["tiny"]
    net = _net(preset, nf)
    sd = {k: v.detach().cpu().clone() for k, v in net.state_dict().items()}
    windows = _windows(nf, N, 2)
    with torch.no_grad():
        outs = net.forward_windows([dict(w) for w in windows])
        for i, w in enumerate(windows):
            ref = O.full_forward(dict(sd), {k: v.cpu() for k, v in w.items()}, O.default_conf(**preset),
                                 O.default_diffuser_conf(1.0))
            for key in ("rigid_update", "rigids", "trans_score"):
                err = (ref[key].double() - outs[i][key].cpu().double()).flatten(2).norm(dim=-1).max().item()
                assert err < 1e-4, (i, key, err)


def test_forward_windows_keeps_autograd_per_window():
    """The gradient of window 0's loss alone does not depend on window 1's inputs being present (no coupling)."""
    preset, nf, N = SHAPES["tiny"]
    net = _net(preset, nf)
    windows = _windows(nf, N, 2)
    outs = net.forward_windows([dict(w) for w in windows])
    loss = syn.surrogate_loss(outs[0])
    loss.backward()
    g_batched = {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None}
    net.zero_grad(set_to_none=True)
    syn.surrogate_loss(net(dict(windows[0]))).backward()
    for n, p in net.named_parameters():
        if p.grad is None:
            continue
        ref = p.grad.double()
        rel = ((g_batched[n].double() - ref).norm() / ref.norm().clamp(min=1e-30)).item()
        assert rel < 1e-4 or ref.norm().item() < 1e-12, (n, rel)


# --------------------------------------------------------------------------------------------------
# TrainStep(batched=True)
# --------------------------------------------------------------------------------------------------
TS_SHAPES = {"tiny": (syn.PRESET_TINY, 3, 40), "A": (syn.PRESET_A, 8, 64)}


def _step(preset_name, windows, **kw):
    preset, nf, _ = TS_SHAPES[preset_name]
    ts = TrainStep(_net(preset, nf), syn.surrogate_loss, windows[0], lr=kw.pop("lr", 0.0), warmup=2, **kw)
    assert ts.graph is not None or not kw.get("graph", True), ts.graph_error
    for i, w in enumerate(windows[:ts.accumulate]):
        ts.load(w, slot=i)
    return ts


@pytest.mark.parametrize("preset,k", [("tiny", 2), ("tiny", 4), ("A", 2), ("A", 4)])
def test_batched_step_gradient_equals_accumulate(preset, k):
    """At lr = 0 both steps see the same weights.  accumulate=k sums k per-window gradients; batched=True reduces every
    layer's weight gradient over the stacked rows of all k windows in one GEMM (and the convolutions' in one launch per
    use), so each element is the same sum of products in another fp32 order.  Bound: that of
    test_gpu_train_recipe.py::test_accumulated_gradient_is_the_window_mean for the k-window sum, k u sum_i |g_i|, plus,
    for the reordered reduction over R = k * nf * N stacked rows, 2 sqrt(R) u times the parameter tensor's largest
    sum_i |g_i| (the tensor-core chunks are summed with round-to-nearest adds, whose error grows as sqrt of the count)."""
    _, nf, N = TS_SHAPES[preset]
    windows = _windows(nf, N, k)
    ref = _step(preset, windows, accumulate=k)
    ref()
    torch.cuda.synchronize()
    g_ref, loss_ref = ref.flat_grad.clone(), ref.loss.clone()
    gabs = torch.zeros_like(g_ref, dtype=torch.float64)
    layout = ref.layout
    del ref
    # per-window gradients (accumulate=1 steps) for sum_i |g_i|
    one = _step(preset, windows, accumulate=1)
    for w in windows:
        one.load(w)
        one()
        gabs += one.flat_grad.double().abs()
    del one
    ts = _step(preset, windows, accumulate=k, batched=True)
    ts()
    torch.cuda.synchronize()
    first = ts.flat_grad.clone()
    R = k * nf * N
    scale = torch.zeros_like(gabs)
    for off, shp in zip(layout.offsets, layout.shapes):
        if off is not None:
            scale[off:off + shp.numel()] = gabs[off:off + shp.numel()].max()
    bound = k * U * gabs + 2 * math.sqrt(R) * U * scale
    _within(f"batched k={k} {preset} gradient", (first.double() - g_ref.double()).abs(), bound, "batched")
    assert _bits(ts.loss, loss_ref), (float(ts.loss), float(loss_ref))
    ts()                                                     # same weights, same windows: the same bits again
    torch.cuda.synchronize()
    assert _bits(first, ts.flat_grad)


def test_batched_replay_equals_eager_and_k1_equals_default():
    _, nf, N = TS_SHAPES["tiny"]
    windows = _windows(nf, N, 2)
    outs = {}
    for name, kw in (("graph", dict(accumulate=2, batched=True)), ("eager", dict(accumulate=2, batched=True, graph=False)),
                     ("k1", dict(accumulate=1, batched=True)), ("default", dict(accumulate=1))):
        ts = _step("tiny", windows, lr=1e-3, **kw)
        for _ in range(3):
            ts()
        torch.cuda.synchronize()
        outs[name] = (ts.flat_param.clone(), ts.flat_grad.clone(), ts.loss.clone())
        del ts
    for a, b in (("graph", "eager"), ("k1", "default")):
        for x, y in zip(outs[a], outs[b]):
            assert _bits(x, y), (a, b)


# --------------------------------------------------------------------------------------------------
# Trainer(batched=True)
# --------------------------------------------------------------------------------------------------
def test_trainer_batched_trains_like_accumulate(tmp_path, caplog):
    """Same csv, config and seeds: batched=True trains the windows accumulate=2 trains, in the same order, logs the same
    lines (the first one's values, taken before any update, agree to 1e-4: the gradient order aside, a linear layer with
    fewer than 32 rows per window may run on the other kernel when its rows double), writes the same checkpoint files, and
    each checkpoint resumes into a fresh batched Trainer."""
    import logging
    from tests import test_gpu_trainer as T
    from dynamicpdb_b200.trainer import Trainer
    csv_path, _ = T._files(tmp_path)
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    runs = {}
    for batched in (False, True):
        ck = str(tmp_path / f"ck{int(batched)}")
        conf = T._conf(csv_path, batch_size=2, num_epoch=3, log_freq=1, ckpt_freq=1, ckpt_dir=ck)
        caplog.clear()
        with caplog.at_level(logging.INFO, logger="dynamicpdb_b200.trainer"):
            tr = Trainer(conf, T._net(), diffuser, accumulate=2, batched=batched)
            assert tr.step.graph is not None and tr.step.batched == batched, tr.step.graph_error
            order = [tr.windows(e) for e in range(3)]
            tr.train()
        torch.cuda.synchronize()
        lines = [m for m in caplog.messages if m.startswith("Epoch[")]
        files = sorted(os.listdir(ck))
        runs[batched] = (order, [l.split(": total_loss=")[0] for l in lines], files,
                         [float(v.split("=")[1].rstrip(",")) for v in lines[0].split(": ", 2)[2].split()[:4]])
        resumed = Trainer(conf, T._net(seed=99), diffuser, accumulate=2, batched=batched)
        resumed.resume(os.path.join(ck, files[-1]))
        assert (resumed.trained_epochs, resumed.trained_steps) == (3, tr.trained_steps)
        assert _bits(resumed.step.flat_param, tr.step.flat_param)
        assert set(T.LOGGED) <= set(tr.step.aux)
        del tr, resumed
    assert runs[True][0] == runs[False][0]
    assert runs[True][1] == runs[False][1] and runs[True][2] == runs[False][2] and runs[True][2]
    for a, b in zip(runs[True][3], runs[False][3]):
        assert abs(a - b) <= 1e-4 * max(1.0, abs(b)) + 1e-4, (runs[True][3], runs[False][3])
