"""-m gpu: the explicit-width split-bf16 GEMM entry points (dfold_gemm_bf16x3_bn, dfold_gemm_wgrad_bf16x3_bn) and the
tile width the 5x5 convolution picks with them.

  * At the convolution GEMMs of one preset-A training step (64 frames x 256 residues, full and cropped layers; forward,
    data gradient and weight gradient) both widths give the same bits, and the same bits as the entry point that picks
    its width itself.  Each output element is one CTA's fixed-order k loop either way, so a difference would mean the
    tensor core's in-MMA reduction depends on the tile width.
  * On reduced shapes that keep every tap, both widths pass the float64 bounds of test_gpu_gemm.py, leave a NaN sentinel
    outside the valid region untouched, give the same bits twice, and launch the CTA count of the width asked for.
  * conv5x5 and its backward launch the width kernels.TILE_COST chooses, counted in CTAs.
"""
import math

import pytest
import torch

from dynamicpdb_b200 import kernels as K
from tests import test_gpu_gemm as G

pytestmark = pytest.mark.gpu
DEV = "cuda"
BM = 128
TAPS = 25


def cdiv(a, b):
    return -(-a // b)


class ConvGemm:
    """One GEMM of a 5x5 convolution layer ci -> co over f_in frames of n residues that produces only the last
    f_in - crop output frames, as kernels._Conv5x5Fn calls it, on random operand planes.  kind: fwd, dgrad or wgrad."""

    def __init__(self, kind, ci, co, f_in, crop, n, seed=0):
        self.kind, self.ci, self.co, self.f_in, self.crop, self.n = kind, ci, co, f_in, crop, n
        fo = f_in - crop
        self.flop = 2.0 * TAPS * fo * n * ci * co
        g = torch.Generator(device=DEV).manual_seed(seed + 2)
        if kind == "fwd":
            a, b = G.Op(f_in * n * ci, seed), G.Op(TAPS * co * ci, seed + 1, scale=1.0 / math.sqrt(TAPS * ci))
            bias, res = torch.randn(co, generator=g, device=DEV), torch.randn(fo * n * co, generator=g, device=DEV)
            self.entry, self.n_out, self.row_tiles, self.num_kb = "dfold_gemm_bf16x3", co, fo * cdiv(n, BM), TAPS * cdiv(ci, 64)
            self.out_numel = fo * n * co
            self.args = lambda out: (a.hi, a.lo, f_in, fo, crop, n, ci, ci, b.hi, b.lo, co, ci, 5, 5, out, co, bias, res, co,
                                     1.0, 1.0, 1)
        elif kind == "dgrad":
            a, b = G.Op(fo * n * co, seed), G.Op(TAPS * ci * co, seed + 1, scale=1.0 / math.sqrt(TAPS * co))
            self.entry, self.n_out, self.row_tiles, self.num_kb = "dfold_gemm_bf16x3", ci, f_in * cdiv(n, BM), TAPS * cdiv(co, 64)
            self.out_numel = f_in * n * ci
            self.args = lambda out: (a.hi, a.lo, fo, f_in, -crop, n, co, co, b.hi, b.lo, ci, co, 5, 5, out, ci, None, None, 0,
                                     1.0, 0.0, 0)
        else:
            a, b = G.Op(fo * n * co, seed), G.Op(f_in * n * ci, seed + 1, scale=1.0 / math.sqrt(fo * n))
            self.entry, self.n_out, self.row_tiles, self.num_kb = "dfold_gemm_wgrad_bf16x3", ci, cdiv(co, BM) * TAPS, fo * cdiv(n, 64)
            self.out_numel = TAPS * co * ci
            self.args = lambda out: (a.hi, a.lo, co, co, b.hi, b.lo, ci, ci, fo, f_in, crop, n, 5, 5, out, ci, 1.0)
        self.name = f"{kind} {ci}->{co} F{f_in}" + (f" crop{crop}" if crop else "")

    def tiles(self, bn):
        return cdiv(self.n_out, bn) * self.row_tiles

    def launch(self, out, bn=None):
        """Into `out`; bn None: the entry point that picks the width, else the explicit-width one."""
        if bn is None:
            K.launch(self.entry, *self.args(out))
        else:
            K.launch(self.entry + "_bn", *self.args(out), bn)

    def run(self, bn=None):
        out = torch.full((self.out_numel,), float("nan"), device=DEV)
        self.launch(out, bn)
        return out


def step_conv_gemms(frames=64, n=256, dim=1280):
    """(kind, ci, co, f_in, crop) of every distinct convolution GEMM of one training step: the full ConvNet of the first and
    last blocks alternates dim -> dim / 2 -> dim, and the middle blocks run layer k on 17 - 2k frames cropped by 2."""
    layers = [(dim, dim // 2, frames, 0), (dim // 2, dim, frames, 0)]
    layers += [((dim, dim // 2) if k % 2 == 0 else (dim // 2, dim)) + (17 - 2 * k, 2) for k in range(8)]
    return [(kind,) + layer for layer in layers for kind in ("fwd", "dgrad", "wgrad")]


STEP = step_conv_gemms()


@pytest.mark.parametrize("case", STEP, ids=lambda c: f"{c[0]}-{c[1]}to{c[2]}-F{c[3]}-crop{c[4]}")
def test_same_bits_at_either_width(case):
    g = ConvGemm(*case, n=256, seed=STEP.index(case))
    ref = g.run()
    for bn in (64, 128):
        got = g.run(bn)
        torch.cuda.synchronize()
        assert not torch.isnan(got).any(), f"{g.name} BN {bn}: output not written"
        diff = int((got.view(torch.int32) != ref.view(torch.int32)).sum())
        assert diff == 0, f"{g.name}: BN = {bn} differs from {g.entry} in {diff} of {ref.numel()} elements"


class _FixedWidth:
    """The C-ABI library with its self-choosing GEMM entry points routed to the explicit-width ones at width `bn`."""

    def __init__(self, lib, bn):
        self._lib, self._bn = lib, bn

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def dfold_gemm_bf16x3(self, *args):
        return self._lib.dfold_gemm_bf16x3_bn(*args[:-1], self._bn, args[-1])

    def dfold_gemm_wgrad_bf16x3(self, *args):
        return self._lib.dfold_gemm_wgrad_bf16x3_bn(*args[:-1], self._bn, args[-1])


@pytest.fixture(params=[64, 128])
def width(request, monkeypatch):
    """test_gpu_gemm's float64 harness, run at one tile width: its launches go to the explicit-width entry points and
    the width it checks the CTA count against is this one."""
    lib = _FixedWidth(K.lib(), request.param)
    monkeypatch.setattr(K, "lib", lambda: lib)
    monkeypatch.setattr(G, "pick_bn", lambda n_out, row_tiles: request.param)
    return request.param


# every 5x5 case of test_gpu_gemm.py (halo-only pixels, row / column / K tails, cropped frames) plus a cropped layer of
# the step's channel counts, reduced to a few frames
CONV_CASES = [c for c in G.GEMM_CASES if c[4] == (5, 5)] + [
    (4, 256, 1280, 640, (5, 5), 2, 2, None),          # cropped forward, dim -> dim / 2
    (2, 256, 640, 1280, (5, 5), 4, -2, None),         # its data gradient
]
WGRAD_CASES = [c for c in G.WGRAD_CASES if c[4] == (5, 5)] + [
    (640, 1280, 2, 256, (5, 5), 4, 2, None, None, None),   # cropped weight gradient of dim -> dim / 2
]


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: f"F{c[0]}N{c[1]}K{c[2]}n{c[3]}fs{c[6]}")
def test_conv_bounds(width, case):
    F, Nr, Kd, n_out, taps, F_out, f_start, lda = case
    _, bn = G.run_gemm(F, Nr, Kd, n_out, taps, F_out, f_start, lda, ldo=n_out + 8, out_ofs=2, seed=CONV_CASES.index(case),
                       bscale=1.0 / math.sqrt(Kd * TAPS))
    assert bn == width


@pytest.mark.parametrize("act", [0, 1])
def test_conv_epilogue_bounds(width, act):
    """bias, ReLU and residual on both widths' column loops, with a column tail in either tile"""
    G.run_gemm(3, 40, 64, 200, taps=(5, 5), F_out=2, f_start=1, ldo=201, out_ofs=1, bias=True, res=True, alpha=1.25,
               beta=0.5, act=act, seed=40 + act, bscale=0.025)


@pytest.mark.parametrize("case", WGRAD_CASES, ids=lambda c: f"M{c[0]}n{c[1]}F{c[2]}N{c[3]}add{c[6]}")
def test_wgrad_bounds(width, case):
    M, Nn, F, Nr, taps, Fb, b_f_add, lda, ldb, ldo = case
    _, bn = G.run_wgrad(M, Nn, F, Nr, taps, Fb, b_f_add, lda, ldb, Nn + 3 if ldo is None else ldo, alpha=0.75,
                        seed=200 + WGRAD_CASES.index(case))
    assert bn == width


def test_other_widths_rejected():
    a = G.Op(2 * 64 * 136, 1)
    b = G.Op(25 * 64 * 136, 2)
    s = K._stream()
    for bn in (0, 32, 96, 192, 256):
        G._rejected(lambda L, o: L.dfold_gemm_bf16x3_bn(K._ptr(a.hi), K._ptr(a.lo), 1, 1, 0, 16, 64, 64, K._ptr(b.hi),
                                                        K._ptr(b.lo), 16, 64, 5, 5, o, 16, None, None, 0, 1.0, 0.0, 0, bn, s),
                    "tile width must be 64 or 128")
        G._rejected(lambda L, o: L.dfold_gemm_wgrad_bf16x3_bn(K._ptr(a.hi), K._ptr(a.lo), 16, 16, K._ptr(b.hi), K._ptr(b.lo),
                                                              16, 16, 1, 1, 0, 16, 5, 5, o, 16, 1.0, bn, s),
                    "tile width must be 64 or 128")


# --------------------------------------------------------------------------------------------------
# the width the convolution launches
# --------------------------------------------------------------------------------------------------
def model_bn(n_out, row_tiles):
    """The width with the least waves x TILE_COST on this device, ties to 128 (kernels._conv_bn)."""
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    cost = {bn: cdiv(cdiv(n_out, bn) * row_tiles, sms) * K.TILE_COST[bn] for bn in (64, 128)}
    return 64 if cost[64] < cost[128] else 128


def _ctas(fn):
    """CTAs of the one GEMM launch `fn` makes (every other launch of it is not a GEMM)."""
    stats = torch.zeros(4 * 200000, dtype=torch.int64, device=DEV)
    torch.cuda.synchronize()
    K.lib().dfold_debug_gemm_stats(K._ptr(stats))
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        K.lib().dfold_debug_gemm_stats(None)
    return int((stats.view(-1, 4)[:, 0] != 0).sum())


@pytest.mark.parametrize("case", STEP, ids=lambda c: f"{c[0]}-{c[1]}to{c[2]}-F{c[3]}-crop{c[4]}")
def test_conv_launches_the_model_width(case):
    kind, ci, co, f_in, crop = case
    g = ConvGemm(kind, ci, co, f_in, crop, n=256)
    want = model_bn(g.n_out, g.row_tiles)
    gen = torch.Generator(device=DEV).manual_seed(5)
    x = torch.randn(f_in, 256, ci, generator=gen, device=DEV, requires_grad=kind == "dgrad")
    w = (torch.randn(co, ci, 5, 5, generator=gen, device=DEV) / math.sqrt(25 * ci)).requires_grad_(kind == "wgrad")
    b = torch.randn(co, generator=gen, device=DEV)
    if kind == "fwd":
        with torch.no_grad():
            ran = _ctas(lambda: K.conv5x5(x, w, b, crop=crop))
    else:
        y = K.conv5x5(x, w, b, crop=crop)
        dy = torch.randn_like(y)
        ran = _ctas(lambda: y.backward(dy))
    assert ran == g.tiles(want), (f"{g.name}: {ran} CTAs ran; the model picks BN = {want} ({g.tiles(want)} CTAs; "
                                  f"BN = {192 - want}: {g.tiles(192 - want)})")
