"""-m gpu: the four split-bf16 wgmma GEMM entry points of csrc/gemm_sm90.cu, called directly through the C ABI and
compared element by element with float64.

The operand planes are built here with torch (hi = bf16(x), lo = bf16(x - hi), round to nearest, as csrc/simt.cu), so
the tests do not depend on dfold_split2d.  Every output element is held to its own error scale S = |A|.|B|, the same
contraction (taps, batching and strides included) over absolute values:

  |C - R3| <= C_ACC * S               R3 = hi.hi + hi.lo + lo.hi in float64, what the kernel is specified to compute
  |C - R|  <= (SPLIT + C_ACC) * S     R  = the float64 product of the fp32 inputs (adds the split-precision error,
                                          SPLIT ~ 3 * 2^-16, derived below)

A max-normalised metric cannot see an element that is wrong by 100 % of its own small value (a dropped k-block, a wrong
tap shift at the image border, a wrong batch slice); this one does.  Each case also
  * checks which tile width ran (dfold_debug_gemm_stats counts the CTAs) against the width `pick_bn` chooses on this
    device, and every entry point has cases of both widths;
  * fills the output with a NaN sentinel first and requires every element outside the valid rows / columns to keep it;
  * launches twice and requires the same bits.
Buffers are filled with random values INCLUDING the padding past the valid columns, so a read past K shows up.
"""
import json
import math
import os

import pytest
import torch
import torch.nn.functional as TF

from dynamicpdb_b200 import kernels as K

pytestmark = pytest.mark.gpu
DEV = "cuda"
BM = 128

# Accumulation error bound, relative to S.  Measured on an H100 80GB HBM3 (400 W power limit): worst |C - R3| / S over
# every case here 1.64e-6 (weight gradient, all-positive operands, K = 256), 1.26e-6 at K = 16384 and 1.20e-6 at
# K = 32000.  The bound is 2.3x the worst measurement.
C_ACC = 2.0 ** -18
# Split error.  x = hi + lo + e with |lo| <= 2^-8 |x| and |e| <= 2^-8 |lo| <= 2^-16 |x| (two round-to-nearest bf16
# roundings, 8 significant bits each), so  a b - (hi_a hi_b + hi_a lo_b + lo_a hi_b) = lo_a lo_b + e_a b + (a - e_a) e_b
# is at most (2^-16 + 2^-16 + 2^-16 (1 + 2^-16)) |a||b|.  Measured worst |C - R| / S: 2.30e-5.
SPLIT = 3.0 * 2.0 ** -16 * (1 + 2.0 ** -16)
# fp32 rounding of the epilogue (alpha scale, bias add, __expf in SiLU for |x| < 10, residual add), relative to the
# magnitudes that enter it
EPI = 2.0 ** -19


def cdiv(a, b):
    return -(-a // b)


def pad8(n):
    return cdiv(n, 8) * 8


def pick_bn(n_out, row_tiles):
    """The tile width gemm_sm90.cu's pick_bn chooses on this device: the smallest waves x BN, ties to 128."""
    if n_out <= 64:
        return 64
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    c128 = cdiv(cdiv(n_out, 128) * row_tiles, sms) * 128
    c64 = cdiv(cdiv(n_out, 64) * row_tiles, sms) * 64
    return 64 if c64 < c128 else 128


class Op:
    """A flat fp32 operand buffer (padding included) and its bf16 hi / lo planes."""

    def __init__(self, numel, seed, positive=False, scale=1.0):
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.x = torch.rand(numel, generator=g, device=DEV) if positive else torch.randn(numel, generator=g, device=DEV)
        self.x *= scale
        hi = self.x.to(torch.bfloat16)
        lo = (self.x - hi.float()).to(torch.bfloat16)
        self.hi, self.lo = hi.view(torch.int16), lo.view(torch.int16)

    def f64(self, dev):
        x = self.x.to(dev, torch.float64)
        hi = self.hi.view(torch.bfloat16).to(dev, torch.float64)
        lo = self.lo.view(torch.bfloat16).to(dev, torch.float64)
        return {"x": x, "hi": hi, "lo": lo, "hl": hi + lo, "abs": x.abs()}


def _refs(contract, a, b, dev):
    """(R3, R, S) of a bilinear contraction of two operands, in float64 on `dev`."""
    A, B = a.f64(dev), b.f64(dev)
    r3 = contract(A["hl"], B["hi"]) + contract(A["hi"], B["lo"])
    return r3, contract(A["x"], B["x"]), contract(A["abs"], B["abs"])


def _ref_dev(*ops):
    return DEV if sum(o.x.numel() for o in ops) > (1 << 21) else "cpu"


def _shift(X, n_frames, f_off, dn):
    """Y[f, n] = X[f + f_off, n + dn] for f < n_frames, zero outside X (the TMA out-of-bounds fill)."""
    F, Nr = X.shape[:2]
    Y = X.new_zeros((n_frames, Nr) + tuple(X.shape[2:]))
    f0, f1 = max(0, -f_off), min(n_frames, F - f_off)
    n0, n1 = max(0, -dn), min(Nr, Nr - dn)
    if f0 < f1 and n0 < n1:
        Y[f0:f1, n0:n1] = X[f0 + f_off:f1 + f_off, n0 + dn:n1 + dn]
    return Y


def _record(**kw):
    """Appends one case's measured error ratios to the JSON-lines file DFOLD_GEMM_ERRORS names (calibration aid)."""
    path = os.environ.get("DFOLD_GEMM_ERRORS")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(kw) + "\n")


def _launch(fn, out_numel, out_ofs, ctas):
    """Runs fn(out_ptr) twice into NaN-filled buffers, the first time with the CTA-cycle hook on.
    Returns (out, number of CTAs that ran)."""
    L = K.lib()
    outs = []
    stats = torch.zeros(4 * ctas + 64, dtype=torch.int64, device=DEV)
    for rep in range(2):
        buf = torch.full((out_numel + out_ofs + 8,), float("nan"), device=DEV)
        if rep == 0:
            L.dfold_debug_gemm_stats(K._ptr(stats))
        try:
            rc = fn(K._ptr(buf, out_ofs))
        finally:
            L.dfold_debug_gemm_stats(None)
        assert rc == 0, L.dfold_last_error().decode()
        torch.cuda.synchronize()
        outs.append(buf)
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), "second launch gave different bits"
    ran = int((stats.view(-1, 4)[:, 0] != 0).sum())
    return outs[0], ran


def _check_width(ran, bn, n_cols, row_tiles_z, what):
    expect = cdiv(n_cols, bn) * row_tiles_z
    other = cdiv(n_cols, 192 - bn) * row_tiles_z
    assert ran == expect, f"{what}: {ran} CTAs ran; BN = {bn} launches {expect} (BN = {192 - bn}: {other})"


def _outside_untouched(what, buf, out_ofs, pos):
    keep = torch.ones(buf.numel(), dtype=torch.bool, device=DEV)
    keep[out_ofs:][pos.to(DEV).reshape(-1)] = False
    assert torch.isnan(buf[keep]).all(), f"{what}: {int((~torch.isnan(buf[keep])).sum())} elements outside the output were written"


def _compare(what, buf, out_ofs, pos, r3, r, s, *, alpha=1.0, epi=None, lip=1.0, outside=True):
    """Every element at flat positions `pos` against its references; everything else must still be NaN.
    epi(y) maps a pre-activation reference to (output, extra tolerance for the fp32 rounding of the epilogue)."""
    dev = r3.device
    got = buf[out_ofs:][pos.to(DEV)].to(dev, torch.float64)
    assert torch.isfinite(got).all(), f"{what}: non-finite outputs"
    scale = abs(alpha) * s * lip
    if epi is None:
        w3, w, extra = alpha * r3, alpha * r, 0.0
    else:
        (w3, extra), (w, _) = epi(alpha * r3), epi(alpha * r)
    e3 = (got - w3).abs()
    e = (got - w).abs()
    ratio3 = ((e3 - extra).clamp(min=0) / scale.clamp(min=1e-300)).max().item()
    ratio = ((e - extra).clamp(min=0) / scale.clamp(min=1e-300)).max().item()
    _record(case=what, r3_over_s=ratio3, r_over_s=ratio, epilogue=epi is not None)
    bad3 = e3 > C_ACC * scale + extra
    assert not bad3.any(), (f"{what}: {int(bad3.sum())} elements off R3 by more than C_ACC * S (worst |C-R3|/S = {ratio3:.3e}); "
                            f"first at flat index {int(pos.reshape(-1)[bad3.reshape(-1).nonzero()[0]])}")
    bad = e > (SPLIT + C_ACC) * scale + extra
    assert not bad.any(), f"{what}: {int(bad.sum())} elements off R by more than (SPLIT + C_ACC) * S (worst {ratio:.3e})"
    if outside:
        _outside_untouched(what, buf, out_ofs, pos)
    return ratio3


# --------------------------------------------------------------------------------------------------
# dfold_gemm_bf16x3: linear layers and the 5x5 convolution (K-major)
# --------------------------------------------------------------------------------------------------
def run_gemm(F, Nr, Kd, n_out, taps=(1, 1), F_out=None, f_start=0, lda=None, ldb=None, ldo=None, out_ofs=0,
             bias=False, res=False, alpha=1.0, beta=0.0, act=0, positive=False, seed=0, bscale=1.0):
    F_out = F if F_out is None else F_out
    lda = pad8(Kd) if lda is None else lda
    ldb = pad8(Kd) if ldb is None else ldb
    ldo = n_out if ldo is None else ldo
    tf, tn = taps
    T = tf * tn
    a = Op(F * Nr * lda, seed, positive)
    b = Op(T * n_out * ldb, seed + 1, positive, bscale)
    g =torch.Generator(device=DEV).manual_seed(seed + 2)
    bias_t = torch.randn(n_out, generator=g, device=DEV) if bias else None
    ldr = n_out + 5
    res_t = torch.randn(F_out * Nr * ldr, generator=g, device=DEV) if res else None
    rows = F_out * Nr
    row_tiles = F_out * cdiv(Nr, BM)
    bn = pick_bn(n_out, row_tiles)
    L = K.lib()

    def fn(out_ptr):
        return L.dfold_gemm_bf16x3(K._ptr(a.hi), K._ptr(a.lo), F, F_out, f_start, Nr, Kd, lda, K._ptr(b.hi), K._ptr(b.lo),
                                   n_out, ldb, tf, tn, out_ptr, ldo, K._ptr(bias_t), K._ptr(res_t), ldr,
                                   alpha, beta, act, K._stream())
    buf, ran = _launch(fn, rows * ldo, out_ofs, cdiv(n_out, 64) * row_tiles)
    what = f"gemm F{F}->{F_out} f_start{f_start} Nr{Nr} K{Kd} lda{lda} n{n_out} taps{tf}x{tn} ldo{ldo}+{out_ofs} act{act}"
    _check_width(ran, bn, n_out, row_tiles, what)

    dev = _ref_dev(a, b)

    def contract(A, B):
        A3 = A.as_strided((F, Nr, Kd), (Nr * lda, lda, 1))
        B3 = B.as_strided((T, n_out, Kd), (n_out * ldb, ldb, 1))
        out = A.new_zeros(rows, n_out)
        for t in range(T):
            df, dn = t // tn - tf // 2, t % tn - tn // 2
            out += _shift(A3, F_out, f_start + df, dn).reshape(rows, Kd) @ B3[t].T
        return out
    r3, r, s = _refs(contract, a, b, dev)
    pos = (torch.arange(rows, device=dev)[:, None] * ldo + torch.arange(n_out, device=dev)[None, :])
    epi, lip = None, 1.0
    if bias or res or act:
        bd = bias_t.to(dev, torch.float64) if bias else torch.zeros(n_out, dtype=torch.float64, device=dev)
        rd = (res_t.to(dev, torch.float64).reshape(rows, ldr)[:, :n_out] * beta) if res else 0.0
        lip = 1.1 if act == 2 else 1.0       # max |d silu / dx| = 1.0998

        def epi(pre):
            y = pre + bd
            mag = y.abs() + bd.abs() + pre.abs()
            if act == 1:
                y = y.clamp(min=0)
            elif act == 2:
                y = TF.silu(y)
            y = y + rd
            return y, EPI * (mag + (rd.abs() if res else 0.0))
    return _compare(what, buf, out_ofs, pos, r3, r, s, alpha=alpha, epi=epi, lip=lip), bn


GEMM_CASES = [
    # (F, Nr, K, n_out, taps, F_out, f_start, lda)
    (1, 100, 64, 96, (1, 1), None, 0, None),          # num_kb = 1
    (1, 300, 512, 200, (1, 1), None, 0, None),        # num_kb = 8 (0 mod 4); row tail; column tail at both widths
    (1, 300, 320, 8, (1, 1), None, 0, None),          # num_kb = 5 (1 mod 4); n_out = 8
    (1, 5, 448, 72, (1, 1), None, 0, None),           # num_kb = 7 (3 mod 4); Nr < 8
    (1, 130, 200, 136, (1, 1), None, 0, 208),         # K tail (200 = 3 x 64 + 8), lda > K
    (1, 64, 72, 64, (1, 1), None, 0, 96),             # K tail, 2 k-blocks, lda > K + 8
    (1, 5000, 136, 256, (1, 1), None, 0, 144),        # BN = 128, K tail
    (1, 1, 64, 80, (5, 5), None, 0, None),            # 5x5: one pixel, every tap but the centre in the halo
    (2, 2, 64, 72, (5, 5), None, 0, None),            # 5x5: F = 2, Nr = 2
    (1, 3, 128, 64, (5, 5), None, 0, None),           # 5x5: Nr = 3, 50 k-blocks
    (7, 40, 64, 128, (5, 5), 5, 2, None),             # cropped forward: the last 5 of 7 frames
    (5, 40, 64, 96, (5, 5), 7, -2, None),             # its data gradient (f_start < 0)
    (3, 130, 88, 136, (5, 5), None, 0, 96),           # 5x5 with a K tail, row and column tails
    (8, 256, 64, 640, (5, 5), None, 0, None),         # 5x5 at BN = 128
    (2, 20, 64, 40, (1, 5), None, 0, None),           # 1 x 5 taps
]


@pytest.mark.parametrize("case", GEMM_CASES, ids=lambda c: f"F{c[0]}N{c[1]}K{c[2]}n{c[3]}t{c[4][0]}{c[4][1]}fs{c[6]}")
def test_gemm(case):
    F, Nr, Kd, n_out, taps, F_out, f_start, lda = case
    run_gemm(F, Nr, Kd, n_out, taps, F_out, f_start, lda, seed=GEMM_CASES.index(case),
             bscale=1.0 / math.sqrt(Kd * taps[0] * taps[1]))


@pytest.mark.parametrize("act,odd", [(0, False), (1, True), (2, False), (2, True), (1, False)])
def test_gemm_epilogue(act, odd):
    """bias, activation, alpha != 1, beta * residual; an odd ldo with an output pointer one float off 8-byte alignment
    takes the scalar store path."""
    n_out = 200
    run_gemm(1, 300, 200, n_out, lda=208, ldo=n_out + 1 if odd else n_out + 8, out_ofs=1 if odd else 0,
             bias=True, res=True, alpha=0.8125, beta=-0.625, act=act, seed=11 + act, bscale=1.0 / math.sqrt(200))
    run_gemm(3, 40, 64, 72, taps=(5, 5), F_out=2, f_start=1, ldo=73 if odd else 72, out_ofs=1 if odd else 0,
             bias=True, res=True, alpha=1.25, beta=0.5, act=act, seed=21 + act, bscale=0.025)


def test_gemm_widths_covered():
    """The parametrisation above runs both tile widths on this device (each case checks the width that ran)."""
    widths = {pick_bn(c[3], (c[5] or c[0]) * cdiv(c[1], BM)) for c in GEMM_CASES}
    assert widths == {64, 128}, widths


# --------------------------------------------------------------------------------------------------
# dfold_gemm_wgrad_bf16x3: weight gradients (MN-major, K = pixels)
# --------------------------------------------------------------------------------------------------
def run_wgrad(M, Nn, F, Nr, taps=(1, 1), Fb=None, b_f_add=0, lda=None, ldb=None, ldo=None, alpha=1.0, positive=False, seed=0):
    Fb = F if Fb is None else Fb
    lda = pad8(M) if lda is None else lda
    ldb = pad8(Nn) if ldb is None else ldb
    ldo = Nn if ldo is None else ldo
    tf, tn = taps
    T = tf * tn
    a = Op(F * Nr * lda, seed, positive)
    b = Op(Fb * Nr * ldb, seed + 1, positive)
    rt = cdiv(M, BM) * T
    bn = pick_bn(Nn, rt)
    L = K.lib()

    def fn(out_ptr):
        return L.dfold_gemm_wgrad_bf16x3(K._ptr(a.hi), K._ptr(a.lo), M, lda, K._ptr(b.hi), K._ptr(b.lo), Nn, ldb,
                                         F, Fb, b_f_add, Nr, tf, tn, out_ptr, ldo, alpha, K._stream())
    buf, ran = _launch(fn, T * M * ldo, 0, cdiv(Nn, 64) * rt)
    what = f"wgrad M{M} n{Nn} F{F}/{Fb}+{b_f_add} Nr{Nr} taps{tf}x{tn} lda{lda} ldb{ldb} ldo{ldo}"
    _check_width(ran, bn, Nn, rt, what)

    def contract(A, B):
        A2 = A.as_strided((F, Nr, M), (Nr * lda, lda, 1)).reshape(F * Nr, M)
        B3 = B.as_strided((Fb, Nr, Nn), (Nr * ldb, ldb, 1))
        outs = []
        for t in range(T):
            df, dn = t // tn - tf // 2, t % tn - tn // 2
            outs.append(A2.T @ _shift(B3, F, b_f_add + df, dn).reshape(F * Nr, Nn))
        return torch.stack(outs)
    dev = _ref_dev(a, b)
    r3, r, s = _refs(contract, a, b, dev)
    ar = lambda n: torch.arange(n, device=dev)
    pos = ar(T)[:, None, None] * (M * ldo) + ar(M)[None, :, None] * ldo + ar(Nn)[None, None, :]
    _outside_untouched(what, buf, 0, pos)
    # tap by tap, so that a failure names the tap
    worst = max(_compare(f"{what} tap {t}", buf, 0, pos[t], r3[t], r[t], s[t], alpha=alpha, outside=False) for t in range(T))
    return worst, bn


WGRAD_CASES = [
    # (M, Nn, F, Nr, taps, Fb, b_f_add, lda, ldb, ldo)
    (96, 200, 1, 64, (1, 1), None, 0, None, None, None),       # num_kb = 1
    (200, 72, 1, 300, (1, 1), None, 0, None, None, None),      # num_kb = 5, K (pixel) tail, row tail
    (64, 8, 7, 64, (1, 1), None, 0, None, None, None),         # num_kb = 7; Nn = 8
    (130, 136, 2, 256, (1, 1), None, 0, 136, 144, 141),        # num_kb = 8; padded planes, odd ldo
    (40, 64, 1, 5, (1, 1), None, 0, None, None, None),         # 5 pixels
    (64, 80, 1, 1, (5, 5), None, 0, None, None, None),         # 5x5, one pixel: every tap but the centre reads the halo
    (72, 64, 2, 2, (5, 5), None, 0, None, None, None),         # 5x5, F = 2, Nr = 2
    (64, 72, 1, 3, (5, 5), None, 0, None, None, None),         # 5x5, Nr = 3
    (64, 96, 5, 40, (5, 5), 7, 2, None, None, None),           # cropped: A frame f pairs with B frame f + 2
    (136, 72, 3, 70, (5, 5), None, 0, None, None, None),       # 5x5, row / column / pixel tails
    (256, 256, 2, 64, (5, 5), None, 0, None, None, None),      # 5x5 at BN = 128
]


@pytest.mark.parametrize("case", WGRAD_CASES, ids=lambda c: f"M{c[0]}n{c[1]}F{c[2]}N{c[3]}t{c[4][0]}add{c[6]}")
def test_wgrad(case):
    M, Nn, F, Nr, taps, Fb, b_f_add, lda, ldb, ldo = case
    run_wgrad(M, Nn, F, Nr, taps, Fb, b_f_add, lda, ldb, ldo, alpha=0.75, seed=100 + WGRAD_CASES.index(case))


def test_wgrad_widths_covered():
    widths = {pick_bn(c[1], cdiv(c[0], BM) * c[4][0] * c[4][1]) for c in WGRAD_CASES}
    assert widths == {64, 128}, widths


# --------------------------------------------------------------------------------------------------
# dfold_gemm_bf16x3_batched (K-major) and dfold_gemm_wgrad_bf16x3_batched (MN-major)
# --------------------------------------------------------------------------------------------------
def run_batched(q, seed=0):
    """q: the call's arguments by name (plus the operand / output sizes a_numel, b_numel, out_numel, out_ofs)."""
    a = Op(q["a_numel"], seed)
    b = Op(q["b_numel"], seed + 1)
    nb, Nr, Kd, n_out = q["n_batches"], q["Nr"], q["K"], q["n_out"]
    rt = nb * cdiv(Nr, BM)
    bn = pick_bn(n_out, rt)
    L = K.lib()

    def fn(out_ptr):
        return L.dfold_gemm_bf16x3_batched(
            K._ptr(a.hi), K._ptr(a.lo), q["a_frames"], Nr, q["a_cols"], q["lda"], nb, q["bmod"], q["a_f_div"],
            q["a_k_bstride"], Kd, K._ptr(b.hi), K._ptr(b.lo), q["b_z"], q["b_rows"], q["b_cols"], q["ldb"], q["b_k_ofs"],
            q["b_k_bstride"], q["b_z_bstride"], n_out, out_ptr, q["ldo"], q["out_rows"], q["o_f_div"], q["o_col_bstride"],
            q["alpha"], K._stream())
    out_ofs = q.get("out_ofs", 0)
    buf, ran = _launch(fn, q["out_numel"], out_ofs, cdiv(n_out, 64) * rt)
    what = "batched " + q["name"]
    _check_width(ran, bn, n_out, rt, what)
    dev = _ref_dev(a, b)
    ar = lambda n: torch.arange(n, device=dev)
    bi = ar(nb)
    hb = bi % q["bmod"]
    ka = hb * q["a_k_bstride"]
    kb = q["b_k_ofs"] + hb * q["b_k_bstride"]

    def contract(A, B):
        A3 = A.as_strided((q["a_frames"], Nr, q["a_cols"]), (Nr * q["lda"], q["lda"], 1))
        B3 = B.as_strided((q["b_z"], q["b_rows"], q["b_cols"]), (q["b_rows"] * q["ldb"], q["ldb"], 1))
        # zero past the valid columns / rows (TMA out-of-bounds fill)
        A3 = TF.pad(A3, (0, max(0, int(ka.max()) + Kd - q["a_cols"])))
        B3 = TF.pad(B3, (0, max(0, int(kb.max()) + Kd - q["b_cols"]), 0, max(0, n_out - q["b_rows"])))[:, :n_out]
        As = torch.gather(A3[bi // q["a_f_div"]], 2, (ka[:, None] + ar(Kd)[None, :])[:, None, :].expand(nb, Nr, Kd))
        Bs = torch.gather(B3[hb * q["b_z_bstride"]], 2, (kb[:, None] + ar(Kd)[None, :])[:, None, :].expand(nb, n_out, Kd))
        return As @ Bs.transpose(1, 2)                                      # [nb, Nr, n_out]
    r3, r, s = _refs(contract, a, b, dev)
    rows = (bi // q["o_f_div"])[:, None] * Nr + ar(Nr)[None, :]
    cols = hb[:, None] * q["o_col_bstride"] + ar(n_out)[None, :]
    pos = rows[:, :, None] * q["ldo"] + cols[:, None, :]
    ok = (rows < q["out_rows"])[:, :, None].expand_as(pos)
    return _compare(what, buf, out_ofs, pos[ok], r3[ok], r[ok], s[ok], alpha=q["alpha"]), bn


def run_batched_mn(q, seed=0):
    a = Op(q["a_numel"], seed)
    b = Op(q["b_numel"], seed + 1)
    M, Nn, Fk, Nr, Z = q["M"], q["Nn"], q["Fk"], q["Nr"], q["zcount"]
    rt = cdiv(M, BM) * Z
    bn = pick_bn(Nn, rt)
    L = K.lib()

    def fn(out_ptr):
        return L.dfold_gemm_wgrad_bf16x3_batched(
            K._ptr(a.hi), K._ptr(a.lo), M, q["a_mid"], q["a_outer"], q["lda"], q["a_ostride"],
            K._ptr(b.hi), K._ptr(b.lo), q["b_cols"], q["b_mid"], q["b_outer"], q["ldb"], q["b_ostride"],
            Nn, Fk, Nr, Z, q["a_f_mul"], q["a_z_mul"], q["b_f_mul"], q["b_z_mul"], q["b_n_zmul"],
            out_ptr, q["ldo"], q["out_z_stride"], q["alpha"], K._stream())
    out_ofs = q.get("out_ofs", 0)
    buf, ran = _launch(fn, q["out_numel"], out_ofs, cdiv(Nn, 64) * rt)
    what = "batched_mn " + q["name"]
    _check_width(ran, bn, Nn, rt, what)
    dev = _ref_dev(a, b)
    ar = lambda n: torch.arange(n, device=dev)
    zi, fi = ar(Z), ar(Fk)
    ao = fi[None, :] * q["a_f_mul"] + zi[:, None] * q["a_z_mul"]          # [Z, Fk]
    bo = fi[None, :] * q["b_f_mul"] + zi[:, None] * q["b_z_mul"]
    cols = zi[:, None] * q["b_n_zmul"] + ar(Nn)[None, :]                   # [Z, Nn]

    def contract(A, B):
        A3 = A.as_strided((q["a_outer"], q["a_mid"], M), (q["a_ostride"], q["lda"], 1))
        B3 = B.as_strided((q["b_outer"], q["b_mid"], q["b_cols"]), (q["b_ostride"], q["ldb"], 1))
        A3 = TF.pad(A3, (0, 0, 0, max(0, Nr - q["a_mid"]), 0, max(0, int(ao.max()) + 1 - q["a_outer"])))[:, :Nr]
        B3 = TF.pad(B3, (0, max(0, int(cols.max()) + 1 - q["b_cols"]), 0, max(0, Nr - q["b_mid"]),
                         0, max(0, int(bo.max()) + 1 - q["b_outer"])))[:, :Nr]
        As = A3[ao]                                                        # [Z, Fk, Nr, M]
        Bs = torch.gather(B3[bo], 3, cols[:, None, None, :].expand(Z, Fk, Nr, Nn))
        return torch.einsum("zfjm,zfjn->zmn", As, Bs)
    r3, r, s = _refs(contract, a, b, dev)
    pos = zi[:, None, None] * q["out_z_stride"] + ar(M)[None, :, None] * q["ldo"] + ar(Nn)[None, None, :]
    return _compare(what, buf, out_ofs, pos, r3, r, s, alpha=q["alpha"]), bn


def _ipa_calls(F, N, H=8, C=256, Pv=12, Cp=32):
    """The batched GEMM calls of kernels._IpaAttnTCFn, argument for argument, at preset-A head geometry."""
    n8, D = pad8(N), H * (C + 8 * Pv + Cp)
    D8, PV3, c8, g8 = pad8(D), 3 * Pv, pad8(Cp), pad8(3 * Pv)
    FH = F * H
    km = dict(alpha=1.0)
    kmaj = {
        "PV": dict(km, a_numel=FH * N * n8, a_frames=FH, Nr=N, a_cols=N, lda=n8, n_batches=FH, bmod=H, a_f_div=1,
                   a_k_bstride=0, K=N, b_numel=H * C * n8, b_z=H, b_rows=C, b_cols=N, ldb=n8, b_k_ofs=0, b_k_bstride=0,
                   b_z_bstride=1, n_out=C, out_numel=F * N * D, ldo=D, out_rows=F * N, o_f_div=H, o_col_bstride=C),
        "dP": dict(km, a_numel=F * N * D8, a_frames=F, Nr=N, a_cols=D, lda=D8, n_batches=FH, bmod=H, a_f_div=H,
                   a_k_bstride=C, K=C, b_numel=N * H * 2 * C, b_z=1, b_rows=N, b_cols=H * 2 * C, ldb=H * 2 * C, b_k_ofs=C,
                   b_k_bstride=2 * C, b_z_bstride=0, n_out=N, out_numel=FH * N * N, ldo=N, out_rows=FH * N, o_f_div=1,
                   o_col_bstride=0),
        "Tz": dict(km, a_numel=N * FH * c8, a_frames=N, Nr=FH, a_cols=Cp, lda=c8, n_batches=N, bmod=N, a_f_div=1,
                   a_k_bstride=0, K=Cp, b_numel=N * N * c8, b_z=N, b_rows=N, b_cols=Cp, ldb=c8, b_k_ofs=0, b_k_bstride=0,
                   b_z_bstride=1, n_out=N, out_numel=N * FH * N, ldo=N, out_rows=N * FH, o_f_div=1, o_col_bstride=0),
        "Tog": dict(km, a_numel=FH * N * g8, a_frames=FH, Nr=N, a_cols=PV3, lda=g8, n_batches=FH, bmod=FH, a_f_div=1,
                    a_k_bstride=0, K=PV3, b_numel=FH * N * g8, b_z=FH, b_rows=N, b_cols=PV3, ldb=g8, b_k_ofs=0,
                    b_k_bstride=0, b_z_bstride=1, n_out=N, out_numel=FH * N * N, ldo=N, out_rows=FH * N, o_f_div=1,
                    o_col_bstride=0),
        "dSKpts": dict(km, a_numel=FH * N * n8, a_frames=FH, Nr=N, a_cols=N, lda=n8, n_batches=FH, bmod=FH, a_f_div=1,
                       a_k_bstride=0, K=N, b_numel=FH * 32 * n8, b_z=FH, b_rows=32, b_cols=N, ldb=n8, b_k_ofs=0,
                       b_k_bstride=0, b_z_bstride=1, n_out=32, out_numel=FH * N * 32, ldo=32, out_rows=FH * N, o_f_div=1,
                       o_col_bstride=0),
    }
    z1 = dict(Fk=1, a_f_mul=0, a_z_mul=1, b_f_mul=0, b_z_mul=1, b_n_zmul=0, alpha=1.0)
    mn = {
        "dV": dict(alpha=1.0, a_numel=FH * N * n8, M=N, a_mid=N, a_outer=FH, lda=n8, a_ostride=N * n8,
                   b_numel=F * N * D8, b_cols=D, b_mid=N, b_outer=F, ldb=D8, b_ostride=N * D8,
                   Nn=C, Fk=F, Nr=N, zcount=H, a_f_mul=H, a_z_mul=1, b_f_mul=1, b_z_mul=0, b_n_zmul=C,
                   out_numel=N * H * 2 * C - C, out_ofs=C, ldo=H * 2 * C, out_z_stride=2 * C),
        "dVpts": dict(z1, a_numel=FH * N * n8, M=N, a_mid=N, a_outer=FH, lda=n8, a_ostride=N * n8,
                      b_numel=FH * N * g8, b_cols=PV3, b_mid=N, b_outer=FH, ldb=g8, b_ostride=N * g8,
                      Nn=PV3, Nr=N, zcount=FH, out_numel=FH * N * PV3, ldo=PV3, out_z_stride=N * PV3),
        "dZ": dict(z1, a_numel=FH * N * n8, M=N, a_mid=FH, a_outer=N, lda=N * n8, a_ostride=n8,
                   b_numel=N * FH * c8, b_cols=Cp, b_mid=FH, b_outer=N, ldb=c8, b_ostride=FH * c8,
                   Nn=Cp, Nr=FH, zcount=N, out_numel=N * N * Cp, ldo=Cp, out_z_stride=N * Cp),
        "dSTQ": dict(z1, a_numel=FH * N * n8, M=N, a_mid=N, a_outer=FH, lda=n8, a_ostride=N * n8,
                     b_numel=FH * N * 32, b_cols=32, b_mid=N, b_outer=FH, ldb=32, b_ostride=N * 32,
                     Nn=32, Nr=N, zcount=FH, out_numel=FH * N * 32, ldo=32, out_z_stride=N * 32),
    }
    return kmaj, mn


IPA_SIZES = [(2, 40), (2, 200), (1, 1024)]

# every offset / stride of the K-major batched GEMM non-trivial: 6 batches, hb = b % 3, A frame b // 2, output rows
# (b // 3) * Nr, output columns hb * 80 of an odd-strided buffer, K slices of A and B that move with hb
BATCHED_GENERIC = [
    dict(name="generic", alpha=-0.75, a_numel=3 * 150 * 432, a_frames=3, Nr=150, a_cols=424, lda=432, n_batches=6, bmod=3,
         a_f_div=2, a_k_bstride=128, K=128, b_numel=3 * 72 * 584, b_z=3, b_rows=72, b_cols=576, ldb=584, b_k_ofs=64,
         b_k_bstride=192, b_z_bstride=1, n_out=72, out_numel=300 * 241, ldo=241, out_rows=300, o_f_div=3, o_col_bstride=80),
    # a K tail (200 = 3 x 64 + 8) inside rows that are wider than K: the sum stops at K
    dict(name="ktail_wide_rows", alpha=1.0, a_numel=2 * 136 * 216, a_frames=2, Nr=136, a_cols=216, lda=216, n_batches=2,
         bmod=1, a_f_div=1, a_k_bstride=0, K=200, b_numel=96 * 224, b_z=1, b_rows=96, b_cols=224, ldb=224, b_k_ofs=0,
         b_k_bstride=0, b_z_bstride=0, n_out=96, out_numel=272 * 96, ldo=96, out_rows=272, o_f_div=1, o_col_bstride=0),
    # fewer output rows than row tiles produce: the rows past out_rows stay unwritten
    dict(name="out_rows_cut", alpha=1.0, a_numel=3 * 100 * 64, a_frames=3, Nr=100, a_cols=64, lda=64, n_batches=3, bmod=1,
         a_f_div=1, a_k_bstride=0, K=64, b_numel=8 * 64, b_z=1, b_rows=8, b_cols=64, ldb=64, b_k_ofs=0, b_k_bstride=0,
         b_z_bstride=0, n_out=8, out_numel=300 * 8, ldo=8, out_rows=250, o_f_div=1, o_col_bstride=0),
]

# a_z_mul, b_z_mul and b_n_zmul all non-zero; A stored [mid][outer][M] (a_ostride < lda, the dZ layout); row / column / K
# tails; odd ldo and z stride
BATCHED_MN_GENERIC = [
    dict(name="generic", alpha=0.5, a_numel=150 * 680, M=130, a_mid=150, a_outer=5, lda=680, a_ostride=136,
         b_numel=6 * 150 * 120, b_cols=120, b_mid=150, b_outer=6, ldb=120, b_ostride=150 * 120,
         Nn=40, Fk=2, Nr=150, zcount=3, a_f_mul=2, a_z_mul=1, b_f_mul=1, b_z_mul=2, b_n_zmul=40,
         out_numel=3 * (130 * 45 + 7), ldo=45, out_z_stride=130 * 45 + 7),
]


def _bcases():
    out = [pytest.param(q, id=q["name"]) for q in BATCHED_GENERIC]
    for F, N in IPA_SIZES:
        for name, q in _ipa_calls(F, N)[0].items():
            out.append(pytest.param(dict(q, name=f"{name}_F{F}_N{N}"), id=f"{name}-F{F}-N{N}"))
    return out


def _mncases():
    out = [pytest.param(q, id=q["name"]) for q in BATCHED_MN_GENERIC]
    for F, N in IPA_SIZES:
        for name, q in _ipa_calls(F, N)[1].items():
            out.append(pytest.param(dict(q, name=f"{name}_F{F}_N{N}"), id=f"{name}-F{F}-N{N}"))
    return out


@pytest.mark.parametrize("q", _bcases())
def test_batched(q):
    run_batched(q, seed=len(q["name"]))


@pytest.mark.parametrize("q", _mncases())
def test_batched_mn(q):
    run_batched_mn(q, seed=len(q["name"]))


def test_batched_widths_covered():
    widths = {pick_bn(p.values[0]["n_out"], p.values[0]["n_batches"] * cdiv(p.values[0]["Nr"], BM)) for p in _bcases()}
    assert widths == {64, 128}, widths
    widths = {pick_bn(p.values[0]["Nn"], cdiv(p.values[0]["M"], BM) * p.values[0]["zcount"]) for p in _mncases()}
    assert widths == {64, 128}, widths


# --------------------------------------------------------------------------------------------------
# accumulator promotion: all-positive operands, long reductions
# --------------------------------------------------------------------------------------------------
def test_promotion_flat_in_k():
    """With operands uniform in [0, 1) every rounding bias of the accumulation adds up instead of cancelling, and
    S = R3: |C - R3| / S is the relative error.  The tensor core's accumulation is not round-to-nearest, so without the
    promotion every kChunk k-blocks that error would grow with K; with it the error must stay within C_ACC for a
    weight gradient over K = F * Nr = 256 ... 16384 pixels and a 5x5 forward over K = 25 * 64 ... 25 * 1280 = 32000."""
    ratios = {}
    for F in (1, 4, 16, 64):
        ratios[f"wgrad K={F * 256}"] = run_wgrad(128, 128, F, 256, positive=True, seed=F)[0]
    for Ci in (64, 320, 1280):
        ratios[f"conv K={25 * Ci}"] = run_gemm(2, 128, Ci, 128, taps=(5, 5), positive=True, seed=Ci)[0]
    _record(case="promotion", **ratios)
    assert max(ratios.values()) <= C_ACC, ratios


# --------------------------------------------------------------------------------------------------
# arguments the host wrappers reject: nothing is launched
# --------------------------------------------------------------------------------------------------
def _rejected(call, needle):
    L = K.lib()
    out = torch.full((4096,), float("nan"), device=DEV)
    rc = call(L, K._ptr(out))
    torch.cuda.synchronize()
    msg = L.dfold_last_error().decode()
    assert rc != 0, "accepted"
    assert needle in msg, msg
    assert torch.isnan(out).all(), "a rejected call wrote its output"


def test_rejected_arguments():
    a = Op(2 * 64 * 136, 1)
    b = Op(25 * 64 * 136, 2)
    s = K._stream()
    # lda not a multiple of 8
    _rejected(lambda L, o: L.dfold_gemm_bf16x3(K._ptr(a.hi), K._ptr(a.lo), 1, 1, 0, 16, 64, 68, K._ptr(b.hi), K._ptr(b.lo),
                                               16, 64, 1, 1, o, 16, None, None, 0, 1.0, 0.0, 0, s), "multiples of 8")
    _rejected(lambda L, o: L.dfold_gemm_wgrad_bf16x3(K._ptr(a.hi), K._ptr(a.lo), 16, 20, K._ptr(b.hi), K._ptr(b.lo), 16, 16,
                                                     1, 1, 0, 16, 1, 1, o, 16, 1.0, s), "multiples of 8")
    # even tap grid
    _rejected(lambda L, o: L.dfold_gemm_bf16x3(K._ptr(a.hi), K._ptr(a.lo), 1, 1, 0, 16, 64, 64, K._ptr(b.hi), K._ptr(b.lo),
                                               16, 64, 4, 5, o, 16, None, None, 0, 1.0, 0.0, 0, s), "tap grid must be odd")
    # a K slice of a wider row whose length is not a multiple of 64
    _rejected(lambda L, o: L.dfold_gemm_bf16x3_batched(K._ptr(a.hi), K._ptr(a.lo), 1, 16, 192, 192, 2, 2, 1, 96, 96,
                                                       K._ptr(b.hi), K._ptr(b.lo), 1, 16, 192, 192, 0, 96, 0, 16,
                                                       o, 32, 16, 1, 16, 1.0, s), "multiple of 64")
    # base pointer not 16-byte aligned
    _rejected(lambda L, o: L.dfold_gemm_bf16x3(K._ptr(a.hi, 1), K._ptr(a.lo), 1, 1, 0, 16, 64, 64, K._ptr(b.hi), K._ptr(b.lo),
                                               16, 64, 1, 1, o, 16, None, None, 0, 1.0, 0.0, 0, s), "16-byte aligned")
    _rejected(lambda L, o: L.dfold_gemm_wgrad_bf16x3_batched(K._ptr(a.hi), K._ptr(a.lo), 16, 16, 1, 16, 256,
                                                             K._ptr(b.hi, 4), K._ptr(b.lo), 16, 16, 1, 16, 256,
                                                             16, 1, 16, 1, 0, 0, 0, 0, 0, o, 16, 256, 1.0, s), "16-byte aligned")
