"""-m gpu: the CUDA-core kernels of csrc/simt.cu, called directly through the C ABI and compared element by element with
a reference of the same operation.

Where a kernel's arithmetic is fully specified the reference is bit-exact, emulated here in torch (whose fp32 / bf16
element-wise ops round to nearest like the kernels):
  * dfold_split2d planes: hi = bf16_rn(x), lo = bf16_rn(x - hi), after relu(x) and the gate (x if gate > 0 else 0);
  * the dfold_conv_weight_prep permutations (forward [T][O][ldi], dgrad [T-1-t][I][ldo]);
  * dfold_taps_to_param, which is one fp32 add per element;
  * the fixed-order column sums (colsum_kernel, and d(bias) of row_ln_wgrad_kernel): an fp32 accumulator [32, C], row
    block k adds rows 32 k + ty in turn, the 32 lane sums are then added in lane order into a zero, and that total is
    added (+=) onto the initial colsum.
Bits are compared with +0 and -0 treated as equal.

Everything else is held per element to a bound derived from the kernel's own operation order (the derivations sit next
to each bound below; u = 2^-24 is the fp32 unit roundoff).  A max-normalised metric cannot see an element that is wrong by
100 % of its own small value; these bounds can.  The worst measured ratio |err| / bound of each kernel family, on an
H100 80GB HBM3 at a 400 W power limit, is listed next to its bound (DFOLD_SIMT_ERRORS names a JSON-lines file that
receives every case's ratio).

Every case also
  * launches twice and requires the same bits (the fixed-order reductions are what makes a training step reproducible);
  * pre-fills the outputs with a sentinel (NaN for fp32, 0x5A5A for bf16 planes) and requires every element outside the
    region the kernel owns to keep it: past ldo / ldt, past cpad / rpad, and outside the conv planes' I / O extent
    (the caller zero-fills that padding once).
The float64 references run on the CPU for small cases and on the GPU for large ones, where their peak device memory is
held under REF_PEAK_BYTES because the device is shared.
"""
import json
import math
import os

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from dynamicpdb_b200 import kernels as K

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24                      # fp32 unit roundoff
UD = 2.0 ** -53                     # float64 unit roundoff
SENT16 = 0x5A5A                     # fills the bf16 planes first: elements a kernel must not write keep it
REF_PEAK_BYTES = 16 << 30


def cdiv(a, b):
    return -(-a // b)


def _record(**kw):
    """Appends one case's worst |err| / bound to the JSON-lines file DFOLD_SIMT_ERRORS names (calibration aid)."""
    path = os.environ.get("DFOLD_SIMT_ERRORS")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(kw) + "\n")


def _ok(rc):
    assert rc == 0, K.lib().dfold_last_error().decode()


def _gen(seed, dev=DEV):
    return torch.Generator(device=dev).manual_seed(seed)


def _wide(n, seed, lo_exp=-130, hi_exp=100, zeros=0.05):
    """fp32 values with magnitudes 2^lo_exp ... 2^hi_exp (subnormals below 2^-126), both signs, and exact +-0."""
    g = _gen(seed)
    e = torch.randint(lo_exp, hi_exp + 1, (n,), generator=g, device=DEV).double()
    m = 1 + torch.rand(n, generator=g, device=DEV, dtype=torch.float64)
    s = torch.where(torch.rand(n, generator=g, device=DEV) < 0.5, -1.0, 1.0)
    x = (s.double() * m * torch.pow(2.0, e)).float()
    return torch.where(torch.rand(n, generator=g, device=DEV) < zeros, s.float() * 0.0, x)


def _gate_values(n, seed):
    """ReLU-backward gates: positive, 0, -0, negative, and the smallest subnormals of both signs."""
    g = _gen(seed)
    pool = torch.tensor([1.0, 0.0, -0.0, -1.0, 2.0 ** -149, -(2.0 ** -149), 3.5, -2.0], device=DEV)
    v = pool[torch.randint(0, pool.numel(), (n,), generator=g, device=DEV)]
    return v * (1 + torch.rand(n, generator=g, device=DEV))


def _planes(v):
    """bf16 hi / lo planes (int16 bits) of fp32 v, round to nearest as split_pack in simt.cu."""
    hi = v.to(torch.bfloat16)
    lo = (v - hi.float()).to(torch.bfloat16)
    return hi.view(torch.int16), lo.view(torch.int16)


def _bits16(t):
    return torch.where(t == -32768, torch.zeros_like(t), t)         # -0 (0x8000) == +0


def _bits32(t):
    return torch.where(t == 0, torch.zeros_like(t), t).view(torch.int32)


def _same_bits(what, got, exp):
    f = _bits16 if got.dtype == torch.int16 else _bits32
    a, b = f(got), f(exp)
    bad = a != b
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} elements differ from the emulation; first at flat index "
                           f"{int(bad.nonzero()[0])}: got {int(a[bad][0])}, expected {int(b[bad][0])}")


def _twice(make, launch):
    """make() -> fresh sentinel-filled output buffers; launch(bufs) -> rc.  Runs twice, requires identical bits."""
    outs = []
    for _ in range(2):
        bufs = make()
        _ok(launch(bufs))
        torch.cuda.synchronize()
        outs.append(bufs)
    for i, (a, b) in enumerate(zip(*outs)):
        if a is not None:
            w = torch.int16 if a.dtype == torch.int16 else (torch.int64 if a.dtype == torch.float64 else torch.int32)
            assert torch.equal(a.view(w), b.view(w)), f"output {i}: the second launch gave different bits"
    return outs[0]


def _kernels_launched(fn):
    """Names of the CUDA kernels fn() launches (torch.profiler sees every kernel of the process)."""
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events()]


class _RefPeak:
    """Asserts that the float64 reference computed inside the block stays under REF_PEAK_BYTES of device memory."""

    def __init__(self, what):
        self.what = what

    def __enter__(self):
        torch.cuda.synchronize()
        self.base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - self.base
        if exc[0] is None:
            assert peak < REF_PEAK_BYTES, f"{self.what}: the float64 reference took {peak / 2**30:.1f} GB of device memory"
        return False


def _within(what, err, bound, family):
    """err, bound: float64 tensors of the same shape.  Records and asserts max(err / bound) <= 1."""
    err, bound = err.reshape(-1), bound.reshape(-1)
    assert torch.isfinite(err).all(), f"{what}: non-finite outputs"
    ratio = torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err > 0, float("inf"), 0.0))
    worst = ratio.max().item() if ratio.numel() else 0.0
    _record(family=family, case=what, worst_ratio=worst)
    bad = ratio > 1
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} elements outside their bound (worst |err| / bound = "
                           f"{worst:.3e}, first at flat index {int(bad.nonzero()[0])})")
    return worst


def _colsum_emul(v, init):
    """colsum_kernel's order: acc[32, C] fp32, row block k adds rows 32 k + ty; then the 32 lane sums in lane order into a
    zero, and that total += init."""
    R, C = v.shape
    nb = cdiv(R, 32)
    if nb * 32 != R:
        v = torch.cat([v, v.new_zeros(nb * 32 - R, C)])        # +0 added to a sum that started at +0 changes nothing
    v = v.reshape(nb, 32, C)
    acc = torch.zeros(32, C, dtype=torch.float32, device=v.device)
    for k in range(nb):
        acc += v[k]
    t = torch.zeros(C, dtype=torch.float32, device=v.device)
    for i in range(32):
        t += acc[i]
    return init + t


# --------------------------------------------------------------------------------------------------
# dfold_split2d
# --------------------------------------------------------------------------------------------------
def run_split2d(R, C, *, ld=None, ldg=None, gate=False, pre_relu=False, planes=True, ldo=None, cpad=None, trans=False,
                ldt=None, rpad=None, colsum=False, x_off=0, g_off=0, p_off=0, seed=0, wide=True):
    """One dfold_split2d call against the emulation.  Returns (hi, lo) [R, C] of the planes it wrote (or None)."""
    ld = C if ld is None else ld
    ldg = C if ldg is None else ldg
    cpad = C if cpad is None else cpad
    ldo = cpad if ldo is None else ldo
    rpad = R if rpad is None else rpad
    ldt = rpad if ldt is None else ldt
    # the [R, C] values depend on the seed only, not on the layout, so calls that differ in layout see the same matrix;
    # the rest of each buffer (the gaps past C, the leading offset) holds other values of the same kind
    mk = (lambda k, s: _wide(k, s)) if wide else (lambda k, s: torch.randn(k, generator=_gen(s), device=DEV))
    xbuf = mk(x_off + (R - 1) * ld + C + 8, seed + 7)
    x = xbuf[x_off:x_off + (R - 1) * ld + C].as_strided((R, C), (ld, 1))
    x.copy_(mk(R * C, seed).view(R, C))
    gbuf = gv = None
    if gate:
        gbuf = _gate_values(g_off + (R - 1) * ldg + C + 8, seed + 8)
        gv = gbuf[g_off:g_off + (R - 1) * ldg + C].as_strided((R, C), (ldg, 1))
        gv.copy_(_gate_values(R * C, seed + 1).view(R, C))
    v = x.clamp(min=0) if pre_relu else x
    if gate:
        v = torch.where(gv > 0, v, torch.zeros_like(v))
    hi, lo = _planes(v) if planes or trans else (None, None)
    init = torch.randn(C, generator=_gen(seed + 2), device=DEV) if colsum else None

    exp = []
    if planes:
        e = torch.full((p_off + R * ldo + 16,), SENT16, dtype=torch.int16, device=DEV)
        el = e.clone()
        for buf, pl in ((e, hi), (el, lo)):
            view = buf[p_off:p_off + R * ldo].view(R, ldo)
            view[:, :C] = pl
            view[:, C:cpad] = 0
        exp += [e, el]
    if trans:
        e = torch.full((p_off + C * ldt + 16,), SENT16, dtype=torch.int16, device=DEV)
        el = e.clone()
        for buf, pl in ((e, hi), (el, lo)):
            view = buf[p_off:p_off + C * ldt].view(C, ldt)
            view[:, :R] = pl.T
            view[:, R:rpad] = 0
        exp += [e, el]
    if colsum:
        exp.append(torch.cat([_colsum_emul(v, init), torch.full((16,), float("nan"), device=DEV)]))

    def make():
        return [torch.full_like(t, SENT16) if t.dtype == torch.int16 else
                torch.cat([init, torch.full((16,), float("nan"), device=DEV)]) for t in exp]

    def launch(bufs):
        it = iter(bufs)
        h, l = (next(it), next(it)) if planes else (None, None)
        ht, lt = (next(it), next(it)) if trans else (None, None)
        cs = next(it) if colsum else None
        return K.lib().dfold_split2d(K._ptr(xbuf, x_off), R, C, ld, int(pre_relu), K._ptr(gbuf, g_off), ldg if gate else 0,
                                     K._ptr(h, p_off), K._ptr(l, p_off), ldo, cpad, K._ptr(ht, p_off), K._ptr(lt, p_off),
                                     ldt, rpad, K._ptr(cs), K._stream())
    got = _twice(make, launch)
    what = (f"split2d R{R} C{C} ld{ld}+{x_off} gate{int(gate)}/{ldg}+{g_off} relu{int(pre_relu)} planes{int(planes)}/{ldo}/"
            f"{cpad}+{p_off} trans{int(trans)}/{ldt}/{rpad} colsum{int(colsum)}")
    for i, (g_, e_) in enumerate(zip(got, exp)):
        _same_bits(f"{what} output {i}", g_, e_)
    if planes:
        return (got[0][p_off:p_off + R * ldo].view(R, ldo)[:, :C], got[1][p_off:p_off + R * ldo].view(R, ldo)[:, :C])
    return None


def _r4(n):
    return cdiv(n, 4) * 4


SPLIT_SHAPES = [(1, 1), (31, 33), (32, 32), (33, 31), (1, 1037), (1029, 1), (33, 1031), (1031, 33)]


@pytest.mark.parametrize("R,C", SPLIT_SHAPES, ids=lambda v: str(v))
def test_split2d_combinations(R, C):
    """pre_relu x gate x colsum, on a row-major layout that the vectorised kernel takes (16-byte rows, cpad % 4 == 0) and
    on a layout with transposed planes, odd strides, cpad > C, rpad > R and ldo > cpad, which the tile kernel takes."""
    seed = 17 * R + C
    for pre_relu in (False, True):
        for gate in (False, True):
            for colsum in (False, True):
                seed += 3
                kw = dict(gate=gate, pre_relu=pre_relu, colsum=colsum, seed=seed)
                run_split2d(R, C, ld=_r4(C) + 4, ldg=_r4(C) + 8, cpad=_r4(C) + 4, ldo=_r4(C) + 8, **kw)
                run_split2d(R, C, ld=C + 1, ldg=C + 3, cpad=C + 3, ldo=C + 5, trans=True, ldt=R + 7, rpad=R + 3, **kw)
                run_split2d(R, C, planes=False, trans=True, ldt=R + 2, rpad=R + 1, x_off=1, g_off=3, **kw)


def test_split2d_paths():
    """Calls that differ in one vectorisation condition each give identical planes, and the condition picks the kernel
    that is expected to run.  A call with column sums only launches colsum_kernel and nothing else."""
    R, C = 37, 1001
    base = dict(ld=1004, ldg=1008, cpad=1004, ldo=1012, gate=True, pre_relu=True, seed=5)
    variants = {
        "x offset by one float": dict(x_off=1),
        "odd ld": dict(ld=1005),
        "odd ldg": dict(ldg=1009),
        "cpad % 4 != 0": dict(cpad=1006),
        "odd ldo": dict(ldo=1013),
        "transposed planes": dict(trans=True),
        "plane pointers offset by 2 bytes": dict(p_off=1),
    }
    names = _kernels_launched(lambda: run_split2d(R, C, **base))
    assert any("split2d_vec_kernel" in n for n in names) and not any("split2d_kernel" in n for n in names), names
    ref_hi, ref_lo = run_split2d(R, C, **base)
    for what, kw in variants.items():
        q = dict(base, **kw)
        names = _kernels_launched(lambda: run_split2d(R, C, **q))
        assert any("split2d_kernel" in n for n in names) and not any("split2d_vec_kernel" in n for n in names), (what, names)
        hi, lo = run_split2d(R, C, **q)
        assert torch.equal(_bits16(hi), _bits16(ref_hi)) and torch.equal(_bits16(lo), _bits16(ref_lo)), what
    # column sums only: no split kernel reads x for nothing
    names = _kernels_launched(lambda: run_split2d(R, C, planes=False, colsum=True, gate=True, seed=9))
    assert any("colsum_kernel" in n for n in names), names
    assert not any("split2d" in n for n in names), names


@pytest.mark.parametrize("R", [65536, 1048576])
@pytest.mark.parametrize("C", [128, 384])
def test_split2d_colsum_long(R, C):
    """Bias-gradient column sums at the EdgeTransition's R = N^2 rows (N = 256 and 1024) and widths, with the ReLU gate
    and a nonzero initial colsum: bit-exact against the documented order, up to 32768 sequential adds per lane."""
    run_split2d(R, C, planes=False, gate=True, colsum=True, seed=R + C, wide=False)
    if R == 65536:
        run_split2d(R, C, ldo=C + 8, cpad=C + 8, colsum=True, seed=R + C + 1, wide=False)


# --------------------------------------------------------------------------------------------------
# dfold_conv_weight_prep
# --------------------------------------------------------------------------------------------------
def run_conv_prep(O, I, T, ldi=None, ldo=None, dgrad=True, seed=0):
    ldi = cdiv(I, 8) * 8 if ldi is None else ldi
    ldo = cdiv(O, 8) * 8 if ldo is None else ldo
    w = _wide(O * I * T, seed, -40, 40)
    hi, lo = _planes(w)
    hi, lo = hi.view(O, I, T), lo.view(O, I, T)
    exp = []
    for pl in (hi, lo):
        e = torch.full((T * O * ldi + 16,), SENT16, dtype=torch.int16, device=DEV)
        e[:T * O * ldi].view(T, O, ldi)[:, :, :I] = pl.permute(2, 0, 1)
        exp.append(e)
    if dgrad:
        for pl in (hi, lo):
            e = torch.full((T * I * ldo + 16,), SENT16, dtype=torch.int16, device=DEV)
            e[:T * I * ldo].view(T, I, ldo)[:, :, :O] = pl.permute(2, 1, 0).flip(0)      # tap t -> T - 1 - t
            exp.append(e)

    def launch(b):
        d = (K._ptr(b[2]), K._ptr(b[3])) if dgrad else (None, None)
        return K.lib().dfold_conv_weight_prep(K._ptr(w), O, I, T, K._ptr(b[0]), K._ptr(b[1]), ldi, d[0], d[1], ldo, K._stream())
    got = _twice(lambda: [torch.full_like(e, SENT16) for e in exp], launch)
    what = f"conv_weight_prep O{O} I{I} T{T} ldi{ldi} ldo{ldo} dgrad{int(dgrad)}"
    for name, g_, e_ in zip(("f_hi", "f_lo", "d_hi", "d_lo"), got, exp):
        _same_bits(f"{what} {name}", g_, e_)


CONV_PREP_CASES = [
    # (O, I, T, ldi, ldo, dgrad)
    (640, 1280, 25, None, None, True),       # the ConvNet's widths, full tiles (fast path)
    (1280, 640, 25, None, None, True),
    (80, 72, 25, None, None, True),          # partial tiles in both directions
    (8, 8, 25, None, None, True),
    (33, 95, 25, None, None, True),
    (33, 95, 1, None, None, True),
    (33, 95, 9, None, None, True),
    (64, 64, 9, None, None, True),
    (64, 64, 25, 66, 72, True),              # full tiles, ldi % 4 != 0: the scalar path
    (64, 64, 25, 72, 70, True),              # full tiles, ldo % 4 != 0: the scalar path
    (96, 64, 25, None, None, False),         # no dgrad planes, fast path
    (40, 64, 25, 68, None, False),           # no dgrad planes, partial tiles
    (32, 32, 56, None, None, True),          # the largest tap count whose tile fits in shared memory
]


@pytest.mark.parametrize("case", CONV_PREP_CASES, ids=lambda c: "O{}I{}T{}ldi{}ldo{}d{}".format(*c))
def test_conv_weight_prep(case):
    run_conv_prep(*case, seed=CONV_PREP_CASES.index(case))


# --------------------------------------------------------------------------------------------------
# dfold_taps_to_param
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("O,I,T", [(8, 72, 25), (33, 95, 9), (7, 130, 1), (5, 70, 64), (1280, 640, 25)])
@pytest.mark.parametrize("accumulate", [0, 1])
def test_taps_to_param(O, I, T, accumulate):
    """out[o][i][t] = (accumulate ? out : 0) + g[t][o][i]: one fp32 add, bit-exact."""
    n = O * I * T
    g = torch.randn(n, generator=_gen(O + I + T), device=DEV)
    init = torch.randn(n, generator=_gen(O + I + T + 1), device=DEV)
    nan = torch.full((16,), float("nan"), device=DEV)
    base = init if accumulate else torch.zeros(n, device=DEV)
    exp = torch.cat([base + g.view(T, O, I).permute(1, 2, 0).reshape(-1), nan])

    def make():
        return [torch.cat([init if accumulate else torch.full((n,), float("nan"), device=DEV), nan])]
    got = _twice(make, lambda b: K.lib().dfold_taps_to_param(K._ptr(g), O, I, T, K._ptr(b[0]), accumulate, K._stream()))
    _same_bits(f"taps_to_param O{O} I{I} T{T} acc{accumulate}", got[0], exp)


# --------------------------------------------------------------------------------------------------
# dfold_sgemm
# --------------------------------------------------------------------------------------------------
# Accumulation: acc = sum_k a_k b_k with one fp32 fma per k in a fixed k order, so |acc - AB| <= gamma_K S with
# gamma_K = K u / (1 - K u) <= (K + 1) u for K u < 1/2, S = |A|.|B|.  ksplit > 1 adds up to ksplit partials of alpha acc
# atomically: + ksplit u.  The epilogue x = alpha acc (u |x|), + bias (u |x + bias|), SiLU x / (1 + expf(-x)) (expf
# <= 2 ulp = 4 u, the add and the divide u each: 6 u |silu|, and it scales the error already there by at most
# max |silu'| = 1.0998), + beta R (fma or two roundings: 2 u |beta R| + u |out|).  Everything is covered by
#   |C - ref| <= lip (K + ksplit + 2) u |alpha| S + EPI (|alpha AB| + |bias| + |beta R|),   EPI = 10 u.
# Measured worst |C - ref| / bound (H100 80GB HBM3, 400 W): 0.21 (dpair_frames at N = 200, K = 8), 0.13 with ksplit = 2.
EPI_SG = 10 * U


def run_sgemm(q, seed=0):
    """q: M, N, K, batch, batch2, A / B / C / R = (numel, off, rs, cs, bs, bs2), bias, alpha, beta, act, pre_relu, ksplit."""
    M, N, Kd, nb, nb2 = q["M"], q["N"], q["K"], q.get("batch", 1), q.get("batch2", 1)
    alpha, beta, act, pre_relu, ksplit = q.get("alpha", 1.0), q.get("beta", 1.0), q.get("act", 0), q.get("pre_relu", 0), q.get("ksplit", 1)
    g = _gen(seed)
    A = torch.randn(q["A"][0], generator=g, device=DEV)
    B = torch.randn(q["B"][0], generator=g, device=DEV) * q.get("bscale", 1.0)
    Rb = torch.randn(q["R"][0], generator=g, device=DEV) if q.get("R") else None
    bias = torch.randn(N, generator=g, device=DEV) if q.get("bias") else None
    cn, coff, crs, ccs, cbs, cbs2 = q["C"]
    L = K.lib()

    def arg(t, spec):
        return (K._ptr(t, spec[1]),) + tuple(spec[2:]) if t is not None else (None, 0, 0, 0, 0)

    idx = torch.arange(cn, device=DEV).as_strided((nb, nb2, M, N), (cbs, cbs2, crs, ccs), coff)
    assert idx.unique().numel() == idx.numel(), "output positions overlap"

    def make():
        c = torch.full((cn + 8,), float("nan"), device=DEV)
        if ksplit > 1:
            c[idx.reshape(-1)] = 0.0
        return [c]

    def launch(b):
        return L.dfold_sgemm(*arg(A, q["A"]), *arg(B, q["B"]), K._ptr(b[0], coff), crs, ccs, cbs, cbs2,
                             *arg(Rb, q["R"]) if Rb is not None else (None, 0, 0, 0, 0), K._ptr(bias), nb, nb2, M, N, Kd,
                             alpha, beta, act, pre_relu, ksplit, K._stream())
    if ksplit > 1:                     # atomics: the order varies from run to run, so no bitwise repeat
        bufs = make()
        _ok(launch(bufs))
        torch.cuda.synchronize()
        buf = bufs[0]
    else:
        buf = _twice(make, launch)[0]
    what = f"sgemm {q.get('name', '')} M{M} N{N} K{Kd} b{nb}x{nb2} act{act} relu{pre_relu} ks{ksplit}"
    keep = torch.ones(buf.numel(), dtype=torch.bool, device=DEV)
    keep[idx.reshape(-1)] = False
    assert torch.isnan(buf[keep]).all(), f"{what}: {int((~torch.isnan(buf[keep])).sum())} elements outside C were written"

    dev = DEV if nb * nb2 * M * N * max(Kd, 1) > (1 << 24) else "cpu"
    with _RefPeak(what):
        a_spec, b_spec = q["A"], q["B"]
        A64 = A.to(dev, torch.float64).as_strided((nb, nb2, M, Kd), (a_spec[4], a_spec[5], a_spec[2], a_spec[3]), a_spec[1])
        B64 = B.to(dev, torch.float64).as_strided((nb, nb2, N, Kd), (b_spec[4], b_spec[5], b_spec[2], b_spec[3]), b_spec[1])
        if pre_relu:
            A64 = A64.clamp(min=0)
        ab = alpha * (A64 @ B64.transpose(-1, -2))
        S = abs(alpha) * (A64.abs() @ B64.abs().transpose(-1, -2))
        y = ab + (bias.to(dev, torch.float64) if bias is not None else 0.0)
        mag = ab.abs() + (bias.to(dev, torch.float64).abs() if bias is not None else 0.0)
        if act == 1:
            y = y.clamp(min=0)
        elif act == 2:
            y = torch.nn.functional.silu(y)
        if Rb is not None:
            r = q["R"]
            rr = beta * Rb.to(dev, torch.float64).as_strided((nb, nb2, M, N), (r[4], r[5], r[2], r[3]), r[1])
            y = y + rr
            mag = mag + rr.abs()
        lip = 1.0998 if act == 2 else 1.0
        bound = lip * (Kd + ksplit + 2) * U * S + EPI_SG * mag
        got = buf[idx.reshape(-1)].to(dev, torch.float64).view(nb, nb2, M, N)
        return _within(what, (got - y).abs(), bound, "sgemm")


def _rowmajor(rows, cols, ld=None, off=0, batches=(1, 1), bstr=(0, 0)):
    """(numel, off, rs, cs, bs, bs2) of a row-major [rows][ld] operand, optionally batched."""
    ld = cols if ld is None else ld
    n = off + rows * ld + (batches[0] - 1) * bstr[0] + (batches[1] - 1) * bstr[1] + 4
    return (n, off, ld, 1, bstr[0], bstr[1])


def _colmajor(rows, cols, ld=None, off=0, batches=(1, 1), bstr=(0, 0)):
    """(numel, off, rs, cs, bs, bs2) of an operand stored column-major: element (r, c) at c * ld + r."""
    ld = rows if ld is None else ld
    n = off + cols * ld + (batches[0] - 1) * bstr[0] + (batches[1] - 1) * bstr[1] + 4
    return (n, off, 1, ld, bstr[0], bstr[1])


def _sgemm_generic_cases():
    out = []
    for Kd in (0, 1, 15, 16, 17, 100):
        for a_cm in (False, True):
            for b_cm in (False, True):
                M, N = 70, 130
                A = (_colmajor(M, max(Kd, 1), ld=M + 3, off=5) if a_cm else _rowmajor(M, max(Kd, 1), ld=Kd + 3, off=5))
                B = (_colmajor(N, max(Kd, 1), ld=N + 1, off=2) if b_cm else _rowmajor(N, max(Kd, 1), ld=Kd + 1, off=2))
                out.append(dict(name=f"K{Kd}_A{'cm' if a_cm else 'rm'}_B{'cm' if b_cm else 'rm'}", M=M, N=N, K=Kd, A=A, B=B,
                                C=_rowmajor(M, N, ld=N + 3, off=1), bias=Kd == 17, alpha=0.75))
    # batch x batch2 with every stride and offset non-trivial, output column-major
    M, N, Kd, nb, nb2 = 45, 67, 33, 3, 2
    out.append(dict(name="batched", M=M, N=N, K=Kd, batch=nb, batch2=nb2,
                    A=_rowmajor(M, Kd, ld=Kd + 2, off=3, batches=(nb, nb2), bstr=(2 * M * (Kd + 2) + 7, M * (Kd + 2) + 1)),
                    B=_colmajor(N, Kd, ld=N + 5, off=1, batches=(nb, nb2), bstr=(Kd * (N + 5) + 2, nb * Kd * (N + 5) + 11)),
                    C=(1 + nb * nb2 * N * (M + 2) + 8, 1, 1, M + 2, nb2 * N * (M + 2), N * (M + 2)),
                    R=_rowmajor(M, N, ld=N + 1, off=4, batches=(nb, nb2), bstr=(M * (N + 1), nb * M * (N + 1))),
                    bias=True, alpha=-1.25, beta=0.5, act=1))
    # epilogue combinations on a 64-tile-crossing shape
    for act in (0, 1, 2):
        for pre_relu in (0, 1):
            out.append(dict(name=f"epilogue_act{act}_relu{pre_relu}", M=129, N=65, K=40, A=_rowmajor(129, 40), B=_rowmajor(65, 40),
                            C=_rowmajor(129, 65, ld=66), R=_rowmajor(129, 65, ld=67, off=2), bias=True, alpha=0.8125,
                            beta=-0.625, act=act, pre_relu=pre_relu))
    out.append(dict(name="K0_epilogue", M=20, N=30, K=0, A=_rowmajor(20, 1), B=_rowmajor(30, 1), C=_rowmajor(20, 30),
                    R=_rowmajor(20, 30), bias=True, beta=2.0, act=2))
    return out


def _kernels_py_calls(F, N, H=8, C=256, Pq=8, Pv=12, Cp=32):
    """Every dfold_sgemm call shape kernels.py issues for the IPA logits (_QKLogitsFn) and the CUDA-core IPA backward
    (_IpaAttnFn.backward), argument for argument, for frame index f = F - 1."""
    f = F - 1
    NN, PQ3, PV3 = N * N, 3 * Pq, 3 * Pv
    W = PQ3 + PV3
    D = H * (C + 8 * Pv + Cp)
    q_n, kv_n, l_n = F * N * H * C, F * N * H * 2 * C, F * H * NN
    pm_n = H * F * NN
    return {
        # logit0[f,h] = alpha q k^T + beta b_hm, b_hm a permuted [F, N, N, H] pair bias
        "qk_fwd": dict(M=N, N=N, K=C, batch=H, A=(q_n, f * N * H * C, H * C, 1, C, 0), B=(kv_n, f * N * H * 2 * C, H * 2 * C, 1, 2 * C, 0),
                       C=(l_n, f * H * NN, N, 1, NN, 0), R=(F * NN * H, f * NN * H, N * H, H, 1, 0), alpha=0.125, beta=0.5773),
        "qk_dq": dict(M=N, N=C, K=N, batch=H, A=(l_n, f * H * NN, N, 1, NN, 0), B=(kv_n, f * N * H * 2 * C, 1, H * 2 * C, 2 * C, 0),
                      C=(q_n, f * N * H * C, H * C, 1, C, 0), alpha=0.125),
        "qk_dk": dict(M=N, N=C, K=N, batch=H, A=(l_n, f * H * NN, 1, N, NN, 0), B=(q_n, f * N * H * C, 1, H * C, C, 0),
                      C=(kv_n, f * N * H * 2 * C, H * 2 * C, 1, 2 * C, 0), alpha=0.125),
        "dkv_shared": dict(M=N, N=C, K=F * N, batch=H, A=(pm_n, 0, 1, N, F * NN, 0), B=(F * N * D, 0, 1, D, C, 0),
                           C=(N * H * 2 * C, C, H * 2 * C, 1, 2 * C, 0)),
        "dkv_frames": dict(M=N, N=C, K=N, batch=H, batch2=F, A=(pm_n, 0, 1, N, F * NN, NN), B=(F * N * D, 0, 1, D, C, N * D),
                           C=(F * N * H * 2 * C, C, H * 2 * C, 1, 2 * C, N * H * 2 * C)),
        "dkv_pts": dict(M=N, N=PV3, K=N, batch=H, batch2=F, A=(pm_n, 0, 1, N, F * NN, NN),
                        B=(F * N * H * PV3, 0, 1, H * PV3, PV3, N * H * PV3), C=(F * N * H * W, PQ3, H * W, 1, W, N * H * W)),
        "dpair_shared": dict(M=N, N=Cp, K=H * F, batch=N, A=(pm_n, 0, 1, NN, N, 0), B=(H * F * N * Cp, 0, 1, N * Cp, Cp, 0),
                             C=(NN * Cp, 0, Cp, 1, N * Cp, 0)),
        "dpair_frames": dict(M=N, N=Cp, K=H, batch=F, batch2=N, A=(pm_n, 0, 1, F * NN, NN, N),
                             B=(F * H * N * Cp, 0, 1, N * Cp, H * N * Cp, Cp), C=(F * NN * Cp, 0, Cp, 1, NN * Cp, N * Cp)),
    }


def _sgemm_cases():
    out = [pytest.param(q, id=q["name"]) for q in _sgemm_generic_cases()]
    for N in (40, 200):
        for name, q in _kernels_py_calls(2, N).items():
            out.append(pytest.param(dict(q, name=f"{name}_N{N}"), id=f"{name}-N{N}"))
    return out


@pytest.mark.parametrize("q", _sgemm_cases())
def test_sgemm(q):
    run_sgemm(q, seed=len(q["name"]) + q["K"])


@pytest.mark.parametrize("ksplit", [2, 5])
def test_sgemm_ksplit(ksplit):
    """ksplit > 1 adds K-chunk partials atomically into a zeroed C: held to the same bound (plus ksplit adds), not bitwise."""
    for Kd in (17, 1000):
        run_sgemm(dict(name="ksplit", M=70, N=90, K=Kd, A=_colmajor(70, Kd), B=_rowmajor(90, Kd, ld=Kd + 1), C=_rowmajor(70, 90),
                       alpha=1.5, ksplit=ksplit), seed=Kd)


# --------------------------------------------------------------------------------------------------
# linear on the CUDA-core path (N_out = 8 < 16): forward, data / weight / bias gradients
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [65536, 1000000, 1048576])
def test_linear_simt(M):
    """linear_b's shape (K = 128, N_out = H = 8) at M = N^2 rows: the weight gradient is ks = 128 or 256 partial
    products of kc rows (plus a tail of 64 rows at M = 10^6), added in order.  Bounds:
      y  = x w^T + b       (K + 2) u S + EPI |.|        (one fma chain, then the bias)
      dx = dy w            (N_out + 2) u S
      dw = sum of parts    (kc + ks + 3) u S            (kc fmas per part; the parts' sum adds at most ks + 1 more)
      db = dy.sum(0)       (M + 1) u S                  (torch's reduction, any order)
    with S the same contraction over absolute values.  Measured worst |err| / bound (H100 80GB HBM3, 400 W): y 0.049,
    dx 0.48, dw 2.2e-4, db 2.7e-7."""
    Kd, No = 128, 8
    g = _gen(M)
    x = torch.randn(M, Kd, generator=g, device=DEV)
    w = torch.randn(No, Kd, generator=g, device=DEV) / math.sqrt(Kd)
    b = torch.randn(No, generator=g, device=DEV)
    dy = torch.randn(M, No, generator=g, device=DEV)
    assert not K._use_tensor_cores(M, No, Kd)
    tiles = cdiv(No, 64) * cdiv(Kd, 64)
    ks = max(1, min(M // 512, 4 * K._sm_count(DEV) // tiles, 256))
    kc = M // ks
    runs = []
    for _ in range(2):
        xv, wv, bv = (t.clone().requires_grad_(True) for t in (x, w, b))
        y = K.linear(xv, wv, bv)
        y.backward(dy)
        torch.cuda.synchronize()
        runs.append([y.detach(), xv.grad, wv.grad, bv.grad])
    for a, c in zip(*runs):
        assert torch.equal(a.view(torch.int32), c.view(torch.int32)), "second run gave different bits"
    y, dx, dw, db = runs[0]
    what = f"linear simt M{M} ks{ks} kc{kc} tail{M - ks * kc}"
    with _RefPeak(what):
        x64, w64, b64, dy64 = (t.double() for t in (x, w, b, dy))
        ref = x64 @ w64.T
        _within(f"{what} y", (y.double() - ref - b64).abs(), (Kd + 2) * U * (x64.abs() @ w64.abs().T) + EPI_SG * (ref.abs() + b64.abs()), "linear")
        _within(f"{what} dx", (dx.double() - dy64 @ w64).abs(), (No + 2) * U * (dy64.abs() @ w64.abs()), "linear")
        _within(f"{what} dw", (dw.double() - dy64.T @ x64).abs(), (kc + ks + 3) * U * (dy64.abs().T @ x64.abs()), "linear")
        _within(f"{what} db", (db.double() - dy64.sum(0)).abs(), (M + 1) * U * dy64.abs().sum(0), "linear")


# --------------------------------------------------------------------------------------------------
# dfold_global_layernorm_fwd / bwd (MyLayerNorm: one mean and unbiased variance over the whole tensor)
# --------------------------------------------------------------------------------------------------
# Forward.  mean and the sum of squares are float64 sums; the longest chain of float64 adds is the per-thread stride
# loop (Lc = ceil(n / (blocks * 256)) adds) plus 5 + 5 shuffle / block levels in each of the two kernels, plus 4 + 8 in the
# finalize loop: D = (Lc + 40) 2^-53.  Hence |mean_d - mean| <= D sum|x| / n and
# |var_d - var| <= (D sum x^2 + 2 D |s| sum|x| / n + 2^-52 sum x^2) / (n - 1) =: dV.  The kernel stores mean_f = fp32(mean_d)
# (delta = u |mean| + D sum|x| / n) and rstd_f = fp32(1 / sqrt(var_d + eps)) (rel_r = u + dV / (2 (var + eps)) + 2^-52).
# xhat_f = fl(fl(x - mean_f) rstd_f) is then off xhat by at most
#   E_xh = 1.01 (rstd delta + |xhat| (2 u + rel_r))
# and y = silu(xhat_f) by at most 1.0998 E_xh + 6 u |y| (expf 2 ulp, the add and the divide).
# Backward, g = dy silu'(xhat_f) with silu' = s (1 + xhat (1 - s)), s = 1 / (1 + expf(-xhat)): |silu''| <= 0.5, and the fp32
# evaluation adds at most 16 u |dy| s (1 + |xhat| (1 - s)):  E_g = |dy| (0.5 E_xh + 16 u M1)  (E_g = 0 without SiLU).
# The float64 sums of g and g xhat are off by dS1 = sum E_g + D sum|g| and dS2 = sum (E_g |xhat| + |g| E_xh) + D sum|g xhat|;
# gmean_f = fp32(S1 / n) and gx_f = fp32(S2 / (n - 1)) add u of themselves.  dx = fl(rstd_f fl(fl(g - gmean) - xhat gx)):
#   E_dx = 1.01 (rstd (E_g + E_gmean + E_xh |gx| + |xhat| E_gx + 2 u (|g| + |gmean| + |xhat gx|)) + |dx| (rel_r + u)).
# Measured worst |err| / bound (H100 80GB HBM3, 400 W): y 0.78, mean 0.62, rstd 0.46, dx 0.77 (all at n = 2,097,153 or 3).
GLN_EPS = 1e-4


@pytest.mark.parametrize("n", [2, 3, 2097152, 2097153, 4194304, 4194305, 20971520])
@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("shift", [0.0, 1000.0])
def test_global_layernorm(n, silu, shift):
    """Covers the capped reduction grid (1024 blocks once n > 2,097,152) and the capped apply grid (4096 blocks once
    n > 4,194,304), MyLayerNorm's 64 x 256 x 256 = 4,194,304 input, and |mean| / std = 10^3."""
    g = _gen(n)
    x = shift + torch.randn(n, generator=g, device=DEV)
    dy = torch.randn(n, generator=g, device=DEV)
    L = K.lib()
    nan = lambda k: torch.full((k,), float("nan"), device=DEV)
    ws = torch.empty(2 * 1024 + 2, dtype=torch.float64, device=DEV)

    def fwd(b):
        return L.dfold_global_layernorm_fwd(K._ptr(x), K._ptr(b[0]), K._ptr(b[1]), K._ptr(ws), n, GLN_EPS, int(silu), K._stream())
    y, stats = _twice(lambda: [nan(n + 16), nan(2 + 16)], fwd)
    assert torch.isnan(y[n:]).all() and torch.isnan(stats[2:]).all(), "written past the output"
    st = stats[:2].clone()

    def bwd(b):
        return L.dfold_global_layernorm_bwd(K._ptr(x), K._ptr(dy), K._ptr(st), K._ptr(ws), K._ptr(b[0]), n, int(silu), K._stream())
    dx, = _twice(lambda: [nan(n + 16)], bwd)
    assert torch.isnan(dx[n:]).all(), "written past dx"
    what = f"global_layernorm n{n} silu{int(silu)} shift{shift:g}"
    dev = DEV if n > 65536 else "cpu"
    with _RefPeak(what):
        xd, dyd = x.to(dev, torch.float64), dy.to(dev, torch.float64)
        blocks = min(cdiv(n, 256 * 8), 1024)
        D = (cdiv(n, blocks * 256) + 40) * UD
        s_abs, s_sq, s = xd.abs().sum(), (xd * xd).sum(), xd.sum()
        mean = s / n
        var = ((xd - mean) ** 2).sum() / (n - 1)
        rstd = 1.0 / torch.sqrt(var + GLN_EPS)
        dV = (D * s_sq + 2 * D * s.abs() * s_abs / n + 2 * UD * s_sq) / (n - 1)
        rel_r = U + dV / (2 * (var + GLN_EPS)) + 2 * UD
        delta = U * mean.abs() + D * s_abs / n
        xh = (xd - mean) * rstd
        e_xh = 1.01 * (rstd * delta + xh.abs() * (2 * U + rel_r))
        if silu:
            sg = torch.sigmoid(xh)
            yr = xh * sg
            e_y = 1.0998 * e_xh + 6 * U * yr.abs()
        else:
            yr, e_y = xh, e_xh
        _within(f"{what} y", (y[:n].to(dev, torch.float64) - yr).abs(), e_y, "gln_fwd")
        _within(f"{what} mean", (st[0].to(dev, torch.float64) - mean).abs().reshape(1), delta.reshape(1), "gln_fwd")
        _within(f"{what} rstd", (st[1].to(dev, torch.float64) - rstd).abs().reshape(1), (rel_r * rstd).reshape(1), "gln_fwd")
        if silu:
            m1 = sg * (1 + xh * (1 - sg))
            gr = dyd * m1
            e_g = dyd.abs() * (0.5 * e_xh + 16 * U * sg * (1 + xh.abs() * (1 - sg)))
        else:
            gr, e_g = dyd, torch.zeros_like(dyd)
        gmean = gr.sum() / n
        gx = (gr * xh).sum() / (n - 1)
        e_gmean = (e_g.sum() + D * gr.abs().sum()) / n + U * gmean.abs()
        e_gx = ((e_g * xh.abs() + gr.abs() * e_xh).sum() + D * (gr * xh).abs().sum()) / (n - 1) + U * gx.abs()
        dxr = rstd * (gr - gmean - xh * gx)
        e_dx = 1.01 * (rstd * (e_g + e_gmean + e_xh * gx.abs() + xh.abs() * e_gx + 2 * U * (gr.abs() + gmean.abs() + (xh * gx).abs()))
                       + dxr.abs() * (rel_r + U))
        _within(f"{what} dx", (dx[:n].to(dev, torch.float64) - dxr).abs(), e_dx, "gln_bwd")


# --------------------------------------------------------------------------------------------------
# dfold_row_layernorm_fwd / bwd (per-row LayerNorm with affine)
# --------------------------------------------------------------------------------------------------
# Forward, one warp per row, Lc = ceil(C / 32) fp32 adds per lane and 5 shuffle levels: sum x is off by (Lc + 5) u sum|x|,
# so mean_f is off by delta = (Lc + 6) u sum|x| / C.  The squares are taken about mean_f: sum (x - mean_f)^2 =
# sum (x - mean)^2 + C delta^2, each d = x - mean_f rounds (u), the fma chain adds (Lc + 6) u, / C and + eps one u each:
#   rel_var = ((Lc + 9) u var + delta^2) / (var + eps) + 2 u,  rstd = rsqrtf(.) (2 ulp = 4 u): rel_r = rel_var / 2 + 4 u.
# y = fl(fl(fl(x - mean_f) rstd) w) + b (or an fma):  E_y = 1.01 |w| (rstd delta + |xhat| (rel_r + 2 u)) + u (|xhat w| + |y|).
# Backward against the float64 LayerNorm gradient at the kernel's own (mean, rstd), which is what it consumes:
# xhat_f = fl(fl(x - mean) rstd) (E_xh = 2.01 u |xhat|), g = fl(dy w) (u |g|); s1 = sum g / C and s2 = sum g xhat / C over
# the row, each off by (Lc + 6) u of its sum over |.| plus the propagated E_g / E_xh; dx = fl(rstd fl(fl(g - s1) - xhat s2)):
#   E_dx = 1.01 (rstd (E_g + E_s1 + E_xh |s2| + |xhat| E_s2 + 2 u (|g| + |s1| + |xhat s2|)) + u |dx|).
# dw[c] += sum_r dy xhat_f: ceil(rows / 32) fmas per lane, 32 lane adds, the += onto dw: (ceil(rows / 32) + 33) u (S + |dw0|)
# with S = sum_r |dy xhat|, plus sum_r |dy| E_xh.  db is bit-exact in colsum_kernel's order.
# Measured worst |err| / bound (H100 80GB HBM3, 400 W): y 0.85 (4096 x 256), mean 0.28, rstd 0.24, dx 0.53 (1,048,576 x 128),
# dw 0.043.
ROWLN_EPS = 1e-5


@pytest.mark.parametrize("rows,C", [(1, 1), (37, 96), (4096, 256), (65536, 128), (1048576, 128), (64, 31), (70, 33), (2048, 384)])
def test_row_layernorm(rows, C):
    g = _gen(rows + C)
    x = torch.randn(rows, C, generator=g, device=DEV) * 2 + torch.randn(rows, 1, generator=g, device=DEV) * 3
    w = torch.randn(C, generator=g, device=DEV)
    b = torch.randn(C, generator=g, device=DEV)
    dy = torch.randn(rows, C, generator=g, device=DEV)
    dw0 = torch.randn(C, generator=g, device=DEV)
    db0 = torch.randn(C, generator=g, device=DEV)
    L = K.lib()
    nan = lambda k: torch.full((k,), float("nan"), device=DEV)
    n = rows * C

    def fwd(bf):
        return L.dfold_row_layernorm_fwd(K._ptr(x), K._ptr(w), K._ptr(b), K._ptr(bf[0]), K._ptr(bf[1]), rows, C, ROWLN_EPS, K._stream())
    y, stats = _twice(lambda: [nan(n + 16), nan(2 * rows + 16)], fwd)
    assert torch.isnan(y[n:]).all() and torch.isnan(stats[2 * rows:]).all(), "written past the output"
    st = stats[:2 * rows].clone()

    def bwd(bf):
        return L.dfold_row_layernorm_bwd(K._ptr(x), K._ptr(w), K._ptr(dy), K._ptr(st), K._ptr(bf[0]), K._ptr(bf[1]), K._ptr(bf[2]),
                                         rows, C, K._stream())
    dx, dw, db = _twice(lambda: [nan(n + 16), torch.cat([dw0, nan(16)]), torch.cat([db0, nan(16)])], bwd)
    assert torch.isnan(dx[n:]).all() and torch.isnan(dw[C:]).all() and torch.isnan(db[C:]).all(), "written past the output"
    _same_bits(f"row_layernorm rows{rows} C{C} db", db[:C], _colsum_emul(dy, db0))

    what = f"row_layernorm rows{rows} C{C}"
    dev = DEV if n > 65536 else "cpu"
    Lc = cdiv(C, 32)
    with _RefPeak(what):
        wd, bd = w.to(dev, torch.float64), b.to(dev, torch.float64)
        dw_sum = torch.zeros(C, dtype=torch.float64, device=dev)       # sum_r dy xhat, sum_r |dy xhat|, sum_r |dy| E_xh
        dw_abs, dw_exh = dw_sum.clone(), dw_sum.clone()
        for r0 in range(0, rows, 1 << 17):                             # row chunks keep the float64 reference small
            r1 = min(rows, r0 + (1 << 17))
            sl = slice(r0 * C, r1 * C)
            xd = x[r0:r1].to(dev, torch.float64)
            dyd = dy[r0:r1].to(dev, torch.float64)
            mean = xd.mean(1, keepdim=True)
            var = ((xd - mean) ** 2).mean(1, keepdim=True)
            rstd = 1.0 / torch.sqrt(var + ROWLN_EPS)
            delta = (Lc + 6) * U * xd.abs().sum(1, keepdim=True) / C
            rel_r = (((Lc + 9) * U * var + delta ** 2) / (var + ROWLN_EPS) + 2 * U) / 2 + 4 * U
            xh = (xd - mean) * rstd
            yr = xh * wd + bd
            e_y = 1.01 * wd.abs() * (rstd * delta + xh.abs() * (rel_r + 2 * U)) + U * ((xh * wd).abs() + yr.abs())
            _within(f"{what} y", (y[sl].view(r1 - r0, C).to(dev, torch.float64) - yr).abs(), e_y, "rowln_fwd")
            del xh, yr, e_y
            st64 = st[2 * r0:2 * r1].view(r1 - r0, 2).to(dev, torch.float64)
            _within(f"{what} mean", (st64[:, :1] - mean).abs(), delta, "rowln_fwd")
            _within(f"{what} rstd", (st64[:, 1:] - rstd).abs(), rel_r * rstd, "rowln_fwd")
            # backward at the kernel's own stats
            m_k, r_k = st64[:, :1], st64[:, 1:]
            xk = (xd - m_k) * r_k
            del xd
            e_xh = 2.01 * U * xk.abs()
            gk = dyd * wd
            e_g = U * gk.abs()
            s1 = gk.sum(1, keepdim=True) / C
            s2 = (gk * xk).sum(1, keepdim=True) / C
            e_s1 = ((Lc + 6) * U * gk.abs().sum(1, keepdim=True) + e_g.sum(1, keepdim=True)) / C + U * s1.abs()
            e_s2 = (((Lc + 6) * U * (gk * xk).abs().sum(1, keepdim=True) + (e_g * xk.abs() + gk.abs() * e_xh).sum(1, keepdim=True)) / C
                    + U * s2.abs())
            dxr = r_k * (gk - s1 - xk * s2)
            e_dx = 1.01 * (r_k * (e_g + e_s1 + e_xh * s2.abs() + xk.abs() * e_s2 + 2 * U * (gk.abs() + s1.abs() + (xk * s2).abs()))
                           + U * dxr.abs())
            _within(f"{what} dx", (dx[sl].view(r1 - r0, C).to(dev, torch.float64) - dxr).abs(), e_dx, "rowln_dx")
            del gk, e_g, dxr, e_dx
            dw_sum += (dyd * xk).sum(0)
            dw_abs += (dyd * xk).abs().sum(0)
            dw_exh += (dyd.abs() * e_xh).sum(0)
        dw0d = dw0.to(dev, torch.float64)
        e_dw = (cdiv(rows, 32) + 33) * U * (dw_abs + dw0d.abs()) + dw_exh
        _within(f"{what} dw", (dw[:C].to(dev, torch.float64) - dw0d - dw_sum).abs(), e_dw, "rowln_dw")


# --------------------------------------------------------------------------------------------------
# dfold_adam_amsgrad
# --------------------------------------------------------------------------------------------------
# One step from the fp32 state (p, m, v, vmax) the kernel itself left, against float64 of the same update with the same
# fp32 constants (1 - b1 and 1 - b2 are exact in fp32):
#   g = grad gs (gs = 0.5: exact);  m' = m + (g - m)(1 - b1):  E_m = 2 u (|m'| + (1 - b1) |g - m|)
#   v' = v b2 + (1 - b2) g g (three products / adds, all terms >= 0):  E_v = 4 u v';  vmax' = max(vmax, v'): E_x = E_v
#   bc = 1 - powf(b, t): powf <= 4 ulp (8 u b^t), the subtraction u:  rel_bc = u (8 b^t / bc + 1)
#   step = lr / bc1 (rel_s = rel_bc1 + u);  ib = 1 / sqrtf(bc2) (rel_ib = rel_bc2 / 2 + 2 u)
#   den = fl(sqrtf(vmax') ib + eps):  rel_den = q / den (E_x / (2 vmax') + u + rel_ib + u) + u,  q = sqrt(vmax') ib
#   U = fl(fl(step m') / den):  E_U = |U| (rel_s + rel_den + 2 u) + step E_m / den;  p' = fl(p - U):  E_p = 1.01 E_U + u |p'|
# Measured worst |err| / bound (H100 80GB HBM3, 400 W): p 0.998 (the final rounding of p - U alone reaches u |p'| when p' sits just
# above a power of two), m 0.50, v and vmax 0.74.


def _adam_ref(p, gr, m, v, x, t, lr, b1, b2, eps, gs):
    c1, c2 = 1.0 - b1, 1.0 - b2
    g = gr * gs
    m2 = m + (g - m) * c1
    v2 = v * b2 + c2 * g * g
    x2 = torch.maximum(x, v2)
    bc1, bc2 = 1.0 - b1 ** t, 1.0 - b2 ** t
    step = lr / bc1
    ib = 1.0 / math.sqrt(bc2)
    q = torch.sqrt(x2) * ib
    den = q + eps
    upd = step * m2 / den
    p2 = p - upd
    e_m = 2 * U * (m2.abs() + c1 * (g - m).abs())
    e_v = 4 * U * v2
    rel_bc1 = U * (8 * b1 ** t / bc1 + 1)
    rel_bc2 = U * (8 * b2 ** t / bc2 + 1)
    rel_s, rel_ib = rel_bc1 + U, rel_bc2 / 2 + 2 * U
    rel_den = q / den * (e_v / (2 * x2.clamp(min=1e-300)) + 2 * U + rel_ib) + U
    e_u = upd.abs() * (rel_s + rel_den + 2 * U) + step * e_m / den
    e_p = 1.01 * e_u + U * p2.abs()
    return (p2, m2, v2, x2), (e_p, e_m, e_v, e_v)


@pytest.mark.parametrize("n", [4, 2162688 + 4, 8388612])
def test_adam_amsgrad(n):
    """20 steps with grad_scale = 0.5 and gradient magnitudes 1e-8 ... 1e3; n = 2,162,692 is one float4 past the first
    grid-stride pass on 132 SMs (16 x 132 CTAs of 256 threads).  A run in two chunks (tick only on the first) gives the
    same bits as one call over the whole buffer."""
    f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))
    lr, b1, b2, eps, gs = f32(1e-3), f32(0.9), f32(0.999), f32(1e-8), 0.5
    g = _gen(n)
    L = K.lib()
    nan = torch.full((16,), float("nan"), device=DEV)
    bufs = [torch.cat([torch.randn(n, generator=g, device=DEV), nan])] + [torch.cat([torch.zeros(n, device=DEV), nan]) for _ in range(3)]
    step = torch.zeros(1, device=DEV)
    dev = DEV if n > 65536 else "cpu"
    worst = [0.0] * 4
    for it in range(20):
        scale = torch.pow(10.0, torch.empty(n, device=DEV).uniform_(-8, 3, generator=g))
        grad = torch.randn(n, generator=g, device=DEV) * scale
        before = [b[:n].clone() for b in bufs]
        _ok(L.dfold_adam_amsgrad(*(K._ptr(b) for b in bufs[:1]), K._ptr(grad), *(K._ptr(b) for b in bufs[1:]), n, K._ptr(step), 1,
                                 lr, b1, b2, eps, gs, K._stream()))
        torch.cuda.synchronize()
        assert step.item() == it + 1
        for b in bufs:
            assert torch.isnan(b[n:]).all(), "written past n"
        what = f"adam n{n} step{it + 1}"
        with _RefPeak(what):
            ref, err = _adam_ref(*(t.to(dev, torch.float64) for t in (before[0], grad, before[1], before[2], before[3])),
                                 it + 1, lr, b1, b2, eps, gs)
            for k, (name, r, e) in enumerate(zip(("p", "m", "v", "vmax"), ref, err)):
                worst[k] = max(worst[k], _within(f"{what} {name}", (bufs[k][:n].to(dev, torch.float64) - r).abs(), e, "adam"))
    _record(family="adam", case=f"adam n{n}", worst=worst)

    # chunked: two calls over two parts, tick = 1 on the first only, against one whole call from the same state
    grad = torch.randn(n, generator=g, device=DEV)
    h = (n // 8) * 4 if n > 4 else n
    whole = [b.clone() for b in bufs]
    parts = [b.clone() for b in bufs]
    s_whole, s_parts = step.clone(), step.clone()
    _ok(L.dfold_adam_amsgrad(K._ptr(whole[0]), K._ptr(grad), *(K._ptr(b) for b in whole[1:]), n, K._ptr(s_whole), 1,
                             lr, b1, b2, eps, gs, K._stream()))
    _ok(L.dfold_adam_amsgrad(K._ptr(parts[0]), K._ptr(grad), *(K._ptr(b) for b in parts[1:]), h, K._ptr(s_parts), 1,
                             lr, b1, b2, eps, gs, K._stream()))
    if n > h:
        _ok(L.dfold_adam_amsgrad(K._ptr(parts[0], h), K._ptr(grad, h), *(K._ptr(b, h) for b in parts[1:]), n - h, K._ptr(s_parts), 0,
                                 lr, b1, b2, eps, gs, K._stream()))
    torch.cuda.synchronize()
    assert s_whole.item() == s_parts.item() == 21
    for a, c in zip(whole, parts):
        assert torch.equal(a.view(torch.int32), c.view(torch.int32)), "chunked update differs from the whole-buffer update"


# --------------------------------------------------------------------------------------------------
# arguments the host wrappers reject: nothing is launched
# --------------------------------------------------------------------------------------------------
def _rejected(call, needle):
    L = K.lib()
    out = torch.full((1 << 16,), float("nan"), device=DEV)
    rc = call(L, out)
    torch.cuda.synchronize()
    msg = L.dfold_last_error().decode()
    assert rc != 0, f"accepted ({needle})"
    assert needle in msg, msg
    assert torch.isnan(out).all(), "a rejected call wrote its output"


def test_rejected_arguments():
    x = torch.randn(64 * 64 * 64, device=DEV)
    s = K._stream()
    P = K._ptr
    p16 = lambda o, k=0: K._ptr(o.view(torch.int16), k)
    # split2d: cpad < C, ldo < cpad, rpad < R, an unpaired plane
    _rejected(lambda L, o: L.dfold_split2d(P(x), 8, 40, 40, 0, None, 0, p16(o), p16(o, 4096), 40, 36, None, None, 0, 0, None, s),
              "need C <= cpad <= ldo")
    _rejected(lambda L, o: L.dfold_split2d(P(x), 8, 40, 40, 0, None, 0, p16(o), p16(o, 4096), 40, 48, None, None, 0, 0, None, s),
              "need C <= cpad <= ldo")
    _rejected(lambda L, o: L.dfold_split2d(P(x), 8, 40, 40, 0, None, 0, None, None, 0, 0, p16(o), p16(o, 4096), 8, 7, None, s),
              "need R <= rpad <= ldt")
    _rejected(lambda L, o: L.dfold_split2d(P(x), 8, 40, 40, 0, None, 0, p16(o), None, 40, 40, None, None, 0, 0, None, s),
              "must come in pairs")
    _rejected(lambda L, o: L.dfold_split2d(P(x), 0, 40, 40, 0, None, 0, p16(o), p16(o, 4096), 40, 40, None, None, 0, 0, P(o), s),
              "empty input")
    # conv_weight_prep: the tile of T >= 57 taps does not fit in shared memory; ldi < I
    _rejected(lambda L, o: L.dfold_conv_weight_prep(P(x), 8, 8, 57, p16(o), p16(o, 40000), 8, None, None, 0, s), "1 <= T <= 56")
    _rejected(lambda L, o: L.dfold_conv_weight_prep(P(x), 8, 16, 25, p16(o), p16(o, 40000), 8, None, None, 0, s), "bad leading dims")
    _rejected(lambda L, o: L.dfold_taps_to_param(P(x), 8, 8, 65, P(o), 0, s), "bad shape")
    # sgemm: split-K with an epilogue; batch x batch2 x ksplit > 65535
    _rejected(lambda L, o: L.dfold_sgemm(P(x), 16, 1, 0, 0, P(x), 16, 1, 0, 0, P(o), 16, 1, 0, 0, None, 0, 0, 0, 0, P(x), 1, 1,
                                         16, 16, 16, 1.0, 0.0, 0, 0, 2, s), "split-K takes no epilogue")
    _rejected(lambda L, o: L.dfold_sgemm(P(x), 16, 1, 0, 0, P(x), 16, 1, 0, 0, P(o), 16, 1, 0, 0, None, 0, 0, 0, 0, None, 256, 128,
                                         16, 16, 16, 1.0, 0.0, 0, 0, 2, s), "batch too large")
    _rejected(lambda L, o: L.dfold_sgemm(P(x), 16, 1, 0, 0, P(x), 16, 1, 0, 0, P(o), 16, 1, 0, 0, None, 0, 0, 0, 0, None, 1, 1,
                                         16, 16, -1, 1.0, 0.0, 0, 0, 1, s), "empty problem")
    ws = torch.empty(2050, dtype=torch.float64, device=DEV)
    _rejected(lambda L, o: L.dfold_global_layernorm_fwd(P(x), P(o), P(o, 100), P(ws), 1, 1e-4, 0, s), "at least 2 elements")
    _rejected(lambda L, o: L.dfold_global_layernorm_bwd(P(x), P(x), P(x), P(ws), P(o), 1, 0, s), "at least 2 elements")
    _rejected(lambda L, o: L.dfold_row_layernorm_fwd(P(x), P(x), P(x), P(o), P(o, 100), 0, 8, 1e-5, s), "empty input")
    _rejected(lambda L, o: L.dfold_row_layernorm_bwd(P(x), P(x), P(x), P(x), P(o), P(o, 100), P(o, 200), 8, 0, s), "empty input")
    st = torch.zeros(1, device=DEV)
    _rejected(lambda L, o: L.dfold_adam_amsgrad(P(o), P(x), P(o, 100), P(o, 200), P(o, 300), 6, P(st), 1, 1e-3, 0.9, 0.999,
                                                1e-8, 1.0, s), "multiple of 4")
    assert st.item() == 0.0, "a rejected Adam call advanced the step"
