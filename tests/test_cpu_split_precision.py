"""CPU: the arithmetic contract of the split-precision tensor-core GEMM, emulated with torch.bfloat16.

x = hi + lo with hi = bf16(x), lo = bf16(x - hi); the kernel accumulates hi*hi + hi*lo + lo*hi in fp32 (the lo*lo term,
~2^-18 relative, is dropped).  This pins the ~5e-6 relative error quoted in DESIGN.md against a float64 product, and
shows why a single bf16 / tf32 pass cannot meet the 1e-4 parity bar (SURVEY.md §0 "precision trap")."""
import math

import torch


def split(x):
    hi = x.to(torch.bfloat16).to(torch.float32)
    lo = (x - hi).to(torch.bfloat16).to(torch.float32)
    return hi, lo


def test_split_representation_error():
    x = torch.randn(1 << 16)
    hi, lo = split(x)
    rel = ((hi + lo) - x).abs() / x.abs().clamp_min(1e-30)
    assert rel.max().item() < 2.0 ** -16          # two bf16 mantissas ~ 16+ significant bits


def test_three_product_gemm_error_is_fp32_grade():
    torch.manual_seed(0)
    M, N, K = 64, 48, 4096
    a, b = torch.randn(M, K), torch.randn(N, K) / math.sqrt(K)
    ref = a.double() @ b.double().T
    a_hi, a_lo = split(a)
    b_hi, b_lo = split(b)
    # products of bf16 values are exact in fp32; fp32 accumulation in chunks + register promotion, as the GEMM does
    y3 = (a_lo @ b_hi.T + a_hi @ b_lo.T + a_hi @ b_hi.T).double()
    y1 = (a_hi @ b_hi.T).double()
    rms = lambda e: (e.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()
    assert rms(y3 - ref) < 1.5e-5, rms(y3 - ref)
    assert rms(y1 - ref) > 1e-3                            # a single bf16 pass is 200x worse
    # tf32-like rounding of both operands (10-bit mantissa) is also far from the bar
    t = lambda x: (x.view(torch.int32) & ~0x1FFF).view(torch.float32)
    assert rms((t(a) @ t(b).T).double() - ref) > 1e-4
