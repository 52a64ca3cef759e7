"""CPU: the arithmetic contract of the fused IPA forward kernel (csrc/ipa_fused.cu), emulated step by step in fp32 torch.

The kernel does not compute a whole-row softmax: every lane owns one key per 32-key tile and keeps a running (m, l) pair
per row with ONE exponential per logit, the 32 lanes are combined once at the end (pass 1); pass 2 recomputes the logits
tile by tile, forms p = exp2((s - m) * log2 e) / l, feeds fp32 p to the pair / value-point accumulations and the bf16 hi/lo
split of p (hi*hi + hi*lo + lo*hi against the split V) to the tensor cores.  This test pins that procedure — tile order,
sentinels for out-of-range keys, the split product — against the oracle's direct fp64 evaluation, at the tolerances the
`-m gpu` tests apply to the kernel itself."""
import math

import torch

from oracle import ops as OO
from tests.test_cpu_split_precision import split

LOG2E = 1.4426950408889634
TILE = 32


def _emulate(logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma, Pq, Pv, inf=1e5, eps=1e-8):
    F, N, H = q_pts.shape[:3]
    C = kv.shape[-1] // 2
    f32 = torch.float32
    k_pts, v_pts = kv_pts[..., :Pq, :], kv_pts[..., Pq:, :]
    ntiles = (N + TILE - 1) // TILE
    gam = (-0.5 * gamma).to(f32)

    def logits(j0):                               # [F,H,N,TILE] of one key tile; keys past N get the kernel's sentinel
        j = torch.arange(j0, j0 + TILE)
        ok = j < N
        jc = j.clamp(max=N - 1)
        d = q_pts[:, :, None] - k_pts[:, None, jc]                           # exact fp32 differences
        d2 = (d * d).sum(-1).sum(-1)                                         # [F,i,j,H]
        s = logit0[:, :, :, jc] + (gam * d2).permute(0, 3, 1, 2) + (inf * (mask[:, :, None] * mask[:, None, jc] - 1))[:, None]
        return torch.where(ok, s, torch.full_like(s, -1.0e30)), ok, jc

    # ---- pass 1: per-lane online (m, l) with one exponential per logit, then the cross-lane combine ----
    m = torch.full((F, H, N, TILE), -3.0e38, dtype=f32)
    l = torch.zeros((F, H, N, TILE), dtype=f32)
    for t in range(ntiles):
        s, _, _ = logits(t * TILE)
        e = torch.exp2(-(s - m).abs() * LOG2E)
        up = s > m
        l = torch.where(up, l * e + 1.0, l + e)
        m = torch.where(up, s, m)
    M = m.max(dim=-1, keepdim=True).values
    L = (l * torch.exp2((m - M) * LOG2E)).sum(-1, keepdim=True)
    il = 1.0 / L
    # ---- pass 2: probabilities tile by tile, fp32 accumulations, split-bf16 P V ----
    v = kv[0, :, :, C:]                                                       # [N,H,C]
    v_hi, v_lo = split(v)
    o = torch.zeros((F, N, H, C), dtype=f32)
    o_pair = torch.zeros((F, N, H, pair.shape[-1]), dtype=f32)
    o_pt = torch.zeros((F, N, H, Pv, 3), dtype=f32)
    psum = torch.zeros((F, H, N), dtype=f32)
    for t in range(ntiles):
        s, ok, jc = logits(t * TILE)
        p = torch.exp2((s - M) * LOG2E) * il
        p = torch.where(ok, p, torch.zeros_like(p))
        psum += p.sum(-1)
        p_hi, p_lo = split(p)
        vt_hi, vt_lo = v_hi[jc], v_lo[jc]                                     # [TILE,H,C]
        o += (torch.einsum("fhij,jhc->fihc", p_lo, vt_hi) + torch.einsum("fhij,jhc->fihc", p_hi, vt_lo)
              + torch.einsum("fhij,jhc->fihc", p_hi, vt_hi))
        o_pair += torch.einsum("fhij,ijc->fihc", p, pair[0][:, jc])
        o_pt += torch.einsum("fhij,fjhpx->fihpx", p, v_pts[:, jc])
    return o, o_pair, o_pt, psum


def test_two_pass_tiled_softmax_and_split_product_match_the_oracle():
    torch.manual_seed(0)
    F, N, H, C, Pq, Pv, Cp = 2, 72, 8, 32, 8, 12, 32                        # N = 2 full tiles + a partial one
    R = lambda *s, scale=1.0: torch.randn(*s) * scale
    logit0, kv = R(1, H, N, N), R(1, N, H, 2 * C)
    q_pts, kv_pts = R(F, N, H, Pq, 3, scale=4.0), R(F, N, H, Pq + Pv, 3, scale=4.0)
    pair = R(1, N, N, Cp)
    quat = torch.nn.functional.normalize(R(F, N, 4), dim=-1)
    trans = R(F, N, 3, scale=8.0)
    mask = torch.ones(F, N)
    mask[0, 3] = 0
    mask[:, -2:] = 0
    gamma = torch.rand(H) * 0.2 + 0.05
    o, o_pair, o_pt, psum = _emulate(logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma, Pq, Pv)
    assert (psum - 1.0).abs().max().item() < 5e-6                            # every row is a distribution
    ref = OO.ipa_attention(*[t.double() for t in (logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma)],
                           Pq=Pq, Pv=Pv, dfold=True, inf=1e5, eps=1e-8)
    keep = mask[:, :, None].double()                  # masked query rows carry logits quantised by the -1e5 shift (as in the GPU test)
    HPv = H * Pv
    ref_o = ref[..., :H * C].reshape(F, N, H, C)
    ref_pair = ref[..., H * C + 4 * HPv:H * C + 4 * HPv + H * Cp].reshape(F, N, H, Cp)
    off_g = H * C + 4 * HPv + H * Cp
    ref_pt = torch.stack([ref[..., off_g + c * HPv:off_g + (c + 1) * HPv] for c in range(3)], dim=-1).reshape(F, N, H, Pv, 3)
    rel = lambda a, b, w: ((a.double() - b) * w).abs().max().item() / b.abs().max().item()
    assert rel(o, ref_o, keep[..., None]) < 2e-5                             # split-bf16 product, fp32 accumulate
    assert rel(o_pair, ref_pair, keep[..., None]) < 2e-5
    assert rel(o_pt, ref_pt, keep[..., None, None]) < 2e-5


def test_point_gradients_as_contractions_with_a_ones_column():
    """The backward computes dq_pts / dk_pts as two contractions over dS with a ones column appended to the point operands
    (kernels._IpaAttnTCFn.backward): the row / column sums of dS fall out of the same products.  Checked against the direct
    sum over coordinate differences (as csrc/ipa_attn.cu computes them), with the split-bf16 product error included."""
    torch.manual_seed(1)
    N, PQ3, gam = 96, 24, 0.17
    q, k = torch.randn(N, PQ3) * 6 + 20.0, torch.randn(N, PQ3) * 6 + 20.0     # coordinates far from the origin: cancellation
    P = torch.softmax(torch.randn(N, N) * 2, dim=-1)
    dP = torch.randn(N, N)
    dS = P * (dP - (P * dP).sum(-1, keepdim=True))                             # softmax gradient: rows sum to ~0
    diff = q[:, None, :].double() - k[None, :, :].double()
    dq_ref = -gam * (dS.double()[:, :, None] * diff).sum(1)
    dk_ref = gam * (dS.double()[:, :, None] * diff).sum(0)
    ones = torch.ones(N, 1)
    kt, qn = torch.cat([k, ones], dim=1), torch.cat([q, ones], dim=1)
    s_hi, s_lo = split(dS)

    def mm3(a_hi, a_lo, b):                                                    # hi*hi + hi*lo + lo*hi in fp32
        b_hi, b_lo = split(b)
        return a_lo @ b_hi + a_hi @ b_lo + a_hi @ b_hi
    g1 = mm3(s_hi, s_lo, kt)                                                   # [i, 25]: sum_j dS k | rowsum
    g2 = mm3(s_hi.T.contiguous(), s_lo.T.contiguous(), qn)                     # [j, 25]: sum_i dS q | colsum
    dq = -gam * (q * g1[:, PQ3:] - g1[:, :PQ3])
    dk = gam * (g2[:, :PQ3] - g2[:, PQ3:] * k)
    rel = lambda a, b: (a.double() - b).abs().max().item() / b.abs().max().item()
    assert rel(dq, dq_ref) < 2e-4 and rel(dk, dk_ref) < 2e-4                   # the op-level GPU tolerance
