"""-m gpu: the IPA attention core's five C-ABI entry points -- dfold_ipa_fused_fwd (csrc/ipa_fused.cu), dfold_ipa_ds_bwd
(csrc/ipa_v2.cu), dfold_ipa_attn_fwd, dfold_ipa_attn_bwd and dfold_ipa_pre_bwd (csrc/ipa_attn.cu) -- called directly and
compared element by element with the float64 intermediates of oracle/ipa_reference.py (pinned against autograd of
oracle/ops.py::ipa_attention by tests/test_cpu_ipa_reference.py).

Isolation.  Each entry point gets exact fp32 inputs; a backward entry point gets the fp32 rounding of the reference's own
intermediates (cat and lse for attn_bwd / pre_bwd; P planes split from the float64 P, dP, Tz, Tog and delta for ds_bwd),
never a kernel forward's output, so a bound covers that kernel's arithmetic plus one rounding of each such input.

Bounds, per element, first order in u = 2^-24 (Higham, "Accuracy and Stability of Numerical Algorithms", 2nd ed., §3.1:
a sum of k rounded terms is within k u of the same sum over absolute values, the "plus form"):
  logits   |ds_ij| <= k_s u (|logit0| + gamma/2 d2_ij + inf |m_i m_j - 1|), d2 = sum_p |q_p(i) - k_p(j)|^2.  The squared
           distance costs one rounding per difference (2 u on its square) and one per accumulation: 24 coordinates in two
           12-deep FMA chains plus the joining add in ipa_fused.cu / ipa_v2.cu (k_d = 15), one 3 Pq-deep serial chain in
           ipa_attn.cu (k_d = 3 Pq + 2); the two adds of the pair bias and mask terms give k_s = k_d + 2.  The inf term
           makes masked rows comparable: their logits sit near -1e5, where the fp32 grid is 2^-7, so their bound is loose
           by nature.
  exp      ex2.approx.ftz.f32 (ipa_fused.cu): maximum relative error 2 ulp over the full range (PTX ISA 8.5, ex2), and
           results below 2^-126 flush to zero; expf (ipa_attn.cu, built without --use_fast_math): 2 ulp (CUDA C++
           Programming Guide, 12.x, mathematical functions appendix).  E_EXP = 2^-22 bounds both; FLOOR = 2^-126 absolute
           covers flushed and subnormal probabilities.
  P        |dp_ij| <= p_ij expm1(E_ij) + FLOOR (the exponential of a first-order argument error), with
             softmax kernels (fused forward, attn_fwd):  E_ij = |ds_ij| + sum_k p_ik |ds_ik| + c_a u |s_ij - m_i|
                 + c_b u sum_k p_ik |s_ik - m_i| + n_e E_EXP + n_r u
           c_a u |s - m| is the rounded argument ((s - m) and, in ipa_fused.cu, the product by a rounded log2 e: c_a = 3;
           expf: c_a = 1).  The online row sum rescales earlier terms by exponentials whose arguments telescope to
           m - s_k, hence c_b = 2 c_a; a term passes through at most ntiles + 3 exponentials (n_e) and ntiles + 9 roundings
           of sums, rescales and 1 / l (n_r; ipa_attn.cu adds one per tile: 2 ntiles + 9).
             attn_bwd recomputes p = expf(s - lse) from the rounded lse input: E_ij = |ds_ij| + u |lse_i| + u |s_ij - lse_i|
                 + E_EXP; its rows are not renormalised, so masked rows move with u |lse| ~ 2^-8.
  planes   hi + lo against the float64 P within dp + half an ulp of lo (hi = bf16_rn(p) is exact in fp32 arithmetic,
           r = p - hi is exact, and lo = bf16_rn(r) is within half an ulp of r, which is at most half an ulp of lo; at
           most 2^-17 p.  A lo truncated toward zero can be off by a whole ulp of lo and fails where dp is small: the
           uniform rows, p = fl(1 / N) exactly, at N = 60 and 240), and hi is the nearest bf16: |lo| <= half an ulp of hi
           (2^-134 for subnormal hi).  bf16_rn(hi + lo) == hi is not an invariant: a remainder just below half an ulp can
           round up to exactly half an ulp in lo, and the tie then goes to the even neighbour.  Row sums of the fused
           forward's planes: the kernel normalises by the sum of the same rounded logits it exponentiates, so
           |sum_j (hi + lo)_ij - 1| <= sum_j (p + dp)_ij (9 u (|s_ij - m_i| + 2 max_k |ds_ik|) + (ntiles + 3) E_EXP
           + (ntiles + 9) u) + sum_j half an ulp of lo_ij + N FLOOR, masked rows included.
  sums     an aggregation sum_j p_ij x_j (pair, value points, values) is held to sum_j dp_ij |x_j| + k_a u sum_j p_ij |x_j|,
           k_a = N (one serial chain over all keys) in ipa_fused.cu, N + ntiles + 2 in ipa_attn.cu (rescales, 1 / l).
           The frame transform R^T (og - t) adds |R|^T |dog| + 10 u R+^T (|og| + |t|) (R+ the plus form of
           quat_to_rot: 5 roundings deep, the subtraction 1, the 3-term dot 3, rounded up), the norms
           sum_b |x_b| |dx_b| / n + 4 u n.
  backward every epilogue-backward output (d_og, delta, dquat, dtrans) is held to k u S, S its plus form over the
           absolute values of cat (rounded once on input) and dcat, k its depth counted in _pre_bounds.  dS =
           P (dP + Tog + Tz - delta) is held to |dp| |dP_total - delta| + k u P (|dPv| + |dPog| + |dPz| + |delta|) plus
           the propagated error of its operands; dq / dk to gamma sum |dS_err| |q - k| + k u gamma sum |dS| |q - k|.
  dgamma   the per-head sum of the partials to sum |dS_err| d2 / 2 + k u sum |dS| d2 / 2, k = k_d + 1 + 4 ntiles
           (each lane's FMA chain over its 4 rows) + 5 (warp tree) + 8 (the per-CTA sum of the 8 warps).  The partials'
           slot layout is internal: they are summed per head in float64 here.
No max-normalised metric is used and no element or row is dropped.  Every case also launches twice and requires the same
bits, pre-fills every output and a guard past its end with NaN, and requires what an entry point must not write to keep
it: columns [0, H C) of the concat buffer after dfold_ipa_fused_fwd (the P V GEMM's), the value-point part of dkv_pts
after dfold_ipa_attn_bwd, and the pad columns [N, ldp) of the planes.  The worst |err| / bound of every check goes to
the JSON-lines file DFOLD_IPA_ERRORS names, when it is set.  The reference runs on the GPU frame by frame in blocks of
query rows, its peak under REF_PEAK_BYTES.
"""
import json
import os

import numpy as np
import pytest
import torch

from dynamicpdb_b200 import kernels as K
from oracle import dfold_oracle as O
from oracle.ipa_reference import ipa_reference
from tests.test_gpu_residue_kernels import _grads, _Out, _RefPeak, _rot_plus, _twice

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
E_EXP = 2.0 ** -22
FLOOR = 2.0 ** -126
INF = 1e5
EPS = float(np.float32(1e-8))


def _record(**kw):
    path = os.environ.get("DFOLD_IPA_ERRORS")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(kw) + "\n")


def _within(what, got, ref, bound):
    got, ref, bound = got.double().reshape(-1), ref.double().reshape(-1), bound.double().reshape(-1)
    assert torch.isfinite(got).all(), f"{what}: non-finite outputs"
    err = (got - ref).abs()
    ratio = torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err > 0, float("inf"), 0.0))
    worst = ratio.max().item() if ratio.numel() else 0.0
    k = int(ratio.argmax()) if ratio.numel() else 0
    _record(case=what, worst_ratio=worst, **({"got": got[k].item(), "ref": ref[k].item(), "bound": bound[k].item()} if ratio.numel() else {}))
    bad = ratio > 1
    if bad.any():
        j = int(bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside their bound (worst |err| / bound = "
                             f"{worst:.3e}); first at flat index {j}: got {got[j].item():.17g}, expected {ref[j].item():.17g}, "
                             f"bound {bound[j].item():.3e}")
    return worst


# --------------------------------------------------------------------------------------------------
# inputs
# --------------------------------------------------------------------------------------------------
def _case(F, N, H, C, Pq, Pv, Cp, Fl, Fs, Fz, edge, seed=0):
    """fp32 device inputs and the cotangent dcat.  edge: plain | masked | dominant | uniform | far | coincident | zero_vpts."""
    g = torch.Generator().manual_seed(seed)
    R = lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale
    mask = torch.ones(F, N)
    logit0 = R(Fl, H, N, N)
    q_pts, kv_pts = R(F, N, H, Pq, 3, scale=4.0), R(F, N, H, Pq + Pv, 3, scale=4.0)
    trans = R(F, N, 3, scale=8.0)
    gamma = torch.rand(H, generator=g) * 0.2 + 0.05
    if edge == "masked":                       # masked keys and query rows, and (F > 1) a wholly masked frame
        mask[:, -3:] = 0
        mask[0, 1] = 0
        if F > 1:
            mask[-1] = 0
    elif edge == "dominant":                   # one key per row carries p ~ 1
        idx = torch.randint(0, N, (Fl, H, N), generator=g)
        logit0.scatter_(-1, idx[..., None], 200.0)
    elif edge == "uniform":                    # gamma = 0 and a constant logit0: p = 1 / N in every unmasked row
        logit0.fill_(0.5)
        gamma = torch.zeros(H)
    elif edge == "far":                        # every key 30 A off every query: every logit below -100
        kv_pts[..., :Pq, 0] += 30.0
    elif edge == "coincident":                 # key points equal to query points: d2 = 0 exactly on the diagonal
        kv_pts[..., :Pq, :] = q_pts
    elif edge == "zero_vpts":                  # head 0 aggregates the origin; translations 0: both norms at sqrt(eps)
        kv_pts[:, :, 0, Pq:] = 0.0
        trans.zero_()
    x = dict(logit0=logit0, kv=R(Fs, N, H, 2 * C), q_pts=q_pts, kv_pts=kv_pts, pair=R(Fz, N, N, Cp),
             quat=torch.nn.functional.normalize(R(F, N, 4), dim=-1), trans=trans, mask=mask, gamma=gamma)
    D = H * (C + 8 * Pv + Cp)
    return {k: v.contiguous().to(DEV) for k, v in x.items()}, R(F, N, D).to(DEV)


def _ref(x, dcat, Pq, Pv, dfold):
    D = dcat.shape[-1] if dfold else dcat.shape[-1] - 4 * x["q_pts"].shape[2] * Pv
    dcat = dcat[..., :D].contiguous()
    with _RefPeak():
        r = ipa_reference(*x.values(), dcat, Pq=Pq, Pv=Pv, dfold=dfold, inf=INF, eps=EPS)
    return r, dcat


def _f(t):
    return t.float().contiguous()


def _half_ulp_bf16(x):
    """Half an ulp of bf16 values x (fp32 tensor): 2^(e-9) for 2^(e-1) <= |x| < 2^e, 2^-134 for zero and subnormals."""
    _, e = torch.frexp(x)
    h = torch.ldexp(torch.ones_like(x), e - 9).clamp(min=2.0 ** -134)
    return torch.where(x == 0, torch.full_like(x, 2.0 ** -134), h).double()


# --------------------------------------------------------------------------------------------------
# bounds
# --------------------------------------------------------------------------------------------------
def _ds_bound(x, r, k_s):
    """|ds| per logit [F,H,N,N]."""
    F = r["s"].shape[0]
    l0 = x["logit0"].double().abs().expand(F, -1, -1, -1)
    m = x["mask"].double()
    mm = (m[:, :, None] * m[:, None, :] - 1).abs()[:, None]
    return k_s * U * (l0 + 0.5 * x["gamma"].double()[None, :, None, None] * r["d2"] + INF * mm)


def _dp_softmax(r, ds, c_a, n_e, n_r):
    P, sm = r["P"], (r["s"] - r["s"].amax(-1, keepdim=True)).abs()
    E = ds + (P * ds).sum(-1, keepdim=True) + c_a * U * sm + 2 * c_a * U * (P * sm).sum(-1, keepdim=True) + n_e * E_EXP + n_r * U
    return P * torch.expm1(E) + FLOOR


def _agg(P, dp, xs, eq, k_a):
    """Bound of sum_j p_ij x_j: sum_j dp |x| + k_a u sum_j p |x|."""
    xa = xs.abs()
    return torch.einsum(eq, dp, xa) + k_a * U * torch.einsum(eq, P, xa)


def _fwd_bounds(x, r, dp, k_a, C, Pq, Pv, Cp, dfold):
    """Per-column bounds of the concat buffer [F,N,D] (the value columns included; the fused forward does not write them)."""
    F, H, N = r["P"].shape[:3]
    P = r["P"]
    v = x["kv"].double()[..., C:].expand(F, -1, -1, -1)
    vp = x["kv_pts"].double()[..., Pq:, :]
    z = x["pair"].double().expand(F, -1, -1, -1)
    b_o = _agg(P, dp, v, "fhij,fjhc->fihc", k_a).reshape(F, N, H * C)
    b_og = _agg(P, dp, vp, "fhij,fjhpx->fihpx", k_a)                                         # [F,N,H,Pv,3]
    b_pair = _agg(P, dp, z, "fhij,fijc->fihc", k_a).reshape(F, N, H * Cp)
    q = x["quat"].double()
    Rm = O.quat_to_rot(q)[:, :, None, None]                                                 # [F,N,1,1,3,3]
    Rp = _rot_plus(q.abs())[:, :, None, None]
    t = x["trans"].double()[:, :, None, None]
    HPv = H * Pv
    og = torch.einsum("fhij,fjhpx->fihpx", P, vp)
    ol = torch.einsum("fnhpba,fnhpb->fnhpa", Rm.expand(-1, -1, H, Pv, -1, -1), og - t)
    b_ol = (torch.einsum("fnhpba,fnhpb->fnhpa", Rm.abs().expand(-1, -1, H, Pv, -1, -1), b_og)
            + 10 * U * torch.einsum("fnhpba,fnhpb->fnhpa", Rp.expand(-1, -1, H, Pv, -1, -1), og.abs() + t.abs()))
    nl = torch.sqrt((ol ** 2).sum(-1) + EPS)
    ng = torch.sqrt((og ** 2).sum(-1) + EPS)
    b_nl = (ol.abs() * b_ol).sum(-1) / nl + 4 * U * nl
    b_ng = (og.abs() * b_og).sum(-1) / ng + 4 * U * ng
    cols = lambda a: a.reshape(F, N, HPv, 3).permute(0, 1, 3, 2).reshape(F, N, 3 * HPv)
    parts = [b_o, cols(b_ol), b_nl.reshape(F, N, HPv), b_pair]
    if dfold:
        parts += [cols(b_og), b_ng.reshape(F, N, HPv)]
    return torch.cat(parts, dim=-1)


def _pre_bounds(x, cat, dcat, H, C, Pv, Cp, dfold):
    """Plus forms and depths of the epilogue backward (ipa_bwd_pre_kernel) from |cat| (fp32, rounded once) and |dcat|.
    Returns bounds of d_og [F,N,H,Pv,3], delta [F,H,N], dquat [F,N,4], dtrans [F,N,3], and the plus form of d_og."""
    F, N, _ = cat.shape
    HPv = H * Pv
    oc, gc = cat.double().abs(), dcat.double().abs()
    offLoc, offNl = H * C, H * C + 3 * HPv
    offPair = offNl + HPv
    offG, offNg = offPair + H * Cp, offPair + H * Cp + 3 * HPv
    pts = lambda a, off: a[..., off:off + 3 * HPv].reshape(F, N, 3, H, Pv).permute(0, 1, 3, 4, 2)     # [F,N,H,Pv,3]
    nrm = lambda a, off: a[..., off:off + HPv].reshape(F, N, H, Pv, 1)
    q = x["quat"].double()
    Rp = _rot_plus(q.abs())[:, :, None, None]                                                        # [F,N,1,1,3,3]
    ta = x["trans"].double().abs()[:, :, None, None]
    l, nl, gl, gn = pts(oc, offLoc), nrm(oc, offNl), pts(gc, offLoc), nrm(gc, offNl)
    a = gl + gn / nl * l                                                                            # depth 5
    Rpe = Rp.expand(-1, -1, H, Pv, -1, -1)
    ra = torch.einsum("fnhpab,fnhpb->fnhpa", Rpe, a)                                                # R a: depth 13
    if dfold:
        og = pts(oc, offG)
        dog = ra + pts(gc, offG) + nrm(gc, offNg) / nrm(oc, offNg) * og                               # depth 15
        k_og = 1
    else:
        og = torch.einsum("fnhpab,fnhpb->fnhpa", Rpe, l) + ta                                        # reconstructed: 10
        dog = ra
        k_og = 10
    k_dog = 16
    lanes = lambda n: -(-n // 32)
    chain = lanes(C) + lanes(Cp) + lanes(Pv)
    s_delta_o = (gc[..., :H * C].reshape(F, N, H, C) * oc[..., :H * C].reshape(F, N, H, C)).sum(-1) \
        + (gc[..., offPair:offPair + H * Cp].reshape(F, N, H, Cp) * oc[..., offPair:offPair + H * Cp].reshape(F, N, H, Cp)).sum(-1)
    s_delta_p = (dog * og).sum((-1, -2))
    b_delta = ((2 + chain + 5) * U * s_delta_o + (k_dog + k_og + 1 + chain + 5) * U * s_delta_p).permute(0, 2, 1)
    k_sum = lanes(HPv) + 5
    b_dt = (13 + 1 + k_sum) * U * ra.sum((2, 3))
    u_ = og + ta
    dR = torch.einsum("fnhpa,fnhpb->fnab", u_, a)
    k_dR = k_og + 1 + 5 + 1 + k_sum
    (s_q,) = _grads(_rot_plus, [q.abs()], [dR])
    b_dq = (k_dR + 10) * U * s_q
    return k_dog * U * dog, b_delta, b_dq, b_dt, dog


def _check_pre(what, x, r, cat32, dcat, d_og, delta, dquat, dtrans, H, C, Pv, Cp, dfold):
    b_dog, b_delta, b_dq, b_dt, dog_plus = _pre_bounds(x, cat32, dcat, H, C, Pv, Cp, dfold)
    _within(what + " d_og", d_og, r["d_og"], b_dog)
    _within(what + " delta", delta, r["delta"], b_delta)
    _within(what + " dquat", dquat, r["dquat"], b_dq)
    _within(what + " dtrans", dtrans, r["dtrans"], b_dt)
    return b_dog, b_delta, dog_plus


def _check_points(what, x, r, dS_err, Pq, k_pts, got_dq, got_dk):
    """dq = -gamma sum_j dS (q_i - k_j), dk = gamma sum_i dS (q_i - k_j): bounds from |dS| + its error."""
    gam = x["gamma"].double()
    q = x["q_pts"].double().flatten(-2)                                                              # [F,N,H,3Pq]
    k = x["kv_pts"].double()[..., :Pq, :].flatten(-2)
    dsa = r["dS"].abs()
    # sum_j w_ij |q_i - k_j| per coordinate, without the [F,N,N,H,3Pq] tensor: |q - k| <= |q| + |k| is too loose at
    # coincident points, so the exact absolute differences are summed frame by frame
    F, H, N, _ = dsa.shape
    bq = torch.empty_like(q)
    bk = torch.empty_like(k)
    for f in range(F):
        d = (q[f][:, None] - k[f][None]).abs()                                                      # [N,N,H,3Pq]
        w = (k_pts * U * dsa[f] + dS_err[f]).permute(1, 2, 0)                                      # [N,N,H]
        bq[f] = gam[None, :, None] * torch.einsum("ijh,ijhc->ihc", w, d)
        bk[f] = gam[None, :, None] * torch.einsum("ijh,ijhc->jhc", w, d)
        del d
    _within(what + " dq_pts", got_dq, r["dq_pts"], bq.reshape(r["dq_pts"].shape))
    _within(what + " dk_pts", got_dk, r["dk_pts"], bk.reshape(r["dk_pts"].shape))


def _check_dgamma(what, r, dS_err, k_d, ntiles, partials):
    k = k_d + 1 + 4 * ntiles + 5 + 8
    half = 0.5 * r["d2"]
    b = (dS_err * half).sum((0, 2, 3)) + k * U * (r["dS"].abs() * half).sum((0, 2, 3))
    _within(what + " dgamma", partials.double().sum(1), r["dgamma"], b)


# --------------------------------------------------------------------------------------------------
# tensor-core route: fused forward, dS kernel, epilogue backward
# --------------------------------------------------------------------------------------------------
def _planes_out(F, H, N, ldp):
    o = _Out((F, H, N, ldp // 2))
    o.buf.view(torch.bfloat16).fill_(float("nan"))
    return o


def _bf(o, shape):
    return o.v.view(torch.bfloat16).reshape(shape)


TC_CASES = [
    (64, 256, 1, "masked", 0), (64, 256, 0, "plain", 0), (8, 1024, 1, "plain", 0), (32, 256, 1, "plain", 0),
    (1, 1280, 1, "masked", 0), (2, 8, 1, "masked", 0), (3, 24, 0, "plain", 0), (3, 40, 1, "masked", 0),
    (2, 1000, 1, "plain", 0), (2, 40, 1, "plain", 8), (3, 40, 0, "dominant", 0), (3, 40, 1, "uniform", 0),
    (3, 40, 1, "far", 0), (3, 40, 0, "coincident", 0), (3, 40, 1, "zero_vpts", 0), (3, 40, 0, "zero_vpts", 8),
    # p = fl(1 / N) exactly: the remainders of 1/60 and 1/240 below hi lose more than half an ulp of lo when truncated
    (3, 60, 1, "uniform", 0), (2, 240, 0, "uniform", 0), (4, 256, 1, "uniform", 0), (4, 256, 0, "dominant", 0),
]


@pytest.mark.parametrize("F,N,dfold,edge,pad", TC_CASES)
def test_tensor_core_route(F, N, dfold, edge, pad):
    H, C, Pq, Pv, Cp = 8, 256, 8, 12, 32
    what = f"tc F={F} N={N} dfold={dfold} {edge} ldp=N+{pad}"
    ldp = N + pad
    x, dcat_full = _case(F, N, H, C, Pq, Pv, Cp, 1, 1, 1, edge)
    D = H * (C + (8 if dfold else 4) * Pv + Cp)
    L = K.lib()
    p = lambda t: K._ptr(t)
    fwd = lambda o: L.dfold_ipa_fused_fwd(p(x["logit0"]), p(x["q_pts"]), p(x["kv_pts"]), p(x["pair"]), p(x["quat"]), p(x["trans"]),
                                         p(x["mask"]), p(x["gamma"]), o[0].ptr(), o[1].ptr(), ldp, F, N, H, C, Pq, Pv, Cp, dfold,
                                         INF, EPS, o[2].ptr(), K._stream())
    hi_o, lo_o, cat_o = _twice(what + " fused_fwd", lambda: [_planes_out(F, H, N, ldp), _planes_out(F, H, N, ldp), _Out((F, N, D))], fwd)
    r, dcat = _ref(x, dcat_full, Pq, Pv, dfold)
    hi, lo = _bf(hi_o, (F, H, N, ldp)), _bf(lo_o, (F, H, N, ldp))
    assert torch.isnan(hi[..., N:]).all() and torch.isnan(lo[..., N:]).all(), f"{what}: pad columns [N, ldp) of the planes written"
    hi, lo = hi[..., :N], lo[..., :N]
    assert torch.isnan(cat_o.v[..., :H * C]).all(), f"{what}: fused_fwd wrote the value columns [0, H C) of the concat buffer"
    ntiles = -(-N // 32)
    ds = _ds_bound(x, r, 17)
    dp = _dp_softmax(r, ds, 3, ntiles + 3, ntiles + 9)
    # planes
    hf, lf = hi.float(), lo.float()
    split = _half_ulp_bf16(lf)
    _within(what + " P hi+lo", hf.double() + lf.double(), r["P"], dp + split)
    assert bool((lf.abs().double() <= _half_ulp_bf16(hf)).all()), f"{what}: |lo| above half an ulp of hi: hi is not the nearest bf16"
    P = r["P"]
    sm = (r["s"] - r["s"].amax(-1, keepdim=True)).abs() + 2 * ds.amax(-1, keepdim=True)
    b_sum = ((P + dp) * (9 * U * sm + (ntiles + 3) * E_EXP + (ntiles + 9) * U)).sum(-1) + split.sum(-1) + N * FLOOR
    _within(what + " row sums of the planes", (hf.double() + lf.double()).sum(-1), torch.ones_like(b_sum), b_sum)
    # point and pair columns
    b_cat = _fwd_bounds(x, r, dp, N, C, Pq, Pv, Cp, dfold)
    _within(what + " cat points and pair", cat_o.v[..., H * C:], r["cat"][..., H * C:], b_cat[..., H * C:])
    del b_cat

    # epilogue backward from the rounded reference concat buffer
    cat32 = _f(r["cat"])
    pre = lambda o: L.dfold_ipa_pre_bwd(p(x["quat"]), p(x["trans"]), F, N, H, C, Pv, Cp, dfold, p(cat32), p(dcat), o[0].ptr(),
                                       o[1].ptr(), o[2].ptr(), o[3].ptr(), K._stream())
    d_og, delta, dquat, dtrans = _twice(what + " pre_bwd", lambda: [_Out((F, N, H, Pv, 3)), _Out((F, H, N)), _Out((F, N, 4)),
                                                                     _Out((F, N, 3))], pre)
    _check_pre(what + " pre_bwd", x, r, cat32, dcat, d_og.v, delta.v, dquat.v, dtrans.v, H, C, Pv, Cp, dfold)

    # dS kernel from the planes of the float64 P and the rounded dP, Tz, Tog, delta
    P32 = _f(P)
    phi = P32.bfloat16()
    plo = (P32 - phi.float()).bfloat16()
    pad_to = lambda t: torch.nn.functional.pad(t.view(torch.int16), (0, pad)).contiguous()
    phi_l, plo_l = pad_to(phi), pad_to(plo)
    dPv, Tog = _f(r["dPv"]), _f(r["dPog"])
    Tz = _f(r["dPz"].permute(2, 0, 1, 3).reshape(N, F * H, N))
    delta32 = _f(r["delta"])

    def dsl(o):
        o[1].v.zero_()
        return L.dfold_ipa_ds_bwd(p(x["q_pts"]), p(x["kv_pts"]), p(phi_l), p(plo_l), ldp, F, N, H, Pq, Pv, p(delta32), p(dPv),
                                  p(Tz), p(Tog), o[0].ptr(), o[1].ptr(), K._stream())
    dS_o, part_o = _twice(what + " ds_bwd", lambda: [_Out((F, H, N, N)), _Out((H, F * N))], dsl)
    dpv = U * P + _half_ulp_bf16(plo.float()) + U * P + FLOOR          # fp32 rounding of P, the split, the kernel's hi + lo
    tot = r["dPv"] + r["dPog"] + r["dPz"]
    plus = r["dPv"].abs() + r["dPog"].abs() + r["dPz"].abs() + r["delta"].abs()[..., None]
    dS_err = dpv * (tot - r["delta"][..., None]).abs() + 6 * U * P * plus
    _within(what + " ds_bwd dS", dS_o.v, r["dS"], dS_err)
    _check_dgamma(what + " ds_bwd", r, dS_err, 15, ntiles, part_o.v)


# --------------------------------------------------------------------------------------------------
# CUDA-core route: attn_fwd, attn_bwd, pre_bwd
# --------------------------------------------------------------------------------------------------
GEN_CASES = [
    # F, N, H, C, Pq, Pv, Cp, Fl, Fs, Fz, dfold, edge
    (3, 12, 2, 8, 2, 3, 4, 1, 1, 1, 1, "plain"),            # tiny preset
    (2, 20, 12, 16, 4, 8, 32, 1, 1, 1, 1, "masked"),        # preset B
    (2, 33, 4, 16, 4, 8, 64, 2, 2, 2, 0, "masked"),         # vanilla OpenFold: per-frame s and z
    (3, 70, 2, 8, 2, 3, 4, 3, 3, 1, 1, "masked"),           # per-frame s, shared z
    (1, 1, 2, 8, 2, 3, 4, 1, 1, 1, 1, "plain"),
    (2, 2, 2, 8, 2, 3, 4, 1, 1, 1, 0, "plain"),
    (2, 33, 2, 8, 2, 3, 4, 1, 1, 1, 1, "masked"),
    (1, 1288, 8, 256, 8, 12, 32, 1, 1, 1, 1, "masked"),     # preset A past the tensor-core route's longest N
    (3, 40, 8, 256, 8, 12, 32, 3, 1, 1, 1, "plain"),        # preset A with per-frame logit0
    (2, 40, 4, 64, 16, 6, 16, 1, 1, 1, 1, "plain"),         # Pq = 16: ipa_bwd_pts_kernel<48>
    (2, 136, 4, 64, 8, 6, 16, 1, 1, 1, 0, "masked"),        # C = 64, Pq = 8: <24>
    (3, 40, 4, 64, 8, 12, 32, 1, 1, 1, 1, "dominant"),
    (3, 40, 4, 64, 8, 12, 32, 1, 1, 1, 0, "uniform"),
    (3, 40, 4, 64, 8, 12, 32, 1, 1, 1, 1, "far"),
    (3, 40, 4, 64, 8, 12, 32, 1, 1, 1, 1, "coincident"),
    (3, 40, 4, 64, 8, 12, 32, 1, 1, 1, 0, "zero_vpts"),
    (2, 256, 4, 64, 8, 12, 32, 1, 1, 1, 1, "uniform"),      # p = 1 / N over eight key tiles
    (2, 256, 4, 64, 8, 12, 32, 1, 1, 1, 0, "dominant"),
    (3, 40, 4, 64, 8, 12, 32, 1, 1, 1, 1, "zero_vpts"),
]


@pytest.mark.parametrize("F,N,H,C,Pq,Pv,Cp,Fl,Fs,Fz,dfold,edge", GEN_CASES)
def test_cuda_core_route(F, N, H, C, Pq, Pv, Cp, Fl, Fs, Fz, dfold, edge):
    what = f"cc F={F} N={N} H={H} C={C} Pq={Pq} Pv={Pv} Cp={Cp} Fl={Fl} Fs={Fs} Fz={Fz} dfold={dfold} {edge}"
    x, dcat_full = _case(F, N, H, C, Pq, Pv, Cp, Fl, Fs, Fz, edge)
    D = H * (C + (8 if dfold else 4) * Pv + Cp)
    L = K.lib()
    p = lambda t: K._ptr(t)
    fs = lambda t, per: 0 if t.shape[0] == 1 else per
    head = (p(x["logit0"]), fs(x["logit0"], H * N * N), p(x["kv"]), fs(x["kv"], N * H * 2 * C), p(x["q_pts"]), p(x["kv_pts"]),
            p(x["pair"]), fs(x["pair"], N * N * Cp), p(x["quat"]), p(x["trans"]), p(x["mask"]), p(x["gamma"]),
            F, N, H, C, Pq, Pv, Cp, dfold, INF, EPS)
    cat_o, lse_o = _twice(what + " attn_fwd", lambda: [_Out((F, N, D)), _Out((F, H, N))],
                          lambda o: L.dfold_ipa_attn_fwd(*head, o[0].ptr(), o[1].ptr(), K._stream()))
    r, dcat = _ref(x, dcat_full, Pq, Pv, dfold)
    ntiles = -(-N // 32)
    k_s = 3 * Pq + 4
    ds = _ds_bound(x, r, k_s)
    dp = _dp_softmax(r, ds, 1, ntiles + 3, 2 * ntiles + 9)
    P = r["P"]
    sm = (r["s"] - r["s"].amax(-1, keepdim=True)).abs()
    b_lse = (P * ds).sum(-1) + (P * (2 * U * sm + (ntiles + 3) * E_EXP + (2 * ntiles + 9) * U)).sum(-1) \
        + 2 * U * (r["lse"] - r["s"].amax(-1)).abs() + U * r["lse"].abs()
    _within(what + " attn_fwd lse", lse_o.v, r["lse"], b_lse)
    _within(what + " attn_fwd cat", cat_o.v, r["cat"], _fwd_bounds(x, r, dp, N + ntiles + 2, C, Pq, Pv, Cp, dfold))

    # backward from the rounded reference concat buffer and lse
    cat32, lse32 = _f(r["cat"]), _f(r["lse"])

    def bwd(o):
        o[8].v.zero_()
        return L.dfold_ipa_attn_bwd(*head, p(cat32), p(lse32), p(dcat), *[t.ptr() for t in o], K._stream())
    outs = _twice(what + " attn_bwd", lambda: [_Out((F, N, H, Pv, 3)), _Out((F, H, N)), _Out((H, F, N, N)), _Out((H, F, N, N)),
                                               _Out((F, N, H, Pq, 3)), _Out((F, N, H, Pq + Pv, 3)), _Out((F, N, 4)), _Out((F, N, 3)),
                                               _Out((H, F * N))], bwd)
    d_og, delta, Pm, dS, dq, dkv, dquat, dtrans, part = outs
    assert torch.isnan(dkv.v[..., Pq:, :]).all(), f"{what}: attn_bwd wrote the value-point part of dkv_pts"
    b_dog, b_delta, dog_plus = _check_pre(what + " attn_bwd", x, r, cat32, dcat, d_og.v, delta.v, dquat.v, dtrans.v, H, C, Pv, Cp,
                                          dfold)
    E = ds + U * r["lse"].abs()[..., None] + U * (r["s"] - r["lse"][..., None]).abs() + E_EXP
    dpb = P * torch.expm1(E) + FLOOR
    _within(what + " attn_bwd P", Pm.v.permute(1, 0, 2, 3), P, dpb)
    v = x["kv"].double()[..., C:].expand(F, -1, -1, -1)
    vp = x["kv_pts"].double()[..., Pq:, :].flatten(-2)
    z = x["pair"].double().expand(F, -1, -1, -1)
    dO = dcat.double()[..., :H * C].reshape(F, N, H, C).abs()
    offPair = H * C + 4 * H * Pv
    dOp = dcat.double()[..., offPair:offPair + H * Cp].reshape(F, N, H, Cp).abs()
    plus_dP = (torch.einsum("fihc,fjhc->fhij", dO, v.abs()) + torch.einsum("fihe,fjhe->fhij", dog_plus.flatten(-2), vp.abs())
               + torch.einsum("fihc,fijc->fhij", dOp, z.abs()))
    err_dP = ((C + 3 * Pv + Cp + 3) * U * plus_dP
              + 16 * U * torch.einsum("fihe,fjhe->fhij", dog_plus.flatten(-2), vp.abs()))
    tot = r["dPv"] + r["dPog"] + r["dPz"]
    dS_err = dpb * (tot - r["delta"][..., None]).abs() + P * (err_dP + b_delta[..., None] + 2 * U * r["delta"].abs()[..., None])
    _within(what + " attn_bwd dS", dS.v.permute(1, 0, 2, 3), r["dS"], dS_err)
    _check_points(what + " attn_bwd", x, r, dS_err, Pq, 1 + ntiles + 5 + 2, dq.v, dkv.v[..., :Pq, :])
    _check_dgamma(what + " attn_bwd", r, dS_err, 3 * Pq + 2, ntiles, part.v)

    # the same epilogue backward through its own entry point
    pre = lambda o: L.dfold_ipa_pre_bwd(p(x["quat"]), p(x["trans"]), F, N, H, C, Pv, Cp, dfold, p(cat32), p(dcat), o[0].ptr(),
                                       o[1].ptr(), o[2].ptr(), o[3].ptr(), K._stream())
    d_og2, delta2, dquat2, dtrans2 = _twice(what + " pre_bwd", lambda: [_Out((F, N, H, Pv, 3)), _Out((F, H, N)), _Out((F, N, 4)),
                                                                         _Out((F, N, 3))], pre)
    _check_pre(what + " pre_bwd", x, r, cat32, dcat, d_og2.v, delta2.v, dquat2.v, dtrans2.v, H, C, Pv, Cp, dfold)
