"""-m gpu: the per-residue kernels of csrc/rigid.cu, csrc/epilogue.cu (quat_mul, rot_compose, frames_to_atoms,
reverse_step, score_fwd / score_bwd), csrc/loss.cu and csrc/featurize.cu, called directly through the C ABI at the training step's shapes and
compared element by element with a float64 reference of the same operation.

Bounds.  u = 2^-24 (fp32) and ud = 2^-53 (fp64) are the unit roundoffs.  An fp32 kernel output that is a sum of k
rounded products is within gamma_k * S of the exact value, where S is the same sum over absolute values (Higham,
"Accuracy and Stability of Numerical Algorithms", 2nd ed., §3.1).  Each family builds S by running its reference on
absolute values with every subtraction turned into an addition (the "plus" form; for gradients, the plus form's
autograd with absolute cotangents), and states k next to it, counted from the kernel's operation order.  The fp64
kernels (loss, featurisation, reverse step) are held to ud times their conditioning; where the conditioning has no
closed form it is measured as the spread of the float64 reference when its inputs move by a relative 2^-30.  The
score epilogue (K9) mixes both: its fp32 rotation vector is held to the fp64 oracle's spread under a relative 4 u move of
its inputs, its fp32 series trigonometry to a first-order bound on the error that arithmetic adds (_igso3_err).
No max-normalised metric is used and no residue is dropped.  The worst |err| / bound of every case goes to the
JSON-lines file DFOLD_RESIDUE_ERRORS names, when it is set.

Every case also
  * launches twice and requires the same bits;
  * pre-fills each output, and a guard region past its end, with NaN, and requires every element the kernel does not
    own (the guard, and every output passed as NULL) to keep it.
The float64 references run on the CPU for small cases and on the GPU for large ones (peak under REF_PEAK_BYTES).

Shapes: n = 64*256 and 8*1024 (the training step), 32*256 and 2*1024 (sampler, rollout), 1 and 2, and 257 = one past a
multiple of 8 (warp-per-residue grids) and of 256 (thread-per-residue grids).
"""
import json
import math
import os

import numpy as np
import pytest
import torch

from dynamicpdb_b200 import kernels as K
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.feats import table
from dynamicpdb_b200.loss import score_network_loss
from oracle import dfold_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
UD = 2.0 ** -53
REF_PEAK_BYTES = 16 << 30
GUARD = 67                                     # sentinel elements past the end of every output
N_SHAPES = [64 * 256, 8 * 1024, 32 * 256, 2 * 1024, 1, 2, 257]
ARG, LYS = 1, 11                               # openfold restype order; the residue types with a chi4 group


GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _load(name):
    return torch.load(os.path.join(GOLD, name + ".pt"), weights_only=False)


def _elementwise_close(a, b, rel, floor):
    a, b = a.double(), b.double()
    return bool(((a - b).abs() <= rel * b.abs() + floor).all())


def _record(**kw):
    path = os.environ.get("DFOLD_RESIDUE_ERRORS")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(kw) + "\n")


def _ok(rc):
    assert rc == 0, K.lib().dfold_last_error().decode()


def _gen(seed, dev="cpu"):
    return torch.Generator(device=dev).manual_seed(seed)


def _rdev(n):
    return "cpu" if n <= 4096 else DEV


class _Out:
    """A NaN-filled device buffer of `numel` elements plus GUARD; .v is the [shape] view the kernel writes."""

    def __init__(self, shape, dtype=torch.float32):
        numel = int(np.prod(shape))
        self.buf = torch.full((numel + GUARD,), float("nan"), dtype=dtype, device=DEV)
        self.v = self.buf[:numel].view(shape)
        self.numel = numel

    def ptr(self):
        return K._ptr(self.v)

    def guard_ok(self, what):
        assert torch.isnan(self.buf[self.numel:]).all(), f"{what}: the kernel wrote past the end of its output"


def _twice(what, make, launch):
    """make() -> list of _Out (or None for a NULL output); launch(outs) -> rc.  Runs twice and requires identical bits;
    checks the guards; returns the first run's outputs."""
    runs = []
    for _ in range(2):
        outs = make()
        _ok(launch(outs))
        torch.cuda.synchronize()
        runs.append(outs)
    for i, (a, b) in enumerate(zip(*runs)):
        if a is None:
            continue
        w = torch.int64 if a.buf.dtype == torch.float64 else torch.int32
        assert torch.equal(a.buf.view(w), b.buf.view(w)), f"{what}: output {i}: the second launch gave different bits"
        a.guard_ok(f"{what}: output {i}")
    return runs[0]


def _nan_kept(what, out):
    assert torch.isnan(out.buf).all(), f"{what}: an output passed as NULL, or one the kernel must not write, was written"


class _RefPeak:
    def __enter__(self):
        torch.cuda.synchronize()
        self.base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - self.base
        if exc[0] is None:
            assert peak < REF_PEAK_BYTES, f"the float64 reference took {peak / 2**30:.1f} GB of device memory"
        return False


def _within(what, got, ref, bound, family):
    """Per element: |got - ref| <= bound (float64 tensors of one shape).  Records the worst ratio."""
    got, ref, bound = got.double().reshape(-1), ref.double().to(got.device).reshape(-1), bound.double().to(got.device).reshape(-1)
    assert torch.isfinite(got).all(), f"{what}: non-finite outputs"
    err = (got - ref).abs()
    ratio = torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err > 0, float("inf"), 0.0))
    worst = ratio.max().item() if ratio.numel() else 0.0
    _record(family=family, case=what, worst_ratio=worst)
    bad = ratio > 1
    if bad.any():
        j = int(bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside their bound (worst |err| / bound = "
                             f"{worst:.3e}); first at flat index {j}: got {got[j].item():.17g}, expected {ref[j].item():.17g}, "
                             f"bound {bound[j].item():.3e}")
    return worst


# --------------------------------------------------------------------------------------------------
# plus forms (absolute values, every subtraction an addition)
# --------------------------------------------------------------------------------------------------
def _rot_plus(q):
    w, x, y, z = q.unbind(-1)
    d = w * w + x * x + y * y + z * z
    r = torch.stack([d, 2 * (x * y + w * z), 2 * (x * z + w * y), 2 * (x * y + w * z), d, 2 * (y * z + w * x),
                     2 * (x * z + w * y), 2 * (y * z + w * x), d], dim=-1)
    return r.reshape(q.shape[:-1] + (3, 3))


def _qmul_plus(a, b):
    aw, ax, ay, az = a.unbind(-1)
    bw, bx, by, bz = b.unbind(-1)
    return torch.stack([aw * bw + ax * bx + ay * by + az * bz, aw * bx + ax * bw + ay * bz + az * by,
                        aw * by + ax * bz + ay * bw + az * bx, aw * bz + ax * by + ay * bx + az * bw], dim=-1)


def _grads(f, inputs, cot):
    """Autograd of <cot, f(*inputs)> w.r.t. every input (float64 leaves)."""
    leaves = [x.detach().double().requires_grad_(True) for x in inputs]
    out = f(*leaves)
    out = out if isinstance(out, tuple) else (out,)
    pairs = [(o, c) for o, c in zip(out, cot) if o is not None and c is not None]
    s = sum((o * c.double()).sum() for o, c in pairs)
    return [g if g is not None else torch.zeros_like(x) for g, x in zip(torch.autograd.grad(s, leaves, allow_unused=True), leaves)]


def _quats(n, seed, *, unit=False):
    """Quaternions with norms spread over 1e-2 ... 1e2 (or unit), fp32 on the device."""
    g = _gen(seed)
    q = torch.randn(n, 4, generator=g, dtype=torch.float64)
    q = q / q.norm(dim=-1, keepdim=True)
    if not unit:
        q = q * torch.pow(10.0, torch.rand(n, 1, generator=g, dtype=torch.float64) * 4 - 2)
    return q.float().to(DEV)


def _randn(shape, seed, scale=1.0):
    return (torch.randn(shape, generator=_gen(seed)) * scale).to(DEV)


# --------------------------------------------------------------------------------------------------
# rigid.cu: quat_to_rot
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", N_SHAPES)
def test_quat_to_rot_fwd_bwd(n):
    q = _quats(n, 1)
    dR = _randn((n, 3, 3), 2)
    (R,) = _twice(f"quat_to_rot_fwd n={n}", lambda: [_Out((n, 3, 3))],
                  lambda o: K.lib().dfold_quat_to_rot_fwd(K._ptr(q), o[0].ptr(), n, K._stream()))
    (dq,) = _twice(f"quat_to_rot_bwd n={n}", lambda: [_Out((n, 4))],
                   lambda o: K.lib().dfold_quat_to_rot_bwd(K._ptr(q), K._ptr(dR), o[0].ptr(), n, K._stream()))
    rd = _rdev(n)
    with _RefPeak():
        qd, dRd = q.to(rd).double(), dR.to(rd).double()
        # each entry: at most 4 products and 3 additions (x2 is exact) -> gamma_4 of the plus form
        _within(f"quat_to_rot_fwd n={n}", R.v, O.quat_to_rot(qd), 5 * U * _rot_plus(qd.abs()), "rigid")
        # dq: a 3-term sum times 2w plus a 6-term sum of products (x2 exact) -> at most 9 roundings deep
        (ref,) = _grads(O.quat_to_rot, [qd], [dRd])
        (S,) = _grads(_rot_plus, [qd.abs()], [dRd.abs()])
        _within(f"quat_to_rot_bwd n={n}", dq.v, ref, 10 * U * S, "rigid")


# --------------------------------------------------------------------------------------------------
# rigid.cu: rigid_apply (one warp per frame, lane k takes points k, k + 32, ...)
# --------------------------------------------------------------------------------------------------
def _apply_ref(q, t, p, inverse):
    R = O.quat_to_rot(q)[:, :, None]
    return torch.einsum("...ba,...b->...a", R, p - t[:, :, None]) if inverse else torch.einsum("...ab,...b->...a", R, p) + t[:, :, None]


def _apply_plus(q, t, p, inverse):
    R = _rot_plus(q)[:, :, None]
    return torch.einsum("...ba,...b->...a", R, p + t[:, :, None]) if inverse else torch.einsum("...ab,...b->...a", R, p) + t[:, :, None]


def _run_rigid_apply(F, N, m, inverse, shared, seed=0):
    what = f"rigid_apply F={F} N={N} m={m} inverse={inverse} shared_pts={shared}"
    n = F * N
    q = _quats(n, seed + 1).view(F, N, 4)
    t = _randn((F, N, 3), seed + 2, 8.0)
    Fs = 1 if shared else F
    p = _randn((Fs, N, m, 3), seed + 3, 6.0)
    g = _randn((F, N, m, 3), seed + 4)
    fs = 0 if shared else N * m * 3
    (out,) = _twice(what + " fwd", lambda: [_Out((F, N, m, 3))],
                    lambda o: K.lib().dfold_rigid_apply_fwd(K._ptr(q), K._ptr(t), K._ptr(p), fs, o[0].ptr(), F, N, m, int(inverse),
                                                            K._stream()))
    dp, dq, dt = _twice(what + " bwd", lambda: [_Out((F, N, m, 3)), _Out((F, N, 4)), _Out((F, N, 3))],
                        lambda o: K.lib().dfold_rigid_apply_bwd(K._ptr(q), K._ptr(t), K._ptr(p), fs, K._ptr(g), o[0].ptr(), o[1].ptr(),
                                                                o[2].ptr(), F, N, m, int(inverse), K._stream()))
    rd = _rdev(n * m)
    with _RefPeak():
        qd, td, pd, gd = q.to(rd).double(), t.to(rd).double(), p.to(rd).double().expand(F, N, m, 3), g.to(rd).double()
        # out: R (gamma_4 of the plus form) times p, 3 products + 2 additions, + t (inverse: p - t first) -> 9 (10) deep
        _within(what + " out", out.v, _apply_ref(qd, td, pd, inverse),
                (10 + inverse) * U * _apply_plus(qd.abs(), td.abs(), pd.abs(), inverse), "rigid")
        f = lambda q_, t_, p_: _apply_ref(q_, t_, p_, inverse)
        fp = lambda q_, t_, p_: _apply_plus(q_, t_, p_, inverse)
        r_q, r_t, r_p = _grads(f, [qd, td, pd], [gd])
        s_q, s_t, s_p = _grads(fp, [qd.abs(), td.abs(), pd.abs()], [gd.abs()])
        # dp = R^T g (inverse R g): R plus a 3-term dot -> 8 deep
        _within(what + " dpts", dp.v, r_p, 8 * U * s_p, "rigid")
        # dR, dt: ceil(m / 32) sequential lane terms, then a 5-level warp tree; dq adds quat_to_rot_bwd's 10 and the
        # inverse's p - t rounding
        k = math.ceil(m / 32) + 6
        _within(what + " dquat", dq.v, r_q, (k + 12) * U * s_q, "rigid")
        _within(what + " dtrans", dt.v, r_t, (k + 10) * U * s_t, "rigid")


@pytest.mark.parametrize("m", [1, 31, 32, 33, 48, 64, 144, 160])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("shared", [True, False])
def test_rigid_apply_point_counts(m, inverse, shared):
    """IPA's point counts (presets A and B: 64 query, 160 key/value points per frame) at F = 64 frames of 256 residues."""
    _run_rigid_apply(64, 256, m, inverse, shared, seed=m)


@pytest.mark.parametrize("n", [8 * 1024, 32 * 256, 2 * 1024, 1, 2, 257])
@pytest.mark.parametrize("inverse", [0, 1])
def test_rigid_apply_shapes(n, inverse):
    F = {8 * 1024: 8, 32 * 256: 32, 2 * 1024: 2}.get(n, 1)
    _run_rigid_apply(F, n // F, 33, inverse, shared=(n % 2 == 0), seed=n)


# --------------------------------------------------------------------------------------------------
# rigid.cu: compose_q_update
# --------------------------------------------------------------------------------------------------
def _compose_ref(q, t, u, m):
    r = O.compose_q_update_vec(torch.cat([q, t], -1), u, None if m is None else m[:, None])
    return r[:, :4], r[:, 4:]


def _compose_plus(q, t, u, m, nrm):
    mm = 1.0 if m is None else m[:, None]
    zero = torch.zeros_like(u[:, :1])
    qn = (q + mm * _qmul_plus(q, torch.cat([zero, u[:, :3]], -1))) / nrm
    return qn, t + mm * torch.einsum("...ab,...b->...a", _rot_plus(q), u[:, 3:])


@pytest.mark.parametrize("n", N_SHAPES)
@pytest.mark.parametrize("kind", ["mask", "nomask", "large"])
def test_compose_q_update(n, kind):
    what = f"compose_q_update n={n} {kind}"
    q = _quats(n, 11, unit=True)
    t = _randn((n, 3), 12, 8.0)
    u = _randn((n, 6), 13, 10.0 if kind == "large" else 0.4)
    m = (torch.rand(n, generator=_gen(14)) > 0.3).float().to(DEV) if kind == "mask" else None
    gq, gt = _randn((n, 4), 15), _randn((n, 3), 16)
    qo, to = _twice(what + " fwd", lambda: [_Out((n, 4)), _Out((n, 3))],
                    lambda o: K.lib().dfold_compose_q_update_fwd(K._ptr(q), K._ptr(t), K._ptr(u), K._ptr(m), o[0].ptr(), o[1].ptr(), n,
                                                                 K._stream()))
    dq, dt, du = _twice(what + " bwd", lambda: [_Out((n, 4)), _Out((n, 3)), _Out((n, 6))],
                        lambda o: K.lib().dfold_compose_q_update_bwd(K._ptr(q), K._ptr(u), K._ptr(m), K._ptr(gq), K._ptr(gt), o[0].ptr(),
                                                                     o[1].ptr(), o[2].ptr(), n, K._stream()))
    rd = _rdev(n)
    with _RefPeak():
        qd, td, ud, gqd, gtd = (x.to(rd).double() for x in (q, t, u, gq, gt))
        md = None if m is None else m.to(rd).double()
        rq, rt = _compose_ref(qd, td, ud, md)
        mm = 1.0 if md is None else md[:, None]
        nrm = (qd + mm * O.quat_mul(qd, torch.cat([torch.zeros_like(ud[:, :1]), ud[:, :3]], -1))).norm(dim=-1, keepdim=True)
        sq, st = _compose_plus(qd.abs(), td.abs(), ud.abs(), None if md is None else md.abs(), nrm)
        # q: the un-normalised product is 4 deep; |.|^2 (4), sqrt, 1/x and the product add 7 more
        _within(what + " quat", qo.v, rq, 12 * U * sq, "compose")
        # t: R (4) times v (3 products, 2 additions), times m, plus t -> 10 deep
        _within(what + " trans", to.v, rt, 11 * U * st, "compose")
        f = lambda q_, t_, u_: _compose_ref(q_, t_, u_, md)
        r_q, r_t, r_u = _grads(f, [qd, td, ud], [gqd, gtd])
        # through the normalisation: (g - o <o, g>) / |n| -- the plus cotangent is |g| + |o| <|o|, |g|>
        cq = gqd.abs() + rq.abs() * (rq.abs() * gqd.abs()).sum(-1, keepdim=True)
        fp = lambda q_, t_, u_: _compose_plus(q_, t_, u_, None if md is None else md.abs(), nrm)
        s_q, s_t, s_u = _grads(fp, [qd.abs(), td.abs(), ud.abs()], [cq, gtd.abs()])
        # dq: 1/|n| (7), <o, g> (4), the projection (2), the product's transpose (4) and quat_to_rot_bwd (10)
        _within(what + " dquat", dq.v, r_q, 30 * U * s_q, "compose")
        _within(what + " dtrans", dt.v, r_t, torch.zeros_like(r_t), "compose")          # a copy
        _within(what + " dupd", du.v, r_u, 16 * U * s_u, "compose")


# --------------------------------------------------------------------------------------------------
# epilogue.cu: quat_mul, rot_compose
# --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", N_SHAPES)
@pytest.mark.parametrize("b_is_vec", [0, 1])
@pytest.mark.parametrize("null", [None, "da", "db"])
def test_quat_mul(n, b_is_vec, null):
    what = f"quat_mul n={n} b_is_vec={b_is_vec} null={null}"
    a = _quats(n, 21)
    b = _randn((n, 3), 22, 2.0) if b_is_vec else _quats(n, 23)
    g = _randn((n, 4), 24)
    (out,) = _twice(what + " fwd", lambda: [_Out((n, 4))],
                    lambda o: K.lib().dfold_quat_mul_fwd(K._ptr(a), K._ptr(b), o[0].ptr(), n, b_is_vec, K._stream()))
    da, db = _twice(what + " bwd", lambda: [_Out((n, 4)), _Out((n, 3 if b_is_vec else 4))],
                    lambda o: K.lib().dfold_quat_mul_bwd(K._ptr(a), K._ptr(b), K._ptr(g), None if null == "da" else o[0].ptr(),
                                                         None if null == "db" else o[1].ptr(), n, b_is_vec, K._stream()))
    rd = _rdev(n)
    with _RefPeak():
        ad, bd, gd = a.to(rd).double(), b.to(rd).double(), g.to(rd).double()
        lift = (lambda v: torch.cat([torch.zeros_like(v[:, :1]), v], -1)) if b_is_vec else (lambda v: v)
        f = lambda a_, b_: O.quat_mul(a_, lift(b_))
        fp = lambda a_, b_: _qmul_plus(a_, lift(b_))
        # 4 products, 3 additions
        _within(what + " out", out.v, f(ad, bd), 5 * U * fp(ad.abs(), bd.abs()), "quat_mul")
        r_a, r_b = _grads(f, [ad, bd], [gd])
        s_a, s_b = _grads(fp, [ad.abs(), bd.abs()], [gd.abs()])
        for name, o, r, s in (("da", da, r_a, s_a), ("db", db, r_b, s_b)):
            if null == name:
                _nan_kept(what + " " + name, o)
            else:
                _within(what + " " + name, o.v, r, 5 * U * s, "quat_mul")


def _rc_ref(Ra, ta, Rb, tb, inverse, plus=False):
    """Ra [na,3,3] (broadcast over rep), Rb [na,rep,3,3], tb [na,rep,3]."""
    A = Ra[:, None]
    Ro = None if Rb is None else A @ Rb
    to = None
    if tb is not None:
        if inverse:
            d = tb if ta is None else (tb + ta[:, None] if plus else tb - ta[:, None])
            to = torch.einsum("...ba,...b->...a", A, d)
        else:
            to = torch.einsum("...ab,...b->...a", A, tb)
            if ta is not None:
                to = to + ta[:, None]
    return Ro, to


@pytest.mark.parametrize("n", N_SHAPES)
@pytest.mark.parametrize("rep", [1, 8, 14, 37])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("null", [None, "ta", "Rb", "tb", "grads"])
def test_rot_compose(n, rep, inverse, null):
    if n > 2048 and (rep > 8 or null not in (None, "grads")):
        pytest.skip("the large shapes run with rep in {1, 8} and every operand present")
    what = f"rot_compose n_a={n} rep={rep} inverse={inverse} null={null}"
    nb = n * rep
    Ra = O.quat_to_rot(_quats(n, 31).double()).float()
    ta = None if null == "ta" else _randn((n, 3), 32, 5.0)
    Rb = None if null == "Rb" else O.quat_to_rot(_quats(nb, 33).double()).float()
    tb = None if null == "tb" else _randn((nb, 3), 34, 5.0)
    gR, gt = _randn((nb, 3, 3), 35), _randn((nb, 3), 36)
    Ro, to = _twice(what + " fwd", lambda: [_Out((nb, 3, 3)), _Out((nb, 3))],
                    lambda o: K.lib().dfold_rot_compose_fwd(K._ptr(Ra), K._ptr(ta), K._ptr(Rb), K._ptr(tb), o[0].ptr(), o[1].ptr(), n,
                                                            rep, inverse, K._stream()))
    skip_g = {"dRa", "dta"} if null == "grads" else set()
    dRa, dta, dRb, dtb = _twice(what + " bwd", lambda: [_Out((n, 3, 3)), _Out((n, 3)), _Out((nb, 3, 3)), _Out((nb, 3))],
                                lambda o: K.lib().dfold_rot_compose_bwd(
                                    K._ptr(Ra), K._ptr(ta), K._ptr(Rb), K._ptr(tb), K._ptr(gR), K._ptr(gt),
                                    None if "dRa" in skip_g else o[0].ptr(), None if "dta" in skip_g else o[1].ptr(),
                                    o[2].ptr(), o[3].ptr(), n, rep, inverse, K._stream()))
    rd = _rdev(nb)
    with _RefPeak():
        dd = lambda x: None if x is None else x.to(rd).double()
        Rad, tad, gRd, gtd = dd(Ra), dd(ta), dd(gR).view(n, rep, 3, 3), dd(gt).view(n, rep, 3)
        Rbd = None if Rb is None else dd(Rb).view(n, rep, 3, 3)
        tbd = None if tb is None else dd(tb).view(n, rep, 3)
        rRo, rto = _rc_ref(Rad, tad, Rbd, tbd, inverse)
        ab = lambda x: None if x is None else x.abs()
        sRo, sto = _rc_ref(ab(Rad), ab(tad), ab(Rbd), ab(tbd), inverse, plus=True)
        # Rout: 3 products, 2 additions; tout: + ta (inverse: tb - ta first)
        if Rb is None:
            _nan_kept(what + " Rout", Ro)
        else:
            _within(what + " Rout", Ro.v, rRo.reshape(nb, 3, 3), 4 * U * sRo.reshape(nb, 3, 3), "rot_compose")
        if tb is None:
            _nan_kept(what + " tout", to)
        else:
            _within(what + " tout", to.v, rto.reshape(nb, 3), 6 * U * sto.reshape(nb, 3), "rot_compose")
        # without ta the kernel still writes dta: the gradient a zero ta would receive
        ins = [Rad, torch.zeros_like(Rad[:, 0]) if tad is None else tad, Rbd, tbd]
        present = [x is not None for x in ins]
        f = lambda *xs: _rc_ref(*_fill(xs, present), inverse)
        fp = lambda *xs: _rc_ref(*_fill(xs, present), inverse, plus=True)
        cot = [gRd if Rb is not None else None, gtd if tb is not None else None]
        r = _grads(f, [x for x in ins if x is not None], cot)
        s = _grads(fp, [x.abs() for x in ins if x is not None], [None if c is None else c.abs() for c in cot])
        r, s = _fill(r, present), _fill(s, present)
        # dRa / dta accumulate rep terms of <= 4 roundings each (the Rb and t parts both land in dRa); dRb / dtb are
        # one 3-term dot
        ka = 4 * rep + 8
        for name, o, i, k, shp in (("dRa", dRa, 0, ka, (n, 3, 3)), ("dta", dta, 1, ka, (n, 3)), ("dRb", dRb, 2, 5, (nb, 3, 3)),
                                   ("dtb", dtb, 3, 5, (nb, 3))):
            if name in skip_g:
                _nan_kept(what + " " + name, o)
                continue
            if r[i] is None:                    # operand absent: the kernel zero-fills its gradient
                _within(what + " " + name, o.v, torch.zeros(shp, dtype=torch.float64), torch.zeros(shp, dtype=torch.float64),
                        "rot_compose")
            else:
                _within(what + " " + name, o.v, r[i].reshape(shp), k * U * s[i].reshape(shp), "rot_compose")


def _fill(xs, present):
    it = iter(xs)
    return [next(it) if p else None for p in present]


# --------------------------------------------------------------------------------------------------
# epilogue.cu: frames_to_atoms (K10)
# --------------------------------------------------------------------------------------------------
def _chain_plus(bb44, alpha, aatype):
    """torsion_angles_to_frames over absolute values: |default| |Rx| products, the chi chain, then |backbone|."""
    tb = O.residue_tables()
    default = tb["default_frames"].to(alpha.device, alpha.dtype)[aatype].abs()
    default[..., 3, 3] = 1
    bb = alpha.new_zeros(alpha.shape[:-2] + (1, 2))
    bb[..., 1] = 1
    al = torch.cat([bb, alpha], dim=-2).abs()
    rot = alpha.new_zeros(al.shape[:-1] + (4, 4))
    rot[..., 0, 0] = 1
    rot[..., 1, 1] = al[..., 1]
    rot[..., 1, 2] = al[..., 0]
    rot[..., 2, 1] = al[..., 0]
    rot[..., 2, 2] = al[..., 1]
    rot[..., 3, 3] = 1
    fr = default @ rot
    chi2 = fr[..., 4, :, :] @ fr[..., 5, :, :]
    chi3 = chi2 @ fr[..., 6, :, :]
    chi4 = chi3 @ fr[..., 7, :, :]
    to_bb = torch.cat([fr[..., :5, :, :], chi2[..., None, :, :], chi3[..., None, :, :], chi4[..., None, :, :]], dim=-3)
    return bb44[..., None, :, :] @ to_bb


def _atoms_plus(frames_plus, aatype):
    tb = O.residue_tables()
    grp = tb["atom14_group"].to(frames_plus.device)[aatype]
    fr = torch.gather(frames_plus, -3, grp[..., None, None].expand(grp.shape + (4, 4)))
    pos = tb["atom14_pos"].to(frames_plus.device, frames_plus.dtype)[aatype].abs()
    out = torch.einsum("...ab,...b->...a", fr[..., :3, :3], pos) + fr[..., :3, 3]
    return out * tb["atom14_mask"].to(frames_plus.device, frames_plus.dtype)[aatype][..., None]


def _bb44(R, t):
    m = R.new_zeros(R.shape[:-2] + (4, 4))
    m[..., :3, :3] = R
    m[..., :3, 3] = t
    m[..., 3, 3] = 1
    return m


@pytest.mark.parametrize("n", N_SHAPES)
@pytest.mark.parametrize("rot_is_matrix", [0, 1])
@pytest.mark.parametrize("null", [None, "frames44", "atom14", "atom37"])
def test_frames_to_atoms(n, rot_is_matrix, null):
    if n in (8 * 1024, 32 * 256, 2 * 1024) and null is not None:
        pytest.skip("the NULL outputs run at the other shapes")
    what = f"frames_to_atoms n={n} rot_is_matrix={rot_is_matrix} null={null}"
    q = _quats(n, 41, unit=True)
    rot = O.quat_to_rot(q.double()).float().reshape(n, 9) if rot_is_matrix else q
    trans = _randn((n, 3), 42, 10.0)
    ang = torch.rand(n, 7, generator=_gen(43), dtype=torch.float64) * 2 * math.pi
    alpha = torch.stack([ang.sin(), ang.cos()], -1).float().to(DEV)
    # every residue type many times; n = 1 and 2 take the two chi4 types
    aatype = (torch.arange(n) % 21 if n > 2 else torch.tensor([ARG, LYS])[:n]).to(DEV)
    tabs = [table(k, DEV) for k in ("default_frames", "atom14_group", "atom14_mask", "atom14_pos", "atom37_to_atom14", "atom37_mask")]
    fr, a14, a37 = _twice(what, lambda: [_Out((n, 8, 4, 4)), _Out((n, 14, 3)), _Out((n, 37, 3))],
                          lambda o: K.lib().dfold_frames_to_atoms_fwd(
                              K._ptr(rot), rot_is_matrix, K._ptr(trans), K._ptr(alpha), K._ptr(aatype), *[K._ptr(x) for x in tabs],
                              None if null == "frames44" else o[0].ptr(), None if null == "atom14" else o[1].ptr(),
                              None if null == "atom37" else o[2].ptr(), n, K._stream()))
    rd = _rdev(n)
    with _RefPeak():
        qd, Rd, td, ald, aa = q.to(rd).double(), O.quat_to_rot(q.to(rd).double()), trans.to(rd).double(), alpha.to(rd).double(), aatype.to(rd)
        if rot_is_matrix:
            Rd = rot.to(rd).double().view(n, 3, 3)
            ref_fr = O.torsion_angles_to_frames(None, ald, aa, bb44=_bb44(Rd, td))
            s_fr = _chain_plus(_bb44(Rd.abs(), td.abs()), ald, aa)
            k_bb = 0
        else:
            ref_fr = O.torsion_angles_to_frames(torch.cat([qd, td], -1), ald, aa)
            s_fr = _chain_plus(_bb44(_rot_plus(qd.abs()), td.abs()), ald, aa)
            k_bb = 4
        ref14 = O.frames_to_atom14(ref_fr, aa)
        ref37, _ = O.atom14_to_atom37(ref14, aa)
        s14 = _atoms_plus(s_fr, aa)
        s37, _ = O.atom14_to_atom37(s14, aa)
        # deepest frame (chi4): Rx (2) + three chain products (4 each: 3 products + the translation's addition) +
        # the backbone product (4) + the quaternion (4)
        k_fr = 2 + 3 * 4 + 4 + k_bb
        if null == "frames44":
            _nan_kept(what + " frames44", fr)
        else:
            _within(what + " frames44", fr.v, ref_fr, (k_fr + 1) * U * s_fr, "frames_to_atoms")
            chi4 = (aa == ARG) | (aa == LYS)
            _within(what + " frames44 chi4 of ARG/LYS", fr.v[chi4.to(DEV)][:, 7], ref_fr[chi4][:, 7],
                    (k_fr + 1) * U * s_fr[chi4][:, 7], "frames_to_atoms")
        # atoms: one more 3-term dot plus the translation
        for name, o, r, s in (("atom14", a14, ref14, s14), ("atom37", a37, ref37, s37)):
            if null == name:
                _nan_kept(what + " " + name, o)
            else:
                _within(what + " " + name, o.v, r, (k_fr + 5) * U * s, "frames_to_atoms")


# --------------------------------------------------------------------------------------------------
# epilogue.cu: reverse_step (one CTA of 256 threads per frame, fp64 arithmetic on fp32 inputs)
# --------------------------------------------------------------------------------------------------
def _ulp32(x):
    """Spacing of fp32 numbers at |x| (the subnormal spacing below 2^-126)."""
    a = x.abs().float().clamp(min=2.0 ** -126)
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


def _rev_inputs(F, N, seed, *, trans_f64, perturb=None):
    g = _gen(seed)
    q = torch.randn(F, N, 4, generator=g)
    q = q * (0.5 + torch.rand(F, N, 1, generator=g))                   # not unit: the kernel normalises
    x = torch.randn(F, N, 3, generator=g) * 12.0
    rs = torch.randn(F, N, 3, generator=g, dtype=torch.float64) * 0.8
    ts = torch.randn(F, N, 3, generator=g, dtype=torch.float64) * 0.5
    zr, zt = torch.randn(F, N, 3, generator=g), torch.randn(F, N, 3, generator=g)
    mask = (torch.rand(F, N, generator=g) > 0.25).float()
    if not trans_f64:
        ts = ts.float()
    return dict(q=q, x=x, rs=rs, ts=ts, zr=zr, zt=zt, mask=mask)


def _rev_consts(t, dt, dc):
    sig = float(O._sigma_of_t(np.array(t), dc))
    g_rot = math.sqrt(2 * (math.exp(dc.max_sigma) - math.exp(dc.min_sigma)) * sig / math.exp(sig))
    b_t = dc.min_b + t * (dc.max_b - dc.min_b)
    return g_rot, math.sqrt(b_t), b_t


@pytest.mark.parametrize("F", [1, 32, 64])
@pytest.mark.parametrize("N", [1, 2, 255, 256, 257, 1024])
@pytest.mark.parametrize("variant", ["center", "no_center", "mask_f32", "no_noise", "tiny", "near_pi", "past_pi", "rot_off",
                                     "trans_off"])
def test_reverse_step(F, N, variant):
    if F == 32 and variant not in ("center", "mask_f32"):
        pytest.skip("F = 32 runs the centred and masked variants")
    what = f"reverse_step F={F} N={N} {variant}"
    t, dt, cs = 0.37, 0.01, 0.1
    dc = O.default_diffuser_conf(cs)
    g_rot, g_trans, b_t = _rev_consts(t, dt, dc)
    c = _rev_inputs(F, N, 1000 * F + N, trans_f64=(variant != "mask_f32"))
    center = variant != "no_center"
    noise = 0.0 if variant in ("no_noise", "tiny", "near_pi", "past_pi") else 0.7
    use_mask = variant == "mask_f32"
    if variant in ("tiny", "near_pi", "past_pi"):
        # rotation perturbation g^2 s dt of norm 1e-13 (below the kernel's 1e-12 series switch), pi - 1e-3, or 2.5 ... 6
        axis = torch.nn.functional.normalize(c["rs"], dim=-1)
        ang = {"tiny": torch.full((F, N, 1), 1e-13, dtype=torch.float64),
               "near_pi": math.pi - 1e-3 + 1e-4 * torch.rand(F, N, 1, generator=_gen(5), dtype=torch.float64),
               "past_pi": 2.5 + 3.5 * torch.rand(F, N, 1, generator=_gen(6), dtype=torch.float64)}[variant]
        c["rs"] = axis * ang / (g_rot * g_rot * dt)
    diffuse_rot, diffuse_trans = variant != "rot_off", variant != "trans_off"
    d = {k: v.to(DEV).contiguous() for k, v in c.items()}
    qo, xo = _twice(what, lambda: [_Out((F, N, 4)), _Out((F, N, 3))],
                    lambda o: K.lib().dfold_reverse_step(
                        K._ptr(d["q"]), K._ptr(d["x"]), K._ptr(d["rs"]), K._ptr(d["ts"]), int(d["ts"].dtype == torch.float64),
                        K._ptr(d["zr"]), K._ptr(d["zt"]), K._ptr(d["mask"]) if use_mask else None, g_rot, g_trans, b_t, dt, noise, cs,
                        int(center), int(diffuse_rot), int(diffuse_trans), o[0].ptr(), o[1].ptr(), F, N, K._stream()))
    qn = torch.nn.functional.normalize(c["q"].double(), dim=-1)
    if diffuse_rot and diffuse_trans:
        ref = O.reverse_step(torch.cat([c["q"], c["x"]], -1), c["rs"].numpy(), c["ts"].double().numpy(), t, dt,
                             c["mask"].numpy() if use_mask else None, c["zr"].double().numpy(), c["zt"].double().numpy(), dc,
                             center=center, noise_scale=noise)
        rq, rx = ref[..., :4].double(), ref[..., 4:].double()
    elif not diffuse_rot:
        ref = O.reverse_step(torch.cat([c["q"], c["x"]], -1), np.zeros((F, N, 3)), c["ts"].double().numpy(), t, dt, None,
                             np.zeros((F, N, 3)), c["zt"].double().numpy(), dc, center=center, noise_scale=noise)
        rq, rx = qn, ref[..., 4:].double()
    else:
        rq, rx = None, c["x"].double()
        ref = O.reverse_step(torch.cat([c["q"], c["x"]], -1), c["rs"].numpy(), np.zeros((F, N, 3)), t, dt, None,
                             c["zr"].double().numpy(), np.zeros((F, N, 3)), dc, center=False, noise_scale=noise)
        rq = ref[..., :4].double()
    got_q, got_x = qo.v.double().cpu(), xo.v.double().cpu()
    # the quaternion up to its sign; both sides round an fp64 value to fp32 (the oracle at its end), so they may differ
    # by one fp32 ulp, plus the fp64 error of the scipy rotation-vector round trips (a few ud of |q| = 1)
    sgn = torch.where((got_q * rq).sum(-1, keepdim=True) < 0, -1.0, 1.0)
    _within(what + " quat", got_q, sgn * rq, _ulp32(rq) + 2.0 ** -44, "reverse_step")
    # translations: one fp32 ulp plus fp64 error relative to the terms of x1 / r3 (x_t, the step and the centre)
    scale = c["x"].double().abs() + rx.abs() + (rx - c["x"].double()).abs()
    _within(what + " trans", got_x, rx, _ulp32(rx) + 2.0 ** -44 * scale, "reverse_step")


# --------------------------------------------------------------------------------------------------
# loss.cu: loss_fwd (one CTA of 256 threads, fp64)
# --------------------------------------------------------------------------------------------------
def _unit2(shape, g):
    a = torch.rand(shape, generator=g, dtype=torch.float64) * 2 * math.pi
    return torch.stack([a.sin(), a.cos()], -1)


def _loss_case(nf, N, seed, *, separate, t=0.5, trans_mean=None, mask=None, zero=False):
    g = _gen(seed)
    gt = _unit2((nf, N, 7), g)
    flip = (torch.rand(nf, N, 7, 1, generator=g) > 0.5).double()
    alt = gt * (1 - 2 * flip)
    x0 = torch.randn(nf, N, 3, generator=g, dtype=torch.float64) * 10
    batch = {"torsion_angles_sin_cos": gt, "alt_torsion_angles_sin_cos": alt,
             "torsion_angles_mask": (torch.rand(nf, N, 7, generator=g) > 0.2).double(),
             "res_mask": (torch.rand(nf, N, generator=g) > 0.1).double(), "fixed_mask": (torch.rand(nf, N, generator=g) < 0.05).double(),
             "rot_score": torch.randn(nf, N, 3, generator=g, dtype=torch.float64) * 0.7,
             "rot_score_scaling": torch.tensor([0.8], dtype=torch.float64), "t": torch.tensor([t], dtype=torch.float64),
             "rigids_0": torch.cat([torch.randn(nf, N, 4, generator=g, dtype=torch.float64), x0], -1)}
    dx = torch.randn(nf, N, 3, generator=g, dtype=torch.float64)
    if trans_mean is not None:                     # every component displaced by the same amount: mean square = trans_mean
        dx = torch.full_like(dx, math.sqrt(trans_mean))
    out = {"angles": torch.randn(nf, N, 7, 2, generator=g, dtype=torch.float64) * 0.8,
           "rot_score": torch.randn(nf, N, 3, generator=g, dtype=torch.float64),
           "rigids": torch.cat([torch.randn(nf, N, 4, generator=g, dtype=torch.float64), x0 + dx], -1)}
    if mask == "last_frame":
        batch["res_mask"][-1] = 0
    elif mask == "all":
        batch["res_mask"][:] = 0
    if zero:                                       # zero-length predictions with alt = gt and alt = -gt, a zero score
        k = min(N, 4)
        out["angles"][-1, :k, 0] = 0
        batch["alt_torsion_angles_sin_cos"][-1, :k:2, 0] = gt[-1, :k:2, 0]
        batch["alt_torsion_angles_sin_cos"][-1, 1:k:2, 0] = -gt[-1, 1:k:2, 0]
        batch["torsion_angles_mask"][-1, :k, 0] = 1
        out["rot_score"][-1, :k] = 0
        batch["res_mask"][-1, :k] = 1
        batch["fixed_mask"][-1, :k] = 0
    return batch, out


def _plus_case(batch, out):
    """The same loss with the torsion and rotation differences turned into sums of magnitudes (targets -|gt|,
    predictions +|.|).  The translations stay as they are, so that the < 100 gates decide as in the real case; the
    translation term's rounding (~ud (|x0| + |x|) / |x0 - x| of itself for coordinates of tens of A) sits inside the
    bound's factor."""
    b = dict(batch)
    b["torsion_angles_sin_cos"] = -batch["torsion_angles_sin_cos"].abs()
    b["alt_torsion_angles_sin_cos"] = -batch["alt_torsion_angles_sin_cos"].abs()
    b["rot_score"] = -batch["rot_score"].abs()
    o = {k: (v if k == "rigids" else v.abs()) for k, v in out.items()}
    return b, o


def _oracle_loss(batch, out, conf, rot_on, dev):
    leaves = {k: out[k].to(dev).clone().requires_grad_(True) for k in ("angles", "rot_score", "rigids")}
    loss, aux = O.loss_fn(leaves, {k: v.to(dev) for k, v in batch.items()}, conf, diffuse_rot=bool(rot_on))
    grads = torch.autograd.grad(loss, list(leaves.values()))
    vals = torch.stack([loss.detach(), aux["rot_loss"], aux["trans_loss"], aux["torsion_loss"], aux["batch_rot_loss"][0],
                        aux["batch_trans_loss"][0], aux["batch_torsion_loss"][0], aux["batch_train_loss"][0]])
    return vals, grads[0][-1], grads[1][-1], grads[2][-1, :, 4:]


def nrm_of(batch):
    """nf / (number of non-empty frames + 1e-10), the denominator formed in fp32 as torch does for an integer count."""
    count = float((batch["res_mask"] != 0).any(-1).sum())
    return batch["res_mask"].shape[0] / float(np.float32(count) + np.float32(1e-10))


def _run_loss(what, nf, N, seed, *, separate, rot_on=1, **kw):
    batch, out = _loss_case(nf, N, seed, separate=separate, **kw)
    conf = O.default_exp_conf(separate_rot_loss=separate)
    d = lambda v: v.to(DEV).contiguous()
    ins = [d(out["angles"][-1]), d(batch["torsion_angles_sin_cos"][-1]), d(batch["alt_torsion_angles_sin_cos"][-1]),
           d(batch["torsion_angles_mask"][-1]), d(out["rot_score"][-1]), d(batch["rot_score"][-1]), d(out["rigids"][-1, :, 4:]),
           d(batch["rigids_0"][-1, :, 4:]), d(batch["res_mask"]), d(batch["fixed_mask"]), d(batch["t"]), d(batch["rot_score_scaling"])]
    res, da, dr, dx = _twice(what, lambda: [_Out((8,), torch.float64), _Out((N, 7, 2), torch.float64), _Out((N, 3), torch.float64),
                                            _Out((N, 3), torch.float64)],
                             lambda o: K.lib().dfold_loss_fwd(*[K._ptr(x) for x in ins], nf, N, conf.torsion_loss_weight,
                                                              conf.rot_loss_weight, conf.trans_loss_weight, conf.rot_loss_t_threshold,
                                                              rot_on, int(separate), *[x.ptr() for x in o], K._stream()))
    rd = _rdev(nf * N)
    with _RefPeak():
        ref = _oracle_loss(batch, out, conf, rot_on, rd)
        plus = _oracle_loss(*_plus_case(batch, out), conf, rot_on, rd)
    # kernel: ceil(N / 256) terms per thread, a 5-level warp tree and 8 warp sums, each term ~30 roundings deep; the fp64
    # oracle's own sums are as deep again.  Every loss term is >= 0, so the plus form bounds the sums' magnitudes.
    k = 2 * (math.ceil(N / 256) + 13 + 30)
    _within(what + " values", res.v, ref[0], k * UD * (ref[0].abs() + plus[0].abs()), "loss")
    # d_rot_score, separate form: the axis term's projection and the angle term (ga - qa) cancel; S takes them apart
    s_rs = ref[2].abs() + plus[2].abs()
    if separate:
        g, q = batch["rot_score"][-1].to(rd), out["rot_score"][-1].to(rd)
        dm = 1 - batch["fixed_mask"][-1].to(rd)
        lm = (batch["res_mask"][-1].to(rd) * dm)[:, None]
        q = q * dm[:, None]
        ga, qa = g.norm(dim=-1, keepdim=True), q.norm(dim=-1, keepdim=True)
        gate1 = float(((batch["rigids_0"][-1, :, 4:] - out["rigids"][-1, :, 4:]) ** 2).mean()) * conf.trans_loss_weight < 100
        k_axis = rot_on / (float(lm.sum()) + 1e-10)
        k_rot = conf.rot_loss_weight * float(batch["t"][0] > conf.rot_loss_t_threshold) * k_axis
        dax = 2 * (g.abs() / (ga + 1e-6) + q.abs() / (qa + 1e-6))
        proj = torch.where(qa > 0, q.abs() * (dax * q.abs()).sum(-1, keepdim=True) / (qa * (qa + 1e-6) ** 2).clamp(min=1e-300), 0 * q)
        ang = torch.where(qa > 0, 2 * (ga + qa) * q.abs() / qa.clamp(min=1e-300), 0 * q) / float(batch["rot_score_scaling"][0]) ** 2
        s_rs = s_rs + (ang * k_rot + (dax / (qa + 1e-6) + proj) * k_axis) * lm * dm[:, None] * gate1 * nrm_of(batch)
    _within(what + " d_rot_score", dr.v, ref[2], 64 * UD * s_rs, "loss")
    # d_angles = k (w / ne - u <w, u> / (n ne^2)), ne = n + 1e-8: the two terms cancel along u, so S takes them apart,
    # with the rounding of w = 2 (v - target) at 2 (|v| + |target|)
    u = out["angles"][-1].to(rd)
    n = u.norm(dim=-1, keepdim=True)
    ne = n + 1e-8
    v = u / ne
    gt, alt = batch["torsion_angles_sin_cos"][-1].to(rd), batch["alt_torsion_angles_sin_cos"][-1].to(rd)
    tgt = torch.where(((v - gt) ** 2).sum(-1, keepdim=True) <= ((v - alt) ** 2).sum(-1, keepdim=True), gt, alt)
    w = 2 * (v - tgt)
    tm = batch["torsion_angles_mask"][-1].to(rd)
    kf = (tm / (tm.sum() + 1e-2) * conf.torsion_loss_weight * nrm_of(batch))[..., None]
    proj = torch.where(n > 0, u.abs() * (w * u).abs().sum(-1, keepdim=True) / (n * ne * ne).clamp(min=1e-300), torch.zeros_like(u))
    s_ang = kf * ((w.abs() + 2 * (v.abs() + tgt.abs())) / ne + proj)
    _within(what + " d_angles", da.v, ref[1], 64 * UD * s_ang, "loss")
    # d_trans = -2 c (x0 - x): the difference carries ud (|x0| + |x|), i.e. the plus form 2 c (|x0| + |x|)
    x0, x = batch["rigids_0"][-1, :, 4:].to(rd), out["rigids"][-1, :, 4:].to(rd)
    dd = (x0 - x).abs()
    s_x = torch.where(dd > 0, ref[3].abs() * (x0.abs() + x.abs()) / dd.clamp(min=1e-300), torch.zeros_like(dd))
    _within(what + " d_trans", dx.v, ref[3], 64 * UD * s_x, "loss")


@pytest.mark.parametrize("nf", [1, 2, 64, 257])
@pytest.mark.parametrize("N", [1, 255, 256, 257, 1024, 4096])
@pytest.mark.parametrize("separate", [0, 1])
def test_loss_shapes(nf, N, separate):
    if nf * N > 64 * 4096:
        pytest.skip("nf x N up to 64 x 4096")
    _run_loss(f"loss nf={nf} N={N} separate={separate}", nf, N, 7 * nf + N, separate=separate, zero=True)


@pytest.mark.parametrize("separate", [0, 1])
@pytest.mark.parametrize("edge", ["rot_off", "t_at_threshold", "trans_99.9", "trans_100.1", "last_frame_masked", "all_masked"])
def test_loss_edges(separate, edge):
    kw = {"rot_off": dict(rot_on=0), "t_at_threshold": dict(t=0.2), "trans_99.9": dict(trans_mean=99.9),
          "trans_100.1": dict(trans_mean=100.1), "last_frame_masked": dict(mask="last_frame"), "all_masked": dict(mask="all")}[edge]
    _run_loss(f"loss {edge} separate={separate}", 3, 300, 91, separate=separate, zero=True, **kw)


@pytest.mark.parametrize("name", syn.LOSS_EDGES)
def test_loss_kernel_matches_reference_edges(name):
    """The kernel against tests/golden/loss_edges.pt, generated from the unmodified Experiment.loss_fn.  The reference
    normalises the fp32 torsion predictions in fp32, the kernel in fp64: elements agree to a relative 1e-6."""
    gold = _load("loss_edges")[name]
    feats, out, separate = syn.loss_edge(name)
    feats = {k: v.to(DEV) for k, v in feats.items()}
    leaves = {k: out[k].to(DEV).requires_grad_(True) for k in ("angles", "rot_score", "rigids")}
    model_out = dict({k: v.to(DEV) for k, v in out.items()}, **leaves)
    loss, aux = score_network_loss(model_out, feats, O.default_exp_conf(separate_rot_loss=separate))
    grads = torch.autograd.grad(loss, list(leaves.values()))
    assert _elementwise_close(loss.detach().cpu(), gold["loss"], 1e-6, 0.0)
    for k in aux:
        assert _elementwise_close(aux[k].cpu(), gold["aux"][k], 1e-6, 0.0), k
    for k, g in zip(leaves, grads):
        ref = gold["grads"][k]
        ref = torch.zeros_like(g.cpu()) if ref is None else ref
        floor = 1e-6 * max(1.0, float(gold["loss"].abs()))     # the gradients' scale (every frame masked: ~1e10)
        assert _elementwise_close(g.cpu(), ref, 1e-6, floor), (k, (g.cpu().double() - ref.double()).abs().max().item())


# --------------------------------------------------------------------------------------------------
# featurize.cu: featurize_window (one thread per (frame, residue), fp64)
# --------------------------------------------------------------------------------------------------
def _axis_rot(axis, theta):
    a = torch.nn.functional.normalize(torch.as_tensor(axis, dtype=torch.float64), dim=-1)
    K_ = torch.tensor([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]], dtype=torch.float64)
    return torch.eye(3, dtype=torch.float64) + math.sin(theta) * K_ + (1 - math.cos(theta)) * (K_ @ K_)


def _target_rotations(seed):
    """Frames that steer the closed-form quaternion into each of its branches: identity (trace 3), pi about x, y and z
    (the x, y, z branches), pi about (1,1,1)/sqrt 3 (the diagonal ties at trace -1), and angles around 2 pi / 3 (the
    trace crosses 0), about random axes."""
    g = _gen(seed)
    Rs = [torch.eye(3, dtype=torch.float64), _axis_rot([1, 0, 0], math.pi), _axis_rot([0, 1, 0], math.pi), _axis_rot([0, 0, 1], math.pi),
          _axis_rot([1, 1, 1], math.pi)]
    for d in (-1e-3, -1e-6, 0.0, 1e-6, 1e-3):
        Rs.append(_axis_rot(torch.randn(3, generator=g, dtype=torch.float64), 2 * math.pi / 3 + d))
    return torch.stack(Rs)


def _window(nf, N, seed, *, prescribed=False):
    """atom37 [nf,N,37,3] (every frame a small displacement of a random chain; frames taken with stride 2 from a
    trajectory of 2 nf), atom_mask [N,37] with missing O, missing side chains and a few residues missing N or C,
    aatype [N] cycling through all 21 types."""
    g = _gen(seed)
    aatype = torch.arange(N) % 21
    ca = torch.cumsum(torch.nn.functional.normalize(torch.randn(N, 3, generator=g, dtype=torch.float64), dim=-1) * 3.8, 0)
    pos = ca[:, None, :] + torch.randn(N, 37, 3, generator=g, dtype=torch.float64) * 1.4
    if prescribed:
        R = _target_rotations(seed)[torch.arange(N) % 10]
        pos[:, 1] = ca
        pos[:, 2] = ca + 1.52 * R[:, :, 0]                                   # C: e0 = (CA - C) / |.| = -R[:, 0]
        pos[:, 0] = ca + 1.33 * R[:, :, 1] - 0.49 * R[:, :, 0]               # N: Gram-Schmidt leaves e1 = R[:, 1]
    traj = pos[None] + torch.randn(2 * nf, N, 37, 3, generator=g, dtype=torch.float64) * 0.05
    if prescribed:
        traj[:, :, :3] = pos[None, :, :3]
    atom37 = traj[1::2].float().contiguous()
    m = O.residue_tables()["atom37_mask"][aatype].float().clone()
    r = torch.rand(N, generator=g)
    m[r < 0.05, 4] = 0                                                       # missing O
    m[(r >= 0.05) & (r < 0.12), 5:] = 0                                      # missing side chain
    if not prescribed:
        m[(r >= 0.12) & (r < 0.14), 0] = 0                                   # CA without N: a degenerate frame
        m[(r >= 0.14) & (r < 0.16), 2] = 0                                   # CA without C
    return atom37, m, aatype


def _feat_oracle(atom37, m, aatype):
    R0, t, sc, alt, mask = O.featurize_window(atom37.double(), m, aatype)
    return R0, t, sc, alt, mask


@pytest.mark.parametrize("nf,N,prescribed", [(64, 1024, False), (8, 1024, False), (32, 256, False), (2, 1024, False), (1, 1, False),
                                             (3, 1, False), (1, 2, False), (1, 257, False), (4, 257, True), (64, 256, True)])
def test_featurize_window(nf, N, prescribed):
    what = f"featurize nf={nf} N={N} prescribed={prescribed}"
    atom37, m, aatype = _window(nf, N, 17 * nf + N, prescribed=prescribed)
    tabs = [table(k, DEV) for k in ("chi_atom_indices", "chi_angles_mask", "chi_pi_periodic")]
    pos_d = atom37.to(DEV)
    # the mask sits behind a guard of ones: a residue 0 that read "its previous residue" would find finite data there
    m_buf = torch.ones(37 + N * 37, device=DEV)
    m_d = m_buf[37:].view(N, 37)
    m_d.copy_(m)
    aa_d = aatype.to(DEV)
    rig, tor, alt, tm = _twice(what, lambda: [_Out((nf, N, 7)), _Out((nf, N, 7, 2), torch.float64), _Out((nf, N, 7, 2), torch.float64),
                                              _Out((nf, N, 7), torch.float64)],
                               lambda o: K.lib().dfold_featurize_window(K._ptr(pos_d), K._ptr(m_d), K._ptr(aa_d), *[K._ptr(x) for x in tabs],
                                                                        nf, N, *[x.ptr() for x in o], K._stream()))
    R0, t0, rsc, ralt, rmask = _feat_oracle(atom37, m, aatype)
    # conditioning: the spread of the oracle when the coordinates move by a relative eps, over two random directions
    eps = 2.0 ** -30
    spread_R = torch.zeros_like(R0)
    spread_t = torch.zeros_like(rsc)
    for s in range(2):
        r = torch.rand(atom37.shape, generator=_gen(100 + s), dtype=torch.float64) * 2 - 1
        P = _feat_oracle(atom37.double() * (1 + eps * r), m, aatype)
        spread_R = torch.maximum(spread_R, (P[0] - R0).abs())
        spread_t = torch.maximum(spread_t, (P[2] - rsc).abs())
    cond_R, cond_t = spread_R / eps, spread_t / eps
    got = rig.v.cpu()
    q = got[..., :4].double()
    # CA, masked, copied exactly
    assert torch.equal(got[..., 4:], (atom37[:, :, 1] * m[None, :, 1, None])), f"{what}: translation is not the masked CA"
    # the frame: residues with N, CA and C; the fp32 quaternion carries u per component into R (4 roundings of |q|^2 terms)
    # on top of the fp64 computation's ud times the conditioning
    bb = (m[:, 0] * m[:, 1] * m[:, 2] > 0)[None].expand(nf, -1)
    assert torch.isfinite(got).all(), f"{what}: non-finite rigids (degenerate frames must stay finite)"
    # R0 itself is orthogonal only up to the 1e-8 under from_3_points' square roots, which a quaternion cannot follow
    defect = (R0 @ R0.transpose(-1, -2) - torch.eye(3, dtype=R0.dtype)).abs().amax((-1, -2))[..., None, None]
    _within(what + " R0", O.quat_to_rot(q)[bb], R0[bb], (10 * U * _rot_plus(q.abs()) + 2 * defect + 256 * UD * cond_R)[bb],
            "featurize")
    _within(what + " |q|", q.norm(dim=-1)[bb], torch.ones_like(q[..., 0])[bb], (3 * U + 2 * defect[..., 0, 0])[bb], "featurize")
    assert torch.equal(tm.v.cpu(), rmask), f"{what}: torsion mask differs"
    # torsions and alternatives where the mask is 1: fp64 both sides, ~30 roundings deep.  A masked torsion is built from
    # zeroed atoms; its (sin, cos) is rounding noise amplified by the 1e-8 guards, only required finite and <= 1 in size
    on = (rmask > 0)[..., None].expand_as(rsc)
    bound = 256 * UD * cond_t + 32 * UD
    _within(what + " torsions", tor.v.cpu()[on], rsc[on], bound[on], "featurize")
    _within(what + " alt torsions", alt.v.cpu()[on], ralt[on], bound[on], "featurize")
    for o in (tor, alt):
        assert torch.isfinite(o.v).all() and (o.v.abs() <= 1 + 1e-12).all(), f"{what}: masked torsions out of range"
    if nf > 1:
        assert (tm.v.cpu()[1:, 0, :2] == 0).all(), f"{what}: residue 0 of a later frame has a pre-omega / phi"


# --------------------------------------------------------------------------------------------------
# epilogue.cu: score_fwd / score_bwd (K9, one warp per residue: fp32 rotation vector and trigonometry, fp64 series)
# --------------------------------------------------------------------------------------------------
K9 = dict(max_sigma=1.5, min_sigma=0.1, min_b=0.1, max_b=20.0, L=1000)
R3, IPA = 0.1, 0.1                             # the r3 and IPA coordinate scalings, as the kernel receives them (fp32)


def _k9_dc():
    return O.default_diffuser_conf(R3)


def _k9_grid():
    return torch.from_numpy(O._sigma_of_t(np.linspace(0.0, 1.0, 1000), _k9_dc()))


def _igso3_err(omega, sigma, L):
    """First-order bounds on the error the kernel's fp32 trigonometry adds to the IGSO(3) series (igso3.cuh) and to
    g = dS / (S + 1e-4) and g' = dg / domega, for the fp32 angle omega [n] (fp64 values): arg = fl(omega h) carries a
    phase error u |arg|, sinf / cosf and products two u each; the weights and sums are fp64.
    Returns (g, g', e_g, e_g')."""
    l = torch.arange(L, dtype=torch.float64, device=omega.device)
    decay = (2 * l + 1) * torch.exp(-l * (l + 1) * sigma * sigma / 2)
    om, h = omega[:, None], l + 0.5
    arg = om * h
    sh, ch = torch.sin(arg), torch.cos(arg)
    lo, dlo = torch.sin(om / 2), 0.5 * torch.cos(om / 2)
    e_sh = U * (arg.abs() * ch.abs() + 2 * sh.abs())
    e_ch = U * (arg.abs() * sh.abs() + 2 * ch.abs())
    e_lo, e_dlo = 2 * U * lo.abs(), 2 * U * dlo.abs()
    dhi = h * ch
    e_dhi = h * e_ch + U * dhi.abs()
    num = lo * dhi - sh * dlo
    e_num = lo.abs() * e_dhi + dhi.abs() * e_lo + dlo.abs() * e_sh + sh.abs() * e_dlo + 2 * U * ((lo * dhi).abs() + (sh * dlo).abs())
    lo2 = lo * lo
    e_lo2 = 2 * lo.abs() * e_lo + U * lo2
    S = (decay * sh / lo).sum(-1)
    dS = (decay * num / lo2).sum(-1)
    d2S = (decay * (sh * (0.25 - h * h) / lo - 2 * dlo * num / (lo2 * lo))).sum(-1)
    eS = (decay * (e_sh / lo.abs() + sh.abs() * e_lo / lo2)).sum(-1)
    edS = (decay * (e_num / lo2 + num.abs() * e_lo2 / (lo2 * lo2))).sum(-1)
    ed2S = (decay * ((0.25 - h * h).abs() * (e_sh / lo.abs() + sh.abs() * e_lo / lo2)
                     + 2 * (e_dlo * num.abs() + dlo.abs() * e_num) / (lo2 * lo.abs()) + 6 * (dlo * num).abs() * e_lo / (lo2 * lo2))).sum(-1)
    D = S + 1e-4
    # where the series cancels, the errors exceed dS itself: the quadratic terms (edS^2 in dS^2 / D^2) are kept
    aS, adS, ad2S = dS.abs() + edS, d2S.abs() + ed2S, dS.abs()
    e_g = edS / D.abs() + aS * eS / (D * D)
    e_gp = ed2S / D.abs() + adS * eS / (D * D) + (2 * ad2S * edS + edS * edS) / (D * D) + 2 * aS * aS * eS / (D * D * D).abs()
    return dS / D, d2S / D - dS * dS / (D * D), e_g, e_gp


def _k9_rotvec(q_pred, q_t):
    q0_inv = q_pred * q_pred.new_tensor([1.0, -1.0, -1.0, -1.0]) / (q_pred * q_pred).sum(-1, keepdim=True)
    return O.quat_to_rotvec(O.quat_mul(q0_inv, q_t))


def _k9_oracle(q_pred, q_t, t, mask, d_rot):
    """fp64 oracle rot_score [n,3] (masked) and, with d_rot, its gradient w.r.t. q_pred."""
    qp = q_pred.double().clone().requires_grad_(d_rot is not None)
    rs = O.rot_score(q_t.double()[None], qp[None], t, _k9_dc())[0] * mask.double()[:, None]
    if d_rot is None:
        return rs.detach(), None
    (g,) = torch.autograd.grad((rs * d_rot).sum(), [qp])
    return rs.detach(), g


def _k9_case(n, seed):
    g = _gen(seed)
    q_pred = torch.randn(n, 4, generator=g) * 1.2                                    # not unit
    rel = torch.logspace(-3, 0.5, n)[:, None] if n > 1 else torch.ones(1, 1)
    q_t = torch.nn.functional.normalize(q_pred + q_pred.norm(dim=-1, keepdim=True) * torch.randn(n, 4, generator=g) * rel, dim=-1)
    k = min(n, 8)
    q_t[0:k:2] = q_pred[0:k:2]                                                       # q_t = +q_pred exactly
    q_t[1:k:2] = -q_pred[1:k:2]                                                      # q_t = -q_pred exactly
    mask = (torch.rand(n, generator=g) > 0.2).float()
    x_pred, x_t = torch.randn(n, 3, generator=g) * 8, torch.randn(n, 3, generator=g) * 30
    d_rot = torch.randn(n, 3, generator=g, dtype=torch.float64)
    d_trs = torch.randn(n, 3, generator=g, dtype=torch.float64)
    return dict(q_pred=q_pred, q_t=q_t, mask=mask, x_pred=x_pred, x_t=x_t, d_rot=d_rot, d_trs=d_trs)


def _run_score(what, n, t, *, trans_f64, seed, null=None):
    c = _k9_case(n, seed)
    d = {k: v.to(DEV).contiguous() for k, v in c.items()}
    tt = torch.tensor([t], dtype=torch.float64)
    t_d, grid_d = tt.to(DEV), _k9_grid().to(DEV)
    d_trs = d["d_trs"] if trans_f64 else d["d_trs"].float()
    tdt = torch.float64 if trans_f64 else torch.float32
    head = lambda: [K._ptr(d["q_pred"]), K._ptr(d["q_t"]), K._ptr(d["x_pred"]), K._ptr(d["x_t"]), K._ptr(t_d), K._ptr(grid_d),
                    grid_d.numel(), K9["max_sigma"], K9["min_sigma"], K9["min_b"], K9["max_b"], R3, IPA, K._ptr(d["mask"]), K9["L"], n]
    rs, ts = _twice(what + " fwd", lambda: [_Out((n, 3), torch.float64), _Out((n, 3), tdt)],
                    lambda o: K.lib().dfold_score_fwd(*head(), None if null == "rot_score" else o[0].ptr(),
                                                      None if null == "trans_score" else o[1].ptr(), int(trans_f64), K._stream()))
    dq, dx = _twice(what + " bwd", lambda: [_Out((n, 4)), _Out((n, 3))],
                    lambda o: K.lib().dfold_score_bwd(*head(), None if null == "d_rot" else K._ptr(d["d_rot"]),
                                                      None if null == "d_trans" else K._ptr(d_trs), int(trans_f64),
                                                      None if null == "dq_pred" else o[0].ptr(), None if null == "dx_pred" else o[1].ptr(),
                                                      K._stream()))
    rd = _rdev(n)
    with _RefPeak():
        qp, qt, m, dr = c["q_pred"].to(rd), c["q_t"].to(rd), c["mask"].to(rd).double(), c["d_rot"].to(rd)
        t_r = tt.to(rd)
        ref_rs, ref_dq = _k9_oracle(qp, qt, t_r, m, dr)
        # the fp32 rotation vector: the spread of the fp64 oracle when q_pred and q_t move by a relative 4 u
        sp_rs, sp_dq = torch.zeros_like(ref_rs), torch.zeros_like(ref_dq)
        for s in range(3):
            r1 = torch.rand(qp.shape, generator=_gen(300 + s), dtype=torch.float64).to(rd) * 2 - 1
            r2 = torch.rand(qp.shape, generator=_gen(400 + s), dtype=torch.float64).to(rd) * 2 - 1
            p_rs, p_dq = _k9_oracle(qp.double() * (1 + 4 * U * r1), qt.double() * (1 + 4 * U * r2), t_r, m, dr)
            sp_rs, sp_dq = torch.maximum(sp_rs, (p_rs - ref_rs).abs()), torch.maximum(sp_dq, (p_dq - ref_dq).abs())
        # the fp32 series: score = c v, c = g / (omega + 1e-6), omega = |v| + 1e-6
        qpd = qp.double().clone().requires_grad_(True)
        v = _k9_rotvec(qpd, qt.double())
        J = torch.stack([torch.autograd.grad(v[:, i].sum(), [qpd], retain_graph=True)[0] for i in range(3)], 1)   # [n,3,4]
        v = v.detach()
        om = v.norm(dim=-1) + 1e-6
        grid = _k9_grid().numpy()
        sigma = float(grid[np.digitize(O._sigma_of_t(np.array([t]), _k9_dc()), grid) - 1][0])
        g, gp, e_g, e_gp = _igso3_err(om, sigma, K9["L"])
        ome = om + 1e-6
        cc, dcc = g / ome, gp / ome - g / (ome * ome)
        e_c = e_g / ome
        e_dc = e_gp / ome + e_g / (ome * ome)
        # the series estimate is first order (a sum of per-term worst cases, where the terms cancel to e^-100 at small
        # sigma and large omega); it carries a factor 8, of which the worst case measured uses about half
        bound_rs = 4 * sp_rs + (8 * e_c[:, None] * v.abs() + 8 * U * ref_rs.abs()) * m[:, None] + 1e-15
        if null == "rot_score":
            _nan_kept(what + " rot_score", rs)
        else:
            _within(what + " rot_score", rs.v, ref_rs, bound_rs, "score")
        gv = dr * m[:, None]
        vn = v.norm(dim=-1, keepdim=True).clamp(min=1e-300)
        e_dv = e_c[:, None] * gv.abs() + (gv * v).sum(-1, keepdim=True).abs() * e_dc[:, None] * v.abs() / vn
        # d vec = c gv + <gv, v> c' v / |v| goes back through the rotation vector and the quaternion algebra in fp32:
        # 32 u of its plus form on top of the series' error, both mapped by |d vec / d q_pred|
        dv_abs = cc.abs()[:, None] * gv.abs() + (gv * v).abs().sum(-1, keepdim=True) * dcc.abs()[:, None] * v.abs() / vn
        s_dq = torch.einsum("nij,ni->nj", J.abs(), 8 * e_dv + 32 * U * dv_abs)
        if null in ("d_rot", "dq_pred"):
            if null == "d_rot":
                _within(what + " dq_pred", dq.v, torch.zeros_like(ref_dq), torch.zeros_like(ref_dq), "score")
            else:
                _nan_kept(what + " dq_pred", dq)
        else:
            _within(what + " dq_pred", dq.v, ref_dq, 4 * sp_dq + s_dq + 32 * U * ref_dq.abs() + 1e-15, "score")
        # translations: a = fl(x_t r3), b = fl(fl(x_pred fl(1 / ipa)) r3), then fp64
        r3, inv_ipa = float(np.float32(R3)), float(np.float32(1.0) / np.float32(IPA))
        beta = t * K9["min_b"] + 0.5 * t * t * (K9["max_b"] - K9["min_b"])
        E, D = math.exp(-0.5 * beta), 1.0 - math.exp(-beta)
        a, b = c["x_t"].to(rd).double() * r3, c["x_pred"].to(rd).double() * inv_ipa * r3
        ref_ts = -(a - E * b) / D * m[:, None]
        bound_ts = (2 * U * a.abs() + 4 * U * E * b.abs()) / D * m[:, None] + (U * ref_ts.abs() if not trans_f64 else 0.0)
        if null == "trans_score":
            _nan_kept(what + " trans_score", ts)
        else:
            _within(what + " trans_score", ts.v, ref_ts, bound_ts, "score")
        dtr = c["d_trs"].to(rd).double() if trans_f64 else c["d_trs"].to(rd).float().double()
        ref_dx = dtr * m[:, None] * E / D * inv_ipa * r3
        if null in ("d_trans", "dx_pred"):
            if null == "d_trans":
                _within(what + " dx_pred", dx.v, torch.zeros_like(ref_dx), torch.zeros_like(ref_dx), "score")
            else:
                _nan_kept(what + " dx_pred", dx)
        else:
            _within(what + " dx_pred", dx.v, ref_dx, 2 * U * ref_dx.abs(), "score")


@pytest.mark.parametrize("t", [float(x) for x in np.linspace(0.01, 1, 100)] + [1.0])
def test_score_schedule(t):
    """The sampler's schedule np.linspace(0.01, 1, 100), and t = 1; alternate translation dtypes."""
    i = int(round((t - 0.01) / 0.01))
    _run_score(f"score t={t:.4f}", 257, t, trans_f64=bool(i % 2), seed=500 + i)


@pytest.mark.parametrize("n", N_SHAPES)
@pytest.mark.parametrize("t", [0.01, 0.5])
def test_score_shapes(n, t):
    _run_score(f"score n={n} t={t}", n, t, trans_f64=(n % 2 == 0), seed=n)


@pytest.mark.parametrize("null", ["rot_score", "trans_score", "d_rot", "d_trans", "dq_pred", "dx_pred"])
@pytest.mark.parametrize("trans_f64", [False, True])
def test_score_null_operands(null, trans_f64):
    _run_score(f"score null={null} f64={trans_f64}", 257, 0.37, trans_f64=trans_f64, seed=77, null=null)
