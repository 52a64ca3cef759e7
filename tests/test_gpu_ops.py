"""-m gpu: every CUDA operator (through the C-ABI) against the plain-torch oracle, forward and backward.

The oracle side runs in float64 on the CPU so the reported error is the CUDA kernel's own error.  Tolerances are
relative to the largest reference magnitude of each tensor:
  * fp32 CUDA-core kernels: 2e-5
  * split-bf16 (x3) tensor-core GEMM / convolution: 1e-4 (hi/lo split keeps ~16 mantissa bits per operand)
"""
import math

import pytest
import torch

from dynamicpdb_b200 import kernels as K
from oracle import ops as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _run(fn, inputs, kwargs, dtype, device, wmask=None):
    xs = []
    for t in inputs:
        if isinstance(t, torch.Tensor) and t.is_floating_point():
            x = t.detach().to(device=device, dtype=dtype).requires_grad_(t.requires_grad)
        elif isinstance(t, torch.Tensor):
            x = t.to(device)
        else:
            x = t
        xs.append(x)
    kw = {}
    for k, v in kwargs.items():
        if isinstance(v, torch.Tensor) and v.is_floating_point():
            v = v.detach().to(device=device, dtype=dtype)
        elif isinstance(v, torch.Tensor):
            v = v.to(device)
        kw[k] = v
    out = fn(*xs, **kw)
    outs = out if isinstance(out, (tuple, list)) else (out,)
    g = torch.Generator().manual_seed(7)
    loss = 0
    for o in outs:
        w = torch.randn(o.shape, generator=g)
        if wmask is not None:
            w = w * wmask.reshape(o.shape)
        w = w.to(device=device, dtype=o.dtype)
        loss = loss + (o * w).sum()
    leaves = [x for x in xs if isinstance(x, torch.Tensor) and x.requires_grad]
    grads = torch.autograd.grad(loss, leaves, allow_unused=True) if leaves else []
    return [o.detach().double().cpu() for o in outs], [None if gr is None else gr.detach().double().cpu() for gr in grads]


def _rel_err(a, b):
    """max |a-b| / max|a| over EVERY element (no outlier allowance)."""
    return (a - b).abs().max().item() / (a.abs().max().item() + 1e-30)


def _safe_gate(pre, tau=1e-3):
    """Output positions whose ReLU pre-activation (fp64 oracle) is further than tau * max|pre| from zero.  The
    upstream gradient of BOTH sides is zeroed elsewhere, so oracle and kernel see the same ReLU gate by construction:
    a pre-activation within rounding of zero may gate differently in fp64 and in the kernel, and that is a property
    of the comparison, not of the kernel.  Every element of every gradient is then compared, none is discarded."""
    pre = pre.detach().double()
    return (pre.abs() > tau * pre.abs().max()).to(torch.float64)


def check(name, inputs, tol, post=None, wmask=None, grad_tol=None, **kwargs):
    fo = getattr(O, name) if post is None else (lambda *a, **k: post(getattr(O, name)(*a, **k), *a))
    fk = getattr(K, name) if post is None else (lambda *a, **k: post(getattr(K, name)(*a, **k), *a))
    ro, rg = _run(fo, inputs, kwargs, torch.float64, "cpu", wmask)
    co, cg = _run(fk, inputs, kwargs, torch.float32, DEV, wmask)
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(ro, co)):
        assert a.shape == b.shape, f"{name} out{i} shape {a.shape} vs {b.shape}"
        err = _rel_err(a, b)
        assert err < tol, f"{name} out{i}: rel err {err:.3e} >= {tol}"
    for i, (a, b) in enumerate(zip(rg, cg)):
        assert (a is None) == (b is None), f"{name} grad{i} presence"
        if a is None:
            continue
        assert a.shape == b.shape, f"{name} grad{i} shape {a.shape} vs {b.shape}"
        err = _rel_err(a, b)
        gt = (grad_tol or {}).get(i, tol)
        assert err < gt, f"{name} grad{i}: rel err {err:.3e} >= {gt}"


def R(*s, grad=True, scale=1.0, seed=None):
    g = torch.Generator().manual_seed(seed if seed is not None else (hash(s) % 1000))
    return (torch.randn(*s, generator=g) * scale).requires_grad_(grad)


def unit(*s, grad=True):
    q = R(*s, grad=False)
    return (q / q.norm(dim=-1, keepdim=True)).requires_grad_(grad)


def test_library_loads():
    assert K.lib().dfold_abi_version() == 3


@pytest.mark.parametrize("M,Kd,N", [(5, 3, 16), (70, 14, 32), (33, 7, 6), (256, 160, 6), (100, 128, 8), (4096, 7, 6), (3000, 14, 32)])
@pytest.mark.parametrize("act,pre_relu,res", [(None, False, False), ("relu", False, False), (None, True, True), ("silu", False, False)])
def test_linear_simt(M, Kd, N, act, pre_relu, res):
    inputs = [R(M, Kd), R(N, Kd, scale=0.3), R(N)]
    check("linear", inputs, 2e-5, act=act, pre_relu=pre_relu, residual=R(M, N) if res else None)


@pytest.mark.parametrize("M,Kd,N", [(128, 64, 64), (256, 256, 2048), (300, 1280, 640), (130, 3072, 256), (4096, 128, 32), (512, 160, 80)])
@pytest.mark.parametrize("act,pre_relu,res", [(None, False, False), ("relu", False, True), (None, True, True)])
def test_linear_tensor_core(M, Kd, N, act, pre_relu, res):
    inputs = [R(M, Kd), R(N, Kd, scale=1.0 / math.sqrt(Kd)), R(N)]
    wmask = None
    if act == "relu":
        with torch.no_grad():
            wmask = _safe_gate(O.linear(*[t.double() for t in inputs], act=None, pre_relu=pre_relu))
    check("linear", inputs, 1e-4, wmask=wmask, act=act, pre_relu=pre_relu, residual=R(M, N) if res else None)


@pytest.mark.parametrize("F,N,Ci,Co", [(2, 16, 160, 80), (3, 12, 80, 160), (5, 130, 64, 128), (8, 256, 320, 256), (1, 40, 256, 640)])
@pytest.mark.parametrize("relu,res", [(True, False), (True, True), (False, False)])
def test_conv5x5(F, N, Ci, Co, relu, res):
    inputs = [R(F, N, Ci), R(Co, Ci, 5, 5, scale=1.0 / math.sqrt(25 * Ci)), R(Co)]
    residual = R(F, N, Co) if res else None
    wmask = None
    if relu:
        with torch.no_grad():
            wmask = _safe_gate(O.conv5x5(*[t.double() for t in inputs], relu=False))
    check("conv5x5", inputs, 1e-4, wmask=wmask, relu=relu, residual=residual)


@pytest.mark.parametrize("shape", [(3, 12, 32), (8, 256, 256), (1, 7, 5)])
@pytest.mark.parametrize("silu", [False, True])
def test_global_layernorm(shape, silu):
    check("global_layernorm", [R(*shape, scale=3.0) + 0.7], 2e-5, eps=1e-4, silu=silu)


def test_row_layernorm():
    check("layer_norm", [R(37, 96), R(96), R(96)], 2e-5, eps=1e-5)


def test_quat_to_rot():
    check("quat_to_rot", [R(4, 33, 4)], 2e-5)     # deliberately non-unit


@pytest.mark.parametrize("inverse", [False, True])
def test_rigid_apply(inverse):
    q, t = R(3, 20, 1, 4), R(3, 20, 1, 3, scale=10.0)
    check("rigid_apply", [q, t, R(3, 20, 17, 3, scale=5.0)], 2e-5, inverse=inverse)
    check("rigid_apply", [R(6, 4), R(6, 3), R(6, 3)], 2e-5, inverse=inverse)


@pytest.mark.parametrize("Fs", [1, 3])
def test_ipa_points(Fs):
    check("ipa_points", [R(Fs, 20, 3 * 4 * 5), unit(3, 20, 4), R(3, 20, 3, scale=10.0), 4], 2e-5)


@pytest.mark.parametrize("masked", [False, True])
def test_compose_q_update(masked):
    m = None
    if masked:
        m = (torch.rand(3, 20, 1) > 0.3).float()
    check("compose_q_update", [unit(3, 20, 4), R(3, 20, 3, scale=10.0), R(3, 20, 6, scale=0.3), m], 2e-5)


@pytest.mark.parametrize("Fs,Fz", [(1, 1), (2, 1), (2, 2)])
def test_qk_logits(Fs, Fz):
    N, H, C = 24, 3, 16
    b = R(Fz, N, N, H).permute(0, 3, 1, 2)       # head-major view, as the module produces it
    check("qk_logits", [R(Fs, N, H, C), R(Fs, N, H, 2 * C), b.detach().requires_grad_(True), 0.25, 0.577], 2e-5)


def _ipa_inputs(F, N, H, C, Pq, Pv, Cp, Fs, Fz, masked):
    mask = torch.ones(F, N)
    if masked:
        mask[:, -3:] = 0
        mask[0, 1] = 0
    return [R(max(Fs, Fz), H, N, N), R(Fs, N, H, 2 * C), R(F, N, H, Pq, 3, scale=4.0), R(F, N, H, Pq + Pv, 3, scale=4.0),
            R(Fz, N, N, Cp), unit(F, N, 4), R(F, N, 3, scale=8.0), mask, (torch.rand(H) * 0.2 + 0.05).requires_grad_(True)]


@pytest.mark.parametrize("F,N,H,C,Pq,Pv,Cp,Fs,Fz,dfold", [
    (3, 12, 2, 8, 2, 3, 4, 1, 1, True),        # tiny preset
    (2, 20, 12, 16, 4, 8, 32, 1, 1, True),     # preset B
    (2, 40, 8, 256, 8, 12, 32, 1, 1, True),    # preset A geometry (tensor-core decomposition)
    (3, 256, 8, 256, 8, 12, 32, 1, 1, True),   # preset A, N = 256
    (1, 32, 8, 256, 8, 12, 32, 1, 1, True),    # fused kernel, exactly one key tile
    (2, 24, 8, 256, 8, 12, 32, 1, 1, True),    # fused kernel, one partial key tile
    (2, 136, 4, 64, 4, 6, 16, 1, 1, False),    # tensor-core path, vanilla layout, N not a multiple of 64
    (2, 33, 4, 16, 4, 8, 64, 2, 2, False),     # vanilla OpenFold, batched z and per-frame s
    (3, 70, 2, 8, 2, 3, 4, 3, 1, True),        # per-frame s, shared z, N not a multiple of the tiles
])
@pytest.mark.parametrize("masked", [False, True])
def test_ipa_attention(F, N, H, C, Pq, Pv, Cp, Fs, Fz, dfold, masked):
    inputs = _ipa_inputs(F, N, H, C, Pq, Pv, Cp, Fs, Fz, masked)
    # rows of masked QUERY residues see every logit shifted by -1e5: in fp32 (reference and kernel alike) that
    # quantises the logits to 2^-7, so those rows are compared only through the unmasked ones
    post = lambda out, *a: out * a[7][:, :, None]
    # d(gamma) [H] (gradient 7: the mask carries none) is a signed sum over all F*N*N pairs of a head whose terms are orders
    # of magnitude larger than the sum: the fp32 rounding of the logits alone moves it by ~2e-4 relative, run to run with the
    # atomic accumulation order, and the split-bf16 value-point term of dS (2^-17 per product) by up to ~7e-4
    check("ipa_attention", inputs, 2e-4, post=post, grad_tol={7: 1.5e-3}, Pq=Pq, Pv=Pv, dfold=dfold, inf=1e5, eps=1e-8)


@pytest.mark.parametrize("F,N,Ci,Co,crop", [(7, 24, 64, 128, 2), (17, 40, 160, 80, 2), (5, 130, 128, 64, 4)])
@pytest.mark.parametrize("relu,res", [(True, True), (False, False)])
def test_conv5x5_cropped(F, N, Ci, Co, crop, relu, res):
    """Only the last F - crop output frames (dead-frame pyramid): forward, data gradient and weight gradient."""
    inputs = [R(F, N, Ci), R(Co, Ci, 5, 5, scale=1.0 / math.sqrt(25 * Ci)), R(Co)]
    residual = R(F - crop, N, Co) if res else None
    wmask = None
    if relu:
        with torch.no_grad():
            wmask = _safe_gate(O.conv5x5(*[t.double() for t in inputs], relu=False, crop=crop))
    check("conv5x5", inputs, 1e-4, wmask=wmask, relu=relu, residual=residual, crop=crop)


# --------------------------------------------------------------------------------------------------
# epilogue kernels (csrc/epilogue.cu): K9 score epilogue, K10 frames -> atoms, quaternion / rotation-matrix algebra
# --------------------------------------------------------------------------------------------------
def _grid():
    import numpy as np
    g = np.log(np.linspace(0.0, 1.0, 1000) * np.exp(1.5) + (1 - np.linspace(0.0, 1.0, 1000)) * np.exp(0.1))
    return torch.from_numpy(g)


@pytest.mark.parametrize("tval,tdtype", [(0.03, torch.float64), (0.5, torch.float64), (1.0, torch.float32), (0.2, torch.float32)])
def test_score_epilogue(tval, tdtype):
    """K9 against the oracle in the reference's own arithmetic (fp32 trigonometry, fp64 series): rot_score fp64 at 1e-4
    per residue (the north-star bar), gradients of both scores w.r.t. the predicted frame."""
    F, N = 3, 70
    gen = torch.Generator().manual_seed(5)
    q_pred = torch.randn(F, N, 4, generator=gen) * 1.2           # non-unit on purpose
    # noised rotation at relative angles from ~0.03 rad to pi.  (Below that the reference formula itself is numerically
    # ill-conditioned in its own fp32 arithmetic — lo*dhi - hi*dlo cancels to (h*omega)^2 of its terms, so3_diffuser.py:
    # 107-113 — and two correct fp32 evaluations differ by O(1); test_score_epilogue_small_angles covers that range.)
    q_t = torch.nn.functional.normalize(q_pred + q_pred.norm(dim=-1, keepdim=True) * torch.randn(F, N, 4, generator=gen)
                                        * torch.logspace(-1.5, 0.5, N)[None, :, None], dim=-1)
    x_pred, x_t = torch.randn(F, N, 3, generator=gen) * 8, torch.randn(F, N, 3, generator=gen)
    mask = (torch.rand(F, N, generator=gen) > 0.2).float()
    t = torch.tensor([tval], dtype=tdtype)
    kw = dict(max_sigma=1.5, min_sigma=0.1, min_b=0.1, max_b=20.0, r3_scale=0.1, ipa_scale=2.0, L=1000)
    w_r = torch.randn(F, N, 3, generator=gen, dtype=torch.float64)
    w_t = torch.randn(F, N, 3, generator=gen, dtype=torch.float64)

    def run(fn, dev):
        qp = q_pred.to(dev).requires_grad_(True)
        xp = x_pred.to(dev).requires_grad_(True)
        rs, ts = fn(qp, q_t.to(dev), xp, x_t.to(dev), t.to(dev), _grid().to(dev), mask.to(dev), **kw)
        loss = (rs * w_r.to(dev)).sum() + (ts.double() * w_t.to(dev)).sum()
        gq, gx = torch.autograd.grad(loss, [qp, xp])
        return rs.detach().cpu(), ts.detach().cpu(), gq.cpu(), gx.cpu()

    # Where is the reference's own arithmetic (fp32 trigonometry + fp64 series, so3_diffuser.py:71-117) well conditioned?
    # At small sigma(t) and large relative angle the series cancels catastrophically (at t = 0.03 the fp32 reference is off
    # the fp64 value by O(1) for omega > 1 rad, where the IGSO(3) density is ~e^-100 and no sample ever lands): residues
    # whose fp32 reference value deviates from its own fp64 evaluation are not compared (their loss weights are zeroed).
    with torch.no_grad():
        r32, _ = O.score_epilogue(q_pred, q_t, None, None, t, _grid(), None, **kw)
        r64, _ = O.score_epilogue(q_pred.double(), q_t.double(), None, None, t, _grid(), None, **kw)
    stable = ((r32 - r64).norm(dim=-1) / r64.norm(dim=-1).clamp(min=1.0)) < 1e-5
    assert stable.float().mean().item() > 0.4, "test data: too few well-conditioned residues"
    w_r = w_r * stable[..., None]
    ro, to_, gqo, gxo = run(O.score_epilogue, "cpu")
    rk, tk, gqk, gxk = run(K.score_epilogue, DEV)
    assert rk.dtype == torch.float64 and tk.dtype == to_.dtype
    err = (((ro - rk).norm(dim=-1) / ro.norm(dim=-1).clamp(min=1.0)) * stable).max().item()
    assert err < 1e-4, f"rot_score per-residue relative L2 {err:.3e}"
    assert _rel_err(to_.double(), tk.double()) < 2e-6
    assert _rel_err(gxo.double(), gxk.double()) < 2e-6
    assert _rel_err(gqo.double(), gqk.double()) < 2e-4, _rel_err(gqo.double(), gqk.double())
    # rotation score alone (the diffuser API, calc_rot_score)
    r2, none = K.score_epilogue(q_pred.to(DEV), q_t.to(DEV), None, None, t.to(DEV), _grid().to(DEV), None, **kw)
    assert none is None and ((r2.cpu() * mask[..., None] - rk) * stable[..., None]).abs().max().item() < 1e-12 * max(1.0, rk.abs().max().item())


def test_score_epilogue_small_angles():
    """Rotation angles down to 1e-6 rad (incl. the small-angle branch of quat_to_rotvec and omega -> eps): finite values
    and gradients, zero where masked."""
    n = 64
    gen = torch.Generator().manual_seed(6)
    q = torch.nn.functional.normalize(torch.randn(1, n, 4, generator=gen), dim=-1)
    q_t = torch.nn.functional.normalize(q + torch.randn(1, n, 4, generator=gen) * torch.logspace(-7, -2, n)[None, :, None], dim=-1)
    q_t[0, 0] = q[0, 0]                                        # exactly equal rotations
    qp = q.to(DEV).requires_grad_(True)
    mask = torch.ones(1, n)
    mask[0, 5] = 0
    kw = dict(max_sigma=1.5, min_sigma=0.1, min_b=0.1, max_b=20.0, r3_scale=1.0, ipa_scale=1.0, L=1000)
    rs, _ = K.score_epilogue(qp, q_t.to(DEV), None, None, torch.tensor([0.5]).to(DEV), _grid().to(DEV), mask.to(DEV), **kw)
    (g,) = torch.autograd.grad(rs.sum(), [qp])
    assert torch.isfinite(rs).all() and torch.isfinite(g).all()
    assert float(rs[0, 5].abs().max()) == 0.0 and float(g[0, 5].abs().max()) == 0.0


@pytest.mark.parametrize("is_mat,want_frames", [(False, False), (True, True), (False, True)])
def test_frames_to_atoms(is_mat, want_frames):
    from dynamicpdb_b200 import feats as FT
    from dynamicpdb_b200 import rigid_utils as ru
    F, N = 2, 45
    gen = torch.Generator().manual_seed(9)
    quat = torch.randn(F, N, 4, generator=gen)
    quat = quat / quat.norm(dim=-1, keepdim=True) * (1.0 + 0.05 * torch.randn(F, N, 1, generator=gen))    # slightly non-unit
    trans = torch.randn(F, N, 3, generator=gen) * 10
    alpha = torch.nn.functional.normalize(torch.randn(F, N, 7, 2, generator=gen), dim=-1) * 1.1
    aatype = torch.randint(0, 21, (F, N), generator=gen)
    rot = O.quat_to_rot(quat) if is_mat else quat
    gws = None

    def run(dev, product):
        nonlocal gws
        r_ = rot.to(dev).requires_grad_(True)
        t_ = trans.to(dev).requires_grad_(True)
        a_ = alpha.to(dev).requires_grad_(True)
        if product:
            rots = ru.Rotation(rot_mats=r_) if is_mat else ru.Rotation(quats=r_, normalize_quats=False)
            outs = FT.frames_to_atoms(ru.Rigid(rots, t_), a_, aatype.to(dev), want_frames=want_frames)
        else:
            outs = O.frames_to_atoms(r_.double(), t_.double(), a_.double(), aatype, None, None, want_frames, is_mat)
        if gws is None:
            gws = [torch.randn(o.shape, generator=gen, dtype=torch.float64) for o in outs]
        loss = sum((o.double() * w.to(dev)).sum() for o, w in zip(outs, gws))
        grads = torch.autograd.grad(loss, [r_, t_, a_])
        return [o.detach().double().cpu() for o in outs], [g.double().cpu() for g in grads]

    oo, og = run("cpu", False)
    ko, kg = run(DEV, True)
    for a, b in zip(oo, ko):
        assert a.shape == b.shape and _rel_err(a, b) < 2e-6
    for a, b in zip(og, kg):
        assert _rel_err(a, b) < 2e-5


@pytest.mark.parametrize("b_is_vec", [False, True])
def test_quat_mul(b_is_vec):
    check("quat_mul", [R(3, 20, 4), R(3, 20, 3 if b_is_vec else 4)], 2e-6, b_is_vec=b_is_vec)
    check("quat_mul", [R(1, 20, 4), R(3, 1, 3 if b_is_vec else 4)], 2e-6, b_is_vec=b_is_vec)      # broadcast both ways


@pytest.mark.parametrize("inverse", [False, True])
def test_rot_compose(inverse):
    first = lambda out, *a: out[0]
    second = lambda out, *a: out[1]
    # rotation product, frame composition, point application with a trailing broadcast (r[..., None].apply(pts))
    check("rot_compose", [R(3, 20, 3, 3), None, R(3, 20, 3, 3), None], 2e-6, post=first)
    if not inverse:
        check("rot_compose", [R(3, 20, 3, 3), R(3, 20, 3), R(3, 20, 3, 3), R(3, 20, 3)], 2e-6)
        check("rot_compose", [R(3, 20, 1, 3, 3), R(3, 20, 1, 3), R(3, 20, 8, 3, 3), R(3, 20, 8, 3)], 2e-6)
    check("rot_compose", [R(3, 20, 1, 3, 3), R(3, 20, 1, 3), None, R(3, 20, 17, 3)], 2e-6, post=second, inverse=inverse)
    check("rot_compose", [R(20, 3, 3), None, None, R(3, 20, 3)], 2e-6, post=second, inverse=inverse)        # leading broadcast
