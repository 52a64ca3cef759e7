"""The float64 IPA intermediates of oracle/ipa_reference.py, which tests/test_gpu_ipa_kernels.py holds the kernels to,
pinned against autograd of oracle/ops.py::ipa_attention at small shapes, for both concat layouts, masked and not.

Every quantity is tied to the oracle by an identity that does not restate the reference's own algebra:
  * cat, and the gradients w.r.t. q_pts, the key points, quat, trans and gamma, equal the oracle's;
  * dS equals the oracle's gradient w.r.t. a per-frame logit0 (logit0 enters the logits with weight one);
  * P = exp(s - lse) sums to one per row, and contracted with v, the value points and z gives the oracle's o, og and
    o_pair columns; d2 equals |q_p(i) - k_p(j)|^2 summed from the inputs;
  * d_og contracted with P over the query rows is the oracle's gradient w.r.t. the value points, and d_og . og,
    dO . o and dO_pair . o_pair per row equal the P-weighted row sums of dPog, dPv and dPz, whose total is delta.
"""
import pytest
import torch

from oracle import ops as OO
from oracle.ipa_reference import ipa_reference

INF, EPS = 1e5, float(torch.tensor(1e-8, dtype=torch.float32))


def _inputs(F, N, H, C, Pq, Pv, Cp, Fs, Fz, masked, seed=0):
    g = torch.Generator().manual_seed(seed)
    R = lambda *s, scale=1.0: torch.randn(*s, generator=g, dtype=torch.float64) * scale
    mask = torch.ones(F, N, dtype=torch.float64)
    if masked:
        mask[:, -2:] = 0
        mask[0, 1] = 0
    quat = torch.nn.functional.normalize(R(F, N, 4), dim=-1)
    return dict(logit0=R(F, H, N, N), kv=R(Fs, N, H, 2 * C), q_pts=R(F, N, H, Pq, 3, scale=2.0),
                kv_pts=R(F, N, H, Pq + Pv, 3, scale=2.0), pair=R(Fz, N, N, Cp), quat=quat, trans=R(F, N, 3, scale=3.0),
                mask=mask, gamma=torch.rand(H, generator=g, dtype=torch.float64) * 0.2 + 0.05)


def _close(a, b, what):
    a, b = a.double(), b.double()
    err = (a - b).abs().max().item()
    assert err <= 1e-10 * max(1.0, b.abs().max().item()), f"{what}: max |err| {err:.3e}"


CASES = [(2, 9, 2, 4, 2, 3, 4, 1, 1), (3, 7, 3, 8, 4, 2, 8, 3, 1), (2, 5, 2, 4, 3, 2, 4, 2, 2)]


@pytest.mark.parametrize("F,N,H,C,Pq,Pv,Cp,Fs,Fz", CASES)
@pytest.mark.parametrize("dfold", [0, 1])
@pytest.mark.parametrize("masked", [False, True])
def test_ipa_reference_matches_oracle(F, N, H, C, Pq, Pv, Cp, Fs, Fz, dfold, masked):
    x = _inputs(F, N, H, C, Pq, Pv, Cp, Fs, Fz, masked)
    kw = dict(Pq=Pq, Pv=Pv, dfold=dfold, inf=INF, eps=EPS)
    leaves = {k: v.clone().requires_grad_(k != "mask") for k, v in x.items()}
    cat = OO.ipa_attention(*leaves.values(), **kw)
    dcat = torch.randn(cat.shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    names = [k for k in leaves if k != "mask"]
    grads = dict(zip(names, torch.autograd.grad((cat * dcat).sum(), [leaves[k] for k in names])))
    # the block size forces several row blocks per frame
    r = ipa_reference(*x.values(), dcat, block_bytes=N * H * Pq * 3 * 8 * 6 * 3, **kw)

    _close(r["cat"], cat, "cat")
    _close(r["dS"], grads["logit0"].reshape(F, H, N, N), "dS")
    _close(r["dq_pts"], grads["q_pts"], "dq_pts")
    _close(r["dk_pts"], grads["kv_pts"][..., :Pq, :], "dk_pts")
    _close(r["dquat"], grads["quat"], "dquat")
    _close(r["dtrans"], grads["trans"], "dtrans")
    _close(r["dgamma"], grads["gamma"], "dgamma")

    P, s = r["P"], r["s"]
    _close(torch.exp(s - r["lse"][..., None]), P, "P = exp(s - lse)")
    _close(P.sum(-1), torch.ones(F, H, N, dtype=torch.float64), "row sums of P")
    d = x["q_pts"][:, :, None] - x["kv_pts"][:, None, :, :, :Pq]
    _close(r["d2"], (d * d).sum((-1, -2)).permute(0, 3, 1, 2), "d2")
    v = x["kv"][..., C:].expand(F, -1, -1, -1)
    vp = x["kv_pts"][..., Pq:, :]
    z = x["pair"].expand(F, -1, -1, -1)
    o = torch.einsum("fhij,fjhc->fihc", P, v)
    og = torch.einsum("fhij,fjhpx->fihpx", P, vp)
    o_pair = torch.einsum("fhij,fijc->fihc", P, z)
    HPv = H * Pv
    off_pair = H * C + 4 * HPv
    _close(o.reshape(F, N, H * C), cat[..., :H * C], "o = P v")
    _close(o_pair.reshape(F, N, H * Cp), cat[..., off_pair:off_pair + H * Cp], "o_pair = P z")
    if dfold:
        off_g = off_pair + H * Cp
        _close(og.reshape(F, N, HPv, 3).permute(0, 1, 3, 2).reshape(F, N, 3 * HPv), cat[..., off_g:off_g + 3 * HPv], "og = P v_pts")
    _close(torch.einsum("fhij,fihpx->fjhpx", P, r["d_og"]), grads["kv_pts"][..., Pq:, :], "P^T d_og")
    do = dcat[..., :H * C].reshape(F, N, H, C)
    dop = dcat[..., off_pair:off_pair + H * Cp].reshape(F, N, H, Cp)
    _close((P * r["dPv"]).sum(-1), (do * o).sum(-1).permute(0, 2, 1), "sum_j P dPv = dO . o")
    _close((P * r["dPz"]).sum(-1), (dop * o_pair).sum(-1).permute(0, 2, 1), "sum_j P dPz = dO_pair . o_pair")
    _close((P * r["dPog"]).sum(-1), (r["d_og"] * og).sum((-1, -2)).permute(0, 2, 1), "sum_j P dPog = d_og . og")
    _close(r["delta"], (P * (r["dPv"] + r["dPog"] + r["dPz"])).sum(-1), "delta")
