"""Float64 statement of the IPA attention core's intermediates, for the tests of the kernels behind
dynamicpdb_b200.kernels.ipa_attention (csrc/ipa_attn.cu, csrc/ipa_fused.cu, csrc/ipa_v2.cu).

ipa_reference() restates the forward of oracle/ops.py::ipa_attention and takes every backward quantity from torch
autograd of <dcat, cat>, never from a hand-derived formula.  It runs frame by frame and in blocks of query rows (every
softmax row is independent), so its memory is bounded by `block_bytes` whatever F and N are; frame-shared logit0 / kv /
pair come with a leading 1, as the kernels take them.  Returned (float64, on the inputs' device):
  s      [F,H,N,N]    logits  logit0 - gamma/2 sum_p |q_p(i) - k_p(j)|^2 + inf (mask_i mask_j - 1)
  d2     [F,H,N,N]    sum_p |q_p(i) - k_p(j)|^2
  lse    [F,H,N]      log sum_j exp(s)
  P      [F,H,N,N]    softmax(s)
  cat    [F,N,D]      the concat buffer, the feature order of oracle/ops.py
  dS     [F,H,N,N]    d<dcat,cat>/ds (retain_grad on the logits)
  dPv, dPog, dPz      [F,H,N,N]  d<dcat,cat>/dP through the value, value-point and pair aggregations, one each
  delta  [F,H,N]      sum_j P (dPv + dPog + dPz)
  d_og   [F,N,H,Pv,3] d<dcat,cat>/d(og), og the aggregated value points in the global frame
  dq_pts [F,N,H,Pq,3], dk_pts [F,N,H,Pq,3], dquat [F,N,4], dtrans [F,N,3], dgamma [H]
"""
import torch

from . import dfold_oracle as O


def ipa_reference(logit0, kv, q_pts, kv_pts, pair, quat, trans, mask, gamma, dcat, *, Pq, Pv, dfold, inf, eps,
                  block_bytes=1 << 30):
    dd = lambda t: t.detach().double()
    F, N, H = q_pts.shape[:3]
    C = kv.shape[-1] // 2
    Cp = pair.shape[-1]
    dev = q_pts.device
    new = lambda *s: torch.empty(s, dtype=torch.float64, device=dev)
    r = {k: new(F, H, N, N) for k in ("s", "d2", "P", "dS", "dPv", "dPog", "dPz")}
    r.update(lse=new(F, H, N), delta=new(F, H, N), cat=new(F, N, dcat.shape[-1]), d_og=new(F, N, H, Pv, 3),
             dq_pts=new(F, N, H, Pq, 3), dk_pts=new(F, N, H, Pq, 3), dquat=new(F, N, 4), dtrans=new(F, N, 3))
    gam = dd(gamma).requires_grad_(True)
    # the [rows, N, H, Pq, 3] differences, their squares and their gradients dominate a block's memory
    nb = max(1, int(block_bytes // (N * H * Pq * 3 * 8 * 6)))
    for f in range(F):
        pick = lambda t: t[f if t.shape[0] > 1 else 0]
        l0, kvf, z = dd(pick(logit0)), dd(pick(kv)), dd(pick(pair))
        v = kvf[..., C:]
        kp = dd(kv_pts[f, :, :, :Pq]).requires_grad_(True)
        vp = dd(kv_pts[f, :, :, Pq:])
        m = dd(mask[f])
        for a in range(0, N, nb):
            b = min(N, a + nb)
            n = b - a
            q = dd(q_pts[f, a:b]).requires_grad_(True)
            qt = dd(quat[f, a:b]).requires_grad_(True)
            tt = dd(trans[f, a:b]).requires_grad_(True)
            d = q[:, None] - kp[None]                                        # [n,N,H,Pq,3]
            d2 = (d * d).sum(-1).sum(-1).permute(2, 0, 1)                    # [H,n,N]
            s = l0[:, a:b] - 0.5 * gam[:, None, None] * d2 + inf * (m[a:b, None] * m[None, :] - 1)
            s.retain_grad()
            P = torch.softmax(s, dim=-1)
            pv, pg, pz = P.clone(), P.clone(), P.clone()
            for t in (pv, pg, pz):
                t.retain_grad()
            o = torch.einsum("hij,jhc->ihc", pv, v).reshape(n, H * C)
            og = torch.einsum("hij,jhpx->ihpx", pg, vp)                      # [n,H,Pv,3]
            og.retain_grad()
            rig = torch.cat([qt, tt], dim=-1)
            ol = O.rigid_invert_apply(rig[:, None, None, :], og)
            nl = torch.sqrt((ol ** 2).sum(-1) + eps).reshape(n, H * Pv)
            ng = torch.sqrt((og ** 2).sum(-1) + eps).reshape(n, H * Pv)
            olr, ogr = ol.reshape(n, H * Pv, 3), og.reshape(n, H * Pv, 3)
            o_pair = torch.einsum("hij,ijc->ihc", pz, z[a:b]).reshape(n, H * Cp)
            feats = [o, olr[..., 0], olr[..., 1], olr[..., 2], nl, o_pair]
            if dfold:
                feats += [ogr[..., 0], ogr[..., 1], ogr[..., 2], ng]
            cat = torch.cat(feats, dim=-1)
            (cat * dd(dcat[f, a:b])).sum().backward()
            with torch.no_grad():
                r["s"][f, :, a:b], r["d2"][f, :, a:b], r["P"][f, :, a:b] = s, d2, P
                r["lse"][f, :, a:b] = torch.logsumexp(s, dim=-1)
                r["dS"][f, :, a:b] = s.grad
                r["dPv"][f, :, a:b], r["dPog"][f, :, a:b], r["dPz"][f, :, a:b] = pv.grad, pg.grad, pz.grad
                r["delta"][f, :, a:b] = (P * (pv.grad + pg.grad + pz.grad)).sum(-1)
                r["cat"][f, a:b] = cat
                r["d_og"][f, a:b] = og.grad
                r["dq_pts"][f, a:b], r["dquat"][f, a:b], r["dtrans"][f, a:b] = q.grad, qt.grad, tt.grad
            del d, d2, s, P, pv, pg, pz, o, og, ol, cat
        r["dk_pts"][f] = kp.grad
    r["dgamma"] = gam.grad
    return r
