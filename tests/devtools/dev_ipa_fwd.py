"""Development probe: time of the IPA forward core (K.ipa_attention) at the benchmark shape with CUDA events on the launching
stream: the fused kernel + P V GEMM, as a training forward (with probability planes kept for the backward) and as an
inference forward.  python tests/devtools/dev_ipa_fwd.py [F N]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch
from dynamicpdb_b200 import kernels as K

F, N = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (64, 256)
H, C, Pq, Pv, Cp = 8, 256, 8, 12, 32
dev = "cuda"
g = torch.Generator(device=dev).manual_seed(0)
R = lambda *s, scale=1.0: torch.randn(*s, device=dev, generator=g) * scale
logit0, kv = R(1, H, N, N), R(1, N, H, 2 * C)
q_pts, kv_pts = R(F, N, H, Pq, 3, scale=4.0), R(F, N, H, Pq + Pv, 3, scale=4.0)
pair = R(1, N, N, Cp)
quat = torch.nn.functional.normalize(R(F, N, 4), dim=-1)
trans, mask = R(F, N, 3, scale=8.0), torch.ones(F, N, device=dev)
gamma = torch.rand(H, device=dev, generator=g) * 0.2 + 0.05
alg = 4.0 * (F * N * (H * (4 * C + 3 * (2 * Pq + Pv) + 8 * Pv + Cp) + 8) + N * N * (H + Cp))


def run(train):
    q = q_pts.detach().requires_grad_(train)
    with torch.set_grad_enabled(train):
        return K.ipa_attention(logit0, kv, q, kv_pts, pair, quat, trans, mask, gamma, Pq=Pq, Pv=Pv, dfold=True, inf=1e5, eps=1e-8).detach()


outs = {}
for name, train in (("fused train", True), ("fused infer", False)):
    for _ in range(3):
        outs[name] = run(train)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 10
    e0.record()
    for _ in range(n):
        run(train)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    print(f"{name}: {ms:.3f} ms/call  {alg / ms / 1e6:.0f} GB/s algorithmic ({alg / 1e6:.0f} MB)")
