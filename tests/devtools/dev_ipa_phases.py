"""Development probe: time of the fused IPA forward with individual phases disabled (DFOLD_IPA_DEBUG_SKIP bit mask:
1 pass 1, 2 distances of pass 2, 4 pair aggregation, 8 value points).  Results are wrong by design."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch
from dynamicpdb_b200 import kernels as K
F, N = 64, 256
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
def run(train):
    q = q_pts.detach().requires_grad_(train)
    with torch.set_grad_enabled(train):
        return K.ipa_attention(logit0, kv, q, kv_pts, pair, quat, trans, mask, gamma, Pq=Pq, Pv=Pv, dfold=True, inf=1e5, eps=1e-8).detach()
for train in (True, False):
    for skip in (0, 1, 2, 3, 4, 8, 12, 16, 15, 31):
        os.environ["DFOLD_IPA_DEBUG_SKIP"] = str(skip)
        for _ in range(2): run(train)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10): run(train)
        e1.record(); torch.cuda.synchronize()
        print(f"train={train} skip={skip:2d}: {e0.elapsed_time(e1) / 10:.3f} ms")

# per-CTA cycle counters (dfold_debug_ipa_stats)
os.environ["DFOLD_IPA_DEBUG_SKIP"] = "0"
ncta = (N // 32) * F
buf = torch.zeros(ncta, 16, dtype=torch.int64, device=dev)
K.lib().dfold_debug_ipa_stats(K._ptr(buf))
run(True); torch.cuda.synchronize()
K.lib().dfold_debug_ipa_stats(None)
m = buf.double().mean(0).tolist()
names = ["ctl total", "ctl wait full", "ctl wait P ready", "ctl wait empty(+issue)", "cmp total", "pass 1", "phase A", "B1", "B2", "barriers", "epilogue"]
for n_, v in zip(names, m): print(f"{n_:24s} {v:12.0f} cycles  ({v / 1.9e3:8.1f} us @1.9 GHz)")
