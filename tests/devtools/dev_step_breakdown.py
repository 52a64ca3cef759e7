"""Development probe: per-shape time of the tensor-core GEMM launches of one eager training step."""
import sys, os, collections
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch
from dynamicpdb_b200 import kernels as K, synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
nf, N = 64, 256
torch.manual_seed(0)
net = FullScoreNetwork(syn.model_conf(nf, **syn.PRESET_A), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
sd = net.state_dict(); syn.dezero_(sd); net.load_state_dict(sd); net = net.cuda()
feats = {k: v.cuda() for k, v in syn.make_feats(nf, N, seed=0).items()}
def step():
    net.zero_grad(set_to_none=True)
    syn.surrogate_loss(net(dict(feats))).backward()
for _ in range(2): step()
torch.cuda.synchronize()
K.PROFILE = []
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(); step(); e1.record()
torch.cuda.synchronize()
prof, K.PROFILE = K.PROFILE, None
agg = collections.OrderedDict()
for name, work, a, b, tag in prof:
    d = agg.setdefault((name, tag), [0, 0.0, 0.0]); d[0] += 1; d[1] += a.elapsed_time(b); d[2] += work
tot = sum(v[1] for v in agg.values())
print(f"eager step {e0.elapsed_time(e1):.1f} ms; timed launches {tot:.1f} ms")
for (name, tag), (n, ms, work) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:40]:
    print(f"{ms:8.3f} ms  x{n:3d}  {ms/n:7.3f} ms/launch  {work/ms/1e9 if ms else 0:7.1f} TF  {name} {tag}")
