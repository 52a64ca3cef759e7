"""Development probe: where do the tensor-core GEMM's producer and consumers wait?  (python tests/devtools/dev_gemm_stats.py)"""
import math, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch
from dynamicpdb_b200 import kernels as K

dev = "cuda"
torch.manual_seed(0)


def run(F, N, Ci, Co, reps=3):
    x = torch.randn(F, N, Ci, device=dev)
    w = torch.randn(Co, Ci, 5, 5, device=dev) / math.sqrt(25 * Ci)
    b = torch.randn(Co, device=dev)
    with torch.no_grad():
        K.conv5x5(x, w, b)
        torch.cuda.synchronize()
        nct = 200000
        stats = torch.zeros(nct, 4, dtype=torch.int64, device=dev)
        K.lib().dfold_debug_gemm_stats(K._ptr(stats))
        K.conv5x5(x, w, b)
        torch.cuda.synchronize()
        K.lib().dfold_debug_gemm_stats(None)
        s = stats[stats[:, 0] > 0].double()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            K.conv5x5(x, w, b)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
    fl = 2.0 * F * N * 25 * Ci * Co
    print(f"conv {F}x{N} {Ci}->{Co}: {ms:.3f} ms  {fl / ms / 1e9:.1f} TFLOP/s fp32-eq  ctas {s.shape[0]}  "
          f"mainloop cyc mean {s[:,0].mean():.0f}  wait_full {100*s[:,1].sum()/s[:,0].sum():.1f}%  "
          f"wait_acc_empty {100*s[:,2].sum()/s[:,0].sum():.1f}%  accwarp_wait {100*s[:,3].sum()/s[:,0].sum():.1f}%")


def run_bwd(F, N, Ci, Co, reps=3):
    x = torch.randn(F, N, Ci, device=dev, requires_grad=True)
    w = (torch.randn(Co, Ci, 5, 5, device=dev) / math.sqrt(25 * Ci)).requires_grad_(True)
    b = torch.randn(Co, device=dev, requires_grad=True)
    y = K.conv5x5(x, w, b)
    g = torch.randn_like(y)
    K.PROFILE = []
    for _ in range(reps + 1):
        torch.autograd.grad(y, [x, w, b], g, retain_graph=True)
    torch.cuda.synchronize()
    prof, K.PROFILE = K.PROFILE, None
    ts = [a.elapsed_time(bb) for (_, _, a, bb, _t) in prof][2:]
    dg, wg = ts[0::2], ts[1::2]
    fl = 2.0 * F * N * 25 * Ci * Co
    print(f"conv bwd {F}x{N} {Ci}->{Co}: dgrad {sum(dg)/len(dg):.3f} ms ({fl/(sum(dg)/len(dg))/1e9:.0f} TF)  "
          f"wgrad {sum(wg)/len(wg):.3f} ms ({fl/(sum(wg)/len(wg))/1e9:.0f} TF)")


run_bwd(64, 256, 1280, 640)
run_bwd(64, 256, 640, 1280)
run_bwd(9, 256, 1280, 640)
run(64, 256, 1280, 640)
run(64, 256, 640, 1280)
run(9, 256, 1280, 640)
run(4, 256, 1280, 640)
