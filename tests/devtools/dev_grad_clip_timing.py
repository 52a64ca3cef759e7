"""Development probe: what global-norm gradient clipping (TrainStep(max_grad_norm=...)) costs at the benchmark shape,
preset A, 64 x 256 (184.4 M parameters), with the GPU's name and power limit.

    python tests/devtools/dev_grad_clip_timing.py [--rounds R] [--steps K] [--launches L]

* the captured step with max_grad_norm None, inf (the norm only) and 0.1 x the unclipped norm (clipping active), timed
  with CUDA events over K replays each, the three alternated R times in one process;
* dfold_grad_norm alone over the 184.4 M-element gradient, and dfold_adam_amsgrad against dfold_adam_amsgrad_clip, with
  CUDA events over L back-to-back launches each (the norm reads 738 MB once; both Adam variants move 36 B per element)."""
import argparse
import math
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

from dynamicpdb_b200 import kernels as K, synthetic as syn  # noqa: E402
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork  # noqa: E402
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser  # noqa: E402
from dynamicpdb_b200.train_step import TrainStep  # noqa: E402

NF, N = 64, 256


def _net():
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(NF, **syn.PRESET_A), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    return net.cuda()


def _events_ms(fn, reps):
    """Mean ms per call of fn over reps back-to-back calls, between two CUDA events on the current stream."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    feats = {k: v.cuda() for k, v in syn.make_feats(NF, N, seed=0).items()}

    steps = {"None": TrainStep(_net(), syn.surrogate_loss, feats, lr=1e-4, graph=True, warmup=2)}
    steps["None"]()
    torch.cuda.synchronize()
    norm = steps["None"].flat_grad.double().norm().item()
    steps["inf"] = TrainStep(_net(), syn.surrogate_loss, feats, lr=1e-4, graph=True, warmup=2, max_grad_norm=math.inf)
    steps["0.1 x norm"] = TrainStep(_net(), syn.surrogate_loss, feats, lr=1e-4, graph=True, warmup=2,
                                    max_grad_norm=0.1 * norm)
    for name, ts in steps.items():
        assert ts.graph is not None, (name, ts.graph_error)
        ts()                                                    # warm replay
    times = {name: [] for name in steps}
    names = list(steps)
    for r in range(args.rounds):
        for name in names[r % 3:] + names[:r % 3]:              # each configuration takes each position in turn
            times[name].append(_events_ms(steps[name], args.steps))
    for name, ts in steps.items():
        extra = "" if ts.grad_norm is None else f", grad_norm {float(ts.grad_norm):.4e}"
        print(f"[{gpu}] step, max_grad_norm {name}: {statistics.median(times[name]):.2f} ms median of "
              f"{', '.join(f'{t:.2f}' for t in times[name])} ms ({args.steps} replays each){extra}")
    print(f"[{gpu}] unclipped norm after one step {norm:.4e}")

    ts = steps["0.1 x norm"]
    n = ts.flat_grad.numel()
    grad = torch.randn(n, device="cuda")
    ws = torch.empty(1024, dtype=torch.float64, device="cuda")
    total, coef = torch.empty((), device="cuda"), torch.empty((), device="cuda")
    ms = _events_ms(lambda: K.launch("dfold_grad_norm", grad, n, 1.0, 1.0, ws, total, coef), args.launches)
    print(f"[{gpu}] dfold_grad_norm over {n / 1e6:.1f} M elements: {ms * 1e3:.1f} us per call, "
          f"{4 * n / (ms * 1e-3) / 1e12:.2f} TB/s of gradient read ({args.launches} launches)")
    bufs = [torch.zeros(n, device="cuda") for _ in range(4)]
    step = torch.zeros((), device="cuda")
    adam = lambda: K.launch("dfold_adam_amsgrad", bufs[0], grad, *bufs[1:], n, step, 1, 1e-4, 0.9, 0.999, 1e-8, 1.0)
    adam_clip = lambda: K.launch("dfold_adam_amsgrad_clip", bufs[0], grad, *bufs[1:], n, step, 1, 1e-4, 0.9, 0.999, 1e-8, 1.0,
                                 coef)
    for name, fn in (("dfold_adam_amsgrad", adam), ("dfold_adam_amsgrad_clip", adam_clip)) * 2:
        ms = _events_ms(fn, args.launches // 4)
        print(f"[{gpu}] {name}: {ms * 1e3:.1f} us per call, {36 * n / (ms * 1e-3) / 1e12:.2f} TB/s at 36 B per element")


if __name__ == "__main__":
    main()
