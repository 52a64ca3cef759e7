"""Development probe: what the moving average of the weights (TrainStep(ema_decay=0.999)) costs at the benchmark shape,
preset A, 64 x 256 (184.4 M parameters), with the GPU's name and power limit.

    python tests/devtools/dev_ema_timing.py [--rounds R] [--steps K] [--launches L]

* the captured step without and with the average, built side by side and timed with CUDA events over K replays each,
  the two alternated R times in one process (median and range);
* dfold_ema_update alone over the 184.4 M-element buffers, with CUDA events over L back-to-back launches (it reads the
  average and the weights and writes the average: 12 B per element)."""
import argparse
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
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    feats = {k: v.cuda() for k, v in syn.make_feats(NF, N, seed=0).items()}
    steps = {"no ema": TrainStep(_net(), syn.surrogate_loss, feats, lr=1e-4, graph=True, warmup=2),
             "ema 0.999": TrainStep(_net(), syn.surrogate_loss, feats, lr=1e-4, graph=True, warmup=2, ema_decay=0.999)}
    for name, ts in steps.items():
        assert ts.graph is not None, (name, ts.graph_error)
        ts()                                                    # warm replay
    times = {name: [] for name in steps}
    names = list(steps)
    for r in range(args.rounds):
        for name in names[r % 2:] + names[:r % 2]:              # each configuration takes each position in turn
            times[name].append(_events_ms(steps[name], args.steps))
    for name in names:
        t = times[name]
        print(f"[{gpu}] step, {name}: {statistics.median(t):.2f} ms median ({min(t):.2f}-{max(t):.2f}) of {args.rounds} "
              f"runs of {args.steps} replays")
    print(f"[{gpu}] difference of the medians: {statistics.median(times['ema 0.999']) - statistics.median(times['no ema']):+.2f} ms")

    ts = steps["ema 0.999"]
    n = ts.ema.numel()
    ms = _events_ms(lambda: K.launch("dfold_ema_update", ts.ema, ts.flat_param, n, ts.ema_factor), args.launches)
    print(f"[{gpu}] dfold_ema_update over {n / 1e6:.1f} M elements: {ms * 1e3:.1f} us per call, "
          f"{12 * n / (ms * 1e-3) / 1e12:.2f} TB/s at 12 B per element ({args.launches} launches)")


if __name__ == "__main__":
    main()
