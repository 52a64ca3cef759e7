"""Development probe: what the training-recipe options of TrainStep cost, with the GPU's name and power limit.

    python tests/devtools/dev_train_recipe_timing.py [--rounds R] [--steps K]

* the captured step at preset A, 64 x 256 (the benchmark shape), without and with lr_schedule=AlphaFoldSchedule() (one
  extra single-thread launch per step, and Adam reads its lr from device memory), and with a schedule whose lr is the
  unscheduled 1e-4 from the second step on;
* one step with accumulate=4 against four single-window steps (accumulate=1) at preset A, frame_time=2 x 256 (the windows
  of the released recipe, run_train.sh: 4 ranks x 1 window).

Each configuration is built once and all are timed side by side: R rounds, in each round every configuration replays K
steps between two CUDA events, and the order of the configurations rotates from round to round.  The accumulate=4 step
is timed per replay and the single-window one per 4 replays, so both numbers cover 4 windows."""
import argparse
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

from dynamicpdb_b200 import synthetic as syn  # noqa: E402
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork  # noqa: E402
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser  # noqa: E402
from dynamicpdb_b200.train_step import AlphaFoldSchedule, TrainStep  # noqa: E402

N = 256


def _net(nf):
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(nf, **syn.PRESET_A), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    return net.cuda()


def _events_ms(fn, reps):
    """ms of reps back-to-back calls of fn, between two CUDA events on the current stream."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def _timed(configs, rounds, steps):
    """{name: [ms per step of each round]} for configs {name: (fn, calls per step)}, order rotated every round."""
    names = list(configs)
    times = {n: [] for n in names}
    for r in range(rounds):
        for n in names[r % len(names):] + names[:r % len(names)]:
            fn, calls = configs[n]
            times[n].append(_events_ms(fn, steps * calls) / steps)
    return times


def _report(gpu, times, what):
    for n, ts in times.items():
        print(f"[{gpu}] {what}, {n}: {statistics.median(ts):.2f} ms median, range {min(ts):.2f} ... {max(ts):.2f} ms "
              f"over {len(ts)} rounds")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]

    feats = {k: v.cuda() for k, v in syn.make_feats(64, N, seed=0).items()}
    steps = {"no schedule": TrainStep(_net(64), syn.surrogate_loss, feats, lr=1e-4, graph=True, warmup=2),
             "AlphaFoldSchedule()": TrainStep(_net(64), syn.surrogate_loss, feats, lr=1e-4, graph=True, warmup=2,
                                              lr_schedule=AlphaFoldSchedule()),
             # the schedule's launches with the unscheduled run's lr from step 2 on: separates their cost from that of
             # the different weights a different lr leads to
             "plateau schedule (lr 0, then 1e-4)": TrainStep(
                 _net(64), syn.surrogate_loss, feats, lr=1e-4, graph=True, warmup=2,
                 lr_schedule=AlphaFoldSchedule(max_lr=1e-4, warmup_no_steps=1, start_decay_after_n_steps=10 ** 9))}
    for name, ts in steps.items():
        assert ts.graph is not None, (name, ts.graph_error)
        ts()
    _report(gpu, _timed({n: (ts, 1) for n, ts in steps.items()}, args.rounds, args.steps), "preset A 64 x 256 step")
    print(f"[{gpu}] lr after {args.rounds * args.steps + 1} scheduled steps: {float(steps['AlphaFoldSchedule()'].current_lr):.6e}")
    del steps, ts, feats
    torch.cuda.empty_cache()

    windows = [{k: v.cuda() for k, v in syn.make_feats(2, N, seed=i).items()} for i in range(4)]
    single = TrainStep(_net(2), syn.surrogate_loss, windows[0], lr=1e-4, graph=True, warmup=2)
    acc = TrainStep(_net(2), syn.surrogate_loss, windows[0], lr=1e-4, graph=True, warmup=2, accumulate=4)
    assert single.graph is not None and acc.graph is not None, (single.graph_error, acc.graph_error)
    for i, w in enumerate(windows):
        acc.load(w, slot=i)
    acc()
    single()
    times = _timed({"accumulate=4, one step": (acc, 1), "accumulate=1, four steps": (single, 4)}, args.rounds, args.steps)
    _report(gpu, times, "preset A frame_time=2 x 256, 4 windows")


if __name__ == "__main__":
    main()
