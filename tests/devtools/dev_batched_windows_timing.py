"""Development probe: what TrainStep(batched=True) gains over accumulate=k, with the GPU's name and power limit.

    python tests/devtools/dev_batched_windows_timing.py [--rounds R] [--steps K] [--nf 2 5] [--k 1 2 4 8 16] [--out DIR]

For each frame count nf (preset A, 256 residues) and each k, a captured step with accumulate=k and one with
accumulate=k, batched=True are built and timed side by side: R rounds, in each round both replay K steps between two
CUDA events, the order alternating from round to round.  Reported: ms per optimizer step (median and range), frames/s
(k * nf frames per step) and the peak memory of building and running each step.  At k = 8 (nf = 2) one eager batched step
runs under torch.profiler, and the kernel time is split between the ConvNet (the split-bf16 GEMM launches of
conv5x5), the IPA kernels and the rest; the trace is written under --out when given."""
import argparse
import gc
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

from dynamicpdb_b200 import synthetic as syn  # noqa: E402
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork  # noqa: E402
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser  # noqa: E402
from dynamicpdb_b200.train_step import TrainStep  # noqa: E402

N = 256


def _net(nf):
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(nf, **syn.PRESET_A), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    return net.cuda()


def _events_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _build(nf, k, batched, windows):
    """The step and the peak memory (GB) that building it and running one replay add to what was allocated before (the
    other configuration's step stays resident while this one is built)."""
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ts = TrainStep(_net(nf), syn.surrogate_loss, windows[0], lr=1e-4, graph=True, warmup=2, accumulate=k, batched=batched)
    assert ts.graph is not None, ts.graph_error
    for i in range(k):
        ts.load(windows[i], slot=i)
    ts()
    torch.cuda.synchronize()
    return ts, (torch.cuda.max_memory_allocated() - base) / 2 ** 30


def _split(nf, k, windows, out_dir):
    """Kernel time of one eager batched step: the total and the IPA kernels (names containing "ipa") from torch.profiler,
    and the ConvNet's GEMMs (the 25-tap launches) from kernels.PROFILE's per-launch events in a second step."""
    from dynamicpdb_b200 import kernels as K
    from torch.profiler import ProfilerActivity, profile
    ts = TrainStep(_net(nf), syn.surrogate_loss, windows[0], lr=1e-4, graph=False, warmup=1, accumulate=k, batched=True)
    for i in range(k):
        ts.load(windows[i], slot=i)
    ts()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ts()
        torch.cuda.synchronize()
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(out_dir, f"batched_nf{nf}_k{k}.pt.trace.json"))
    total = ipa = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
        total += t
        if "ipa" in e.key.lower():
            ipa += t
    K.PROFILE = []
    try:
        ts()
        torch.cuda.synchronize()
        conv = sum(e0.elapsed_time(e1) for _, _, e0, e1, tag in K.PROFILE if "taps25" in tag) * 1000.0
    finally:
        K.PROFILE = None
    return {"ConvNet GEMMs": conv, "IPA kernels": ipa}, total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--nf", type=int, nargs="+", default=[2, 5])
    ap.add_argument("--k", type=int, nargs="+", default=[1, 2, 4, 8, 16])
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-split", action="store_true", help="skip the profiled step")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    print(f"[{gpu}] preset A, {N} residues, {args.rounds} rounds x {args.steps} replays")
    for nf in args.nf:
        for k in args.k:
            windows = [{kk: v.cuda() for kk, v in syn.make_feats(nf, N, seed=i, t=0.1 + 0.05 * i).items()} for i in range(k)]
            steps, peak = {}, {}
            for name, batched in (("accumulate", False), ("batched", True)):
                try:
                    steps[name], peak[name] = _build(nf, k, batched, windows)
                except torch.cuda.OutOfMemoryError:
                    print(f"[{gpu}] nf={nf} k={k} {name}: out of memory")
            times = {n: [] for n in steps}
            names = list(steps)
            for r in range(args.rounds):
                for n in (names if r % 2 == 0 else names[::-1]):
                    times[n].append(_events_ms(steps[n], args.steps))
            for n in names:
                ms = statistics.median(times[n])
                print(f"[{gpu}] nf={nf} k={k} {n:10s}: {ms:8.2f} ms/step (range {min(times[n]):.2f} ... "
                      f"{max(times[n]):.2f}), {1000.0 * k * nf / ms:7.1f} frames/s, peak +{peak[n]:.2f} GB", flush=True)
            del steps
            gc.collect()
            torch.cuda.empty_cache()
    if 2 in args.nf and 8 in args.k and not args.no_split:
        windows = [{kk: v.cuda() for kk, v in syn.make_feats(2, N, seed=i).items()} for i in range(8)]
        fam, total = _split(2, 8, windows, args.out)
        parts = ", ".join(f"{n} {t / 1000:.2f} ms ({100 * t / total:.0f} %)" for n, t in fam.items())
        print(f"[{gpu}] nf=2 k=8 batched eager step, kernel time {total / 1000:.2f} ms: {parts}")


if __name__ == "__main__":
    main()
