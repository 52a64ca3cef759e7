"""Time the evaluation-metric kernels (csrc/metrics.cu) and the host path the reference takes for the same numbers.

    python tests/devtools/dev_eval_metrics.py

Device: window_metrics (eval_fn's row: rigid errors, atom errors, last-frame superposition) and validation_metrics_all
(rmsd_all, rmsd_ca, drmsd_ca, per-frame CA superposition), each timed with CUDA events after warm-up, median of 20.
Host: the reference's route -- copy prot_traj[0] / rigid_pred to the host, synchronise, then the same arithmetic in numpy
and torch-CPU (oracle/metrics_oracle.py, the fp64 restatement; the reference's Bio superposition is an SVD per set too),
median of 5 wall-clock runs.  Prints the card and its power limit with the numbers."""
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from dynamicpdb_b200 import metrics as M  # noqa: E402
from oracle import metrics_cases as C  # noqa: E402
from oracle import metrics_oracle as MO  # noqa: E402

SHAPES = [(5, 256), (32, 256), (64, 256), (8, 1024), (3, 130)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def device_ms(fn, reps=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def host_ms(fn, reps=5):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    assert torch.cuda.is_available(), "dev_eval_metrics needs a CUDA device"
    print(f"[card] {card()}  torch threads {torch.get_num_threads()}")
    for nf, N in SHAPES:
        g_r, p_r = C.rigids(nf, N, 3)
        g_a, p_a, m = C.atoms(nf, N, 4, "loader")
        d = {k: v.cuda() for k, v in dict(g_r=g_r, p_r=p_r, g_a=g_a, p_a=p_a, m=m).items()}
        win = lambda: M.window_metrics(d["p_r"], d["p_a"], d["g_r"], d["g_a"], d["m"])
        val = lambda: M.validation_metrics_all(d["g_a"], d["p_a"], d["m"])
        both = lambda: (win(), val())
        t_win, t_val, t_both = device_ms(win), device_ms(val), device_ms(both)

        def host_path():
            pr, pa = d["p_r"].cpu(), d["p_a"].cpu()        # the D2H copies (synchronising)
            gr, ga, mm = d["g_r"].cpu(), d["g_a"].cpu(), d["m"].cpu()
            MO.window_metrics(pr, pa, gr, ga, mm)
            MO.validation_metrics_all(ga, pa, mm)
        t_host = host_ms(host_path)
        mb = (p_a.numel() * 4 + g_a.numel() * 8 + m.numel() * 8) / 1e6
        print(f"[metrics] {nf} x {N}: window_metrics {t_win:.3f} ms, validation_metrics_all {t_val:.3f} ms, both {t_both:.3f} ms "
              f"(device); host path (copy out + fp64 numpy/torch-CPU) {t_host:.1f} ms; atom37 inputs {mb:.1f} MB")


if __name__ == "__main__":
    main()
