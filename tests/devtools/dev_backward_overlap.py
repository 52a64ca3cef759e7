"""Development probe: where the backward's time goes with the convolution weight gradients on a side stream, at the
benchmark shape (preset A, 64 x 256), with the GPU's name and power limit.

    python tests/devtools/dev_backward_overlap.py OUT_DIR [--reps R]

For the single-stream backward (kernels.PROFILE set: every launch on the current stream) and the overlapped one:
* the backward's wall time (loss.backward() through the side-stream join), CUDA events, median and range over R eager
  steps, and the peak memory allocated during one eager step;
* under torch.profiler (CPU and CUDA activities, one more step; the trace goes to
  OUT_DIR/backward_<mode>.pt.trace.json): the summed kernel time of the backward per stream, and how much of each
  stream's kernel time ran while a kernel of another stream was running."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from dynamicpdb_b200 import kernels as K, synthetic as syn  # noqa: E402
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork  # noqa: E402
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser  # noqa: E402
from dynamicpdb_b200.train_step import TrainStep  # noqa: E402

NF, N = 64, 256


def _step(ts):
    """One eager training step as TrainStep._eager takes it; returns the (start, end) CUDA events around the backward."""
    ts.flat_grad.zero_()
    loss = ts.loss_fn(ts.net(dict(ts.static)))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    K.GRAD_ACCUMULATE_INPLACE = True
    try:
        loss.backward()
    finally:
        K.GRAD_ACCUMULATE_INPLACE = False
        if hasattr(K, "join_side_stream"):
            K.join_side_stream()
    e1.record()
    ts.optimizer_step()
    if K.PROFILE is not None:
        K.PROFILE.clear()
    return e0, e1


def _kernel_stats(trace_path):
    """Per stream, the kernels launched inside the backward's annotation window (by any host thread: autograd launches
    from its device thread): their summed time, and how much of it ran while a kernel of another stream was running."""
    ev = json.load(open(trace_path))["traceEvents"]
    win = [e for e in ev if e.get("name") == "backward_window" and e.get("cat") == "user_annotation"][0]
    lo, hi = win["ts"], win["ts"] + win["dur"]
    corr = {e["args"].get("correlation") for e in ev if e.get("cat") in ("cuda_runtime", "cuda_driver")
            and lo <= e["ts"] <= hi}
    kern = [e for e in ev if e.get("cat") == "kernel" and e["args"].get("correlation") in corr]
    by = {}
    for e in kern:
        by.setdefault(e["args"]["stream"], []).append((e["ts"], e["ts"] + e["dur"]))
    out = {}
    for s, iv in by.items():
        others = sorted(x for t, v in by.items() if t != s for x in v)
        merged = []
        for a, b in others:
            if merged and a <= merged[-1][1]:
                merged[-1][1] = max(merged[-1][1], b)
            else:
                merged.append([a, b])
        busy = sum(b - a for a, b in iv)
        over = 0.0
        for a, b in iv:
            for c, d in merged:
                if c >= b:
                    break
                over += max(0.0, min(b, d) - max(a, c))
        out[str(s)] = {"kernels": len(iv), "kernel_ms": busy / 1e3, "overlapped_ms": over / 1e3,
                       "span_ms": (max(b for _, b in iv) - min(a for a, _ in iv)) / 1e3}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(NF, **syn.PRESET_A), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    net = net.cuda()
    feats = {k: v.cuda() for k, v in syn.make_feats(NF, N, seed=0).items()}
    ts = TrainStep(net, syn.surrogate_loss, feats, lr=1e-4, graph=False, warmup=1)
    report = {"gpu": gpu, "shape": f"preset A {NF} x {N}"}
    for mode in ("single_stream", "overlapped"):
        K.PROFILE = [] if mode == "single_stream" else None
        _step(ts)
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.reps):
            e0, e1 = _step(ts)
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        _step(ts)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        path = os.path.join(args.out, f"backward_{mode}.pt.trace.json")
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            ts.flat_grad.zero_()
            loss = ts.loss_fn(ts.net(dict(ts.static)))
            with torch.profiler.record_function("backward_window"):
                K.GRAD_ACCUMULATE_INPLACE = True
                loss.backward()
                K.GRAD_ACCUMULATE_INPLACE = False
                if hasattr(K, "join_side_stream"):
                    K.join_side_stream()
            ts.optimizer_step()
            torch.cuda.synchronize()
        prof.export_chrome_trace(path)
        if K.PROFILE is not None:
            K.PROFILE.clear()
        report[mode] = {"backward_ms_median": statistics.median(ms), "backward_ms_range": [min(ms), max(ms)],
                        "step_peak_allocated_GB": peak / 2 ** 30, "streams": _kernel_stats(path)}
        print(json.dumps({mode: report[mode]}), flush=True)
    K.PROFILE = None
    with open(os.path.join(args.out, "backward_overlap.json"), "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps(report))


if __name__ == "__main__":
    main()
