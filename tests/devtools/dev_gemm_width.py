"""Development probe: every convolution GEMM of one preset-A training step (64 frames x 256 residues; forward, data
gradient and weight gradient of the full and the cropped layers) timed at tile widths 64 and 128.

    python tests/devtools/dev_gemm_width.py [--out FILE.json]

Each GEMM is launched alone through the explicit-width entry points, warmed up, then timed with CUDA events in rounds
that alternate the two widths, at least ~100 ms per width; the per-launch time is the median over the rounds.  Besides
ms, fp32-equivalent TFLOP/s and tiles, it prints the cost of one tile per k-block, ms / (waves x k-blocks), and that
cost at width 64 relative to width 128: the TILE_COST ratio kernels._conv_bn weighs the waves with.  The card's name,
power limit and the median SM clock over the timed rounds come from the same run."""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import threading

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch

from dynamicpdb_b200 import kernels as K
from tests.test_gpu_gemm_width import ConvGemm, step_conv_gemms

DEV = "cuda"


def cdiv(a, b):
    return -(-a // b)


class SmClock:
    """Samples the SM clock with nvidia-smi every 200 ms while it runs."""

    def __init__(self, index):
        self.mhz = []
        self.proc = subprocess.Popen(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i",
                                      str(index), "-lms", "200"], stdout=subprocess.PIPE, text=True)
        threading.Thread(target=self._read, daemon=True).start()

    def _read(self):
        for line in self.proc.stdout:
            if line.strip().isdigit():
                self.mhz.append(int(line))

    def stop(self):
        self.proc.terminate()
        self.proc.wait()
        return statistics.median(self.mhz) if self.mhz else None


def time_widths(g, target_ms=25.0, rounds=4):
    """Median ms per launch of `g` at each width over `rounds` alternating batches of >= target_ms each."""
    out = torch.empty(g.out_numel, device=DEV)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def batch(bn, reps):
        e0.record()
        for _ in range(reps):
            g.launch(out, bn)
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / reps

    first = max(batch(bn, 3) for bn in (64, 128))          # warm-up, and the batch size
    reps = max(3, math.ceil(target_ms / first))
    ms = {64: [], 128: []}
    for r in range(rounds):
        for bn in ((64, 128) if r % 2 == 0 else (128, 64)):
            ms[bn].append(batch(bn, reps))
    return {bn: statistics.median(v) for bn, v in ms.items()}, reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the table as JSON here")
    args = ap.parse_args()
    idx = torch.cuda.current_device()
    sms = torch.cuda.get_device_properties(idx).multi_processor_count
    name, plimit = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i",
                                   str(idx)], capture_output=True, text=True).stdout.strip().split(", ")
    rows = []
    clock = SmClock(idx)
    try:
        for i, case in enumerate(step_conv_gemms()):
            g = ConvGemm(*case, n=256, seed=i)
            ms, reps = time_widths(g)
            # per step: a full layer runs 4 times in each of blocks 0 and 3, a cropped one once in each of blocks 1 and 2
            row = dict(name=g.name, kind=g.kind, per_step=8 if case[4] == 0 else 2, num_kb=g.num_kb, reps=reps,
                       tflop=g.flop / 1e12)
            for bn in (64, 128):
                tiles = g.tiles(bn)
                waves = cdiv(tiles, sms)
                row[bn] = dict(ms=ms[bn], tflops=g.flop / ms[bn] / 1e9, tiles=tiles, waves=waves,
                               us_per_wave_kb=1e3 * ms[bn] / (waves * g.num_kb))
            row["cost64"] = row[64]["us_per_wave_kb"] / row[128]["us_per_wave_kb"]
            row["pick_bn"] = 64 if g.n_out > 64 and row[64]["waves"] * 64 < row[128]["waves"] * 128 else 128
            row["model_bn"] = K._conv_bn(g.n_out, g.row_tiles, DEV)
            rows.append(row)
            del g
            torch.cuda.empty_cache()
    finally:
        mhz = clock.stop()

    print(f"{name}, power limit {plimit} W, {sms} SMs, median SM clock {mhz} MHz over the timed rounds")
    print(f"{'GEMM':34s} {'kb':>4s} | {'BN=64 ms':>9s} {'TF/s':>6s} {'tiles':>5s} {'wv':>3s} {'us/wv-kb':>8s} | "
          f"{'BN=128 ms':>9s} {'TF/s':>6s} {'tiles':>5s} {'wv':>3s} {'us/wv-kb':>8s} | {'c64/c128':>8s} pick model")
    for r in rows:
        a, b = r[64], r[128]
        print(f"{r['name']:34s} {r['num_kb']:4d} | {a['ms']:9.3f} {a['tflops']:6.1f} {a['tiles']:5d} {a['waves']:3d} "
              f"{a['us_per_wave_kb']:8.3f} | {b['ms']:9.3f} {b['tflops']:6.1f} {b['tiles']:5d} {b['waves']:3d} "
              f"{b['us_per_wave_kb']:8.3f} | {r['cost64']:8.3f} {r['pick_bn']:4d} {r['model_bn']:5d}")
    for kind in ("fwd", "dgrad", "wgrad"):
        c = [r["cost64"] for r in rows if r["kind"] == kind]
        print(f"{kind}: cost of a 64-wide tile per k-block relative to a 128-wide one, median {statistics.median(c):.3f} "
              f"(range {min(c):.3f}-{max(c):.3f})")
    step = {"pick_bn": sum(r["per_step"] * r[r["pick_bn"]]["ms"] for r in rows),
            "model": sum(r["per_step"] * r[r["model_bn"]]["ms"] for r in rows),
            "best": sum(r["per_step"] * min(r[64]["ms"], r[128]["ms"]) for r in rows)}
    print("convolution GEMMs of one step, each launched alone: " + ", ".join(f"{k} {v:.2f} ms" for k, v in step.items()))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=name, power_limit_w=float(plimit), sms=sms, sm_mhz_median=mhz, rows=rows, step_ms=step),
                      f, indent=1)


if __name__ == "__main__":
    main()
