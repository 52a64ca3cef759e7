"""Development probe: device time of the forward diffusion (csrc/diffuse.cu) with CUDA events after warm-up — the IGSO(3)
table build, forward_marginal at 64 x 256 and 8 x 1024 (t = 0.01 / 0.37 / 1.0: small sigma keeps the most series terms),
sample_ref at 64 x 256, and one prefetched window (slice + copy + featurise + noise) — plus the card and its power limit."""
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
import torch
from dynamicpdb_b200 import kernels as K, synthetic as syn
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser

REPS = 20


def timed(fn, reps=REPS):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)), float(np.min(ts))


def main():
    dev = torch.device("cuda", 0)
    name = torch.cuda.get_device_name(dev)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    print(f"device: {name}; power limit, max SM clock: {q}")
    d = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    grid = d.grid(dev)
    med, mn = timed(lambda: K.igso3_tables(grid, d.num_omega, d.L), reps=5)
    print(f"igso3 tables 1000 sigma x 1000 omega (L = 1000): median {med:.3f} ms, min {mn:.3f} ms")
    d.tables(dev)
    for nf, N in ((64, 256), (8, 1024)):
        rig7 = syn.make_feats(nf, N, seed=1)["rigids_0"].to(dev)
        for t in (0.01, 0.37, 1.0):
            tt = torch.tensor([t], dtype=torch.float64, device=dev)
            med, mn = timed(lambda: d.forward_marginal(rig7, tt))
            print(f"forward_marginal {nf} x {N} t={t}: median {med:.3f} ms, min {mn:.3f} ms (draws from the device generator included)")
            n = nf * N
            draws = {"z_axis": torch.randn(n, 3, dtype=torch.float64, device=dev), "u": torch.rand(n, dtype=torch.float64, device=dev),
                     "z_trans": torch.randn(n, 3, dtype=torch.float64, device=dev)}
            med, mn = timed(lambda: d.forward_marginal(rig7, tt, draws=draws))
            print(f"forward_marginal {nf} x {N} t={t}, injected draws: median {med:.3f} ms, min {mn:.3f} ms")
    med, mn = timed(lambda: d.sample_ref(64 * 256, frame_time=64, device=dev))
    print(f"sample_ref 64 x 256: median {med:.3f} ms, min {mn:.3f} ms")

    from oracle import synth_traj
    from dynamicpdb_b200.input_pipeline import TrajectoryStore, WindowPrefetcher
    with tempfile.TemporaryDirectory() as tmp:
        row = synth_traj.write_files(synth_traj.make_trajectory(T=64, N=256), tmp)
        for diffuser in (None, d):
            store = TrajectoryStore(frame_time=64, frame_sample_step=1)
            pf = WindowPrefetcher(store, [row], dev, training=True, diffuser=diffuser)
            pf._make(row)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ts = []
            for _ in range(REPS):
                e0.record(pf.stream)
                _, ev = pf._make(row)
                e1.record(pf.stream)
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            tag = "featurise + noise" if diffuser is not None else "featurise only"
            print(f"prefetched window (synthetic trajectory, 64 x 256, {tag}) side-stream time: median {np.median(ts):.3f} ms")


if __name__ == "__main__":
    main()
