"""Development probe: wall time of save_checkpoint / load_checkpoint for the captured training step at preset A, 64 x 256
(184.4 M parameters; parameters and three Adam moments, about 2.95 GB), with the GPU's name and power limit.

    python tests/devtools/dev_checkpoint_timing.py [--dir DIR] [--repeats R]

The checkpoint goes to a temporary directory (under DIR when given) that is removed afterwards."""
import argparse
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

from dynamicpdb_b200 import checkpoint as C, synthetic as syn  # noqa: E402
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork  # noqa: E402
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser  # noqa: E402
from dynamicpdb_b200.train_step import TrainStep  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", default=None)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    nf, N = 64, 256
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(nf, **syn.PRESET_A), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    feats = {k: v.cuda() for k, v in syn.make_feats(nf, N, seed=0).items()}
    ts = TrainStep(net.cuda(), syn.surrogate_loss, feats, lr=1e-4, graph=True, warmup=2)
    ts()
    torch.cuda.synchronize()
    nbytes = 4 * ts.flat_param.numel() * 4
    with tempfile.TemporaryDirectory(dir=args.dir) as d:
        path = os.path.join(d, "step.pth")
        for r in range(args.repeats):
            t0 = time.perf_counter()
            C.save_checkpoint(path, ts, None, 0, 1)
            t1 = time.perf_counter()
            C.load_checkpoint(path, ts)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            print(f"[{gpu}] repeat {r}: save_checkpoint {t1 - t0:.2f} s, load_checkpoint {t2 - t1:.2f} s, "
                  f"file {os.path.getsize(path) / 1e9:.2f} GB, state {nbytes / 1e9:.2f} GB")
        loss = float(ts())
    print(f"[{gpu}] step after the last load: loss {loss:.6f}, graph {'kept' if ts.graph is not None else 'absent'}")


if __name__ == "__main__":
    main()
