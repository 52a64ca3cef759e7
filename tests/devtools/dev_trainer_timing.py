"""Development probe: frames/s of trainer.Trainer against the bare TrainStep loop on the same windows, with the GPU's
name and power limit.

    python tests/devtools/dev_trainer_timing.py [--rounds R]

Preset A at two shapes: the released recipe (run_train.sh: frame_time=2, N=256, 4 ranks x 1 window, here one rank with
accumulate=4) and 64 x 256 (accumulate=1).  The rows of the csv all name one synthetic trajectory of 256 residues (the
store decodes it once).  For each shape one Trainer and one bare loop (WindowPrefetcher, TrainStep.load, replay: what a
user writes without the trainer, with no log line) are built, run one warm epoch each, then R rounds alternate one epoch
of each, every epoch timed on the host clock up to a device synchronise; both include the prefetch.  The Trainer logs
every 32 steps, as the recipe does."""
import argparse
import os
import statistics
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

from dynamicpdb_b200 import synthetic as syn  # noqa: E402
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork  # noqa: E402
from dynamicpdb_b200.input_pipeline import TrajectoryStore, WindowPrefetcher  # noqa: E402
from dynamicpdb_b200.loss import score_network_loss  # noqa: E402
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser  # noqa: E402
from dynamicpdb_b200.train_step import TrainStep  # noqa: E402
from dynamicpdb_b200.trainer import Trainer, epoch_order  # noqa: E402
from oracle import synth_traj  # noqa: E402

N = 256
SHAPES = {"recipe 2 x 256, accumulate=4": (2, 4, 64), "64 x 256": (64, 1, 12)}     # frame_time, accumulate, csv rows


def _net(nf):
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(nf, **syn.PRESET_A), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    return net.cuda()


def _conf(csv_path, nf, k):
    return {"experiment": {"batch_size": k, "num_epoch": 10 ** 6, "log_freq": 32, "ckpt_freq": 400, "ckpt_dir": None,
                           "learning_rate": 1e-4, "torsion_loss_weight": 1.0, "rot_loss_weight": 7.0,
                           "trans_loss_weight": 100.0, "rot_loss_t_threshold": 0.0, "separate_rot_loss": False},
            "data": {"csv_path": csv_path, "filtering": {"max_len": 256}, "frame_time": nf, "frame_sample_step": 1,
                     "keep_first": None, "min_t": 0.01}}


class _Bare:
    """The loop without the trainer: the same order, windows and step."""

    def __init__(self, tr: Trainer, nf, k):
        self.rows, self.k, self.diffuser = tr.rows, k, tr.diffuser
        self.store = TrajectoryStore(nf)
        example, = list(WindowPrefetcher(self.store, self.rows[:1], "cuda", diffuser=self.diffuser))
        self.ts = TrainStep(_net(nf), lambda out, w: score_network_loss(out, w, tr.exp_conf), example, lr=1e-4,
                            accumulate=k, loss_reads_window=True)

    def epoch(self, e):
        order = epoch_order(len(self.rows), self.k, e)
        it = iter(WindowPrefetcher(self.store, [self.rows[i] for s in zip(*order) for i in s], "cuda", diffuser=self.diffuser))
        for _ in range(len(order[0])):
            for s in range(self.k):
                self.ts.load(next(it), slot=s)
            self.ts()


def _timed(fn, e):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn(e)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    with tempfile.TemporaryDirectory() as tmp:
        row = synth_traj.write_files(synth_traj.make_trajectory(T=72, N=N, seed=3), tmp)
        for name, (nf, k, n_rows) in SHAPES.items():
            csv_path = os.path.join(tmp, f"train_{nf}.csv")
            with open(csv_path, "w") as f:
                f.write("seq_len,atlas_npz,force_path,vel_path,embed_path\n")
                f.writelines(f"{N}," + ",".join(row) + "\n" for _ in range(n_rows))
            tr = Trainer(_conf(csv_path, nf, k), _net(nf), SE3ScoreDiffuser(syn.diffuser_conf(1.0)), accumulate=k)
            bare = _Bare(tr, nf, k)
            frames = len(epoch_order(n_rows, k, 0)[0]) * k * nf
            times = {"Trainer": [], "bare loop": []}
            _timed(tr.train_epoch, 0)
            _timed(bare.epoch, 0)
            for r in range(1, args.rounds + 1):
                order = [("Trainer", tr.train_epoch), ("bare loop", bare.epoch)]
                for what, fn in (order if r % 2 else order[::-1]):
                    times[what].append(_timed(fn, r))
            for what, ts in times.items():
                fps = [frames / t for t in ts]
                print(f"{gpu} | {name} | {what}: {statistics.median(fps):.1f} frames/s "
                      f"({min(fps):.1f}-{max(fps):.1f}) over {len(fps)} epochs of {frames} frames", flush=True)
            del tr, bare
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
