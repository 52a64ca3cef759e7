"""Development probe: time per protein of evaluator.Evaluator.extend, with the GPU's name and power limit.

    python tests/devtools/dev_extension_timing.py [--rounds R]

Preset A, frame_time=2, length=200 (eval_extension's), over a test split of 8 synthetic proteins of 64 to 256 residues,
each of its own length: per protein the window from the prefetcher, 200 eager network forwards with the prediction fed
back, and the 200 horizons scored against the MD frames that follow the window.  Two ways over the whole split:

  extend   Evaluator.extend's device loop (``_run_extension``), prefetch included, timed as a whole;
  bare     the same rollout and scoring per window, from windows made before the clock starts, each window timed on its
           own: the time of the rollout itself at each residue count, without the prefetch worker beside it.

One warm round of each, then R rounds alternate them, each timed on the host clock up to a device synchronise; the median
and range of the rounds are reported per protein and per rolled-out frame, and for bare per residue count.  "held" is
the allocation left once an extend round has finished, above the allocation before it."""
import argparse
import json
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
from dynamicpdb_b200.evaluator import Evaluator  # noqa: E402
from dynamicpdb_b200.metrics import horizon_metrics  # noqa: E402
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser  # noqa: E402
from oracle import synth_traj  # noqa: E402

NF, LENGTH, MIN_T = 2, 200, 0.01
LENGTHS = [64, 256, 96, 224, 128, 192, 160, 80]
START = 1
FRAMES = START + NF + LENGTH - 1


def _net():
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(NF, **syn.PRESET_A), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    return net.cuda()


def _split(root):
    path = os.path.join(root, "test.csv")
    with open(path, "w") as f:
        f.write("name,seq_len,atlas_npz,force_path,vel_path,embed_path,pdb_path\n")
        for i, n in enumerate(LENGTHS):
            row = synth_traj.write_files(synth_traj.make_trajectory(T=FRAMES, N=n, seed=100 + i), root, name=f"p{i}")
            f.write(f"p{i},{n}," + ",".join(row) + ",x.pdb\n")
    return path


def _timed(ev):
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    scores = ev._run_extension(LENGTH, None)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    held = torch.cuda.memory_allocated() - before
    del scores
    return dt / len(LENGTHS), held


def _bare(ev, windows):
    """Seconds per window, in split order: rollout and scoring of each window, timed on its own."""
    out = []
    for w in windows:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        traj = ev.roller.rollout(w, LENGTH, min_t=MIN_T, graph=False)
        horizon_metrics(traj["rigid_traj"], traj["atom_traj"], w["rigids_0"][NF - 2], w["horizon_rigids_0"],
                        w["horizon_atom37_pos"], w["horizon_atom37_mask"])
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dev_extension_timing: needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    with tempfile.TemporaryDirectory() as root:
        csv_path = _split(root)
        net = _net()
        weights = os.path.join(root, "w.pth")
        torch.save({"model": {k: v.cpu() for k, v in net.state_dict().items()}}, weights)
        conf = {"eval": {"weights_path": weights, "eval_batch_size": 1}, "experiment": {"noise_scale": 0.1},
                "data": {"test_csv_path": csv_path, "filtering": {"max_len": 256}, "frame_time": NF,
                         "frame_sample_step": 1, "fix_sample_start": START, "num_t": 10, "min_t": MIN_T}}
        ev = Evaluator(conf, net, SE3ScoreDiffuser(syn.diffuser_conf(1.0)), seed=0)
        windows = list(ev._prefetcher(ev.generators()[0], horizons=LENGTH))
        _timed(ev)
        _bare(ev, windows)
        times, held, bare = [], [], []
        for _ in range(args.rounds):
            dt, h = _timed(ev)
            times.append(dt)
            held.append(h)
            bare.append(_bare(ev, windows))
    per_n = {n: statistics.median(r[i] for r in bare) for i, n in enumerate(LENGTHS)}
    bare_means = [statistics.mean(r) for r in bare]
    res = {"gpu": q, "preset": "A", "frame_time": NF, "length": LENGTH, "lengths": LENGTHS, "rounds": args.rounds,
           "ms_per_protein": round(1e3 * statistics.median(times), 1),
           "ms_per_protein_range": [round(1e3 * min(times), 1), round(1e3 * max(times), 1)],
           "ms_per_frame": round(1e3 * statistics.median(times) / LENGTH, 2),
           "ms_per_protein_all": [round(1e3 * x, 1) for x in times],
           "held_MiB": round(max(held) / 2 ** 20, 1),
           "bare_ms_per_protein": round(1e3 * statistics.median(bare_means), 1),
           "bare_ms_per_protein_range": [round(1e3 * min(bare_means), 1), round(1e3 * max(bare_means), 1)],
           "bare_ms_per_frame_by_residues": {n: round(1e3 * per_n[n] / LENGTH, 2) for n in sorted(per_n)}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
