"""Development probe: time per protein of evaluator.Evaluator against the two other ways of sampling a test split on the
device, and the device memory each leaves held, with the GPU's name and power limit.

    python tests/devtools/dev_evaluator_timing.py [--rounds R]

The shipped evaluation launch (run_eval.sh): preset A, frame_time=2, num_t=10, noise_scale=0.1, batch 1, over a test
split of 8 synthetic proteins of 64 to 256 residues, each of its own length.  Three ways, each over the whole split:

  evaluator  Evaluator.evaluate(): the memoised sampler run eagerly (one trunk pass, num_t x 2 small kernels);
  graphed    metrics.evaluate_window per window with a fresh DeviceReverseDiffusion, so one CUDA graph per length is
             warmed up, captured and replayed once, as a process evaluating a split for the first time does;
  literal    DeviceReverseDiffusion.sample(literal=True): num_t full network evaluations per window, as inference_fn
             runs them, scored with window_metrics.

All three read their windows from the same prefetcher.  The evaluator's prefetch runs inside its timed loop; graphed and
literal take their windows from a list made before the clock starts, because a graph cannot be captured while the
prefetch worker's thread issues CUDA calls (the capture is invalidated).  One warm round of each, then R rounds
alternate them; each is timed on the host clock up to a device synchronise, and the medians are reported per protein.  "held" is the allocation left once the way has finished
while its objects are alive (the graphed sampler keeps its graphs' pools), above the allocation before it."""
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
from dynamicpdb_b200.inference import DeviceReverseDiffusion  # noqa: E402
from dynamicpdb_b200.metrics import eval_sampler_inputs, evaluate_window, window_metrics  # noqa: E402
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser  # noqa: E402
from oracle import synth_traj  # noqa: E402

NF, NUM_T, MIN_T, NOISE = 2, 10, 0.01, 0.1
LENGTHS = [64, 256, 96, 224, 128, 192, 160, 80]
FRAMES, START = 4, 1


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


def _timed(fn):
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    keep = fn()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    held = torch.cuda.memory_allocated() - before
    del keep
    return dt / len(LENGTHS), held


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    with tempfile.TemporaryDirectory() as root:
        csv_path = _split(root)
        net = _net()
        weights = os.path.join(root, "w.pth")
        torch.save({"model": {k: v.cpu() for k, v in net.state_dict().items()}}, weights)
        conf = {"eval": {"weights_path": weights, "eval_batch_size": 1}, "experiment": {"noise_scale": NOISE},
                "data": {"test_csv_path": csv_path, "filtering": {"max_len": 256}, "frame_time": NF,
                         "frame_sample_step": 1, "fix_sample_start": START, "num_t": NUM_T, "min_t": MIN_T}}
        ev = Evaluator(conf, net, SE3ScoreDiffuser(syn.diffuser_conf(1.0)), seed=0)

        def windows():
            return ev._prefetcher(ev.generators()[0])

        def evaluator():
            rows = ev._run()
            return rows

        def graphed(ws):
            sampler = DeviceReverseDiffusion(net)
            rows = [evaluate_window(sampler, w, NUM_T, MIN_T, NOISE)["all_atom_rmsd"] for w in ws]
            return sampler, rows

        def literal(ws):
            sampler = DeviceReverseDiffusion(net)
            gen = ev.generators()[1]
            rows = []
            for w in ws:
                s = sampler.sample(eval_sampler_inputs(w), NUM_T, MIN_T, NOISE, generator=gen, literal=True)
                rows.append(window_metrics(s["rigid_pred"], s["prot_traj"][0], w["rigids_0"], w["atom37_pos"],
                                           w["atom37_mask"])["all_atom_rmsd"])
            return rows

        ways = {"evaluator": evaluator, "graphed": graphed, "literal": literal}
        for fn in ways.values():
            _timed(fn if fn is evaluator else lambda fn=fn: fn(list(windows())))
        times = {k: [] for k in ways}
        held = {k: [] for k in ways}
        for _ in range(args.rounds):
            for k, fn in ways.items():
                ws = None if fn is evaluator else list(windows())
                dt, h = _timed(fn if fn is evaluator else lambda: fn(ws))
                del ws
                times[k].append(dt)
                held[k].append(h)
    res = {"gpu": q, "preset": "A", "frame_time": NF, "num_t": NUM_T, "lengths": LENGTHS, "rounds": args.rounds,
           "ms_per_protein": {k: round(1e3 * statistics.median(v), 2) for k, v in times.items()},
           "ms_per_protein_all": {k: [round(1e3 * x, 2) for x in v] for k, v in times.items()},
           "held_MiB": {k: round(max(v) / 2 ** 20, 1) for k, v in held.items()}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
