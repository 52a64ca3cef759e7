"""Development probe: what the backbone-atom and pair-distance losses (score_network_loss(aux_losses=True)) cost in the
captured training step, preset A (184.4 M parameters), with the GPU's name and power limit.

    python tests/devtools/dev_aux_loss_timing.py [--rounds R] [--steps K] [--shapes 2x256,64x256]

For each shape (frames x residues): two captured steps from the same weights on the same window (t = 0.1, below both
filters, so every aux term is on), one on the default objective and one with aux_losses=True.  After the warm-up of
their construction, the two are timed with CUDA events over K replays each, alternated R times; the median and range
of the per-step time are printed.  Then the peak memory one eager step of each allocates above its resident state."""
import argparse
import copy
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch  # noqa: E402

from dynamicpdb_b200 import synthetic as syn  # noqa: E402
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork  # noqa: E402
from dynamicpdb_b200.loss import score_network_loss  # noqa: E402
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser  # noqa: E402
from dynamicpdb_b200.train_step import TrainStep  # noqa: E402
from oracle import dfold_oracle as O  # noqa: E402

EXP = O.default_exp_conf(bb_atom_loss_weight=1.0, bb_atom_loss_t_filter=0.25, dist_mat_loss_weight=1.0,
                         dist_mat_loss_t_filter=0.25, aux_loss_weight=0.25)


def _net(nf):
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(nf, **syn.PRESET_A), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    return net


def _batch(nf, N):
    b = syn.add_loss_targets(syn.make_feats(nf, N, seed=0, t=0.1, loader_dtypes=True), seed=0)
    return {k: v.cuda() for k, v in b.items()}


def _step(net, batch, aux, graph):
    return TrainStep(net, lambda out: score_network_loss(out, batch, EXP, aux_losses=aux)[0], batch, lr=1e-4,
                     graph=graph, warmup=2)


def _events_ms(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _peak(nf, N, aux):
    batch = _batch(nf, N)
    ts = _step(_net(nf).cuda(), batch, aux, graph=False)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ts()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del ts
    torch.cuda.empty_cache()
    return peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--shapes", default="2x256,64x256")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    print(f"[aux timing] {gpu}")
    for shape in args.shapes.split(","):
        nf, N = (int(v) for v in shape.split("x"))
        base = _net(nf).cuda()
        steps = {}
        for aux in (False, True):
            steps[aux] = _step(copy.deepcopy(base), _batch(nf, N), aux, graph=True)
            assert steps[aux].graph is not None, steps[aux].graph_error
        del base
        times = {False: [], True: []}
        for _ in range(args.rounds):
            for aux in (False, True):
                times[aux].append(_events_ms(steps[aux], args.steps))
        del steps
        torch.cuda.empty_cache()
        for aux in (False, True):
            t = times[aux]
            print(f"[aux timing] {nf} x {N} {'aux' if aux else 'default'}: {statistics.median(t):.2f} ms per step "
                  f"({min(t):.2f}-{max(t):.2f}) over {args.rounds} alternated rounds of {args.steps} replays")
        peaks = {aux: _peak(nf, N, aux) for aux in (False, True)}
        print(f"[aux timing] {nf} x {N} peak memory of one eager step above its resident state: default "
              f"{peaks[False] / 2**20:.1f} MiB, aux {peaks[True] / 2**20:.1f} MiB "
              f"(+{(peaks[True] - peaks[False]) / 2**20:.1f} MiB)")


if __name__ == "__main__":
    main()
