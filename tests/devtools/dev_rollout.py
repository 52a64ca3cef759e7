"""Time the trajectory rollout (dynamicpdb_b200/rollout.py) in its three modes.

    python tests/devtools/dev_rollout.py

Preset A, random weights, at 2 x 256, 5 x 256 and 2 x 1024 (frames x residues):
* graph   -- the default path: one captured (forward + advance) graph replayed per frame;
* eager   -- the same step launched from Python per frame (``graph=False``);
* literal -- the reference's schedule per frame: fresh sample_ref draws and num_t = 100 full forwards
  (``literal=True, num_t=100``).
graph and eager roll L = 200 frames, timed with CUDA events around the whole call after a warm-up rollout, median of 3.
literal rolls L = 3 frames (a 200-frame literal rollout is 20,000 forwards), median of 3; its L = 200 total is printed as
200 x the measured per-frame time and labelled so.  Prints the card and its power limit with the numbers."""
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from dynamicpdb_b200 import synthetic as syn  # noqa: E402
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork  # noqa: E402
from dynamicpdb_b200.rollout import TrajectoryRollout  # noqa: E402
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser  # noqa: E402

SHAPES = [(2, 256), (5, 256), (2, 1024)]
L = 200
L_LITERAL = 3


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def device_ms(fn, reps=3):
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


def main():
    assert torch.cuda.is_available(), "dev_rollout needs a CUDA device"
    print(f"[card] {card()}")
    for nf, N in SHAPES:
        torch.manual_seed(0)
        net = FullScoreNetwork(syn.model_conf(nf, **syn.PRESET_A), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
        sd = net.state_dict()
        syn.dezero_(sd)
        net.load_state_dict(sd)
        net = net.cuda().eval()
        w = {k: v.cuda() for k, v in syn.make_feats(nf, N, seed=1, loader_dtypes=True).items()}
        r = TrajectoryRollout(net)
        t_graph = device_ms(lambda: r.rollout(w, L))
        t_eager = device_ms(lambda: r.rollout(w, L, graph=False))
        t_lit = device_ms(lambda: r.rollout(w, L_LITERAL, literal=True, num_t=100))
        print(f"[rollout] {nf} x {N}: graph {t_graph / L:.3f} ms/frame, {t_graph:.1f} ms for L={L}; "
              f"eager {t_eager / L:.3f} ms/frame, {t_eager:.1f} ms for L={L}; "
              f"literal num_t=100 {t_lit / L_LITERAL:.1f} ms/frame (measured at L={L_LITERAL}), "
              f"{t_lit / L_LITERAL * L / 1e3:.1f} s for L={L} (200 x per-frame)")


if __name__ == "__main__":
    main()
