"""Generate tests/golden/trainer_log.pt from the UNMODIFIED reference (a checkout of it at $DFOLD_REFERENCE_ROOT):

    python oracle/make_trainer_golden.py

Drives ``Experiment.start_training`` / ``train_epoch`` of train_DFOLD_dynamics.py (:591-763), imported through the
trainer-module stubs of oracle/ref_shims.py, on the CPU: the Experiment is built without its constructor (which needs
hydra, data and a GPU census) and given what the loop reads.  ``create_dataset`` returns the reference's own training
loader layout (a ``DataLoader`` of batch size 1 over a ``DistributedSampler(num_replicas=world, rank=rank)``) over a
dataset whose item i is ``{"idx": i}``; ``update_fn`` records the indices it gets and returns seeded ``aux_data`` with the
keys and dtypes of ``Experiment.loss_fn``; ``du.write_checkpoint`` records its path, epoch and step instead of writing.
For every case and rank it stores the log messages, the indices per update, the aux_data returned (as lists; the dtypes
once, in ``aux_dtypes``), and the checkpoints.
"""
import logging
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
AUX_KEYS = ("batch_train_loss", "batch_rot_loss", "batch_trans_loss", "batch_torsion_loss", "total_loss", "rot_loss",
            "trans_loss", "torsion_loss")           # Experiment.loss_fn's aux_data, in its order
# name: (world, dataset size, num_epoch, log_freq, ckpt_freq, trained_epochs, trained_steps) -- several sizes need padding
CASES = {
    "w1": (1, 5, 3, 2, 1, 0, 0),
    "w2_pad": (2, 5, 4, 3, 2, 0, 0),
    "w3_pad": (3, 7, 3, 1, 2, 0, 0),
    "w4": (4, 8, 3, 5, 1, 0, 0),
    "w2_resumed": (2, 6, 5, 2, 3, 2, 7),
    "w4_pad_resumed": (4, 6, 5, 4, 2, 3, 11),
    "w1_rare_log": (1, 9, 2, 100, 1, 0, 0),
}


class _Records(logging.Handler):
    def __init__(self):
        super().__init__()
        self.lines = []

    def emit(self, record):
        self.lines.append(record.getMessage())


def _aux(rng):
    """aux_data with Experiment.loss_fn's keys and dtypes (float64, the translation terms float32), values spanning
    several magnitudes so that the log's 4-decimal rounding is exercised."""
    out = {}
    for k in AUX_KEYS:
        dt = torch.float32 if "trans" in k else torch.float64
        v = torch.tensor(rng.lognormal(0.0, 2.0, size=2 if k.startswith("batch") else ()), dtype=dt)
        out[k] = v
    return out


def run(T, world, rank, n, num_epoch, log_freq, ckpt_freq, trained_epochs, trained_steps, seed):
    exp = object.__new__(T.Experiment)
    handler = _Records()
    exp._log = logging.Logger(f"trainer_golden_{seed}")
    exp._log.addHandler(handler)
    eval_dir = tempfile.mkdtemp()
    exp._exp_conf = types.SimpleNamespace(log_freq=log_freq, num_epoch=num_epoch, ckpt_freq=ckpt_freq, ckpt_dir="ckpt",
                                          eval_dir=eval_dir, use_gpu=False, use_ddp=False, num_gpus=world,
                                          batch_size=world)
    exp._conf = types.SimpleNamespace(name="conf")
    exp._use_tensorboard = False
    exp._model = torch.nn.Linear(1, 1)
    exp._optimizer = torch.optim.Adam(exp._model.parameters(), lr=1e-4, amsgrad=True)
    exp.trained_epochs, exp.trained_steps = trained_epochs, trained_steps
    exp._init_best_eval()
    dataset = [{"idx": i} for i in range(n)]
    sampler = torch.utils.data.distributed.DistributedSampler(dataset, num_replicas=world, rank=rank)
    loader = torch.utils.data.DataLoader(dataset, batch_size=1, shuffle=False, num_workers=0, drop_last=False,
                                         sampler=sampler)
    exp.create_dataset = lambda: (loader, None)
    rng = np.random.default_rng(seed)
    updates, auxes, ckpts = [], [], []

    def update_fn(data):
        updates.append((exp.trained_epochs, int(data["idx"].reshape(-1)[0])))
        aux = _aux(rng)
        auxes.append({k: v.tolist() for k, v in aux.items()})
        return aux["total_loss"], {k: v.clone() for k, v in aux.items()}

    def write_checkpoint(ckpt_path, model, conf, optimizer, epoch, step, logger=None, use_torch=True):
        ckpts.append({"path": ckpt_path, "epoch": epoch, "step": step})

    exp.update_fn = update_fn
    T.du.write_checkpoint = write_checkpoint
    exp.start_training()
    return {"log": handler.lines, "updates": updates, "aux": auxes, "ckpts": ckpts,
            "trained_epochs": exp.trained_epochs, "trained_steps": exp.trained_steps}


def main():
    if not ref_shims.reference_available():
        raise SystemExit("set DFOLD_REFERENCE_ROOT to a checkout of the reference")
    ref_shims.install_trainer_stubs()
    import train_DFOLD_dynamics as T
    T.HydraConfig = types.SimpleNamespace(initialized=lambda: False)      # no hydra run: replica 0
    res = {"cases": {}, "aux_keys": AUX_KEYS, "aux_dtypes": {k: v.dtype for k, v in _aux(np.random.default_rng(0)).items()}}
    for ci, (name, (world, n, num_epoch, log_freq, ckpt_freq, te, ts)) in enumerate(CASES.items()):
        ranks = [run(T, world, r, n, num_epoch, log_freq, ckpt_freq, te, ts, seed=100 * ci + r) for r in range(world)]
        res["cases"][name] = {"world": world, "n": n, "num_epoch": num_epoch, "log_freq": log_freq, "ckpt_freq": ckpt_freq,
                              "trained_epochs": te, "trained_steps": ts, "ranks": ranks}
        r0 = ranks[0]
        print(f"[golden] trainer {name}: {len(r0['updates'])} updates, {sum('trained_steps' in l for l in r0['log'])} "
              f"log lines, checkpoints {[(c['epoch'], c['step']) for c in r0['ckpts']]}")
    torch.save(res, os.path.join(OUT, "trainer_log.pt"))


if __name__ == "__main__":
    main()
