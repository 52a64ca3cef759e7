"""Generate tests/golden/lr_schedule.pt from the UNMODIFIED reference (a checkout of it at $DFOLD_REFERENCE_ROOT):

    python oracle/make_lr_schedule_golden.py

Runs the reference's AlphaFoldLRScheduler (openfold/utils/lr_schedulers.py, imported by train_DFOLD_dynamics.py:56) over
torch.optim.Adam(amsgrad=True), the trainer's optimizer (:412), made constructible by a shim below (torch no longer
takes its ``verbose`` argument).  For each setting it records param_groups[0]['lr'] at last_epoch = s:
  * four settings step by step, optimizer.step() then scheduler.step() as a trainer calls them, s = 0 ... 399:
    TestAF2LRScheduler's defaults, a short recipe (warmup 4, start 7, every 2), and decay_factor 1.0 and 0.5;
  * AlphaFold's defaults at the phase boundaries and up to 10^6, by setting last_epoch to s - 1 and stepping once.
It also records optimizer.state_dict()['param_groups'] of the TestAF2 run at a mid-warmup step (5 of 10).
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402
from oracle.lr_schedule_oracle import ALPHAFOLD_DEFAULTS, TEST_AF2_DEFAULTS  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def alphafold_lr_scheduler_classes():
    """(AlphaFoldLRScheduler, TestAF2LRScheduler) of the UNMODIFIED reference (openfold/utils/lr_schedulers.py), made
    constructible under the installed torch.  Their constructor passes ``verbose`` to ``LRScheduler.__init__``
    (lr_schedulers.py:48-52), a parameter torch has removed, so construction raises TypeError there.  The shim wraps
    ``LRScheduler.__init__`` to accept and drop ``verbose`` (which only ever printed the new lr); nothing else changes."""
    import inspect

    from torch.optim import lr_scheduler as L
    init = L.LRScheduler.__init__
    if "verbose" not in inspect.signature(init).parameters:
        def drop_verbose(self, optimizer, last_epoch=-1, verbose=False):
            init(self, optimizer, last_epoch)
        L.LRScheduler.__init__ = drop_verbose
    ref_shims.install()
    from openfold.utils import lr_schedulers
    return lr_schedulers.AlphaFoldLRScheduler, lr_schedulers.TestAF2LRScheduler
ADAM_LR = 1e-4                      # the optimizer's own lr (the scheduler ignores it; it becomes initial_lr)
STEPS = 400
MID_WARMUP = 5
SETTINGS = {
    "test_af2": None,               # TestAF2LRScheduler with its defaults (TEST_AF2_DEFAULTS)
    "recipe": dict(base_lr=0.0, max_lr=1e-3, warmup_no_steps=4, start_decay_after_n_steps=7, decay_every_n_steps=2,
                   decay_factor=0.95),
    "decay_1.0": dict(base_lr=1e-5, max_lr=5e-4, warmup_no_steps=7, start_decay_after_n_steps=20, decay_every_n_steps=3,
                      decay_factor=1.0),
    "decay_0.5": dict(base_lr=2e-6, max_lr=3e-4, warmup_no_steps=13, start_decay_after_n_steps=13, decay_every_n_steps=2,
                      decay_factor=0.5),
}


def _alphafold_samples():
    w, s, e = (ALPHAFOLD_DEFAULTS[k] for k in ("warmup_no_steps", "start_decay_after_n_steps", "decay_every_n_steps"))
    pts = {0, 1, 2, 3, 10 ** 6, 10 ** 6 - 1, 10 ** 6 + 1}
    for b in (w, s) + tuple(s + k * e for k in range(1, 20)):
        pts |= {b - 1, b, b + 1}
    pts |= set(range(0, w + 1, 7)) | set(range(w, s, 997)) | set(range(s, 10 ** 6, 9973))
    return sorted(pts)


def _adam():
    p = torch.nn.Parameter(torch.zeros(4))
    p.grad = torch.zeros(4)
    return torch.optim.Adam([p], lr=ADAM_LR, amsgrad=True)


def main():
    AF, TestAF = alphafold_lr_scheduler_classes()
    res = {"settings": {}, "torch": str(torch.__version__), "adam_lr": ADAM_LR}
    for name, kw in SETTINGS.items():
        opt = _adam()
        sched = TestAF(opt) if kw is None else AF(opt, **kw)
        lrs = [opt.param_groups[0]["lr"]]
        for s in range(1, STEPS):
            opt.step()
            sched.step()
            assert sched.last_epoch == s
            lrs.append(opt.param_groups[0]["lr"])
            if name == "test_af2" and s == MID_WARMUP:
                res["mid_warmup"] = {"setting": name, "step": s, "param_groups": opt.state_dict()["param_groups"]}
        res["settings"][name] = {"kwargs": dict(TEST_AF2_DEFAULTS if kw is None else kw), "steps": list(range(STEPS)),
                                 "lr": lrs}
    opt = _adam()
    sched = AF(opt)
    opt.step()
    steps = _alphafold_samples()
    lrs = []
    for s in steps:
        sched.last_epoch = s - 1
        sched.step()
        lrs.append(opt.param_groups[0]["lr"])
    res["settings"]["alphafold"] = {"kwargs": dict(ALPHAFOLD_DEFAULTS), "steps": steps, "lr": lrs}
    for name, v in res["settings"].items():
        assert all(type(x) is float for x in v["lr"]), name
        print(f"[golden] lr_schedule {name}: {len(v['steps'])} steps, lr {min(v['lr']):.3e} ... {max(v['lr']):.3e}")
    print(f"[golden] lr_schedule mid-warmup param_groups: {res['mid_warmup']['param_groups']}")
    torch.save(res, os.path.join(OUT, "lr_schedule.pt"))


if __name__ == "__main__":
    main()
