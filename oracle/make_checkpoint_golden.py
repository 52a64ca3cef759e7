"""Generate tests/golden/checkpoint_layout.pt from the UNMODIFIED reference (a checkout of it at $DFOLD_REFERENCE_ROOT):

    python oracle/make_checkpoint_golden.py

Builds the reference network (tiny preset, synthetic.random_state weights, seed 141) and its trainer's optimizer,
torch.optim.Adam(model.parameters(), lr, amsgrad=True) (train_DFOLD_dynamics.py:412), runs two Experiment.update_fn
steps (:660-667) on seeded batches, writes the checkpoint with du.write_checkpoint (src/data/utils.py:324-362) as
train_epoch does (:743-755), reads it back with torch.load(map_location="cpu") as the evaluator does, and records the
file's structure without any weight: the top-level keys, the model's names and shapes, param_groups, each optimizer
state entry's keys / dtypes / devices / shapes, and the parameter indices that have no state entry.
"""
import copy
import os
import sys
import tempfile
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402

ref_shims.install_trainer_stubs()
from src.model import Dfold_network_dynamic as RefNet  # noqa: E402
from src.data import se3_diffuser  # noqa: E402
from src.data import utils as du  # noqa: E402
from dynamicpdb_b200 import synthetic as syn  # noqa: E402
from oracle import dfold_oracle as O  # noqa: E402
from oracle.make_golden import BOUNDARY_EXP_CONF  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
LR = 1e-4


def layout(ckpt):
    """What the checkpoint holds, without any tensor's values."""
    opt = ckpt["optimizer"]
    desc = lambda t: (str(t.dtype), str(t.device), tuple(t.shape))
    state = {int(i): {k: desc(v) for k, v in st.items()} for i, st in opt["state"].items()}
    n = len(opt["param_groups"][0]["params"])
    return {
        "top_keys": list(ckpt),
        "model": {k: tuple(v.shape) for k, v in ckpt["model"].items()},
        "param_groups": [{k: (list(v) if k == "params" else v) for k, v in g.items()} for g in opt["param_groups"]],
        "state_keys": list(opt),
        "state": state,
        "missing": [i for i in range(n) if i not in state],
        "lr": LR,
        "torch": str(torch.__version__),
    }


def main():
    torch.manual_seed(0)
    diffuser = se3_diffuser.SE3Diffuser(syn.diffuser_conf(1.0))
    model_conf = syn.model_conf(3, **syn.PRESET_TINY)
    net = RefNet.FullScoreNetwork(model_conf, diffuser)
    net.load_state_dict(syn.random_state({k: v.shape for k, v in net.state_dict().items()}, seed=141))
    exp = ref_shims.reference_experiment(net, diffuser,
                                         SimpleNamespace(cfg_drop_in_train=True, cfg_drop_rate=0.0,
                                                         embed=SimpleNamespace(embed_self_conditioning=False)),
                                         O.default_exp_conf(**BOUNDARY_EXP_CONF), SimpleNamespace(diffuse_rot=True))
    exp._conf = SimpleNamespace(model=SimpleNamespace(cfg_drop_rate=0.0, cfg_gamma=1.0))
    exp._data_conf = SimpleNamespace(num_t=4, min_t=0.01)
    exp._optimizer = torch.optim.Adam(net.parameters(), lr=LR, amsgrad=True)
    for seed in (141, 142):
        loss, _ = exp.update_fn(syn.add_loss_targets(syn.make_feats(3, 12, seed=seed, loader_dtypes=True), seed=seed))
        print(f"[golden] checkpoint: update_fn loss {float(loss.detach()):.6f}")
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "step_2.pth")
        du.write_checkpoint(path, copy.deepcopy(net.state_dict()), SimpleNamespace(model=model_conf),
                            copy.deepcopy(exp._optimizer.state_dict()), 1, 2, use_torch=True)
        ckpt = torch.load(path, map_location="cpu", weights_only=False)
    res = layout(ckpt)
    torch.save(res, os.path.join(OUT, "checkpoint_layout.pt"))
    print(f"[golden] checkpoint: {len(res['model'])} tensors, {len(res['state'])} state entries, missing {res['missing']}")


if __name__ == "__main__":
    main()
