"""Generate tests/golden/loss_edges.pt from the UNMODIFIED reference (a checkout of it at $DFOLD_REFERENCE_ROOT):

    python oracle/make_loss_edges_golden.py

Runs Experiment.loss_fn (train_DFOLD_dynamics.py:1181-1400) on the edge cases of dynamicpdb_b200.synthetic.LOSS_EDGES
(zero-length predictions, a tie between the torsion targets, t on the rotation gate, masked frames) and stores its value,
aux_data and gradients as tests/golden/loss.pt does.  The inputs are rebuilt by the tests from the same seeds.
"""
import os
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402

ref_shims.install()
from dynamicpdb_b200 import synthetic as syn  # noqa: E402
from oracle import dfold_oracle as O  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def main():
    res = {}
    for name in syn.LOSS_EDGES:
        feats, out, separate = syn.loss_edge(name)
        leaves = {k: out[k].clone().requires_grad_(True) for k in ("angles", "rot_score", "rigids")}
        model_out = dict(out, **leaves)
        exp_conf = O.default_exp_conf(separate_rot_loss=separate, bb_atom_loss_weight=1.0, bb_atom_loss_t_filter=0.25,
                                      dist_mat_loss_weight=1.0, dist_mat_loss_t_filter=0.25, aux_loss_weight=0.25)
        model_conf = SimpleNamespace(cfg_drop_in_train=True, cfg_drop_rate=0.0, embed=SimpleNamespace(embed_self_conditioning=False))
        exp = ref_shims.reference_experiment(lambda batch, drop_ref=False: model_out, None, model_conf, exp_conf,
                                             SimpleNamespace(diffuse_rot=True))
        loss, aux = exp.loss_fn(dict(feats))
        grads = torch.autograd.grad(loss, list(leaves.values()), allow_unused=True)
        res[name] = {"loss": loss.detach(), "aux": {k: a.detach() for k, a in aux.items()},
                     "grads": {k: (g.detach() if g is not None else None) for k, g in zip(leaves, grads)}}
        print(f"[golden] loss_edges/{name}: {float(loss):.6e}")
    torch.save(res, os.path.join(OUT, "loss_edges.pt"))


if __name__ == "__main__":
    main()
