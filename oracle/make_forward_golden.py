"""Generate tests/golden/forward.pt from the UNMODIFIED reference (a checkout of it at $DFOLD_REFERENCE_ROOT):

    python oracle/make_forward_golden.py

SE3Diffuser.forward_marginal / sample_ref (src/data/se3_diffuser.py:47-110, :217-280) on a small seeded window, with
numpy's global stream seeded before each call, and excerpts of the IGSO(3) tables the reference builds on the way
(so3_diffuser.py:132-180; about a minute for the default 1000 x 1000 grid).  The inputs are stored in the fixture; the
draws are regenerated from the seeds by the tests.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims  # noqa: E402

ref_shims.install()
from src.data import se3_diffuser  # noqa: E402
from openfold.utils import rigid_utils as RefRU  # noqa: E402
from dynamicpdb_b200 import synthetic as syn  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
os.makedirs(OUT, exist_ok=True)


FORWARD_CASES = {
    # name: (t, numpy seed, coordinate_scaling, so3 overrides, diffuse_rot, with mask, sample_ref)
    "t037": (0.37, 101, 0.1, {}, True, False, False),
    "t001": (0.01, 102, 0.1, {}, True, False, False),
    "t1": (1.0, 103, 1.0, {}, True, False, False),
    "mask": (0.37, 104, 0.1, {}, True, True, False),
    "norot": (0.37, 105, 0.1, {}, False, False, False),
    "ref": (1.0, 106, 0.1, {}, True, False, True),
    "small_grid": (0.6, 107, 0.1, {"num_omega": 250, "num_sigma": 120}, True, False, False),
}


def run_forward():
    """tests/golden/forward.pt: SE3Diffuser.forward_marginal / sample_ref of the UNMODIFIED reference (se3_diffuser.py:47-110,
    :217-280) on a 3-frame x 11-residue window (synthetic.make_feats seed 9), each case with numpy's global stream seeded
    before the call, and excerpts of the IGSO(3) tables it built (so3_diffuser.py:132-180): the whole score_scaling vector
    and the cdf row of every case's t.  The tests regenerate the draws from the seed in the reference's order."""
    import numpy as np
    nf, N = 3, 11
    rig7 = syn.make_feats(nf, N, seed=9)["rigids_0"]
    mask = torch.ones(nf, N, dtype=torch.float64)
    mask[:, [0, 4, 5]] = 0.0
    res = {"rigids_0": rig7, "mask": mask, "cases": {}, "tables": {}}
    diffusers = {}
    for name, (t, seed, cs, so3_over, rot, with_mask, ref) in FORWARD_CASES.items():
        conf = syn.diffuser_conf(cs)
        for k, v in so3_over.items():
            setattr(conf.so3, k, v)
        conf.diffuse_rot = rot
        conf.dynamics, conf.frame_time = True, nf
        key = (cs, tuple(sorted(so3_over.items())), rot)
        if key not in diffusers:
            diffusers[key] = se3_diffuser.SE3Diffuser(conf)
        diff = diffusers[key]
        so3 = diff._so3_diffuser
        np.random.seed(seed)
        if ref:
            out = diff.sample_ref(n_samples=nf * N, diffuse_mask=None, as_tensor_7=True)
        else:
            out = diff.forward_marginal(rigids_0=RefRU.Rigid.from_tensor_7(rig7), t=t,
                                        diffuse_mask=mask.numpy() if with_mask else None)
        c = {"t": t, "seed": seed, "coordinate_scaling": cs, "so3": dict(num_omega=len(so3.discrete_omega), num_sigma=so3.num_sigma),
             "diffuse_rot": rot, "mask": with_mask, "sample_ref": ref, "sigma_idx": int(so3.t_to_idx(t))}
        c["out"] = {k: (v.clone() if torch.is_tensor(v) else torch.as_tensor(np.asarray(v))) for k, v in out.items()}
        res["cases"][name] = c
        grid = (c["so3"]["num_omega"], c["so3"]["num_sigma"])
        tab = res["tables"].setdefault(grid, {"score_scaling": torch.from_numpy(so3._score_scaling.copy()), "cdf_rows": {}})
        tab["cdf_rows"][c["sigma_idx"]] = torch.from_numpy(so3._cdf[c["sigma_idx"]].copy())
        print(f"[golden] forward/{name}: t={t} sigma_idx={c['sigma_idx']}")
    torch.save(res, os.path.join(OUT, "forward.pt"))


if __name__ == "__main__":
    run_forward()
