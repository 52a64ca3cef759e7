"""CPU: the forward-diffusion oracle (oracle/forward_oracle.py igso3_tables / forward_marginal / sample_ref) pinned against the
UNMODIFIED reference (tests/golden/forward.pt, oracle/make_forward_golden.py), with the draws regenerated from the
fixture's numpy seed in the order the reference consumes them; and the host-side contract of the new device ops."""
import math
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dynamicpdb_b200 import kernels as K
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from oracle import dfold_oracle as O
from oracle import forward_oracle as FO

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FWD = None

# Bounds of the comparisons against the reference (fp64 unit roundoff u = 2^-53 ~ 1.1e-16):
# - rotations: the reference returns R_t through fp32 rotation matrices and an fp32 eigen-decomposition (a few fp32 ulps,
#   ~6e-8 each), so matrices agree to 2e-6;
# - translations: fp64 arithmetic rounded once to fp32, so 1e-6 relative;
# - scores: fp64 on both sides, but the angle is np.interp of a cdf row whose entries may differ by a few u (different
#   summation orders); the angle moves by that over the row's pdf and the score by at most |d score / d omega| (~1/sigma^2)
#   times that.  SCORE_TOL bounds |err| / (1 + |score|);
# - scalings: a table entry (a sum over the row) and a closed form, 1e-12 relative.
ROT_TOL, TRANS_TOL, SCORE_TOL, SCALING_TOL = 2e-6, 1e-6, 1e-9, 1e-12


def forward_fixture():
    global FWD
    if FWD is None:
        FWD = torch.load(os.path.join(GOLD, "forward.pt"), weights_only=False)
    return FWD


def case_conf(c):
    """Oracle diffuser config of a fixture case (synthetic.diffuser_conf with the case's overrides)."""
    dc = O.default_diffuser_conf(c["coordinate_scaling"])
    dc.num_sigma, dc.num_omega = c["so3"]["num_sigma"], c["so3"]["num_omega"]
    return dc


def case_diffuser(c, frame_time=None):
    conf = syn.diffuser_conf(c["coordinate_scaling"])
    conf.so3.num_sigma, conf.so3.num_omega = c["so3"]["num_sigma"], c["so3"]["num_omega"]
    conf.diffuse_rot = c["diffuse_rot"]
    conf.frame_time = frame_time
    return SE3ScoreDiffuser(conf)


def case_draws(c, n):
    """numpy's legacy global stream seeded as the fixture was: so3 randn(n,3), so3 rand(n) (so3_diffuser.py:246,230; absent
    when rotations are not diffused), then r3 normal(size=(n,3)) (r3_diffuser.py:95 / :40)."""
    np.random.seed(c["seed"])
    d = {}
    if c["diffuse_rot"]:
        d["z_axis"] = torch.from_numpy(np.random.randn(n, 3))
        d["u"] = torch.from_numpy(np.random.rand(n))
    d["z_trans"] = torch.from_numpy(np.random.normal(size=(n, 3)))
    return d


def rotmats(rig7):
    return O.quat_to_rot(torch.nn.functional.normalize(rig7[..., :4].double(), dim=-1))


def max_ratio(got, ref, tol, rel_floor=1.0):
    """max |got - ref| / (tol * (rel_floor + |ref|)) over the elements."""
    got, ref = got.double(), ref.double()
    return ((got - ref).abs() / (tol * (rel_floor + ref.abs()))).max().item()


def check_against_reference(out, ref, c):
    """Worst error / bound of each output against the reference's, as a dict (every value must be <= 1)."""
    r = {"rot": (rotmats(out["rigids_t"]) - rotmats(ref["rigids_t"])).abs().max().item() / ROT_TOL}
    xt, xr = out["rigids_t"][..., 4:].double(), ref["rigids_t"][..., 4:].double()
    r["trans"] = ((xt - xr).abs().max() / (TRANS_TOL * max(1.0, xr.abs().max().item()))).item()
    if not c["sample_ref"]:
        for k in ("rot_score", "trans_score"):
            r[k] = max_ratio(out[k], ref[k], SCORE_TOL)
        for k in ("rot_score_scaling", "trans_score_scaling"):
            got = float(out[k]) if not torch.is_tensor(out[k]) else out[k].item()
            r[k] = abs(got - float(ref[k])) / (SCALING_TOL * abs(float(ref[k])))
    return r


def oracle_case(c, rig7, mask, tables=None):
    """The oracle's outputs for fixture case c, with the tables given (default: the oracle's own row for the case)."""
    dc = case_conf(c)
    n = rig7[..., 0].numel()
    draws = case_draws(c, n)
    idx = c["sigma_idx"]
    if tables is None:
        tables = FO.igso3_tables(dc, rows=[idx])
        cdf_row, scaling = tables["cdf"][0], tables["score_scaling"][0]
    else:
        cdf_row, scaling = tables["cdf"][idx], tables["score_scaling"][idx]
    if c["sample_ref"]:
        return {"rigids_t": FO.sample_ref(n, rig7.shape[0], draws, dc, cdf_row)}
    return FO.forward_marginal(rig7, c["t"], draws, dc, cdf_row, float(scaling), diffuse_mask=mask if c["mask"] else None,
                              diffuse_rot=c["diffuse_rot"])


@pytest.mark.parametrize("name", ["t037", "t001", "t1", "mask", "norot", "ref", "small_grid"])
def test_oracle_forward_marginal_matches_reference(name):
    g = forward_fixture()
    c = g["cases"][name]
    out = oracle_case(c, g["rigids_0"], g["mask"])
    ref = c["out"]
    assert out["rigids_t"].shape == ref["rigids_t"].shape
    worst = check_against_reference(out, ref, c)
    assert all(v <= 1.0 for v in worst.values()), worst
    if not c["sample_ref"]:
        assert ref["rot_score"].dtype == torch.float64 and ref["trans_score"].dtype == torch.float64
        assert ref["rigids_t"].dtype == torch.float32
    if c["mask"]:
        fixed = g["mask"] == 0
        assert (out["rot_score"][fixed] == 0).all() and (out["trans_score"][fixed] == 0).all()


def test_oracle_tables_match_reference_excerpts():
    """cdf rows of every case's sigma and the whole score_scaling vector of both grids (so3_diffuser.py:132-180)."""
    g = forward_fixture()
    for (num_omega, num_sigma), tab in g["tables"].items():
        dc = O.default_diffuser_conf(1.0)
        dc.num_sigma, dc.num_omega = num_sigma, num_omega
        rows = sorted(tab["cdf_rows"])
        got = FO.igso3_tables(dc, rows=rows)
        for i, r in enumerate(rows):
            assert (got["cdf"][i] - tab["cdf_rows"][r]).abs().max().item() < 1e-13, (num_omega, r)
        all_rows = FO.igso3_tables(dc, chunk=64)["score_scaling"]
        err = ((all_rows - tab["score_scaling"]).abs() / tab["score_scaling"].abs()).max().item()
        assert err < SCALING_TOL, (num_omega, num_sigma, err)


def test_oracle_interp_is_numpy_interp():
    """Clamps, exact hits, plateaus (repeated xp) and the slope form of np.interp."""
    xp = torch.tensor([0.1, 0.2, 0.2, 0.2, 0.5, 0.9, 0.9], dtype=torch.float64)
    fp = torch.tensor([1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 7.0], dtype=torch.float64)
    x = torch.tensor([0.0, 0.05, 0.1, 0.15, 0.2, 0.3, 0.5, 0.7, 0.9, 0.95, 1.0 - 2.0 ** -53, 0.19999999999999998],
                     dtype=torch.float64)
    ref = np.interp(x.numpy(), xp.numpy(), fp.numpy())
    assert torch.equal(FO.interp(x, xp, fp), torch.from_numpy(ref))
    gen = np.random.default_rng(3)
    xp = np.cumsum(gen.random(200) * (gen.random(200) > 0.2))
    x = np.concatenate([gen.random(500) * xp[-1] * 1.1, xp[:50]])
    ref = np.interp(x, xp, np.arange(200.0))
    assert torch.equal(FO.interp(torch.from_numpy(x), torch.from_numpy(xp), torch.arange(200.0, dtype=torch.float64)),
                       torch.from_numpy(ref))


def test_new_ops_refuse_cpu_tensors():
    d = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    rig = torch.cat([torch.tensor([1.0, 0, 0, 0]).expand(2, 5, 4), torch.zeros(2, 5, 3)], dim=-1)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        d.forward_marginal(rig, 0.3)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        d.sample_ref(10, frame_time=2, device="cpu")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        d.tables("cpu")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        d.score_scaling(torch.tensor([0.5], dtype=torch.float64))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        K.igso3_tables(torch.linspace(0.1, 1.5, 10, dtype=torch.float64), 100)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        K.forward_marginal(rig.reshape(10, 7), torch.zeros(10, 3), torch.zeros(10), torch.zeros(10, 3), None,
                           torch.zeros(1, dtype=torch.float64), torch.zeros(3, dtype=torch.float64), torch.zeros(3, 4),
                           torch.zeros(3), max_sigma=1.5, min_sigma=0.1, min_b=0.1, max_b=20.0, r3_scale=1.0)


def test_sample_ref_and_t_are_checked_before_any_launch():
    d = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    with pytest.raises(ValueError, match="impute"):
        d.sample_ref(10, impute=object(), frame_time=2)
    with pytest.raises(ValueError, match="impute"):
        d.sample_ref(10, diffuse_mask=np.ones(10), frame_time=2)
    with pytest.raises(ValueError, match="frame_time"):
        d.sample_ref(10, frame_time=3)
    with pytest.raises(ValueError, match="frame_time"):
        d.sample_ref(10)
    for bad in (-0.1, 1.5):
        with pytest.raises(ValueError, match="Invalid t"):
            d._t64(bad, "cpu")
    conf = syn.diffuser_conf(1.0)
    conf.diffuse_rot = False
    with pytest.raises(ValueError, match="imputation"):
        SE3ScoreDiffuser(conf).sample_ref(10, frame_time=2)


def test_from_reference_carries_the_forward_settings():
    """num_omega, the diffuse flags and frame_time come from a reference-shaped SE3Diffuser; existing configs default to
    num_omega = 1000 and both diffusions on."""
    so3 = SimpleNamespace(min_sigma=0.1, max_sigma=1.5, num_sigma=120, discrete_omega=np.linspace(0, math.pi, 251)[1:],
                          use_cached_score=False, schedule="logarithmic")
    r3 = SimpleNamespace(min_b=0.1, max_b=20.0, _r3_conf=SimpleNamespace(coordinate_scaling=0.1))
    ref = SimpleNamespace(_so3_diffuser=so3, _r3_diffuser=r3, _diffuse_rot=False, _diffuse_trans=True,
                          _se3_conf=SimpleNamespace(dynamics=True, frame_time=4))
    d = SE3ScoreDiffuser.from_reference(ref)
    assert (d.num_omega, d.num_sigma, d.diffuse_rot, d.diffuse_trans, d.frame_time) == (250, 120, False, True, 4)
    assert d.coordinate_scaling == 0.1
    d0 = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    assert (d0.num_omega, d0.diffuse_rot, d0.diffuse_trans, d0.frame_time) == (1000, True, True, None)
