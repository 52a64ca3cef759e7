"""CPU: the metric oracle (oracle/metrics_oracle.py) pinned against the UNMODIFIED reference (tests/golden/metrics.pt,
oracle/make_metrics_golden.py, inputs rebuilt by oracle/metrics_cases.py), its Kabsch against scipy's independent
Rotation.align_vectors, and the host-side argument checks of the metric entry points and wrappers.

Bounds (shared with tests/test_gpu_metrics.py):
- fp64 sums (MAE, MSE, rmsd_*, drmsd, translation errors, superposition RMSD): |err| <= 1e-12 (1 + |ref|);
- angles: 1e-5 degrees.  An angle is 2 acos(|dot|) of normalised quaternions; in fp64 the dot product carries an error
  of up to ~4u (u = 2^-53: two normalisations and a 4-term sum).  acos is worst conditioned at |dot| = 1, where
  acos(1 - e) ~ sqrt(2 e): an error d in the dot moves acos by at most sqrt(2 d), so the angle by at most
  2 sqrt(2 * 4u) = 6.0e-8 rad = 3.4e-6 degrees (a mean over residues by no more).  Away from |dot| = 1 the error is
  O(u / sin(angle / 2)) and far smaller.  1e-5 degrees covers it with margin;
- fp32 predictions: the reference normalises them in fp32, the kernels in fp64, so the bound is the spread between the
  reference's fp32 and fp64 runs plus the bound above."""
import ctypes
import math
import os
import warnings

import pytest
import torch
from scipy.spatial.transform import Rotation

from dynamicpdb_b200 import kernels as K
from dynamicpdb_b200 import metrics as M
from oracle import metrics_cases as C
from oracle import metrics_oracle as MO

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SUM_TOL, ANGLE_TOL = 1e-12, 1e-5
_FIX = None


def metrics_fixture():
    global _FIX
    if _FIX is None:
        _FIX = torch.load(os.path.join(GOLD, "metrics.pt"), weights_only=False)
    return _FIX


def ratio(got, ref, tol, spread=None):
    """max |got - ref| / bound with bound = tol (1 + |ref|), plus the fp32 / fp64 spread of the reference where given.
    NaN must meet NaN."""
    got, ref = got.detach().double().cpu(), torch.as_tensor(ref).double().cpu()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    assert torch.equal(torch.isnan(got), torch.isnan(ref)), (got, ref)
    ok = ~torch.isnan(ref)
    if not bool(ok.any()):
        return 0.0
    bound = tol * (1.0 + ref.abs())
    if spread is not None:
        bound = bound + torch.as_tensor(spread).double().cpu().abs()
    return float(((got - ref).abs() / bound)[ok].max())


def angle_ratio(got, ref, spread=None):
    got, ref = got.detach().double().cpu(), torch.as_tensor(ref).double().cpu()
    bound = torch.full_like(ref, ANGLE_TOL)
    if spread is not None:
        bound = bound + torch.as_tensor(spread).double().cpu().abs()
    return float(((got - ref).abs() / bound).max())


def rigid_inputs(name):
    nf, N, seed = C.RIGID_CASES[name]
    gt, pred = C.rigids(nf, N, seed)
    assert torch.equal(C.checksum(gt, pred), metrics_fixture()["rigid"][name]["check"])
    return gt, pred


def atom_inputs(name):
    nf, N, seed, kind = C.ATOM_CASES[name]
    gt, pred, mask = C.atoms(nf, N, seed, kind)
    assert torch.equal(C.checksum(gt, pred, mask), metrics_fixture()["atoms"][name]["check"])
    return gt, pred, mask


def kabsch_inputs(name):
    ref, x = C.point_sets(name, C.KABSCH_CASES[name])
    assert torch.equal(C.checksum(ref, x), metrics_fixture()["kabsch"][name]["check"])
    return ref, x


def eval_inputs():
    w = C.eval_window()
    assert torch.equal(C.checksum(*w.values()), metrics_fixture()["eval_window"]["check"])
    return w


def check_rigid(name, got, prec):
    """got = (ave_rot, ave_trans, ref_ave_rot, ref_ave_trans) of the prediction run as `prec` against the fixture."""
    c = metrics_fixture()["rigid"][name]
    ref = c["fp64"]["calc"]
    spread = [a - b for a, b in zip(c["fp32"]["calc"], c["fp64"]["calc"])] if prec == "fp32" else [None] * 4
    return {"ave_rot": angle_ratio(got[0], ref[0], spread[0]), "ave_trans": ratio(got[1], ref[1], SUM_TOL, spread[1]),
            "ref_ave_rot": angle_ratio(got[2], ref[2]), "ref_ave_trans": ratio(got[3], ref[3], SUM_TOL)}


def check_validation(got, c, prec):
    ref = c["fp64"]["validation"]
    out = {}
    for k in ("rmsd_all", "rmsd_ca", "drmsd_ca", "rmsd_ca_aligned"):
        spread = c["fp32"]["validation"][k].double() - ref[k].double() if prec == "fp32" else None
        out[k] = ratio(got[k], ref[k], SUM_TOL, spread)
    return out


def check_eval_row(got, prec):
    c = metrics_fixture()["eval_window"]
    ref = c["fp64"]["eval_fn"]
    sp = (lambda k: c["fp32"]["eval_fn"][k].double() - ref[k].double()) if prec == "fp32" else (lambda k: None)
    return {"ave_rot": angle_ratio(got["ave_rot"], ref["ave_rot"], sp("ave_rot")),
            **{k: ratio(got[k], ref[k], SUM_TOL, sp(k)) for k in ("ave_trans", "all_atom_mae", "all_atom_mse", "all_atom_rmsd")}}


# ------------------------------------------------------------------------------------------------------------------
# the oracle against the reference
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(C.RIGID_CASES))
@pytest.mark.parametrize("prec", ["fp32", "fp64"])
def test_oracle_rot_trans_error_matches_reference(name, prec):
    gt, pred = rigid_inputs(name)
    c = metrics_fixture()["rigid"][name]
    got = MO.rot_trans_error(pred if prec == "fp32" else pred.double(), gt)
    worst = check_rigid(name, got, prec)
    assert all(v <= 1.0 for v in worst.values()), worst
    # the direct calls agree with the method (the method is these two calls)
    assert torch.equal(c[prec]["quat"], c[prec]["calc"][0]) and torch.equal(c[prec]["trans"], c[prec]["calc"][1])


@pytest.mark.parametrize("name", list(C.ATOM_CASES))
@pytest.mark.parametrize("prec", ["fp32", "fp64"])
def test_oracle_validation_metrics_match_reference(name, prec):
    gt, pred, mask = atom_inputs(name)
    c = metrics_fixture()["atoms"][name]
    p = pred if prec == "fp32" else pred.double()
    worst = check_validation(MO.validation_metrics_all(gt, p, mask), c, prec)
    assert all(v <= 1.0 for v in worst.values()), worst
    assert ratio(MO.drmsd(p[..., 1, :] * mask[..., 1, None], gt[..., 1, :] * mask[..., 1, None], mask[..., 1]),
                 c[prec]["drmsd_ca"], SUM_TOL) <= 1.0
    assert ratio(MO.drmsd(p[..., 1, :], gt[..., 1, :]), c[prec]["drmsd_ca_nomask"], SUM_TOL) <= 1.0


def test_fixture_covers_the_traps():
    """The masks of the atom cases differ between frames (so n = min over frames matters), one frame is empty (NaN MAE,
    dRMSD 0), and rmsd_* carry the +1e-4 (an exact recomputation without it differs)."""
    gt, pred, mask = atom_inputs("atoms_24")
    counts = mask[..., 1].sum(-1)
    assert float(counts.min()) < float(counts.max())
    v = metrics_fixture()["atoms"]["atoms_24"]["fp64"]["validation"]
    d = gt * mask[..., None] - pred.double() * mask[..., None]
    no_eps = torch.sqrt((d ** 2).sum(dim=(-1, -2, -3)) / mask.sum(dim=(-1, -2)))
    assert float(((no_eps - v["rmsd_all"]).abs() / v["rmsd_all"]).max()) > 1e-9
    e = metrics_fixture()["atoms"]["atoms_empty_frame"]["fp64"]["validation"]
    assert float(e["drmsd_ca"].abs().max()) == 0.0
    _, _, m2 = atom_inputs("atoms_empty_frame")
    assert torch.isnan(MO.atom_errors(pred, gt, m2)["mae"][1])


@pytest.mark.parametrize("name", list(C.KABSCH_CASES))
def test_oracle_kabsch_matches_reference_rmsdalign(name):
    ref, x = kabsch_inputs(name)
    g = metrics_fixture()["kabsch"][name]
    sup, rmsd, R, _ = MO.kabsch(ref, x)
    assert ratio(rmsd, g["rmsd"], SUM_TOL) <= 1.0
    assert abs(float(torch.linalg.det(R)) - 1.0) < 1e-12
    if float(MO.key_matrix_gap(ref, x)) > 1e-6:          # a unique optimum: the coordinates agree too
        assert ratio(sup, g["superimposed"], SUM_TOL) <= 1.0


def test_oracle_window_metrics_match_eval_fn():
    w = eval_inputs()
    for prec in ("fp32", "fp64"):
        cast = (lambda t: t) if prec == "fp32" else (lambda t: t.double())
        got = MO.window_metrics(cast(w["rigid_pred"]), cast(w["atom37_pred"]), w["rigids_0"], w["atom37_pos"], w["atom37_mask"])
        worst = check_eval_row(got, prec)
        assert all(v <= 1.0 for v in worst.values()), (prec, worst)
        vm = MO.validation_metrics_all(w["atom37_pos"], cast(w["atom37_pred"]), w["atom37_mask"])
        worst = check_validation(vm, metrics_fixture()["eval_window"], prec)
        assert all(v <= 1.0 for v in worst.values()), (prec, worst)
    # the quirk: without it the mask keeps one more atom and MAE moves
    got = MO.window_metrics(w["rigid_pred"], w["atom37_pred"], w["rigids_0"], w["atom37_pos"], w["atom37_mask"], drop_last_atom=False)
    assert w["atom37_mask"][-1, -1, -1] == 1.0
    assert float(got["all_atom_mae"][0]) != float(metrics_fixture()["eval_window"]["fp32"]["eval_fn"]["all_atom_mae"][0])


# ------------------------------------------------------------------------------------------------------------------
# the oracle's Kabsch against scipy
# ------------------------------------------------------------------------------------------------------------------
def _scipy_rmsd(ref, x, w=None):
    ref, x = ref.double(), x.double()
    w = torch.ones(ref.shape[0], dtype=torch.float64) if w is None else w.double()
    W = w.sum()
    rc = ref - (w[:, None] * ref).sum(0) / W
    xc = x - (w[:, None] * x).sum(0) / W
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", UserWarning)
        rot, _ = Rotation.align_vectors(rc.numpy(), xc.numpy(), weights=w.numpy())
    y = xc @ torch.from_numpy(rot.as_matrix()).mT
    return torch.sqrt((w * ((y - rc) ** 2).sum(-1)).sum() / W)


@pytest.mark.parametrize("name", list(C.KABSCH_CASES))
def test_oracle_kabsch_matches_scipy(name):
    ref, x = kabsch_inputs(name)
    _, rmsd, R, t = MO.kabsch(ref, x)
    if ref.shape[0] == 1:                    # one point: nothing to rotate (scipy refuses zero vectors)
        assert float(rmsd) == 0.0
        return
    want = _scipy_rmsd(ref, x)
    assert abs(float(rmsd) - float(want)) <= 1e-12 * max(float(want), 1e-300) + 1e-13, (float(rmsd), float(want))
    assert torch.allclose(R @ R.mT, torch.eye(3, dtype=torch.float64), atol=1e-13)


def test_oracle_kabsch_weights_and_empty():
    ref, x = kabsch_inputs("random")
    w = (torch.arange(ref.shape[0]) % 3 != 0).double()
    _, rmsd, _, _ = MO.kabsch(ref, x, w)
    sel = w > 0
    _, rsel, _, _ = MO.kabsch(ref[sel], x[sel])
    assert abs(float(rmsd) - float(rsel)) <= 1e-12 * float(rsel)
    assert abs(float(rmsd) - float(_scipy_rmsd(ref, x, w))) <= 1e-12 * float(rsel)
    sup, rmsd0, R0, t0 = MO.kabsch(ref, x, torch.zeros(ref.shape[0], dtype=torch.float64))
    assert math.isnan(float(rmsd0)) and torch.equal(R0, torch.eye(3, dtype=torch.float64)) and torch.equal(sup, x)
    assert float(t0.abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------------------------
# host-side contract
# ------------------------------------------------------------------------------------------------------------------
def test_metric_wrappers_refuse_cpu_tensors():
    r = torch.zeros(3, 4, 7)
    a = torch.zeros(3, 4, 37, 3)
    m = torch.ones(3, 4, 37)
    for call in (lambda: M.rot_trans_error(r, r), lambda: M.atom_errors(a, a, m), lambda: M.superimpose(a[0, 0], a[0, 0]),
                 lambda: M.drmsd(a[..., 1, :], a[..., 1, :], m[..., 1]), lambda: M.validation_metrics_all(a, a, m),
                 lambda: M.window_metrics(r, a, r, a, m)):
        with pytest.raises(RuntimeError, match="CUDA"):
            call()


def test_evaluate_window_needs_the_targets():
    with pytest.raises(ValueError, match="atom37_pos"):
        M.evaluate_window(None, {"rigids_0": torch.zeros(2, 3, 7)}, 2, 0.01)


def test_metric_entry_points_validate_arguments():
    """Rejected before anything touches a device (fake non-null pointers are never dereferenced)."""
    L = K.lib()
    P = ctypes.c_void_p(16)
    cases = [
        (lambda: L.dfold_rot_trans_error(None, 0, P, 0, 3, 4, 1, P, None), "null pointer"),
        (lambda: L.dfold_rot_trans_error(P, 0, P, 0, 0, 4, 0, P, None), "nf >= 1"),
        (lambda: L.dfold_rot_trans_error(P, 0, P, 0, 3, 4, 3, P, None), "ref_frame 3 outside"),
        (lambda: L.dfold_rot_trans_error(P, 0, P, 0, 3, 4, -1, P, None), "ref_frame -1 outside"),
        (lambda: L.dfold_atom_errors(P, 0, P, 0, P, 0, 3, 4, 1, 1, P, None), "A = 1"),
        (lambda: L.dfold_atom_errors(P, 0, P, 0, None, 0, 3, 4, 37, 1, P, None), "null pointer"),
        (lambda: L.dfold_superimpose(P, 0, P, 0, 12, 3, None, 0, 4, 1, 1, 2, 4, P, None, None, None, None), "needs a mask"),
        (lambda: L.dfold_superimpose(P, 0, P, 0, 12, 3, P, 0, 4, 1, 3, 2, 4, P, None, None, None, None), "mask_mode 3"),
        (lambda: L.dfold_superimpose(P, 0, P, 0, 12, 2, None, 0, 0, 0, 0, 2, 4, P, None, None, None, None), "bad strides"),
        (lambda: L.dfold_superimpose(P, 0, P, 0, 12, 3, None, 0, 0, 0, 0, 2, 0, P, None, None, None, None), "P >= 1"),
        (lambda: L.dfold_drmsd(P, 0, P, 0, 12, 3, None, 0, 0, 0, 1, 2, 4, P, P, None), "premul needs a mask"),
        (lambda: L.dfold_drmsd(P, 0, P, 0, 12, 3, None, 0, 0, 0, 0, 70000, 4, P, P, None), "exceeds 65535"),
        (lambda: L.dfold_drmsd(P, 0, P, 0, 12, 3, None, 0, 0, 0, 0, 2, 4, None, P, None), "null pointer"),
    ]
    for call, msg in cases:
        assert call() == 1
        assert msg in L.dfold_last_error().decode() or pytest.fail(f"{msg!r} not in {L.dfold_last_error().decode()!r}")
