"""-m gpu: the metric kernels (csrc/metrics.cu) through dynamicpdb_b200/metrics.py against the fp64 oracle
(oracle/metrics_oracle.py) at the evaluation shapes, and against the unmodified reference (tests/golden/metrics.pt);
large offsets, reproducible bits, guard regions, graph capture, and the prefetcher -> sampler -> metrics loop.
Bounds and their derivation: tests/test_cpu_metrics.py (fp64 sums 1e-12 (1 + |ref|), angles 1e-5 degrees, fp32
predictions within the reference's own fp32 / fp64 spread plus those).  Rotations are compared to 1e-10 where the top
two eigenvalues of the key matrix are separated (relative gap > 1e-6); elsewhere only the RMSD is."""
import numpy as np
import pytest
import torch

from dynamicpdb_b200 import metrics as M
from oracle import metrics_cases as C
from oracle import metrics_oracle as MO
from tests.test_cpu_metrics import (SUM_TOL, angle_ratio, atom_inputs, check_eval_row, check_rigid, check_validation,
                                    eval_inputs, kabsch_inputs, metrics_fixture, ratio, rigid_inputs)

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROT_TOL = 1e-10
SHAPES = [(5, 256), (32, 256), (64, 256), (8, 1024), (3, 130), (3, 1), (3, 2)]


def _window(nf, N, seed):
    g_r, p_r = C.rigids(nf, N, seed)
    g_a, p_a, m = C.atoms(nf, N, seed + 1, "per_frame")
    return {k: v.to(DEV) for k, v in dict(rigids_0=g_r, rigid_pred=p_r, atom37_pos=g_a, atom37_pred=p_a, atom37_mask=m).items()}


def _worst(d, into):
    for k, v in d.items():
        into[k] = max(into.get(k, 0.0), v)


WORST = {}


@pytest.mark.parametrize("nf,N", SHAPES)
@pytest.mark.parametrize("prec", ["fp32", "fp64"])
def test_kernels_match_oracle(nf, N, prec):
    w = _window(nf, N, 1000 + nf + N)
    cast = (lambda t: t) if prec == "fp32" else (lambda t: t.double())
    rp, ap = cast(w["rigid_pred"]), cast(w["atom37_pred"])
    got = M.rot_trans_error(rp, w["rigids_0"])
    ref = MO.rot_trans_error(rp, w["rigids_0"])
    r = {"ave_rot": angle_ratio(got[0], ref[0]), "ave_trans": ratio(got[1], ref[1], SUM_TOL),
         "ref_ave_rot": angle_ratio(got[2], ref[2]), "ref_ave_trans": ratio(got[3], ref[3], SUM_TOL)}
    for drop in (False, True):
        ge, re_ = M.atom_errors(ap, w["atom37_pos"], w["atom37_mask"], drop), MO.atom_errors(ap, w["atom37_pos"], w["atom37_mask"], drop)
        for k in ge:
            r[k] = max(r.get(k, 0.0), ratio(ge[k], re_[k], SUM_TOL))
    gv, rv = M.validation_metrics_all(w["atom37_pos"], ap, w["atom37_mask"]), MO.validation_metrics_all(w["atom37_pos"], ap, w["atom37_mask"])
    for k in rv:
        r[k] = ratio(gv[k], rv[k], SUM_TOL)
    gw = M.window_metrics(rp, ap, w["rigids_0"], w["atom37_pos"], w["atom37_mask"])
    ow = MO.window_metrics(rp, ap, w["rigids_0"], w["atom37_pos"], w["atom37_mask"])
    r["all_atom_rmsd"] = ratio(gw["all_atom_rmsd"], ow["all_atom_rmsd"], SUM_TOL)
    for k in ow["per_frame"]:
        assert gw["per_frame"][k].shape == (nf,) and gw["per_frame"][k].dtype == torch.float64
    # dRMSD without a mask and superposition of every frame's CA set (rotations where unique)
    ca_g, ca_p = w["atom37_pos"][..., 1, :], ap[..., 1, :]
    r["drmsd_nomask"] = ratio(M.drmsd(ca_p, ca_g), MO.drmsd(ca_p, ca_g), SUM_TOL)
    sup, rmsd, R, t = M.superimpose(ca_g, ca_p, w["atom37_mask"][..., 1], return_transform=True)
    osup, ormsd, oR, ot = MO.kabsch(ca_g, ca_p, w["atom37_mask"][..., 1])
    r["sup_rmsd"] = ratio(rmsd, ormsd, SUM_TOL)
    gap = MO.key_matrix_gap(ca_g, ca_p, w["atom37_mask"][..., 1])
    uniq = gap > 1e-6
    if bool(uniq.any()):
        r["rotation_abs"] = float((R - oR).abs()[uniq].max()) / ROT_TOL
        assert ratio(sup[uniq], osup[uniq], 1e-10) <= 1.0
    _worst(r, WORST)
    print(f"[metrics vs oracle] {nf}x{N} {prec}: {r}")
    assert all(v <= 1.0 for v in r.values()), r


@pytest.mark.parametrize("name", list(C.RIGID_CASES))
@pytest.mark.parametrize("prec", ["fp32", "fp64"])
def test_rot_trans_error_matches_reference(name, prec):
    gt, pred = rigid_inputs(name)
    got = M.rot_trans_error((pred if prec == "fp32" else pred.double()).to(DEV), gt.to(DEV))
    worst = check_rigid(name, got, prec)
    print(f"[metrics vs reference] rigid {name} {prec}: {worst}")
    assert all(v <= 1.0 for v in worst.values()), worst


@pytest.mark.parametrize("name", list(C.ATOM_CASES))
@pytest.mark.parametrize("prec", ["fp32", "fp64"])
def test_validation_metrics_match_reference(name, prec):
    gt, pred, mask = atom_inputs(name)
    c = metrics_fixture()["atoms"][name]
    p = (pred if prec == "fp32" else pred.double()).to(DEV)
    g, m = gt.to(DEV), mask.to(DEV)
    worst = check_validation(M.validation_metrics_all(g, p, m), c, prec)
    worst["drmsd_ca"] = max(worst["drmsd_ca"], ratio(M.drmsd(p[..., 1, :] * m[..., 1, None], g[..., 1, :] * m[..., 1, None], m[..., 1]),
                                                     c[prec]["drmsd_ca"], SUM_TOL))
    worst["drmsd_nomask"] = ratio(M.drmsd(p[..., 1, :], g[..., 1, :]), c[prec]["drmsd_ca_nomask"], SUM_TOL)
    print(f"[metrics vs reference] atoms {name} {prec}: {worst}")
    assert all(v <= 1.0 for v in worst.values()), worst


@pytest.mark.parametrize("name", list(C.KABSCH_CASES))
def test_superimpose_matches_reference_rmsdalign(name):
    ref, x = kabsch_inputs(name)
    g = metrics_fixture()["kabsch"][name]
    sup, rmsd, R, t = M.superimpose(ref.to(DEV), x.to(DEV), return_transform=True)
    worst = {"rmsd": ratio(rmsd, g["rmsd"], SUM_TOL)}
    Rc = R.cpu()
    assert float((Rc @ Rc.mT - torch.eye(3, dtype=torch.float64)).abs().max()) < 1e-13
    assert abs(float(torch.linalg.det(Rc)) - 1.0) < 1e-13
    assert ratio(sup, x.to(DEV) @ R.mT + t, 1e-13) <= 1.0
    if float(MO.key_matrix_gap(ref, x)) > 1e-6:
        worst["superimposed"] = ratio(sup, g["superimposed"], SUM_TOL)
    print(f"[metrics vs reference] kabsch {name}: {worst}")
    assert all(v <= 1.0 for v in worst.values()), worst


def test_window_metrics_match_eval_fn():
    w = {k: v.to(DEV) for k, v in eval_inputs().items()}
    for prec in ("fp32", "fp64"):
        cast = (lambda t: t) if prec == "fp32" else (lambda t: t.double())
        got = M.window_metrics(cast(w["rigid_pred"]), cast(w["atom37_pred"]), w["rigids_0"], w["atom37_pos"], w["atom37_mask"])
        worst = check_eval_row(got, prec)
        worst.update(check_validation(M.validation_metrics_all(w["atom37_pos"], cast(w["atom37_pred"]), w["atom37_mask"]),
                                      metrics_fixture()["eval_window"], prec))
        print(f"[metrics vs reference] eval window {prec}: {worst}")
        assert all(v <= 1.0 for v in worst.values()), (prec, worst)


@pytest.mark.parametrize("offset", [1e3, 1e5])
def test_superimpose_large_offsets(offset):
    """Centroids and covariance in separate passes: moving both sets far from the origin leaves the RMSD (to 1e-9 A) and
    the rotation unchanged, and an exact rotated copy superimposes to below 1e-9 A."""
    rs = np.random.RandomState(7)
    ref = torch.from_numpy(rs.randn(64, 256, 3) * 10.0).to(DEV)
    x = ref + torch.from_numpy(rs.randn(64, 256, 3) * 0.5).to(DEV)
    _, r0, R0, _ = M.superimpose(ref, x, return_transform=True)
    shift = torch.tensor([offset, -0.7 * offset, 0.3 * offset], dtype=torch.float64, device=DEV)
    _, r1, R1, _ = M.superimpose(ref + shift, x + shift, return_transform=True)
    assert float((r1 - r0).abs().max()) < 1e-9
    assert float((R1 - R0).abs().max()) < 1e-9
    Rt = torch.from_numpy(np.stack([C._rotmats(rs, 1)[0] for _ in range(64)])).to(DEV)
    y = torch.einsum("bij,bpj->bpi", Rt, ref) + shift
    sup, r2 = M.superimpose(ref + shift, y)
    assert float(r2.max()) < 1e-9, float(r2.max())
    assert float((sup - (ref + shift)).abs().max()) < 1e-9 * 10


def test_reproducible_bits_and_guards():
    """Two launches give the same bits; outputs written into NaN-filled oversized buffers leave everything else NaN."""
    w = _window(64, 256, 5)
    calls = lambda: (M.rot_trans_error(w["rigid_pred"], w["rigids_0"]),
                     M.validation_metrics_all(w["atom37_pos"], w["atom37_pred"], w["atom37_mask"]),
                     M.window_metrics(w["rigid_pred"], w["atom37_pred"], w["rigids_0"], w["atom37_pos"], w["atom37_mask"]),
                     M.superimpose(w["atom37_pos"][..., 1, :], w["atom37_pred"][..., 1, :]))
    flat = lambda o: torch.cat([t.reshape(-1) for t in _leaves(o)])
    a, b = flat(calls()), flat(calls())
    assert torch.equal(a.view(torch.int64), b.view(torch.int64))
    # guard regions: call the entry points on buffers with NaN margins through the raw ABI
    from dynamicpdb_b200 import kernels as K
    nf, N = 64, 256
    g = w["rigids_0"].contiguous()
    p = w["rigid_pred"].contiguous()
    buf = torch.full((4 * nf + 64,), float("nan"), dtype=torch.float64, device=DEV)
    assert K.lib().dfold_rot_trans_error(K._ptr(p), 0, K._ptr(g), 1, nf, N, nf - 2, K._ptr(buf, 32), K._stream()) == 0
    assert bool(torch.isnan(buf[:32]).all()) and bool(torch.isnan(buf[32 + 4 * nf:]).all())
    assert bool(torch.isfinite(buf[32:32 + 4 * nf]).all())
    ca_g = w["atom37_pos"][..., 1, :].contiguous()
    ca_p = w["atom37_pred"][..., 1, :].contiguous()
    T = (N + 63) // 64
    part = torch.full((nf * T * T + 64,), float("nan"), dtype=torch.float64, device=DEV)
    out = torch.full((nf + 64,), float("nan"), dtype=torch.float64, device=DEV)
    assert K.lib().dfold_drmsd(K._ptr(ca_p), 0, K._ptr(ca_g), 1, 3 * N, 3, None, 0, 0, 0, 0, nf, N, K._ptr(part, 32), K._ptr(out, 32),
                               K._stream()) == 0
    assert bool(torch.isnan(part[:32]).all()) and bool(torch.isnan(part[32 + nf * T * T:]).all())
    assert bool(torch.isnan(out[:32]).all()) and bool(torch.isnan(out[32 + nf:]).all()) and bool(torch.isfinite(out[32:32 + nf]).all())
    rm = torch.full((nf + 64,), float("nan"), dtype=torch.float64, device=DEV)
    co = torch.full((nf * N * 3 + 64,), float("nan"), dtype=torch.float64, device=DEV)
    assert K.lib().dfold_superimpose(K._ptr(ca_g), 1, K._ptr(ca_p), 0, 3 * N, 3, None, 0, 0, 0, 0, nf, N, K._ptr(rm, 32), None, None,
                                     K._ptr(co, 32), K._stream()) == 0
    assert bool(torch.isnan(rm[:32]).all()) and bool(torch.isnan(rm[32 + nf:]).all())
    assert bool(torch.isnan(co[:32]).all()) and bool(torch.isnan(co[32 + nf * N * 3:]).all())
    am = torch.full((6 * nf + 64,), float("nan"), dtype=torch.float64, device=DEV)
    assert K.lib().dfold_atom_errors(K._ptr(w["atom37_pred"]), 0, K._ptr(w["atom37_pos"]), 1, K._ptr(w["atom37_mask"]), 1, nf, N, 37, 1,
                                     K._ptr(am, 32), K._stream()) == 0
    assert bool(torch.isnan(am[:32]).all()) and bool(torch.isnan(am[32 + 6 * nf:]).all())


def _leaves(o):
    if torch.is_tensor(o):
        return [o]
    if isinstance(o, dict):
        return [x for v in o.values() for x in _leaves(v)]
    return [x for v in o for x in _leaves(v)]


def test_empty_and_degenerate_sets():
    ref = torch.randn(4, 5, 3, dtype=torch.float64, device=DEV) * 10
    x = torch.randn(4, 5, 3, dtype=torch.float64, device=DEV) * 10
    mask = torch.ones(4, 5, dtype=torch.float64, device=DEV)
    mask[1] = 0.0
    mask[2, 1:] = 0.0                 # one point
    mask[3, 2:] = 0.0                 # two points
    sup, rmsd, R, t = M.superimpose(ref, x, mask, return_transform=True)
    assert torch.isnan(rmsd[1]) and torch.equal(R[1], torch.eye(3, dtype=torch.float64, device=DEV)) and torch.equal(sup[1], x[1])
    _, ormsd, _, _ = MO.kabsch(ref, x, mask)
    assert ratio(rmsd, ormsd, SUM_TOL) <= 1.0
    assert float(rmsd[2]) < 1e-12
    # dRMSD: n <= 1 gives 0
    m1 = torch.zeros(2, 5, dtype=torch.float64, device=DEV)
    m1[:, 0] = 1.0
    assert float(M.drmsd(ref[:2], x[:2], m1).abs().max()) == 0.0


def test_metrics_capture_in_a_cuda_graph():
    w = _window(32, 256, 9)
    static = {k: v.clone() for k, v in w.items()}
    run = lambda d: (M.window_metrics(d["rigid_pred"], d["atom37_pred"], d["rigids_0"], d["atom37_pos"], d["atom37_mask"]),
                     M.validation_metrics_all(d["atom37_pos"], d["atom37_pred"], d["atom37_mask"]))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run(static)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        res = run(static)
    w2 = _window(32, 256, 10)
    for k, v in w2.items():
        static[k].copy_(v)
    g.replay()
    eager = run(w2)
    a, b = torch.cat([t.reshape(-1) for t in _leaves(res)]), torch.cat([t.reshape(-1) for t in _leaves(eager)])
    assert torch.equal(a.view(torch.int64), b.view(torch.int64))


@pytest.mark.timeout(600)
def test_prefetcher_targets_and_evaluate_window(tmp_path):
    from dynamicpdb_b200 import synthetic as syn
    from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
    from dynamicpdb_b200.inference import DeviceReverseDiffusion
    from dynamicpdb_b200.input_pipeline import TrajectoryStore, WindowPrefetcher
    from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
    from oracle import synth_traj
    row = synth_traj.write_files(synth_traj.make_trajectory(), str(tmp_path))
    store = TrajectoryStore(frame_time=3, frame_sample_step=2, keep_first=8)
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    plain = list(WindowPrefetcher(store, [row], DEV, training=False, diffuser=diffuser))[0]
    it = list(WindowPrefetcher(store, [row], DEV, training=False, diffuser=diffuser, targets=True))[0]
    assert set(it) - set(plain) == {"atom37_pos", "atom37_mask"}
    assert it["atom37_pos"].shape == (3, 17, 37, 3) and it["atom37_pos"].dtype == torch.float64
    assert it["atom37_mask"].shape == (3, 17, 37) and it["atom37_mask"].dtype == torch.float64
    assert set(plain) == {"rigids_0", "torsion_angles_sin_cos", "alt_torsion_angles_sin_cos", "torsion_angles_mask", "res_mask",
                          "aatype", "seq_idx", "residue_index", "force", "vel", "node_repr", "edge_repr", "fixed_mask", "sc_ca_t",
                          "rigids_t", "t"}
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(3, **syn.PRESET_TINY), SE3ScoreDiffuser(syn.diffuser_conf(1.0))).to(DEV)
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    sampler = DeviceReverseDiffusion(net)
    got = M.evaluate_window(sampler, it, 4, 0.01)
    # the same sampler output through the oracle: the graph's result buffers still hold this call's sample
    (_, static, _, res), = sampler._graphs.values()
    assert "atom37_pos" not in static and "atom37_mask" not in static
    assert torch.equal(static["seq_idx"][0].cpu(), torch.arange(1, 18))
    want = MO.window_metrics(res["rigid_pred"], res["prot_traj"][0], it["rigids_0"], it["atom37_pos"], it["atom37_mask"])
    for k in ("ave_rot", "ave_trans", "all_atom_mae", "all_atom_mse", "all_atom_rmsd"):
        assert got[k].shape == (1,) and got[k].is_cuda
        tol = angle_ratio(got[k], want[k]) if k == "ave_rot" else ratio(got[k], want[k], SUM_TOL)
        assert tol <= 1.0, (k, tol)
