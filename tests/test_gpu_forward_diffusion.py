"""-m gpu: forward diffusion on the device (csrc/diffuse.cu): the IGSO(3) tables, forward_marginal and sample_ref against the
unmodified reference (tests/golden/forward.pt, same numpy draws injected) and against the fp64 oracle at the training
shapes; np.interp's edge rules, the sampled distributions, determinism, graph capture, and the noising prefetcher feeding
a training step and the sampler."""
import math

import numpy as np
import pytest
import torch

from dynamicpdb_b200 import kernels as K
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from oracle import dfold_oracle as O
from oracle import forward_oracle as FO
from tests.test_cpu_forward_diffusion import (SCORE_TOL, SCALING_TOL, case_diffuser, case_draws, check_against_reference,
                                              forward_fixture, max_ratio, rotmats)

pytestmark = pytest.mark.gpu
DEV = "cuda"
WORST = {}


def _dev(d):
    return {k: v.to(DEV) for k, v in d.items()}


@pytest.mark.parametrize("name", ["t037", "t001", "t1", "mask", "norot", "ref", "small_grid"])
def test_kernel_matches_reference_golden(name):
    g = forward_fixture()
    c = g["cases"][name]
    rig7 = g["rigids_0"]
    n = rig7[..., 0].numel()
    draws = _dev(case_draws(c, n))
    if c["sample_ref"]:
        d = case_diffuser(c, frame_time=rig7.shape[0])
        out = d.sample_ref(n, draws=draws)
    else:
        d = case_diffuser(c)
        out = d.forward_marginal(rig7.to(DEV), c["t"], diffuse_mask=g["mask"].to(DEV) if c["mask"] else None, draws=draws)
        assert out["rot_score"].dtype == torch.float64 and out["trans_score"].dtype == torch.float64
        assert out["rot_score_scaling"].dtype == torch.float64 and out["rot_score_scaling"].shape == ()
    assert out["rigids_t"].dtype == torch.float32 and out["rigids_t"].shape == c["out"]["rigids_t"].shape
    q = out["rigids_t"][..., :4].double()
    assert float((q.norm(dim=-1) - 1).abs().max()) < 1e-6
    if c["diffuse_rot"]:                     # noised rotations come out with w >= 0; kept ones are rigids_0's own bits
        noised = g["mask"].to(DEV) > 0.5 if c["mask"] else torch.ones(q.shape[:-1], dtype=torch.bool, device=DEV)
        assert bool((q[..., 0][noised] >= 0).all())
    worst = check_against_reference({k: v.cpu() if torch.is_tensor(v) else v for k, v in out.items()}, c["out"], c)
    WORST[name] = worst
    print(f"[forward parity] {name}: worst |err|/bound {worst}")
    assert all(v <= 1.0 for v in worst.values()), worst


@pytest.mark.parametrize("grid", [(1000, 1000), (250, 120)])
def test_tables_match_oracle_and_are_reproducible(grid):
    num_omega, num_sigma = grid
    dc = O.default_diffuser_conf(1.0)
    dc.num_sigma, dc.num_omega = num_sigma, num_omega
    sig = torch.from_numpy(FO.discrete_sigma(dc)).to(DEV)
    cdf, sc = K.igso3_tables(sig, num_omega)
    cdf2, sc2 = K.igso3_tables(sig, num_omega)
    assert torch.equal(cdf, cdf2) and torch.equal(sc, sc2)
    ref = FO.igso3_tables(dc, device=DEV, chunk=32)
    # cdf entries are probabilities built from sums of up to L terms of size <= (2l+1): absolute 1e-12 covers the
    # different summation orders (sequential here, pairwise in torch) with a wide margin; score_scaling relative 1e-11
    err_cdf = (cdf - ref["cdf"]).abs().max().item()
    err_sc = ((sc - ref["score_scaling"]).abs() / ref["score_scaling"].abs()).max().item()
    print(f"[tables {grid}] max |cdf err| {err_cdf:.3e}, max rel score_scaling err {err_sc:.3e}")
    assert err_cdf < 1e-12 and err_sc < 1e-11
    # rows are non-decreasing up to a few ulps of 1: the rounding noise of the plateau where the pdf underflows (as in the
    # reference)
    assert (cdf[:, :-1] - cdf[:, 1:]).max().item() < 16 * 2.0 ** -52


def _oracle_vs_kernel(d, rig7, t, mask, draws, dc):
    out = d.forward_marginal(rig7, t, diffuse_mask=mask, draws=draws)
    cdf, sc = d.tables(DEV)
    idx = FO.sigma_idx(t, dc)
    ref = FO.forward_marginal(rig7, t, draws, dc, cdf[idx], float(sc[idx]), diffuse_mask=mask, diffuse_rot=d.diffuse_rot,
                             diffuse_trans=d.diffuse_trans)
    return out, ref


@pytest.mark.parametrize("shape", [(64, 256), (8, 1024), (3, 130)])
@pytest.mark.parametrize("variant", ["plain", "mask", "norot", "notrans"])
def test_kernel_matches_oracle_at_training_shapes(shape, variant):
    nf, N = shape
    conf = syn.diffuser_conf(0.1)
    conf.diffuse_rot, conf.diffuse_trans = variant != "norot", variant != "notrans"
    d = SE3ScoreDiffuser(conf)
    dc = O.default_diffuser_conf(0.1)
    rig7 = syn.make_feats(nf, N, seed=nf + N)["rigids_0"].to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(nf * N)
    n = nf * N
    draws = {"z_axis": torch.randn(n, 3, dtype=torch.float64, device=DEV, generator=gen),
             "u": torch.rand(n, dtype=torch.float64, device=DEV, generator=gen),
             "z_trans": torch.randn(n, 3, dtype=torch.float64, device=DEV, generator=gen)}
    mask = None
    if variant == "mask":
        mask = (torch.rand(nf, N, device=DEV, generator=gen) > 0.3).double()
    for t in (0.37, 0.01):
        out, ref = _oracle_vs_kernel(d, rig7, t, mask, draws, dc)
        # kernel and oracle share the cdf row and the draws: both sides are fp64 up to the final fp32 rounding of rigids_t
        assert (rotmats(out["rigids_t"]) - rotmats(ref["rigids_t"])).abs().max().item() < 1e-6
        xr = ref["rigids_t"][..., 4:]
        assert (out["rigids_t"][..., 4:].double() - xr).abs().max().item() < 1e-6 * max(1.0, xr.abs().max().item())
        assert max_ratio(out["rot_score"], ref["rot_score"], SCORE_TOL) <= 1.0
        assert max_ratio(out["trans_score"], ref["trans_score"], SCORE_TOL) <= 1.0
        assert abs(out["rot_score_scaling"].item() - ref["rot_score_scaling"]) <= SCALING_TOL * ref["rot_score_scaling"]
        assert abs(out["trans_score_scaling"].item() - ref["trans_score_scaling"]) <= SCALING_TOL * ref["trans_score_scaling"]
        if variant == "norot":
            assert torch.equal(out["rigids_t"][..., :4], rig7[..., :4]) and bool((out["rot_score"] == 0).all())
            assert out["rot_score_scaling"].item() == 1.0
        if variant == "notrans":
            assert torch.equal(out["rigids_t"][..., 4:], rig7[..., 4:]) and bool((out["trans_score"] == 0).all())
            assert out["trans_score_scaling"].item() == 1.0
        if mask is not None:
            fixed = mask == 0
            assert torch.equal(out["rigids_t"][fixed], rig7[fixed])
            assert bool((out["rot_score"][fixed] == 0).all()) and bool((out["trans_score"][fixed] == 0).all())


def _angles(rig7):
    q = rig7[..., :4].double()
    return 2 * torch.atan2(q[..., 1:].norm(dim=-1), q[..., 0])


@pytest.mark.parametrize("t", [0.01, 0.37])
def test_interp_edges_match_numpy(t):
    """u = 0 -> omega_0; u = 1 - 2^-53 -> pi where the row ends below it (t = 0.01; at t = 0.37 the row's rectangle-rule
    sum ends above 1 and u lies inside); exact cdf hits -> their node; midpoints -> the slope form; all as np.interp gives
    them from the kernel's own cdf row.  Points inside the underflow plateau (where the row moves by rounding noise only)
    are left out: there np.interp's guessed search and a plain bisection may pick different plateau nodes."""
    d = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    cdf, _ = d.tables(DEV)
    dc = O.default_diffuser_conf(1.0)
    row = cdf[FO.sigma_idx(t, dc)].cpu().numpy()
    om = np.linspace(0, np.pi, 1001)[1:]
    rising = np.nonzero(np.diff(row) > 1e-12)[0]
    u = np.concatenate([[0.0, 1.0 - 2.0 ** -53], row[rising], (row[rising] + row[rising + 1]) / 2])
    u = u[u < 1.0]
    n = u.size
    rig7 = torch.cat([torch.tensor([1.0, 0, 0, 0]).expand(n, 4), torch.zeros(n, 3)], -1).to(DEV)
    draws = {"z_axis": torch.tensor([[0.0, 0.0, 1.0]], dtype=torch.float64).expand(n, 3).to(DEV),
             "u": torch.from_numpy(u).to(DEV), "z_trans": torch.zeros(n, 3, dtype=torch.float64, device=DEV)}
    out = d.forward_marginal(rig7, t, draws=draws)
    got = _angles(out["rigids_t"].cpu()).numpy()
    want = np.interp(u, row, om)
    assert want[0] == om[0]
    if row.max() <= 1.0 - 2.0 ** -53:
        assert want[1] == np.pi
    assert np.abs(got - want).max() < 1e-6, np.abs(got - want).max()       # fp32 quaternion output: ~1e-7 rad


@pytest.mark.parametrize("t", [0.01, 0.37, 1.0])
def test_sampled_distribution(t):
    """2^20 draws from the device generator: the angles against the cdf row (KS), the axes isotropic, the translations with
    the marginal's mean and variance.  Thresholds: 6 standard deviations (KS: the alpha = 1e-8 quantile) at this n."""
    n = 1 << 20
    cs = 0.1
    d = SE3ScoreDiffuser(syn.diffuser_conf(cs))
    dc = O.default_diffuser_conf(cs)
    x0 = torch.tensor([1.0, -2.0, 3.0])
    rig7 = torch.cat([torch.tensor([1.0, 0, 0, 0]), x0]).expand(n, 7).contiguous().to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(123)
    out = d.forward_marginal(rig7, t, generator=gen)
    r = out["rigids_t"].double()
    ang = _angles(r).cpu().numpy()
    cdf, _ = d.tables(DEV)
    row = cdf[FO.sigma_idx(t, dc)].cpu().numpy()
    om = np.linspace(0, np.pi, 1001)[1:]
    x = np.sort(ang)
    F = np.where(x >= np.pi - 1e-5, 1.0, np.interp(x, om, row))
    i = np.arange(1, n + 1)
    D = max((i / n - F).max(), (F - (i - 1) / n).max())
    ks_thr = math.sqrt(-math.log(1e-8 / 2) / (2 * n))
    assert D < ks_thr, (D, ks_thr)
    axis = r[:, 1:4] / r[:, 1:4].norm(dim=-1, keepdim=True)
    assert axis.mean(0).abs().max().item() < 6 / math.sqrt(3 * n)
    second = (axis[:, :, None] * axis[:, None, :]).mean(0) - torch.eye(3, dtype=torch.float64, device=DEV) / 3
    assert second.abs().max().item() < 6 * math.sqrt(4 / 45) / math.sqrt(n)
    beta = t * dc.min_b + 0.5 * t * t * (dc.max_b - dc.min_b)
    sd = math.sqrt(1 - math.exp(-beta)) / cs
    xt = r[:, 4:]
    mean_err = (xt.mean(0).cpu() - math.exp(-beta / 2) * x0.double()).abs().max().item()
    assert mean_err < 6 * sd / math.sqrt(n)
    var_err = (xt.var(0).cpu() / sd ** 2 - 1).abs().max().item()
    assert var_err < 6 * math.sqrt(2 / n)


def test_two_launches_same_bits_and_nothing_else_written():
    """Raw C-ABI calls into NaN-filled buffers with guard regions on both sides: equal bits twice, guards untouched."""
    nf, N, pad = 4, 130, 64
    n = nf * N
    d = SE3ScoreDiffuser(syn.diffuser_conf(0.1))
    cdf, sc = d.tables(DEV)
    grid = d.grid(torch.device(DEV, torch.cuda.current_device()))
    rig7 = syn.make_feats(nf, N, seed=2)["rigids_0"].reshape(n, 7).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(9)
    za = torch.randn(n, 3, dtype=torch.float64, device=DEV, generator=gen)
    u = torch.rand(n, dtype=torch.float64, device=DEV, generator=gen)
    zt = torch.randn(n, 3, dtype=torch.float64, device=DEV, generator=gen)
    t64 = torch.tensor([0.37], dtype=torch.float64, device=DEV)
    outs = []
    for _ in range(2):
        rig = torch.full((n * 7 + 2 * pad,), float("nan"), device=DEV)
        rs = torch.full((n * 3 + 2 * pad,), float("nan"), dtype=torch.float64, device=DEV)
        ts = torch.full_like(rs, float("nan"))
        scal = torch.full((2 + 2 * pad,), float("nan"), dtype=torch.float64, device=DEV)
        K.launch("dfold_forward_marginal", rig7, za, u, zt, None, t64, grid, cdf, sc, grid.numel(), cdf.shape[1], 1000, 1.5, 0.1,
                 0.1, 20.0, 0.1, 1, 1, 0, K._ptr(rig, pad), K._ptr(rs, pad), K._ptr(ts, pad), K._ptr(scal, pad),
                 K._ptr(scal, pad + 1), n)
        for buf, m in ((rig, n * 7), (rs, n * 3), (ts, n * 3), (scal, 2)):
            assert bool(torch.isnan(buf[:pad]).all()) and bool(torch.isnan(buf[pad + m:]).all())
            assert bool(torch.isfinite(buf[pad:pad + m]).all())
        outs.append((rig, rs, ts, scal))
    for a, b in zip(*outs):
        assert torch.equal(a[pad:-pad].view(torch.int64 if a.dtype == torch.float64 else torch.int32),
                           b[pad:-pad].view(torch.int64 if b.dtype == torch.float64 else torch.int32))


def test_graph_capture():
    nf, N = 8, 64
    d = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    rig7 = syn.make_feats(nf, N, seed=5)["rigids_0"].to(DEV)
    t = torch.tensor([0.37], dtype=torch.float64, device=DEV)
    gen = torch.Generator(device=DEV).manual_seed(4)
    n = nf * N
    static = {"z_axis": torch.randn(n, 3, dtype=torch.float64, device=DEV, generator=gen),
              "u": torch.rand(n, dtype=torch.float64, device=DEV, generator=gen),
              "z_trans": torch.randn(n, 3, dtype=torch.float64, device=DEV, generator=gen)}
    eager = d.forward_marginal(rig7, t, draws=static)
    d.forward_marginal(rig7, t)                             # warm-up of the device-draw path outside the capture
    torch.cuda.synchronize()
    g1, g2 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.graph(g1):
        fresh = d.forward_marginal(rig7, t)                 # default CUDA generator: graph-aware, new draws per replay
    with torch.cuda.graph(g2):
        fixed = d.forward_marginal(rig7, t, draws=static)
    g1.replay()
    a = {k: v.clone() for k, v in fresh.items()}
    g1.replay()
    assert not torch.equal(a["rigids_t"], fresh["rigids_t"])
    for o in (a, fresh):
        assert bool(torch.isfinite(o["rigids_t"]).all()) and bool(torch.isfinite(o["rot_score"]).all())
        assert float((o["rigids_t"][..., :4].norm(dim=-1) - 1).abs().max()) < 1e-6
    g2.replay()
    for k in eager:
        assert torch.equal(fixed[k], eager[k]), k


def _synth_row(tmp_path):
    from oracle import synth_traj
    return synth_traj.write_files(synth_traj.make_trajectory(), str(tmp_path))


@pytest.mark.timeout(300)
def test_prefetcher_training_items_feed_a_train_step(tmp_path):
    from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
    from dynamicpdb_b200.input_pipeline import TrajectoryStore, WindowPrefetcher
    from dynamicpdb_b200.loss import score_network_loss
    from dynamicpdb_b200.train_step import TrainStep
    row = _synth_row(tmp_path)
    store = TrajectoryStore(frame_time=3, frame_sample_step=2, keep_first=8)
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    np.random.seed(5)
    gen = torch.Generator(device=DEV).manual_seed(11)
    items = list(WindowPrefetcher(store, [row] * 4, DEV, training=True, diffuser=diffuser, min_t=0.2, generator=gen))
    nf, N = 3, 17
    shapes = {"rigids_t": ((nf, N, 7), torch.float32), "rot_score": ((nf, N, 3), torch.float64),
              "trans_score": ((nf, N, 3), torch.float64), "rot_score_scaling": ((), torch.float64),
              "trans_score_scaling": ((), torch.float64), "t": ((1,), torch.float64)}
    ts_seen = []
    for it in items:
        for k, (shp, dt) in shapes.items():
            assert tuple(it[k].shape) == shp and it[k].dtype == dt and it[k].is_cuda, k
        t = it["t"].item()
        ts_seen.append(t)
        assert 0.2 <= t <= 1.0
        assert bool(torch.isfinite(it["rot_score"]).all()) and bool(torch.isfinite(it["rigids_t"]).all())
    assert len(set(ts_seen)) == len(ts_seen)
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(nf, **syn.PRESET_TINY), SE3ScoreDiffuser(syn.diffuser_conf(1.0))).to(DEV)
    keys = ("rigids_t", "rigids_0", "t", "rot_score", "trans_score", "rot_score_scaling", "trans_score_scaling", "res_mask",
            "fixed_mask", "seq_idx", "aatype", "torsion_angles_sin_cos", "alt_torsion_angles_sin_cos", "torsion_angles_mask",
            "sc_ca_t", "node_repr", "edge_repr", "force", "vel")
    # the loss reads its targets from `batch`; the network reads the step's static copy: both are refilled per item
    batch = {k: items[0][k].contiguous().clone() for k in keys if k in items[0]}
    exp_conf = O.default_exp_conf()
    step = TrainStep(net, lambda out: score_network_loss(out, batch, exp_conf)[0], batch, lr=1e-4, graph=True, warmup=2)
    for it in items[1:]:
        for k in batch:
            batch[k].copy_(it[k])
        step.load(batch)
        loss = float(step())
        assert math.isfinite(loss), loss


@pytest.mark.timeout(300)
def test_prefetcher_eval_item_feeds_the_sampler(tmp_path):
    from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
    from dynamicpdb_b200.inference import DeviceReverseDiffusion
    from dynamicpdb_b200.input_pipeline import TrajectoryStore, WindowPrefetcher
    row = _synth_row(tmp_path)
    store = TrajectoryStore(frame_time=3, frame_sample_step=2, keep_first=8)
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    items = list(WindowPrefetcher(store, [row], DEV, training=False, diffuser=diffuser))
    it = items[0]
    assert it["rigids_t"].shape == (3, 17, 7) and it["rigids_t"].dtype == torch.float32 and it["t"].item() == 1.0
    assert "rot_score" not in it
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(3, **syn.PRESET_TINY), SE3ScoreDiffuser(syn.diffuser_conf(1.0))).to(DEV)
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    feats = {k: v.contiguous() for k, v in it.items()}
    out = DeviceReverseDiffusion(net).sample_graphed(feats, 4, 0.01)
    assert bool(torch.isfinite(out["rigids"]).all()) and out["prot_traj"].shape[:3] == (4, 3, 17)
