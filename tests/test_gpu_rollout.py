"""-m gpu: the trajectory rollout (dynamicpdb_b200/rollout.py, csrc/rollout.cu).

* dfold_rollout_advance against a torch emulation, bit for bit, with sentinel-filled guard regions around every output, and
  no write at all once the counter has reached L;
* the default path (one graphed forward + advance per frame) against ``literal=True`` (the reference's schedule: fresh
  sample_ref draws and num_t full forwards per frame): the same bits;
* graph replay against the eager step, two rollouts against each other, and in-place weight changes between rollouts;
* the unmodified reference's eval_extension loop (tests/golden/rollout.pt): each stored input window gives the reference's
  next frame within the network bar (atoms: the atom37 bar), and a free-running rollout stays within the bars of
  tests/test_cpu_rollout.py;
* rollout lengths of 200 at the evaluation shapes, and the prefetcher -> rollout -> metrics loop against later MD frames."""
import pytest
import torch

from dynamicpdb_b200 import kernels as K
from dynamicpdb_b200 import metrics as M
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.rollout import TrajectoryRollout
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from oracle import metrics_oracle as MO
from tests.test_cpu_rollout import (ATOM_TOL, CASES, DRIFT_TOL, FREE_STEPS, NET_TOL, atom_l2, case_shapes,
                                    rollout_fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENTINEL = -7.125e5
GUARD_ROWS = 3


def _net(nf, preset, seed=0):
    torch.manual_seed(seed)
    net = FullScoreNetwork(syn.model_conf(nf, **preset), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    return net.to(DEV).eval()


def _window(nf, N, seed):
    return {k: v.to(DEV) for k, v in syn.make_feats(nf, N, seed=seed, loader_dtypes=True).items()}


def _guarded(shape, dtype=torch.float32, fill=SENTINEL):
    """A tensor of `shape` inside a buffer with GUARD_ROWS rows of `fill` before and after it (rows of shape[1:])."""
    buf = torch.full((shape[0] + 2 * GUARD_ROWS, *shape[1:]), fill, dtype=dtype, device=DEV)
    return buf, buf[GUARD_ROWS:GUARD_ROWS + shape[0]]


def _guards_intact(buf, n):
    return bool((buf[:GUARD_ROWS] == SENTINEL).all()) and bool((buf[GUARD_ROWS + n:] == SENTINEL).all())


@pytest.mark.parametrize("nf,N,A,L", [(2, 256, 37, 5), (5, 130, 37, 3), (3, 1, 37, 2), (2, 7, 14, 1), (4, 1024, 37, 2)])
def test_advance_kernel_matches_emulation(nf, N, A, L):
    g = torch.Generator(device=DEV).manual_seed(nf * 1000 + N)
    rand = lambda *s: torch.randn(*s, generator=g, device=DEV)
    r0_buf, rigids_0 = _guarded((nf, N, 7))
    rigids_0.copy_(rand(nf, N, 7))
    rt_buf, rigid_traj = _guarded((L, N, 7))
    at_buf, atom_traj = _guarded((L, N, A, 3))
    st_buf, step = _guarded((1,), torch.int64, fill=-99)
    step.zero_()
    want_r0, want_rt, want_at = rigids_0.clone(), rigid_traj.clone(), atom_traj.clone()
    for s in range(L + 2):                               # two calls past the end must write nothing
        rigid_pred, atom37 = rand(nf, N, 7), rand(nf, N, A, 3) * 10.0
        before = [t.clone() for t in (rigids_0, rigid_traj, atom_traj)]
        K.rollout_advance(rigid_pred, atom37, rigids_0, rigid_traj, atom_traj, step)
        if s < L:
            want_r0 = torch.cat([rigid_pred[1:], rigid_pred[-1:]])
            want_rt[s], want_at[s] = rigid_pred[-1], atom37[-1]
            assert int(step) == s + 1
        else:
            assert int(step) == L
            for b, t in zip(before, (rigids_0, rigid_traj, atom_traj)):
                assert torch.equal(b, t), s
        assert torch.equal(rigids_0, want_r0) and torch.equal(rigid_traj, want_rt) and torch.equal(atom_traj, want_at), s
        assert _guards_intact(r0_buf, nf) and _guards_intact(rt_buf, L) and _guards_intact(at_buf, L), s
        assert bool((st_buf[:GUARD_ROWS] == -99).all()) and bool((st_buf[GUARD_ROWS + 1:] == -99).all())
    # the row comes from the device counter: starting at L - 1 writes the last row only
    step.fill_(L - 1)
    rigid_pred, atom37 = rand(nf, N, 7), rand(nf, N, A, 3)
    K.rollout_advance(rigid_pred, atom37, rigids_0, rigid_traj, atom_traj, step)
    assert int(step) == L and torch.equal(rigid_traj[L - 1], rigid_pred[-1]) and torch.equal(atom_traj[L - 1], atom37[-1])


def test_advance_kernel_refuses_aliasing_and_bad_buffers():
    r = torch.zeros(2, 4, 7, device=DEV)
    a = torch.zeros(2, 4, 37, 3, device=DEV)
    rt, at, st = torch.zeros(3, 4, 7, device=DEV), torch.zeros(3, 4, 37, 3, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
    with pytest.raises(RuntimeError, match="aliases"):
        K.rollout_advance(r, a, r, rt, at, st)
    with pytest.raises(ValueError, match="int64"):
        K.rollout_advance(r, a, r.clone(), rt, at, st.int())
    with pytest.raises(ValueError, match="fp32"):
        K.rollout_advance(r, a, r.clone().double(), rt, at, st)
    with pytest.raises(ValueError, match="contiguous"):
        K.rollout_advance(r, a, r.clone(), torch.zeros(4, 3, 7, device=DEV).transpose(0, 1), at, st)
    with pytest.raises(ValueError, match="atom_traj"):
        K.rollout_advance(r, a, r.clone(), rt, at[:2], st)
    assert int(st) == 0


def test_default_path_is_bit_identical_to_literal():
    """One forward at t = min_t per frame == the reference's num_t-step sampler per frame (DESIGN §5.5)."""
    nf, N, L = 2, 256, 8
    net = _net(nf, syn.PRESET_A)
    w = _window(nf, N, 11)
    r = TrajectoryRollout(net)
    a = r.rollout(w, L)
    b = r.rollout(w, L, literal=True, num_t=3)
    assert a["rigid_traj"].shape == (L, N, 7) and a["atom_traj"].shape == (L, N, 37, 3)
    assert a["rigid_traj"].dtype == torch.float32 and a["atom_traj"].dtype == torch.float32
    assert torch.equal(a["rigid_traj"], b["rigid_traj"]) and torch.equal(a["atom_traj"], b["atom_traj"])
    assert float((a["rigid_traj"][-1] - a["rigid_traj"][0]).abs().max()) > 0       # the trajectory moves


def test_graphed_matches_eager_and_is_deterministic():
    nf, N, L = 3, 64, 6
    net = _net(nf, syn.PRESET_A, seed=1)
    r = TrajectoryRollout(net)
    for seed in (21, 22):                                # the second window is a pure replay from the static buffers
        w = _window(nf, N, seed)
        before = {k: v.clone() for k, v in w.items()}
        a, b = r.rollout(w, L), r.rollout(w, L)
        c = r.rollout(w, L, graph=False)
        for k in a:
            assert torch.equal(a[k], b[k]) and torch.equal(a[k], c[k]), (seed, k)
        for k in before:
            assert torch.equal(before[k], w[k]), k       # the caller's window is never modified
    assert len(r._graphs) == 1


def test_weight_changes_between_rollouts_take_effect():
    nf, N, L = 2, 48, 4
    net = _net(nf, syn.PRESET_A, seed=2)
    r = TrajectoryRollout(net)
    w = _window(nf, N, 23)
    a = r.rollout(w, L)
    with torch.no_grad():
        for name, p in net.named_parameters():
            if "bb_update" in name or "angle_resnet" in name:
                p.mul_(1.25)
    K.invalidate_weight_cache()
    b = r.rollout(w, L)
    c = r.rollout(w, L, graph=False)
    assert not torch.equal(a["rigid_traj"], b["rigid_traj"])
    assert torch.equal(b["rigid_traj"], c["rigid_traj"]) and torch.equal(b["atom_traj"], c["atom_traj"])


def _fixture_net(g):
    c = g["case"]
    net = FullScoreNetwork(syn.model_conf(c["nf"], **syn.PRESET_TINY, coordinate_scaling=c["cs"]),
                           SE3ScoreDiffuser(syn.diffuser_conf(c["cs"])))
    net.load_state_dict(syn.random_state(case_shapes(c), seed=c["wseed"]))
    return net.to(DEV).eval(), _window(c["nf"], c["N"], c["seed"])


@pytest.mark.parametrize("name", CASES)
def test_single_steps_match_reference(name):
    """Teacher-forced: each stored input window of the reference, rolled one frame, gives the reference's frame."""
    g = rollout_fixture()["cases"][name]
    net, w = _fixture_net(g)
    r = TrajectoryRollout(net)
    for i, j in enumerate(g["steps"]):
        out = r.rollout(dict(w, rigids_0=g["rigids_0"][i].to(DEV)), 1)
        err = float((out["rigid_traj"][0].double().cpu() - g["rigid_traj"][j].double()).norm(dim=-1).max())
        assert err < NET_TOL, (name, j, err)
        if j in g["atom_steps"]:
            ref = g["atom_traj"][g["atom_steps"].index(j)].double()
            assert atom_l2(out["atom_traj"][0].cpu(), ref) < ATOM_TOL, (name, j)


@pytest.mark.parametrize("name", CASES)
def test_free_running_rollout_matches_reference(name):
    g = rollout_fixture()["cases"][name]
    net, w = _fixture_net(g)
    out = TrajectoryRollout(net).rollout(w, 200)
    err = (out["rigid_traj"].double().cpu() - g["rigid_traj"].double()).norm(dim=-1).amax(dim=-1)
    assert float(err[:FREE_STEPS].max()) < NET_TOL, err[:FREE_STEPS]
    assert float(err.max()) < DRIFT_TOL, float(err.max())
    ref_atoms = g["atom_traj"][0].double()
    assert atom_l2(out["atom_traj"][0].cpu(), ref_atoms) < ATOM_TOL


@pytest.mark.timeout(900)
@pytest.mark.parametrize("nf,N", [(2, 256), (5, 256), (2, 1024), (3, 130)])
def test_long_rollouts_at_evaluation_shapes(nf, N):
    """L = 200: the graph replays every frame, rows fill in order, and the result equals the eager step bit for bit."""
    L = 200
    net = _net(nf, syn.PRESET_A, seed=3)
    w = _window(nf, N, 30 + nf)
    r = TrajectoryRollout(net)
    a = r.rollout(w, L)
    b = r.rollout(w, L, graph=False)
    assert a["rigid_traj"].shape == (L, N, 7) and a["atom_traj"].shape == (L, N, 37, 3)
    assert bool(torch.isfinite(a["rigid_traj"]).all()) and bool(torch.isfinite(a["atom_traj"]).all())
    assert torch.equal(a["rigid_traj"], b["rigid_traj"]) and torch.equal(a["atom_traj"], b["atom_traj"])
    assert bool((a["rigid_traj"][1:] != a["rigid_traj"][:-1]).any(dim=-1).any(dim=-1).all())   # every row was written


@pytest.mark.timeout(600)
def test_prefetcher_window_rolled_out_and_scored_against_md(tmp_path):
    from dynamicpdb_b200.input_pipeline import TrajectoryStore, WindowPrefetcher, featurize_window
    from oracle import synth_traj
    row = synth_traj.write_files(synth_traj.make_trajectory(), str(tmp_path))
    nf, T = 3, 9
    store = TrajectoryStore(frame_time=nf, frame_sample_step=1)
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    it = list(WindowPrefetcher(store, [row], DEV, training=False, diffuser=diffuser, targets=True))[0]
    net = _net(nf, syn.PRESET_TINY, seed=4)
    L = T - nf                                           # the MD frames after the window (it starts at frame 0)
    out = TrajectoryRollout(net).rollout(it, L)
    ent = store.protein(*row)
    md = ent["atom37"][nf:nf + L].to(DEV)
    mask = ent["atom_mask"].to(DEV)
    gt = featurize_window(md, mask, ent["aatype"].to(DEV))
    rot, tr, _, _ = M.rot_trans_error(out["rigid_traj"], gt["rigids_0"])
    m37 = mask.double().unsqueeze(0).expand(L, -1, -1)
    err = M.atom_errors(out["atom_traj"], md.double(), m37)
    want = MO.rot_trans_error(out["rigid_traj"], gt["rigids_0"])
    want_e = MO.atom_errors(out["atom_traj"], md.double(), m37)
    for got_v, want_v in ((rot, want[0]), (tr, want[1]), (err["mae"], want_e["mae"]), (err["rmsd_all"], want_e["rmsd_all"])):
        assert got_v.shape == (L,) and bool(torch.isfinite(got_v).all())
        assert float((got_v - want_v.to(got_v)).abs().max()) <= 1e-5 * (1 + float(want_v.abs().max()))
