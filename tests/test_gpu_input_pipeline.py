"""-m gpu: the featurisation kernel (csrc/featurize.cu) and the prefetching window iterator (SURVEY.md §8 f4) against the
fixtures generated from the unmodified loader and against the oracle.

Every prefetched window is also held bit for bit against the same window built one at a time on the current stream from
the public pieces (``TrajectoryStore.window_index``, ``featurize_window``, the diffuser with a fresh generator), across
proteins of different lengths and ring depths, and under two timings that a list() of the items never produces: a
consumer whose stream runs behind its host thread, and a side stream stalled behind one window."""
import threading

import numpy as np
import pytest
import torch

from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.input_pipeline import TrajectoryStore, WindowPrefetcher, featurize_window
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from oracle import dfold_oracle as O
from oracle import synth_traj
from tests.test_cpu_oracle import close, load

pytestmark = pytest.mark.gpu
DEV = "cuda"
T = 12                                                          # frames per synthetic trajectory
PROTEINS = {"A": (17, 31), "B": (23, 32), "C": (40, 33)}        # name: (residues, seed)
MIN_T = 0.2


def _check_against_gold(feats, gold):
    q = feats["rigids_0"][..., :4].double().cpu()
    assert feats["rigids_0"].dtype == torch.float32
    assert close(q.norm(dim=-1), torch.ones(q.shape[:-1], dtype=torch.float64), 1e-6)
    assert close(O.quat_to_rot(q), gold["rot_0"].double(), 2e-6)                    # same rotation (the reference's sign is arbitrary)
    assert close(feats["rigids_0"][..., 4:].cpu(), gold["rigids_0"][..., 4:], 1e-6)
    for k in ("torsion_angles_sin_cos", "alt_torsion_angles_sin_cos"):
        assert feats[k].dtype == gold[k].dtype and close(feats[k].cpu(), gold[k], 1e-6), k
    assert torch.equal(feats["torsion_angles_mask"].cpu(), gold["torsion_angles_mask"])
    assert close(feats["res_mask"].cpu().double(), gold["res_mask"].double(), 0)


def test_featurize_kernel_matches_reference_loader(tmp_path):
    traj = synth_traj.make_trajectory()
    row = synth_traj.write_files(traj, str(tmp_path))
    store = TrajectoryStore(frame_time=3, frame_sample_step=2, keep_first=8)
    ent = store.protein(*row)
    np.random.seed(5)
    sl = store.window_index(ent["atom37"].shape[0], training=True)
    feats = featurize_window(ent["atom37"][sl].to(DEV), ent["atom_mask"].to(DEV), ent["aatype"].to(DEV))
    _check_against_gold(feats, load("loader"))
    with pytest.raises(RuntimeError):
        featurize_window(ent["atom37"][sl], ent["atom_mask"], ent["aatype"])        # no CPU path


@pytest.mark.timeout(120)
def test_prefetcher_yields_reference_windows(tmp_path):
    """Three windows of the same protein through the worker thread + side stream; the first equals the golden window."""
    traj = synth_traj.make_trajectory()
    row = synth_traj.write_files(traj, str(tmp_path))
    store = TrajectoryStore(frame_time=3, frame_sample_step=2, keep_first=8)
    np.random.seed(5)
    items = list(WindowPrefetcher(store, [row, row, row], DEV, training=True))
    assert len(items) == 3
    gold = load("loader")
    _check_against_gold(items[0], gold)
    assert close(items[0]["force"].cpu(), gold["force"], 0) and items[0]["force"].dtype == torch.float64
    for it in items:
        assert it["node_repr"].shape == (17, 256) and it["edge_repr"].shape == (17, 17, 128) and it["aatype"].shape == (3, 17)
        assert it["rigids_0"].is_cuda and bool(torch.isfinite(it["rigids_0"]).all())


def _rows(tmp_path, order, n):
    """The csv rows of ``n`` windows cycling through ``order`` (protein names of PROTEINS), each protein written once."""
    files = {}
    for name in sorted(set(order)):
        N, seed = PROTEINS[name]
        files[name] = synth_traj.write_files(synth_traj.make_trajectory(T=T, N=N, seed=seed), str(tmp_path), name=name)
    return [files[order[i % len(order)]] for i in range(n)]


def _reference(conf, rows, training, diffuser, gen_seed, np_seed, targets):
    """Every window built one at a time on the current stream from the public pieces, in the prefetcher's draw order."""
    store = TrajectoryStore(pin=False, **conf)
    gen = torch.Generator(DEV).manual_seed(gen_seed)
    np.random.seed(np_seed)
    out = []
    for row in rows:
        ent = store.protein(*row)
        sl = store.window_index(ent["atom37"].shape[0], training)
        atom37, mask, aa = ent["atom37"][sl].to(DEV), ent["atom_mask"].to(DEV), ent["aatype"].to(DEV)
        nf, N = atom37.shape[:2]
        assert nf == conf["frame_time"]
        f = featurize_window(atom37, mask, aa)
        rix = ent["residue_index"].to(DEV).unsqueeze(0).expand(nf, -1)
        f.update(aatype=aa.unsqueeze(0).expand(nf, -1), seq_idx=rix, residue_index=rix,
                 force=ent["force"][sl].to(DEV), vel=ent["vel"][sl].to(DEV),
                 node_repr=ent["node_repr"].to(DEV), edge_repr=ent["edge_repr"].to(DEV),
                 fixed_mask=torch.zeros(nf, N, dtype=torch.float64, device=DEV),
                 sc_ca_t=torch.zeros(nf, N, 3, dtype=torch.float32, device=DEV))
        if targets:
            f["atom37_pos"] = atom37.double()
            f["atom37_mask"] = mask.double().unsqueeze(0).expand(nf, -1, -1)
        if diffuser is not None and training:
            t = MIN_T + (1.0 - MIN_T) * torch.rand(1, dtype=torch.float64, device=DEV, generator=gen)
            f.update(diffuser.forward_marginal(f["rigids_0"], t, generator=gen), t=t)
        elif diffuser is not None:
            f.update(diffuser.sample_ref(nf * N, frame_time=nf, generator=gen, device=DEV),
                     t=torch.ones(1, dtype=torch.float64, device=DEV))
        out.append(f)
    torch.cuda.synchronize()
    return out


def _assert_windows_equal(got, want):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert set(g) == set(w), (i, set(g) ^ set(w))
        for k in w:
            assert g[k].dtype == w[k].dtype and g[k].shape == w[k].shape and g[k].device == w[k].device, (i, k)
            assert torch.equal(g[k], w[k]), f"window {i}: {k} differs from the window built on its own"


def _prefetcher(cls, conf, rows, training, diffuser, gen_seed, np_seed, targets, depth, **kw):
    np.random.seed(np_seed)
    gen = torch.Generator(DEV).manual_seed(gen_seed)
    return cls(TrajectoryStore(**conf), rows, DEV, training=training, depth=depth, diffuser=diffuser, min_t=MIN_T,
               generator=gen, targets=targets, **kw)


_CYCLES_PER_MS = []


def _sleep_cycles(ms):
    """torch.cuda._sleep cycles that spin about ``ms`` milliseconds on this device (measured once with CUDA events)."""
    if not _CYCLES_PER_MS:
        c = 2_000_000
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(c)
        e0.record()
        torch.cuda._sleep(c)
        e1.record()
        torch.cuda.synchronize()
        _CYCLES_PER_MS.append(c / e0.elapsed_time(e1))
    return int(ms * _CYCLES_PER_MS[0])


# (mode, frame_sample_step, keep_first, fix_sample_start, depth, protein order)
MATRIX = [
    ("train", 1, None, 0, 1, "A"),
    ("train", 2, 9, 0, 3, "AB"),
    ("train_diffuser", 2, 10, 0, 2, "ABAB"),
    ("train_diffuser_targets", 1, 8, 0, 1, "AABA"),
    ("eval_diffuser", 2, None, 3, 3, "AABA"),
    ("eval_diffuser_targets", 1, 6, 5, 2, "ABC"),
]


@pytest.mark.timeout(120)
@pytest.mark.parametrize("mode,k,keep_first,fix_start,depth,order", MATRIX,
                         ids=[f"{m}-k{k}-keep{kf}-depth{d}-{o}" for m, k, kf, _, d, o in MATRIX])
def test_prefetched_windows_equal_windows_built_one_at_a_time(tmp_path, mode, k, keep_first, fix_start, depth, order):
    """Every field of every item, bit for bit, over enough windows that every ring of depth + 1 wraps three times."""
    training, targets = mode.startswith("train"), mode.endswith("targets")
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0)) if "diffuser" in mode else None
    conf = dict(frame_time=3, frame_sample_step=k, keep_first=keep_first, fix_sample_start=fix_start)
    rows = _rows(tmp_path, order, 3 * (depth + 1))
    want = _reference(conf, rows, training, diffuser, 7, 3, targets)
    got = list(_prefetcher(WindowPrefetcher, conf, rows, training, diffuser, 7, 3, targets, depth))
    _assert_windows_equal(got, want)


@pytest.mark.timeout(120)
def test_lagging_consumer_reads_windows_the_worker_has_not_overwritten(tmp_path):
    """The consumer's stream runs ~40 ms behind its host thread on every item, which it drops before taking the next, as a
    training loop that never waits on the host does: what its stream reads must still be the window it was handed.  One
    protein, so that every window's device memory fits the next one's and no staging buffer is shared across lengths."""
    conf = dict(frame_time=3, frame_sample_step=2)
    depth = 2
    rows = _rows(tmp_path, "A", 3 * (depth + 1))
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    want = _reference(conf, rows, True, diffuser, 5, 2, False)
    cycles = _sleep_cycles(40)
    got = []
    for item in _prefetcher(WindowPrefetcher, conf, rows, True, diffuser, 5, 2, False, depth):
        torch.cuda._sleep(cycles)
        got.append({key: v.clone() for key, v in item.items()})
        del item
    torch.cuda.synchronize()
    _assert_windows_equal(got, want)


class _StalledPrefetcher(WindowPrefetcher):
    """Test only: the side stream sleeps before window ``stall_at`` is made, so that window's copies wait behind the sleep
    while the worker thread goes on making the next windows."""

    def __init__(self, *args, stall_at, cycles, **kw):
        super().__init__(*args, **kw)
        self.stall_at, self.cycles, self.made = stall_at, cycles, 0

    def _make(self, row):
        if self.made == self.stall_at:
            with torch.cuda.stream(self.stream):
                torch.cuda._sleep(self.cycles)
        self.made += 1
        return super()._make(row)


@pytest.mark.timeout(120)
def test_stalled_side_stream_keeps_each_window_its_own_frames(tmp_path):
    """Rows A B A B of two lengths with depth 2: window 3 is made while window 1's copies still wait behind the stall."""
    conf = dict(frame_time=3, frame_sample_step=2)
    depth = 2
    rows = _rows(tmp_path, "AB", 3 * (depth + 1))
    want = _reference(conf, rows, True, None, 0, 1, False)
    assert not torch.equal(want[1]["force"], want[3]["force"])      # windows 1 and 3 take different frames
    pf = _prefetcher(_StalledPrefetcher, conf, rows, True, None, 0, 1, False, depth, stall_at=1, cycles=_sleep_cycles(100))
    for row in rows:
        pf.store.protein(*row)                                       # decoded before the stall: the host races ahead of it
    _assert_windows_equal(list(pf), want)


@pytest.mark.timeout(120)
def test_evaluation_window_reaches_past_keep_first_as_the_reference_loader(tmp_path):
    """tests/golden/loader_eval.pt: an evaluation window from frame 4, every 2nd frame, with keep_first=8 reads frame 8."""
    gold = load("loader_eval")
    c = gold["case"]
    row = synth_traj.write_files(synth_traj.make_trajectory(T=c["T"]), str(tmp_path))
    store = TrajectoryStore(frame_time=c["frame_time"], frame_sample_step=c["frame_sample_step"], keep_first=c["keep_first"],
                            fix_sample_start=c["fix_sample_start"])
    item, = list(WindowPrefetcher(store, [row], DEV, training=False, targets=True))
    for key in ("aatype", "seq_idx", "force", "vel", "atom37_mask"):
        assert item[key].dtype == gold[key].dtype and torch.equal(item[key].cpu(), gold[key]), key
    assert item["atom37_pos"].dtype == gold["atom37_pos"].dtype        # coordinates of the atoms in the mask
    assert torch.equal((item["atom37_pos"] * item["atom37_mask"][..., None]).cpu(), gold["atom37_pos"])
    _check_against_gold(item, gold)


@pytest.mark.timeout(60)
def test_leaving_the_loop_early_stops_the_worker(tmp_path):
    """A consumer that breaks after the first item (an evaluation of part of a split) leaves no worker thread behind."""
    row = synth_traj.write_files(synth_traj.make_trajectory(), str(tmp_path))
    pf = WindowPrefetcher(TrajectoryStore(frame_time=3), [row] * 8, DEV, depth=1)
    before = set(threading.enumerate())
    for _ in pf:
        workers = [th for th in threading.enumerate() if th not in before]
        break
    assert len(workers) == 1
    workers[0].join(timeout=5)
    assert not workers[0].is_alive(), "the worker thread is still blocked after the consumer left"
    assert pf._thread is workers[0]
