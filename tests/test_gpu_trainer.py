"""-m gpu: dynamicpdb_b200.trainer and TrainStep(loss_reads_window=True) on windows the input pipeline builds from
trajectory files in the reference loader's formats (oracle/synth_traj.py), tiny preset.

  * accumulate=2: the gradient buffer is the sum of score_network_loss's gradients over the two windows, each slot's
    loss reading its own window's targets;
  * TrainStep.aux is eager score_network_loss's aux_data on slot 0's window at the same weights, captured and eager;
  * two epochs of Trainer equal a hand-written TrainStep loop over the same windows, bit for bit;
  * two epochs, a checkpoint and resume() into a fresh Trainer, then the third epoch equal three epochs straight;
  * data parallel: spawned ranks each train their DistributedSampler shard (gloo with eager steps on one GPU; NCCL with
    captured steps, one rank per GPU, skipped below two GPUs).
"""
import copy
import datetime
import logging
import os
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.input_pipeline import TrajectoryStore, WindowPrefetcher
from dynamicpdb_b200.loss import score_network_loss
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from dynamicpdb_b200.train_step import TrainStep
from dynamicpdb_b200.trainer import LOGGED, Trainer, epoch_order
from oracle import synth_traj
from tests.test_cpu_oracle import close

pytestmark = pytest.mark.gpu
DEV = "cuda"
NF, N, T = 3, 17, 9
N_PROTEINS = 3


def _files(root):
    """N_PROTEINS trajectories of N residues and their training csv."""
    rows = [synth_traj.write_files(synth_traj.make_trajectory(T=T, N=N, seed=31 + i), str(root), name=f"p{i}")
            for i in range(N_PROTEINS)]
    path = os.path.join(str(root), "train.csv")
    with open(path, "w") as f:
        f.write("name,seq_len,atlas_npz,force_path,vel_path,embed_path\n")
        for i, r in enumerate(rows):
            f.write(f"p{i},{N}," + ",".join(r) + "\n")
    return path, rows


def _conf(csv_path, batch_size=1, num_epoch=2, log_freq=2, ckpt_freq=1, ckpt_dir=None):
    return {"experiment": {"batch_size": batch_size, "num_epoch": num_epoch, "log_freq": log_freq, "ckpt_freq": ckpt_freq,
                           "ckpt_dir": ckpt_dir, "learning_rate": 1e-3, "torsion_loss_weight": 1.0, "rot_loss_weight": 0.5,
                           "trans_loss_weight": 1.0, "rot_loss_t_threshold": 0.2, "separate_rot_loss": False},
            "data": {"csv_path": csv_path, "filtering": {"max_len": 256}, "frame_time": NF, "frame_sample_step": 1,
                     "keep_first": None, "min_t": 0.01}}


def _net(seed=7):
    net = FullScoreNetwork(syn.model_conf(NF, **syn.PRESET_TINY), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    state = syn.random_state({k: v.shape for k, v in net.state_dict().items()}, seed=seed)
    state["score_model.angle_resnet.linear_out.bias"] = state["score_model.angle_resnet.linear_out.bias"] + 0.5
    net.load_state_dict(state, strict=True)
    return net.to(DEV)


def _windows(rows, k):
    store = TrajectoryStore(frame_time=NF)
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    return list(WindowPrefetcher(store, [rows[i % len(rows)] for i in range(k)], DEV, diffuser=diffuser))


class _Exp:
    torsion_loss_weight, rot_loss_weight, trans_loss_weight = 1.0, 0.5, 1.0
    rot_loss_t_threshold, separate_rot_loss = 0.2, False


def _loss(out, window):
    return score_network_loss(out, window, _Exp)


def _state(ts):
    return [ts.flat_param, ts.exp_avg, ts.exp_avg_sq, ts.max_exp_avg_sq, ts.step_count]


def _assert_same_state(a, b, what):
    for x, y, name in zip(_state(a), _state(b), ("parameters", "exp_avg", "exp_avg_sq", "max_exp_avg_sq", "step")):
        assert torch.equal(x, y), f"{what}: {name} differ, max |diff| {(x - y).abs().max().item():.3e}"


@pytest.mark.parametrize("graph", [True, False], ids=["captured", "eager"])
def test_each_slot_trains_on_its_own_window(graph, tmp_path):
    """accumulate=2 with loss_reads_window: the gradient buffer is the sum over the two windows of score_network_loss's
    gradient taken with plain autograd, each on its own window's targets.  The bar is that of
    test_gpu_training_objective's single-window comparison (2e-5 of the largest element of a parameter's gradient, per
    window), which the accumulation bound of DESIGN.md §7 (k u sum |g_i|) is far inside.  Also: `loss` is the mean of the
    two windows' losses and `aux` is slot 0's aux_data."""
    _, rows = _files(tmp_path)
    w0, w1 = _windows(rows, 2)
    net = _net()
    ref = copy.deepcopy(net)
    ts = TrainStep(net, _loss, w0, lr=0.0, graph=graph, warmup=2, accumulate=2, loss_reads_window=True)
    assert not graph or ts.graph is not None, ts.graph_error
    ts.load(w0, slot=0)
    ts.load(w1, slot=1)
    ts()
    torch.cuda.synchronize()
    losses, auxes, per = [], [], []
    for w in (w0, w1):
        for q in ref.parameters():
            q.grad = None
        loss, aux = score_network_loss(ref(dict(w)), w, _Exp)
        loss.backward()
        losses.append(float(loss.detach()))
        auxes.append(aux)
        per.append([torch.zeros_like(q) if q.grad is None else q.grad.clone() for q in ref.parameters()])
    assert abs(losses[0] - losses[1]) > 1e-6 * abs(losses[0])              # the windows are told apart
    off = 0
    for (name, p), g0, g1 in zip(net.named_parameters(), *per):
        n = p.numel()
        got = ts.flat_grad[off:off + n].view_as(p)
        off += n
        scale = (g0.abs() + g1.abs()).max().item()
        assert (got - (g0 + g1)).abs().max().item() <= 2e-5 * max(1e-6, scale) + 1e-9, name
    mean = (losses[0] + losses[1]) / 2
    assert abs(float(ts.loss) - mean) <= 1e-6 * max(1.0, abs(mean))
    for k, v in auxes[0].items():
        assert ts.aux[k].shape == v.shape and ts.aux[k].dtype == v.dtype, k
        assert close(ts.aux[k].cpu(), v.cpu(), 1e-5), (k, ts.aux[k], v)


def test_aux_follows_every_step(tmp_path):
    """TrainStep.aux is the aux_data of eager score_network_loss on slot 0's window at the weights the step starts from,
    step after step of captured replays, in the same static tensors; nothing of the capture window is kept."""
    _, rows = _files(tmp_path)
    wins = _windows(rows, 4)
    net = _net()
    ref = copy.deepcopy(net)
    ts = TrainStep(net, _loss, wins[0], lr=1e-3, graph=True, warmup=2, loss_reads_window=True)
    assert ts.graph is not None, ts.graph_error
    ptrs = {k: v.data_ptr() for k, v in ts.aux.items()}
    seen = []
    for w in wins[1:]:
        with torch.no_grad():
            for q, p in zip(ref.parameters(), net.parameters()):
                q.copy_(p)
            want = score_network_loss(ref(dict(w)), w, _Exp)[1]
        ts.load(w)
        ts()
        assert {k: v.data_ptr() for k, v in ts.aux.items()} == ptrs
        for k, v in want.items():
            assert ts.aux[k].dtype == v.dtype and close(ts.aux[k].cpu(), v.cpu(), 1e-5), k
        seen.append(float(ts.aux["total_loss"]))
    assert len(set(seen)) == 3


def test_plain_loss_keeps_no_aux(tmp_path):
    _, rows = _files(tmp_path)
    w, = _windows(rows, 1)
    ts = TrainStep(_net(), lambda out: score_network_loss(out, w, _Exp)[0], w, lr=1e-3, graph=False, warmup=1)
    ts()
    assert ts.aux is None


def _hand_loop(csv_rows, epochs, accumulate, net):
    """The loop a user would write: the Trainer's example window, seeding and per-epoch DistributedSampler order over
    `accumulate` stand-in ranks, WindowPrefetcher, load, replay."""
    store = TrajectoryStore(frame_time=NF)
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    example, = list(WindowPrefetcher(store, csv_rows[:1], DEV, diffuser=diffuser, min_t=0.01))
    ts = TrainStep(net, _loss, example, lr=1e-3, accumulate=accumulate, loss_reads_window=True)
    np.random.seed(0)
    torch.manual_seed(0)
    for epoch in range(epochs):
        order = epoch_order(len(csv_rows), accumulate, epoch)
        seq = [csv_rows[i] for step in zip(*order) for i in step]
        it = iter(WindowPrefetcher(store, seq, DEV, diffuser=diffuser, min_t=0.01))
        for _ in range(len(order[0])):
            for s in range(accumulate):
                ts.load(next(it), slot=s)
            ts()
    torch.cuda.synchronize()
    return ts


def test_two_epochs_equal_a_hand_written_loop(tmp_path, caplog):
    csv_path, rows = _files(tmp_path)
    with caplog.at_level(logging.INFO, logger="dynamicpdb_b200.trainer"):
        tr = Trainer(_conf(csv_path, batch_size=2, log_freq=1), _net(), SE3ScoreDiffuser(syn.diffuser_conf(1.0)),
                     accumulate=2)
        assert tr.step.graph is not None, tr.step.graph_error
        tr.train()
    torch.cuda.synchronize()
    steps = 2 * -(-N_PROTEINS // 2)
    assert (tr.trained_epochs, tr.trained_steps) == (1, steps) and float(tr.step.step_count) == steps
    ts = _hand_loop(rows, 2, 2, _net())
    _assert_same_state(tr.step, ts, "Trainer against the hand-written loop")
    lines = [m for m in caplog.messages if m.startswith("Epoch[")]
    assert len(lines) == steps and lines[-1].startswith(f"Epoch[1/2] trained_steps: [{steps}]: total_loss=")
    assert all(f"{k}=" in lines[0] for k in LOGGED)
    # the last line shows the last step's slot 0 (log_freq 1): the hand-written step's aux
    last = {k: float(v) for k, v in zip(LOGGED, tr.logged.tolist())}
    assert all(abs(last[k] - float(ts.aux[k])) == 0.0 for k in LOGGED)


def test_resume_continues_as_one_run(tmp_path):
    """Epochs 0 and 1, the checkpoint written at the end of epoch 1, resume() into a fresh Trainer built from other
    weights, then epoch 2: the same weights, moments, step and counters as three epochs straight, with the data streams
    re-seeded the same way before epoch 2 in both runs."""
    csv_path, _ = _files(tmp_path)
    conf = _conf(csv_path, num_epoch=3, ckpt_freq=1, ckpt_dir=str(tmp_path / "ckpt"))
    diffuser = SE3ScoreDiffuser(syn.diffuser_conf(1.0))
    straight = Trainer(conf, _net(), diffuser)
    straight.train_epoch(0)
    straight.train_epoch(1)
    path = os.path.join(str(tmp_path / "ckpt"), f"step_{2 * N_PROTEINS}.pth")
    assert os.listdir(str(tmp_path / "ckpt")) == [os.path.basename(path)]       # none after epoch 0, as the reference
    ck = torch.load(path, weights_only=False)
    assert (ck["epoch"], ck["step"]) == (1, 2 * N_PROTEINS) and ck["conf"] == conf
    np.random.seed(11)
    torch.manual_seed(11)
    straight.train_epoch(2)
    torch.cuda.synchronize()
    resumed = Trainer(conf, _net(seed=99), diffuser)
    resumed.resume(path)
    assert (resumed.trained_epochs, resumed.trained_steps) == (2, 2 * N_PROTEINS)
    np.random.seed(11)
    torch.manual_seed(11)
    resumed.train()
    torch.cuda.synchronize()
    assert (resumed.trained_epochs, resumed.trained_steps) == (straight.trained_epochs, straight.trained_steps) == (2, 9)
    _assert_same_state(straight.step, resumed.step, "resumed against straight")


# --------------------------------------------------------------------------------------------------
# data parallel
# --------------------------------------------------------------------------------------------------
WORLD = 2
EPOCHS = 2


def _worker(rank, backend, store_path, csv_path, out_dir):
    try:
        dev = rank if backend == "nccl" else 0
        torch.cuda.set_device(dev)
        if backend == "nccl":
            os.environ["TORCH_NCCL_ASYNC_ERROR_HANDLING"] = "0"
        dist.init_process_group(backend, store=dist.FileStore(store_path, WORLD), rank=rank, world_size=WORLD,
                                timeout=datetime.timedelta(seconds=300),
                                **({"device_id": torch.device("cuda", dev)} if backend == "nccl" else {}))
        global DEV
        DEV = f"cuda:{dev}"
        tr = Trainer(_conf(csv_path, batch_size=WORLD, num_epoch=EPOCHS), _net(), SE3ScoreDiffuser(syn.diffuser_conf(1.0)),
                     world_size=WORLD, rank=rank, graph=backend == "nccl", warmup=1)
        shards = []
        for epoch in range(EPOCHS):
            shards.append([s[0] for s in tr.windows(epoch)])
            tr.train_epoch(epoch)
        torch.cuda.synchronize()
        torch.save({"shards": shards, "state": [t.cpu() for t in _state(tr.step)], "steps": tr.trained_steps,
                    "graph": tr.step.graph is not None}, os.path.join(out_dir, f"rank{rank}.pt"))
    except BaseException:                                                  # noqa: BLE001  (reported by the parent)
        with open(os.path.join(out_dir, f"rank{rank}.err"), "w") as f:
            f.write(traceback.format_exc())
        os._exit(1)
    if backend == "nccl":
        os._exit(0)                 # destroy_process_group blocks on a communicator a graph has captured (DESIGN.md §7)
    dist.destroy_process_group()


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_ranks_train_their_sampler_shards(backend, tmp_path):
    """Each rank trains DistributedSampler(num_replicas=2, rank=r)'s shard of every epoch, on windows drawn from its own
    seeded streams, and the all-reduced update leaves both ranks with the same weights, moments and step, bit for bit,
    away from the weights they started from."""
    if backend == "nccl" and torch.cuda.device_count() < WORLD:
        pytest.skip("the NCCL arm needs one GPU per rank")
    csv_path, rows = _files(tmp_path)
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_worker, args=(r, backend, str(tmp_path / "store"), csv_path, str(tmp_path)))
             for r in range(WORLD)]
    for p in procs:
        p.start()
    try:
        for p in procs:
            p.join(600)
    finally:
        late = [r for r, p in enumerate(procs) if p.is_alive()]
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    errors = {r: open(tmp_path / f"rank{r}.err").read() for r in range(WORLD) if (tmp_path / f"rank{r}.err").exists()}
    assert not errors, "\n".join(f"rank {r}:\n{e}" for r, e in errors.items())
    assert not late, f"ranks {late} still running: killed"
    res = [torch.load(tmp_path / f"rank{r}.pt") for r in range(WORLD)]
    for epoch in range(EPOCHS):
        assert [r["shards"][epoch] for r in res] == epoch_order(N_PROTEINS, WORLD, epoch)
    steps = EPOCHS * -(-N_PROTEINS // WORLD)
    for r in res:
        assert r["steps"] == steps and float(r["state"][4]) == steps and r["graph"] == (backend == "nccl")
    for a, b in zip(res[0]["state"], res[1]["state"]):
        assert torch.equal(a, b)
    start = torch.cat([p.detach().reshape(-1).cpu() for p in _net().parameters()])
    assert not torch.equal(res[0]["state"][0][:start.numel()], start)
