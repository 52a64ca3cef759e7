#!/usr/bin/env python
"""Benchmark of the DFOLDv2 score-network training step (BASELINE.json metric: frames/s, fwd+bwd, N_res=256,
64 trajectory frames per sample), one process per GPU.

    python bench.py --gpus N --steps K --warmup W            # the CUDA path (this repo)
    python bench.py --impl reference --steps K --warmup W    # the CPU oracle port, timed on the host cores

A step = zero_grad + forward + surrogate loss + backward (+ one flat NCCL gradient all-reduce when N > 1)
+ Adam(amsgrad) step, captured in one CUDA graph (dynamicpdb_b200/train_step.py), on ONE protein window of `--frames` frames x `--res` residues per rank (the only shape the
reference executes in one forward, SURVEY.md §8d).  Weak scaling: every rank processes its own window.
Prints ONE JSON line on rank 0.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

METRIC = "DFOLDv2 frames/sec (fwd+bwd, N_res=256, batch=64)"


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-graph", action="store_true", help="launch the step eagerly instead of replaying a CUDA graph")
    ap.add_argument("--no-literal", action="store_true", help="skip the extra measurement with dead-frame elimination off")
    ap.add_argument("--cpu-frames", type=int, default=4, help="frames in the bounded CPU sample")
    ap.add_argument("--no-extra", action="store_true", help="skip the secondary configs (100-step inference, N_res=1024)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed step computed to DIR/<name>.npy")
    return ap.parse_args()


# --------------------------------------------------------------------------------------------------
# clocks sampling during the timed region
# --------------------------------------------------------------------------------------------------
class ClockSampler:
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-i", str(self.index), "-lms", "200"], stdout=subprocess.PIPE, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["unavailable"]}
        self.proc.terminate()
        sm = sorted(float(r[1]) for r in self.rows if len(r) > 8 and r[1].replace(".", "").isdigit())
        mx = [float(r[2]) for r in self.rows if len(r) > 8 and r[2].replace(".", "").isdigit()]
        reasons = set()
        for r in self.rows:
            if len(r) > 8:
                for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[5:9]):
                    if v.lower().startswith("active"):
                        reasons.add(name)
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


# --------------------------------------------------------------------------------------------------
# CPU arm (reference arm / cpu_baseline): the reference's own PyTorch-CPU path, or the oracle port of it
# --------------------------------------------------------------------------------------------------
def _cgroup_cpu_limit():
    """CPU quota of this container in cores (cgroup v2 cpu.max, v1 cfs quota), or None when unlimited / unknown."""
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if q != "max":
            return float(q) / float(p)
    except Exception:       # noqa: BLE001
        pass
    for base in ("/sys/fs/cgroup/cpu", "/sys/fs/cgroup/cpu,cpuacct"):
        try:
            q = int(open(base + "/cpu.cfs_quota_us").read())
            p = int(open(base + "/cpu.cfs_period_us").read())
            if q > 0 and p > 0:
                return q / p
        except Exception:   # noqa: BLE001
            pass
    return None


def pick_host_threads():
    """Thread count for the CPU arm: bounded by the affinity mask AND the cgroup CPU quota (sched_getaffinity alone
    reports every core of the host and oversubscribes a quota-limited container 10x), then calibrated: a short GEMM +
    elementwise probe is timed at each candidate count and the fastest wins."""
    try:
        cap = len(os.sched_getaffinity(0))
    except Exception:       # noqa: BLE001
        cap = os.cpu_count() or 1
    lim = _cgroup_cpu_limit()
    if lim:
        cap = max(1, min(cap, int(lim + 0.999)))
    cands = sorted({c for c in (4, 8, 16, 24, 32, 48, 64, 96, 128, cap) if c <= cap}) or [1]
    a = torch.randn(1536, 1536)
    b = torch.randn(1536, 1536)
    e = torch.randn(8, 256, 256, 24)
    best, best_t = cands[0], float("inf")
    for c in cands:
        torch.set_num_threads(c)
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            (a @ b).sum()
            ((e - 0.5) ** 2).sum(-1).exp().sum()
            ts.append(time.perf_counter() - t0)
        t = min(ts[1:])
        if t < best_t * 0.95:          # prefer fewer threads unless more are clearly faster
            best, best_t = c, t
    torch.set_num_threads(best)
    return best, {"affinity_or_quota_cap": cap, "cgroup_quota": lim}


def _reference_root():
    """Where an unmodified reference checkout is importable from: $DFOLD_REFERENCE_ROOT, if set."""
    cand = os.environ.get("DFOLD_REFERENCE_ROOT")
    if cand and os.path.isdir(os.path.join(cand, "src", "model")):
        return cand
    return None


def cpu_step_fn(frames, n_res):
    """-> (step, kind, what): `step()` runs one forward + backward of one window of `frames` x `n_res` on the CPU.
    kind "reference": the UNMODIFIED reference modules (src.model.Dfold_network_dynamic.FullScoreNetwork with the
    reference's SE3Diffuser), imported through oracle/ref_shims.py; kind "port": the oracle restatement."""
    from dynamicpdb_b200 import synthetic as syn
    torch.manual_seed(0)
    conf = syn.model_conf(frames, **syn.PRESET_A)
    feats = syn.make_feats(frames, n_res, seed=0)
    root = _reference_root()
    if root is not None and os.environ.get("DFOLD_CPU_ARM", "") != "port":
        try:
            os.environ["DFOLD_REFERENCE_ROOT"] = root
            from oracle import ref_shims
            ref_shims.REFERENCE_ROOT = root
            ref_shims.install()
            from src.model import Dfold_network_dynamic as RefNet
            from src.data import se3_diffuser
            net = RefNet.FullScoreNetwork(conf, se3_diffuser.SE3Diffuser(syn.diffuser_conf(1.0)))
            sd = net.state_dict()
            syn.dezero_(sd)
            net.load_state_dict(sd)

            def step():
                net.zero_grad(set_to_none=True)
                out = net(dict(feats))
                syn.surrogate_loss(out).backward()
            return step, "reference", f"unmodified reference modules from {root} (PyTorch CPU)"
        except Exception as e:      # noqa: BLE001
            print(f"[bench] live reference unavailable ({type(e).__name__}: {str(e)[:120]}); using the oracle port",
                  file=sys.stderr)
    from oracle import dfold_oracle as O
    from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
    from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
    net = FullScoreNetwork(conf, SE3ScoreDiffuser(syn.diffuser_conf(1.0)))      # only used to draw the weights
    sd = net.state_dict()
    syn.dezero_(sd)
    p = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
    del net
    oc, dc = O.default_conf(**syn.PRESET_A), O.default_diffuser_conf(1.0)
    leaves = [v for v in p.values() if v.requires_grad]

    def step():
        out = O.full_forward(p, feats, oc, dc)
        torch.autograd.grad(O.surrogate_loss(out), leaves, allow_unused=True)
    return step, "port", "oracle/dfold_oracle.py (CPU restatement of the reference path)"


def cpu_arm(frames, n_res, steps, warmup, budget_s):
    """Times the CPU arm inside a wall-clock budget: the first step is always run (and counted as warm-up); how many
    more warm-up / timed steps follow is derived from its duration so the whole call ends within `budget_s`."""
    t_begin = time.perf_counter()
    threads, tinfo = pick_host_threads()
    step, kind, what = cpu_step_fn(frames, n_res)
    t0 = time.perf_counter()
    step()
    first = time.perf_counter() - t0
    left = budget_s - (time.perf_counter() - t_begin)
    afford = max(1, int(left // max(first, 1e-3)))
    n_timed = max(1, min(steps, afford))
    n_warm = max(0, min(warmup - 1, afford - n_timed))
    for _ in range(n_warm):
        step()
    times = []
    for _ in range(n_timed):
        t0 = time.perf_counter()
        step()
        times.append(time.perf_counter() - t0)
    ms = 1e3 * sum(times) / len(times)
    return {"fps": frames / (ms / 1e3), "ms": ms, "threads": threads, "thread_info": tinfo, "kind": kind, "what": what,
            "steps_timed": n_timed, "warmup_run": n_warm + 1, "first_step_s": first,
            "wall_s": time.perf_counter() - t_begin}


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    frames = args.cpu_frames
    r = cpu_arm(frames, args.res, args.steps, args.warmup, float(os.environ.get("DFOLD_REF_BUDGET_S", "240")))
    sample = (f"{r['steps_timed']} timed fwd+bwd steps (after {r['warmup_run']} warm-up) of one window of {frames} frames x "
              f"{args.res} residues each, {r['what']}; per-frame cost is linear in the frame count; "
              f"wall-clock budget bounded ({r['wall_s']:.0f} s)")
    line = {
        "impl": "reference", "metric": METRIC, "value": r["fps"], "unit": "frames/s", "n_gpus": args.gpus,
        "steps": r["steps_timed"], "warmup": r["warmup_run"], "steps_requested": args.steps, "warmup_requested": args.warmup,
        "ms_per_step": r["ms"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": {"workload": f"DFOLDv2 training step fwd+bwd, N_res={args.res}, PyTorch CPU (bounded sample of configs[2])",
                   "frames_per_step": frames, "n_res": args.res, "preset": "train_DFOLDv2.yaml"},
        "cpu_baseline": {"value": r["fps"], "unit": "frames/s", "cores": r["threads"], "kind": r["kind"], "sample": sample,
                         "thread_info": r["thread_info"]},
        "e2e": {"value": r["fps"], "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line), file=_REAL_STDOUT, flush=True)


# --------------------------------------------------------------------------------------------------
# the CUDA path
# --------------------------------------------------------------------------------------------------
def _log(msg):
    if os.environ.get("DFOLD_BENCH_VERBOSE", "0") == "1":
        print(f"[bench rank {os.environ.get('RANK', '0')} t={time.perf_counter():.1f}] {msg}", file=sys.stderr, flush=True)



def time_ipa_core(dev, nf, N, iters=20):
    """Fused IPA forward core alone at the benchmark shape (preset A), CUDA events on the launching stream around `iters`
    back-to-back calls after 3 warm-up calls.  Inputs (q/k/v, points, pair, bias: 659 MB at nf=64) exceed the 50 MB L2."""
    from dynamicpdb_b200 import kernels as K
    H, C, Pq, Pv, Cp = 8, 256, 8, 12, 32
    g = torch.Generator(device=dev).manual_seed(0)
    R = lambda *s, scale=1.0: torch.randn(*s, device=dev, generator=g) * scale
    logit0, kv = R(1, H, N, N), R(1, N, H, 2 * C)
    q_pts, kv_pts = R(nf, N, H, Pq, 3, scale=4.0), R(nf, N, H, Pq + Pv, 3, scale=4.0)
    pair = R(1, N, N, Cp)
    quat = torch.nn.functional.normalize(R(nf, N, 4), dim=-1)
    trans, mask = R(nf, N, 3, scale=8.0), torch.ones(nf, N, device=dev)
    gamma = torch.rand(H, device=dev, generator=g) * 0.2 + 0.05
    alg = 4.0 * (nf * N * (H * (4 * C + 3 * (2 * Pq + Pv) + 8 * Pv + Cp) + 8) + N * N * (H + Cp))

    def run(train):
        q = q_pts.detach().requires_grad_(train)      # training forward: the op also writes the probability planes for backward
        with torch.set_grad_enabled(train):
            return K.ipa_attention(logit0, kv, q, kv_pts, pair, quat, trans, mask, gamma, Pq=Pq, Pv=Pv, dfold=True,
                                   inf=1e5, eps=1e-8).detach()
    res = {}
    for train in (True, False):
        for _ in range(3):
            run(train)
        torch.cuda.synchronize()
        K.LAUNCH_COUNT = 0
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            run(train)
        e1.record()
        torch.cuda.synchronize()
        res[train] = (e0.elapsed_time(e1) / iters, K.LAUNCH_COUNT // iters)
    return res[True][0], alg, res[True][1], res[False][0]


def _fresh_net(nf, dev):
    from dynamicpdb_b200 import synthetic as syn
    from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
    from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(nf, **syn.PRESET_A), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    return net.to(dev)


def extra_configs(dev, graph):
    """BASELINE.json configs[1] (100-step reverse diffusion, N_res=256, 32 frames) and configs[4] (N_res=1024, 8 frames,
    fwd+bwd+Adam) on one GPU.  Secondary lines: wall time of whole jobs, CUDA events, inputs resident."""
    from dynamicpdb_b200 import synthetic as syn
    from dynamicpdb_b200.inference import DeviceReverseDiffusion
    from dynamicpdb_b200.train_step import TrainStep
    out = {}
    try:
        nf, N, num_t = 32, 256, 100
        net = _fresh_net(nf, dev).eval()
        feats = {k: v.to(dev) for k, v in syn.make_feats(nf, N, seed=1).items()}
        gen = torch.Generator(device=dev).manual_seed(0)
        sampler = DeviceReverseDiffusion(net)
        res = {}
        for name, literal, reps in (("memoised", False, 3), ("literal", True, 1)):
            sampler.memo.reset()
            sampler.sample(feats, 3, 0.01, generator=gen, literal=literal)        # warm-up
            sampler.memo.reset()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                sampler.memo.reset()
                sampler.sample(feats, num_t, 0.01, generator=gen, literal=literal)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            res[name] = {"ms_per_sample": ms, "frames_per_s": nf / (ms * 1e-3), "denoise_steps_per_s": num_t / (ms * 1e-3)}
        try:
            sampler.memo.reset()
            sampler.sample_graphed(feats, num_t, 0.01)              # capture (trunk + 100 steps in one CUDA graph)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(3):
                sampler.sample_graphed(feats, num_t, 0.01)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 3
            res["memoised_graph"] = {"ms_per_sample": ms, "frames_per_s": nf / (ms * 1e-3), "denoise_steps_per_s": num_t / (ms * 1e-3)}
        except Exception as e:      # noqa: BLE001
            res["memoised_graph"] = {"error": f"{type(e).__name__}: {str(e)[:160]}"}
        out["inference_100step"] = {
            "workload": "configs[1]: 100-step reverse diffusion, N_res=256, 32 frames, 1 GPU", **res,
            "note": "memoised = one trunk pass + 100 x (score-epilogue kernel + reverse-step kernel) on the device; memoised_graph = the "
                    "same work replayed from one CUDA graph (input copies included); literal = the "
                    "reference's schedule (whole network at every step) with the device reverse step"}
        del net, sampler, feats
        torch.cuda.empty_cache()
    except Exception as e:      # noqa: BLE001
        out["inference_100step"] = {"error": f"{type(e).__name__}: {str(e)[:200]}"}
    try:
        nf, N = 8, 1024
        net = _fresh_net(nf, dev)
        feats = {k: v.to(dev) for k, v in syn.make_feats(nf, N, seed=2).items()}
        ts = TrainStep(net, syn.surrogate_loss, feats, lr=1e-4, world_size=1, graph=graph, warmup=2)
        for _ in range(2):
            ts()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 5
        e0.record()
        for _ in range(n):
            ts()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        ipa_ms, alg, _, _ = time_ipa_core(dev, nf, N, iters=5)
        out["long_chain_1024"] = {
            "workload": "configs[4]: training step fwd+bwd+Adam, N_res=1024, 8 frames, 1 GPU", "ms_per_step": ms,
            "frames_per_s": nf / (ms * 1e-3), "cuda_graph": ts.graph is not None,
            "ipa_core_fwd": {"ms": ipa_ms, "algorithmic_GBs": alg / ipa_ms / 1e6, "algorithmic_MB": alg / 1e6}}
        del net, ts, feats
        torch.cuda.empty_cache()
    except Exception as e:      # noqa: BLE001
        out["long_chain_1024"] = {"error": f"{type(e).__name__}: {str(e)[:200]}"}
    try:
        # SURVEY.md 8 f4: one training window (64 frames x 256 residues) from pinned host trajectories to device features
        from dynamicpdb_b200.input_pipeline import featurize_window
        nf, N, T = 64, 256, 512
        g = torch.Generator().manual_seed(0)
        traj = torch.randn(T, N, 37, 3, generator=g).pin_memory()
        amask = torch.ones(N, 37).to(dev)
        aatype = torch.randint(0, 20, (N,), generator=g).to(dev)
        def one(start):
            return featurize_window(traj[start:start + nf].to(dev, non_blocking=True), amask, aatype)
        for i in range(3):
            one(i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 20
        e0.record()
        for i in range(n):
            one(7 * i)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        out["input_pipeline"] = {"workload": "window of 64 frames x 256 residues: H2D of the fp32 atom37 slice (7.3 MB, pinned) + "
                                             "featurize_window (rigids_0, torsion features)", "ms_per_window": ms,
                                 "frames_per_s": nf / (ms * 1e-3)}
    except Exception as e:      # noqa: BLE001
        out["input_pipeline"] = {"error": f"{type(e).__name__}: {str(e)[:200]}"}
    return out


def run_ours(args):
    import torch.distributed as dist
    from dynamicpdb_b200 import kernels as K
    from dynamicpdb_b200 import synthetic as syn
    from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
    from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert torch.cuda.is_available(), "bench.py needs a CUDA device (no CPU fallback)"
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        os.environ.setdefault("TORCH_NCCL_ASYNC_ERROR_HANDLING", "0")   # required for capturing NCCL in a CUDA graph
        dist.init_process_group("nccl", device_id=dev)
    K.lib()
    _log("process group + library ready")

    nf, N = args.frames, args.res
    torch.manual_seed(0)
    conf = syn.model_conf(nf, **syn.PRESET_A)
    net = FullScoreNetwork(conf, SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    net = net.to(dev)
    _log("model on device")
    from dynamicpdb_b200.train_step import TrainStep
    host = syn.make_feats(nf, N, seed=rank)                             # one protein window per rank
    host = {k: v.pin_memory() for k, v in host.items()}
    h2d_bytes = sum(v.numel() * v.element_size() for v in host.values())
    resident = {k: v.to(dev, non_blocking=True) for k, v in host.items()}
    loss_host = torch.zeros((), dtype=torch.float32).pin_memory()
    # forward + loss + backward + flat NCCL gradient all-reduce + Adam(amsgrad), captured in one CUDA graph
    ts = TrainStep(net, syn.surrogate_loss, resident, lr=1e-4, world_size=world, graph=not args.no_graph,
                   warmup=max(3, args.warmup))

    graph_on, graph_err = ts.graph is not None, ts.graph_error
    _log(f"train step ready (graph={graph_on}, err={graph_err})")

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(n, e2e):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            if e2e:
                ts.load(host)                                          # H2D of this step's inputs (pinned host memory)
                loss = ts()
                loss_host.copy_(loss, non_blocking=True)               # D2H of the step's result
            else:
                ts()
        e1.record()
        barrier()
        ms = e0.elapsed_time(e1) / n
        if world > 1:
            t = torch.tensor([ms], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = float(t.item())
        return ms

    for _ in range(args.warmup):
        ts()
    sampler = ClockSampler(local) if rank == 0 else None
    if sampler:
        sampler.start()
    ms = timed(args.steps, e2e=False)
    _log(f"timed region done: {ms:.1f} ms/step")
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, ts)
    ms_e2e = timed(args.steps, e2e=True)
    _log("e2e region done")
    clocks = sampler.stop() if sampler else None
    # per-kernel durations: the same step, launched eagerly with CUDA events around the C-ABI launches
    K.LAUNCH_COUNT = 0
    K.PROFILE = [] if rank == 0 else None
    prof_steps = 2
    for _ in range(prof_steps):
        ts._eager()
    torch.cuda.synchronize()
    launches = K.LAUNCH_COUNT // prof_steps
    prof, K.PROFILE = K.PROFILE, None

    # transparency: the same step with the reference's literal schedule (ConvNet on every frame in every block,
    # i.e. dead-frame elimination off) — every rank takes part (the step contains the gradient all-reduce)
    literal = None
    if not args.no_literal:
        try:
            from dynamicpdb_b200 import ipa_pytorch_dynamic as ipd
            if ipd._DEAD_FRAME_SKIP:
                ipd._DEAD_FRAME_SKIP = False
                ts_main, ts = ts, None
                ts = TrainStep(net, syn.surrogate_loss, resident, lr=1e-4, world_size=world, graph=not args.no_graph, warmup=2)
                ms_lit = timed(max(2, min(3, args.steps)), e2e=False)
                literal = {"value": world * nf / (ms_lit * 1e-3), "unit": "frames/s", "ms_per_step": ms_lit,
                           "note": "DFOLD_NO_DEAD_FRAME_SKIP=1 schedule: all 64 frames through the ConvNet in all 4 blocks"}
                ts = ts_main
                ipd._DEAD_FRAME_SKIP = True
        except Exception as e:      # noqa: BLE001
            literal = {"error": f"{type(e).__name__}: {str(e)[:160]}"}
    if rank != 0:
        _finish(world, dist)
        return

    # ---- roofline of the dominant kernel (the split-bf16 tensor-core GEMM) and of the fused IPA forward ----
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    tf_peak, tf_src = (peaks.get("bf16_tflops_sustained"), "measured (sustained)") if peaks.get("bf16_tflops_sustained") \
        else (989.0, "H100 SXM data sheet, dense BF16 at 700 W")
    hbm_peak, hbm_src = (peaks.get("hbm_gbs"), "measured") if peaks.get("hbm_gbs") else (3350.0, "H100 SXM data sheet")
    agg = {}
    for name, work, a, b, _tag in prof:
        t = a.elapsed_time(b) * 1e-3
        d = agg.setdefault(name, [0.0, 0.0, 0])
        d[0] += work
        d[1] += t
        d[2] += 1
    roof = None
    if "gemm_bf16x3" in agg:
        w, t, n = agg["gemm_bf16x3"]
        ach = w / t / 1e12
        roof = {"kernel": "gemm_bf16x3_kernel (implicit 5x5 conv / linear, 3 bf16 MMAs per fp32 product)",
                "bound": "tensor", "achieved": ach, "peak": tf_peak, "unit": "TFLOP/s", "frac": ach / tf_peak,
                "peak_source": tf_src, "launches_timed": n, "avg_launch_ms": 1e3 * t / n,
                "share_of_step": (t / prof_steps) / (ms * 1e-3), "tensor_pipe_frac": 3 * ach / tf_peak,
                "timed_in": "eager instrumented steps right after the timed (graph-replayed) region",
                "note": "achieved counts fp32-equivalent FLOPs; the split issues 3 bf16 MMAs per product, so frac <= 1/3"}
    roof_ipa = None
    try:
        ipa_ms, ipa_alg, ipa_launches, ipa_infer_ms = time_ipa_core(dev, nf, N)
        ach = ipa_alg / ipa_ms / 1e6
        in_step = None
        if "ipa_fwd" in agg:
            w, t, n = agg["ipa_fwd"]
            in_step = {"launches_timed": n, "avg_ms_eager_events": 1e3 * t / n,
                       "note": "event pairs around the op inside the eager instrumented steps; includes host launch gaps"}
        roof_ipa = {"kernel": "ipa_fused_fwd_kernel + P.V GEMM (fused IPA forward core, SURVEY.md 8d)", "bound": "hbm",
                    "achieved": ach, "peak": hbm_peak, "unit": "GB/s", "frac": ach / hbm_peak, "peak_source": hbm_src,
                    "algorithmic_bytes": ipa_alg,
                    "avg_launch_ms": ipa_ms, "inference_ms": ipa_infer_ms, "kernels_per_call": ipa_launches, "calls_per_step": 4,
                    "share_of_step": 4 * ipa_ms / ms, "in_step": in_step,
                    "timed_in": "20 back-to-back calls of the op at the benchmark shape, CUDA events on the launching stream, "
                                "inputs (659 MB) larger than L2",
                    "note": "training forward (also writes the 134 MB of bf16 probability planes the backward GEMMs read); inference_ms = "
                            "the same kernel without the planes; algorithmic bytes per SURVEY.md 8(d) (per-frame q/k/v formulation)"}
    except Exception as e:      # noqa: BLE001
        roof_ipa = {"error": f"{type(e).__name__}: {str(e)[:200]}"}

    cpu = None
    if not args.no_cpu_baseline and world == 1:
        r = cpu_arm(args.cpu_frames, N, 1, 2, float(os.environ.get("DFOLD_CPU_BASELINE_BUDGET_S", "90")))
        cpu = {"value": r["fps"], "unit": "frames/s", "cores": r["threads"], "kind": r["kind"],
               "sample": f"{r['steps_timed']} fwd+bwd of {args.cpu_frames} frames x {N} residues ({r['ms'] / 1e3:.1f} s each, "
                         f"after {r['warmup_run']} warm-up), {r['what']}", "thread_info": r["thread_info"]}

    extra = None
    if world == 1 and not args.no_extra:
        del ts
        torch.cuda.empty_cache()
        extra = extra_configs(dev, not args.no_graph)
        ts = None

    line = {
        "metric": METRIC, "value": world * nf / (ms * 1e-3), "unit": "frames/s", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32 (bf16x3 split on wgmma, fp32 accumulate)", "data": "synthetic",
        "config": {"workload": f"DFOLDv2 training step fwd+bwd+Adam, N_res={N}, batch={nf} frames per rank (configs[2])",
                   "frames_per_rank": nf, "n_res": N, "preset": "train_DFOLDv2.yaml (c_s 256, c_z 128, C 256, H 8, Pq 8, Pv 12, 4 blocks)",
                   "parallelism": f"dp{world}", "l2": "working set (weights 738 MB + activations) exceeds the 50 MB L2",
                   "gpu": torch.cuda.get_device_name(dev),
                   "cuda_graph": graph_on, "cuda_graph_error": graph_err,
                   "dead_frame_elimination": os.environ.get("DFOLD_NO_DEAD_FRAME_SKIP", "0") != "1"},
        "e2e": {"value": world * nf / (ms_e2e * 1e-3), "unit": "frames/s", "ms_per_step": ms_e2e,
                "h2d_bytes_per_step": h2d_bytes, "d2h_bytes_per_step": 4},
        "gpu_launches": launches, "clocks": clocks, "roofline": roof, "roofline_ipa": roof_ipa, "cpu_baseline": cpu,
        "literal_schedule": literal, "extra_configs": extra,
    }
    print(json.dumps(line), file=_REAL_STDOUT, flush=True)
    _finish(world, dist)


DUMP_SAMPLE = 1 << 21      # elements kept of each flat parameter-sized array


def dump_outputs(out_dir, ts):
    """What the last timed step handed back, as float32 / float64 .npy files: the loss it returns, and the updated
    parameters and gradients it leaves in place, as a fixed seeded sample of 2^21 positions of the flat arrays (their
    indices in `flat_index.npy`) -- 32 MB in all.  The inputs are seeded, so two builds run with the same arguments can
    be compared array for array."""
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    torch.cuda.synchronize()
    params = torch.cat([p.detach().reshape(-1) for p in ts.params])
    grads = torch.cat([(p.grad if p.grad is not None else torch.zeros_like(p)).detach().reshape(-1) for p in ts.params])
    n = params.numel()
    g = torch.Generator().manual_seed(0)
    idx = torch.randint(0, n, (min(n, DUMP_SAMPLE),), generator=g).sort().values
    np.save(os.path.join(out_dir, "loss.npy"), np.asarray([float(ts.loss)], dtype=np.float64))
    np.save(os.path.join(out_dir, "flat_index.npy"), idx.double().numpy())
    np.save(os.path.join(out_dir, "params_sample.npy"), params[idx.to(params.device)].float().cpu().numpy())
    np.save(os.path.join(out_dir, "grads_sample.npy"), grads[idx.to(grads.device)].float().cpu().numpy())
    del params, grads


def _finish(world, dist):
    """Leave without tearing the NCCL communicator down: destroy_process_group() blocks while a captured CUDA graph
    still references the communicator.  Every rank has finished measuring (the timed regions end with barriers)."""
    sys.stdout.flush()
    sys.stderr.flush()
    _REAL_STDOUT.flush()
    if world > 1:
        try:
            dist.barrier()
        except Exception:       # noqa: BLE001
            pass
        torch.cuda.synchronize()
        os._exit(0)


def _json_only_stdout():
    """Library banners (e.g. NCCL's version line) go to fd 1; keep fd 1 for the ONE JSON line by pointing it at stderr
    for the rest of the process and returning a private handle to the real stdout."""
    sys.stdout.flush()
    real = os.fdopen(os.dup(1), "w")
    os.dup2(2, 1)
    return real


if __name__ == "__main__":
    _REAL_STDOUT = _json_only_stdout()
    a = parse()
    if a.impl == "reference":
        run_reference(a)
    else:
        run_ours(a)
