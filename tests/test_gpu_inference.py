"""-m gpu: reverse-diffusion sampling on the device (SURVEY.md §8 f2, BASELINE.json configs[1])."""
import pytest
import torch

from dynamicpdb_b200 import kernels as K
from dynamicpdb_b200 import rigid_utils as ru
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork
from dynamicpdb_b200.inference import DeviceReverseDiffusion, MemoizedScoreNetwork
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from oracle import dfold_oracle as O
from tests.test_cpu_oracle import close, load, reverse_case

pytestmark = pytest.mark.gpu
DEV = "cuda"


def test_reverse_step_kernel_matches_reference_golden_and_oracle():
    """The reverse-step kernel through the diffuser-shaped API (reference signature) against SE3Diffuser.reverse of the
    unmodified reference (tests/golden/reverse.pt) with the same normal draws, and against the oracle without a mask."""
    c = reverse_case()
    d = SE3ScoreDiffuser(syn.diffuser_conf(c["cs"]))
    rig = ru.Rigid.from_tensor_7(c["rig"].to(DEV))
    out = d.reverse(rig, c["rot_score"].numpy(), c["trans_score"].numpy(), c["t"], c["dt"], diffuse_mask=c["mask"].numpy(),
                    center=True, noise_scale=c["noise_scale"], z_rot=c["z_rot"].float(), z_trans=c["z_trans"].float()).to_tensor_7()
    out = torch.cat([torch.where(out[..., :1] < 0, -out[..., :4], out[..., :4]), out[..., 4:]], dim=-1).cpu()
    assert close(out, load("reverse")["rigids_t_1"], 5e-6)
    for center in (True, False):
        o2 = d.reverse(rig, c["rot_score"].to(DEV), c["trans_score"].float().to(DEV), 0.9, 0.05, diffuse_mask=None, center=center,
                       noise_scale=1.0, z_rot=c["z_rot"].float(), z_trans=c["z_trans"].float()).to_tensor_7().cpu()
        o2 = torch.cat([torch.where(o2[..., :1] < 0, -o2[..., :4], o2[..., :4]), o2[..., 4:]], dim=-1)
        ref = O.reverse_step(c["rig"], c["rot_score"], c["trans_score"].float(), 0.9, 0.05, None, c["z_rot"].float(), c["z_trans"].float(),
                             O.default_diffuser_conf(c["cs"]), center=center, noise_scale=1.0)
        assert close(o2, ref, 5e-6)


def _net(nf, preset):
    torch.manual_seed(0)
    net = FullScoreNetwork(syn.model_conf(nf, **preset), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    sd = net.state_dict()
    syn.dezero_(sd)
    net.load_state_dict(sd)
    return net.to(DEV).eval()


def test_device_sampler_matches_literal_loop(monkeypatch):
    """One trunk pass + per-step score / reverse kernels == evaluating the whole network at every step (same noise).
    The comparison of two runs relies on the kernels' fixed accumulation order (run-to-run rounding noise would be amplified
    without bound by u / |u| of a near-zero torsion)."""
    nf, N, num_t = 3, 24, 7
    net = _net(nf, syn.PRESET_TINY)
    feats = {k: v.to(DEV) for k, v in syn.make_feats(nf, N, seed=6).items()}
    feats["fixed_mask"][:, 0] = 1
    g = torch.Generator().manual_seed(1)
    noise = (torch.randn(num_t, nf, N, 3, generator=g).to(DEV), torch.randn(num_t, nf, N, 3, generator=g).to(DEV))
    s = DeviceReverseDiffusion(net)
    a = s.sample(feats, num_t, 0.01, noise_scale=0.5, noise=noise)
    b = s.sample(feats, num_t, 0.01, noise_scale=0.5, noise=noise, literal=True)
    assert a["prot_traj"].shape == (num_t, nf, N, 37, 3)
    for k in a:
        assert close(a[k].cpu(), b[k].cpu(), 1e-6), k
    assert float((a["rigids"][:, 0, 4:] - feats["rigids_t"][:, 0, 4:]).abs().max()) > 0     # last step returns the prediction


def test_graphed_sampler_replays_match_eager(monkeypatch):
    """The trunk pass + every score / reverse step captured in one CUDA graph: replays with new inputs reproduce the eager
    loop (injected noise, fixed accumulation order)."""
    nf, N, num_t = 3, 24, 6
    net = _net(nf, syn.PRESET_TINY)
    g = torch.Generator().manual_seed(2)
    noise = (torch.randn(num_t, nf, N, 3, generator=g).to(DEV), torch.randn(num_t, nf, N, 3, generator=g).to(DEV))
    s = DeviceReverseDiffusion(net)
    for seed in (6, 7):                                      # second window: a pure replay from the static buffers
        feats = {k: v.to(DEV) for k, v in syn.make_feats(nf, N, seed=seed).items()}
        a = s.sample_graphed(feats, num_t, 0.01, noise_scale=0.5, noise=noise)
        s.memo.reset()
        b = s.sample(feats, num_t, 0.01, noise_scale=0.5, noise=noise)
        for k in b:
            assert a[k].shape == b[k].shape and close(a[k].cpu(), b[k].cpu(), 1e-6), (seed, k)
    assert len(s._graphs) == 1
    c = s.sample_graphed(feats, num_t, 0.01, noise_scale=0.5)    # device-generated noise: its own graph, finite output
    assert len(s._graphs) == 2 and bool(torch.isfinite(c["rigids"]).all())


def test_memoized_network_on_gpu_and_cache_invalidation(monkeypatch):
    """MemoizedScoreNetwork on CUDA: a new window allocated at the same address must NOT hit the cache (ADVICE r1)."""
    nf, N = 3, 16
    net = _net(nf, syn.PRESET_TINY)
    memo = MemoizedScoreNetwork(net)
    outs = []
    for seed in (3, 4):
        feats = {k: v.to(DEV) for k, v in syn.make_feats(nf, N, seed=seed).items()}
        with torch.no_grad():
            full = net(dict(feats))
        fast1 = memo(dict(feats))
        feats2 = dict(feats)
        feats2["t"] = torch.tensor([0.2], device=DEV)
        feats2["rigids_t"] = syn.make_feats(nf, N, seed=50 + seed)["rigids_t"].to(DEV)
        with torch.no_grad():
            full2 = net(dict(feats2))
        fast2 = memo(dict(feats2))                                   # trunk inputs unchanged -> cached trunk, fresh scores
        for k in full:
            assert close(fast1[k].cpu(), full[k].cpu(), 1e-6), k
            assert close(fast2[k].cpu(), full2[k].cpu(), 1e-6), k
        outs.append(full["rigids"].cpu())
        del feats, feats2                                           # the next window may land on the same addresses
    assert not close(outs[0], outs[1], 1e-3)
    # weights changed in place -> the cache must miss
    feats = {k: v.to(DEV) for k, v in syn.make_feats(nf, N, seed=3).items()}
    a = memo(dict(feats))["rigids"].clone()
    with torch.no_grad():
        for p_ in net.score_model.trunk["bb_update_3"].parameters():
            p_.mul_(2.0)
    b = memo(dict(feats))["rigids"]
    assert float((a - b).abs().max()) > 1e-6
