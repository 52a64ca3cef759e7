"""Argument checks of the batched-windows path, all raised before any device work (no GPU needed):
kernels.conv5x5(windows=...), kernels.global_layernorm(segments=...), FullScoreNetwork.forward_windows, and the
``batched`` flag of TrainStep and Trainer."""
import pytest
import torch

from dynamicpdb_b200 import kernels as K
from dynamicpdb_b200 import synthetic as syn
from dynamicpdb_b200.Dfold_network_dynamic import FullScoreNetwork, check_windows
from dynamicpdb_b200.score_epilogue import SE3ScoreDiffuser
from dynamicpdb_b200.train_step import TrainStep


@pytest.mark.parametrize("windows,msg", [(0, "positive integer"), (-2, "positive integer"), (True, "positive integer"),
                                         (2.0, "positive integer"), (4, "does not divide the 6 frames")])
def test_conv_refuses_bad_windows(windows, msg):
    x, w = torch.zeros(6, 4, 8), torch.zeros(8, 8, 5, 5)
    with pytest.raises(ValueError, match=msg):
        K.conv5x5(x, w, windows=windows)


def test_conv_refuses_a_crop_that_empties_the_windows():
    x, w = torch.zeros(6, 4, 8), torch.zeros(8, 8, 5, 5)
    with pytest.raises(ValueError, match="removes every frame of the 3-frame windows"):
        K.conv5x5(x, w, crop=3, windows=2)


@pytest.mark.parametrize("segments,msg", [(0, "positive integer"), (False, "positive integer"), (1.5, "positive integer"),
                                          (5, "does not divide the 6 rows"), (6, "at least 2 elements")])
def test_layer_norm_refuses_bad_segments(segments, msg):
    with pytest.raises(ValueError, match=msg):
        K.global_layernorm(torch.zeros(6, 1), segments=segments)


def test_windowed_ops_keep_refusing_cpu_tensors():
    with pytest.raises(RuntimeError, match="need CUDA tensors"):
        K.conv5x5(torch.zeros(4, 4, 8), torch.zeros(8, 8, 5, 5), windows=2)
    with pytest.raises(RuntimeError, match="need CUDA tensors"):
        K.global_layernorm(torch.zeros(4, 3), segments=2)


def _w(nf=3, n=16, seed=0, **kw):
    return syn.make_feats(nf, n, seed=seed, **kw)


def test_windows_must_share_residue_and_frame_counts():
    check_windows([_w(), _w(seed=1, t=0.9)])                         # distinct proteins and t: accepted
    with pytest.raises(ValueError, match="window 1 has 20 residues and window 0 has 16"):
        check_windows([_w(), _w(n=20)])
    with pytest.raises(ValueError, match="window 1 has 4 frames and window 0 has 3"):
        check_windows([_w(), _w(nf=4)])
    with pytest.raises(ValueError, match="non-empty list"):
        check_windows([])
    with pytest.raises(ValueError, match="non-empty list"):
        check_windows(_w())
    with pytest.raises(ValueError, match="dict of input tensors"):
        check_windows([_w(), 3])
    other = _w()
    other["force"] = other["force"].double()
    with pytest.raises(ValueError, match="'force' of window 1"):
        check_windows([_w(), other])
    missing = _w()
    del missing["vel"]
    with pytest.raises(ValueError, match="keys"):
        check_windows([_w(), missing])


def test_forward_windows_refuses_before_any_device_work(monkeypatch):
    """The check runs before the first kernel: with every launch made to fail, the ValueError still comes first."""
    net = FullScoreNetwork(syn.model_conf(3, **syn.PRESET_TINY), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))

    def no_launch(*a, **kw):
        raise AssertionError("device work before the argument check")
    monkeypatch.setattr(K, "launch", no_launch)
    monkeypatch.setattr(K, "linear", no_launch)
    with pytest.raises(ValueError, match="residues"):
        net.forward_windows([_w(), _w(n=20)])


def test_train_step_refuses_bad_batched():
    net = FullScoreNetwork(syn.model_conf(3, **syn.PRESET_TINY), SE3ScoreDiffuser(syn.diffuser_conf(1.0)))
    with pytest.raises(ValueError, match="batched must be True or False"):
        TrainStep(net, syn.surrogate_loss, _w(), batched=1)
    with pytest.raises(ValueError, match="needs a network with forward_windows"):
        TrainStep(torch.nn.Linear(2, 2), syn.surrogate_loss, _w(), batched=True)


def test_trainer_refuses_bad_batched():
    from dynamicpdb_b200.trainer import Trainer
    with pytest.raises(ValueError, match="batched must be True or False"):
        Trainer({}, None, None, batched="yes")
