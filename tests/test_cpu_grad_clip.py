"""TrainStep(max_grad_norm=...) refuses what it cannot honour before it touches a device: a value that is not a positive
number, and clipping combined with the chunked all-reduce (DFOLD_ALLREDUCE_CHUNKS > 1 on more than one rank), which
updates each piece of the gradient before the global norm exists."""
import math

import pytest
import torch

from dynamicpdb_b200.train_step import TrainStep, _check_max_grad_norm


def _make(**kw):
    return TrainStep(torch.nn.Linear(4, 4), lambda out: out, {}, **kw)


@pytest.mark.parametrize("bad", [0, 0.0, -1.0, -math.inf, math.nan, "1.0", True, torch.tensor(1.0), [1.0]])
def test_bad_max_grad_norm_is_refused(bad):
    with pytest.raises(ValueError, match="max_grad_norm"):
        _make(max_grad_norm=bad)


def test_good_max_grad_norm_values():
    assert _check_max_grad_norm(None) is None
    assert _check_max_grad_norm(1) == 1.0 and isinstance(_check_max_grad_norm(1), float)
    assert _check_max_grad_norm(0.25) == 0.25
    assert _check_max_grad_norm(math.inf) == math.inf


def test_clipping_with_chunked_all_reduce_is_refused(monkeypatch):
    monkeypatch.setenv("DFOLD_ALLREDUCE_CHUNKS", "2")
    monkeypatch.setenv("DFOLD_TORCH_ADAM", "0")
    for max_grad_norm in (1.0, math.inf):
        with pytest.raises(ValueError, match="DFOLD_ALLREDUCE_CHUNKS"):
            _make(world_size=2, max_grad_norm=max_grad_norm)
