"""Checkpoints of the captured training step (train_step.TrainStep) in the reference trainer's format.

The reference writes ``{'model', 'conf', 'optimizer', 'epoch', 'step'}`` with ``du.write_checkpoint``
(train_DFOLD_dynamics.py:743-755, src/data/utils.py:324-362): ``model`` is the network's state_dict (``module.``-prefixed
under DDP) and ``optimizer`` is ``torch.optim.Adam(model.parameters(), lr, amsgrad=True).state_dict()`` (:412), whose
``state`` is keyed by the parameter's index in ``model.parameters()`` order and has no entry for a parameter that never
received a gradient.  ``TrainStep`` keeps the same state in flat device buffers (the trained parameters back to back, padded
to a multiple of four elements); the functions here map between those buffers, taken to the host, and that dict, and
validate a dict before anything is written, so that a refused load leaves the step untouched.  A step that keeps a
moving average of the weights (``TrainStep(ema_decay=...)``) adds OpenFold's ``ema`` entry,
``ExponentialMovingAverage.state_dict()``.
"""
import numbers
import os
import pickle
import tempfile
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple

import torch

ADAM_BETAS = (0.9, 0.999)
ADAM_EPS = 1e-8
STATE_KEYS = ("step", "exp_avg", "exp_avg_sq", "max_exp_avg_sq")
MOMENTS = STATE_KEYS[1:]


class FlatLayout(NamedTuple):
    """Where each parameter of ``net.parameters()`` sits in the flat buffers (offset None: the step does not train it)."""
    names: List[str]
    shapes: List[torch.Size]
    offsets: List[Optional[int]]
    numel: int                                     # the buffers' length: the trained elements rounded up to a multiple of 4


def flat_layout(net: torch.nn.Module) -> FlatLayout:
    names, shapes, offsets, off = [], [], [], 0
    for name, p in net.named_parameters():
        names.append(name)
        shapes.append(p.shape)
        offsets.append(off if p.requires_grad else None)
        off += p.numel() if p.requires_grad else 0
    return FlatLayout(names, shapes, offsets, (off + 3) // 4 * 4)


def views(layout: FlatLayout, flat: torch.Tensor) -> List[Optional[torch.Tensor]]:
    """Per-parameter views of one flat buffer, None for the parameters it does not hold."""
    return [None if o is None else flat[o:o + s.numel()].view(s) for s, o in zip(layout.shapes, layout.offsets)]


def adam_param_groups(n_params: int, lr: float) -> list:
    """``param_groups`` of ``torch.optim.Adam(params, lr, amsgrad=True).state_dict()`` over n_params parameters, taken from
    such an optimizer so that the installed torch's field set is reproduced exactly."""
    dummies = [torch.nn.Parameter(torch.empty(0)) for _ in range(n_params)]
    return torch.optim.Adam(dummies, lr=lr, betas=ADAM_BETAS, eps=ADAM_EPS, amsgrad=True).state_dict()["param_groups"]


def optimizer_state_dict(layout: FlatLayout, exp_avg: torch.Tensor, exp_avg_sq: torch.Tensor, max_exp_avg_sq: torch.Tensor,
                         step: float, lr: float, indices: Optional[Sequence[int]] = None,
                         initial_lr: Optional[float] = None) -> dict:
    """Host flat moment buffers -> the state_dict of ``torch.optim.Adam(net.parameters(), lr, amsgrad=True)``.  Every
    trained parameter gets an entry (``indices``: only those), each with its own float32 ``step`` tensor (torch increments
    them one by one) and views of the flat buffers for the moments.  ``initial_lr``: the optimizer's lr before a
    learning-rate scheduler took over, which torch's LRScheduler adds to the param group."""
    keep = None if indices is None else set(indices)
    per = [views(layout, b) for b in (exp_avg, exp_avg_sq, max_exp_avg_sq)]
    state = {}
    for i, o in enumerate(layout.offsets):
        if o is None or (keep is not None and i not in keep):
            continue
        state[i] = {"step": torch.tensor(float(step), dtype=torch.float32),
                    **{k: v[i] for k, v in zip(MOMENTS, per)}}
    groups = adam_param_groups(len(layout.names), lr)
    if initial_lr is not None:
        groups[0]["initial_lr"] = initial_lr
    return {"state": state, "param_groups": groups}


def strip_module_prefix(model: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Names as the un-wrapped network has them: DDP prefixes every key with ``module.`` (removed on load as
    train_DFOLD_dynamics.py:481 and eval_DFOLD_dynamics.py:133 do)."""
    return {(k[len("module."):] if k.startswith("module.") else k): v for k, v in model.items()}


def _names(keys, limit=4):
    keys = sorted(keys, key=str)
    return ", ".join(map(str, keys[:limit])) + (f" and {len(keys) - limit} more" if len(keys) > limit else "")


def check_model(sd: dict, model_shapes: Dict[str, torch.Size]) -> Dict[str, torch.Tensor]:
    """Validates the ``model`` state_dict of a checkpoint dict against a network's ``{name: shape}`` and returns its
    tensors by the network's own names (``module.`` stripped).  Raises ValueError naming the unknown or missing keys, or
    the first tensor whose shape differs, so that a strict ``load_state_dict`` of the result cannot fail half-way."""
    if not isinstance(sd, dict) or not isinstance(sd.get("model"), dict):
        raise ValueError("checkpoint has no 'model' state_dict")
    return _check_params(sd["model"], model_shapes, "model")


def _check_params(params: dict, model_shapes: Dict[str, torch.Size], what: str) -> Dict[str, torch.Tensor]:
    model = strip_module_prefix(params)
    unknown, missing = set(model) - set(model_shapes), set(model_shapes) - set(model)
    if unknown or missing:
        raise ValueError(f"checkpoint {what} does not match the network: unknown keys [{_names(unknown)}], "
                         f"missing keys [{_names(missing)}]")
    for k, shape in model_shapes.items():
        if not torch.is_tensor(model[k]) or tuple(model[k].shape) != tuple(shape):
            got = tuple(model[k].shape) if torch.is_tensor(model[k]) else type(model[k]).__name__
            raise ValueError(f"checkpoint {what} '{k}' has shape {got}, the network {tuple(shape)}")
    return model


def check_ema(sd: dict, model_shapes: Dict[str, torch.Size], decay: Optional[float] = None
              ) -> Optional[Dict[str, torch.Tensor]]:
    """Validates the ``ema`` entry of a checkpoint dict, OpenFold's ``ExponentialMovingAverage.state_dict()``
    (``{'params': the averaged net.state_dict(), 'decay': float}``), and returns its tensors by the network's own names
    (``module.`` stripped), or None when the checkpoint has no ``ema``.  Raises ValueError for unknown or missing keys, a
    shape that differs, a tensor that is not float32, or, when ``decay`` is given, a decay other than it."""
    ema = sd.get("ema") if isinstance(sd, dict) else None
    if ema is None:
        return None
    if not isinstance(ema, dict) or not isinstance(ema.get("params"), dict):
        raise ValueError("checkpoint ema has no 'params' state_dict")
    d = ema.get("decay")
    if isinstance(d, bool) or not isinstance(d, numbers.Real):
        raise ValueError(f"checkpoint ema decay must be a number, got {d!r}")
    params = _check_params(ema["params"], model_shapes, "ema")
    for k in model_shapes:
        if params[k].dtype != torch.float32:
            raise ValueError(f"checkpoint ema '{k}' is {params[k].dtype}; the average is kept in torch.float32")
    if decay is not None and float(d) != decay:
        raise ValueError(f"checkpoint ema decay {d!r} differs from the training step's {decay!r}: construct "
                         f"TrainStep(ema_decay={d!r}) to resume this checkpoint")
    return params


def check_state(sd: dict, layout: FlatLayout, model_shapes: Dict[str, torch.Size], lr: float, schedule=None
                ) -> Tuple[Dict[str, torch.Tensor], Optional[Dict[int, dict]], float]:
    """Validates a checkpoint dict against the step it is to be loaded into and returns (model tensors by the network's
    own names, optimizer state entries by parameter index or None for a weights-only load, the common step).  Raises
    ValueError, naming the problem, for anything that would resume a different optimisation than the one saved.
    ``schedule`` (train_step.AlphaFoldSchedule or None): the checkpoint's lr must be ``schedule.lr(step)``, the lr a
    scheduler stepped once per optimizer step leaves in the param group, instead of ``lr``."""
    model = check_model(sd, model_shapes)
    opt = sd.get("optimizer")
    if opt is None:
        return model, None, 0.0
    groups = opt.get("param_groups") if isinstance(opt, dict) else None
    if not isinstance(groups, list) or len(groups) != 1:
        raise ValueError(f"checkpoint optimizer has {len(groups) if isinstance(groups, list) else 'no'} param groups; "
                         "the training step has a single one")
    g = groups[0]
    if schedule is None and g.get("lr") != lr:
        raise ValueError(f"checkpoint lr {g.get('lr')!r} differs from the training step's {lr!r}; the lr is part of the "
                         f"captured step: construct TrainStep(lr={g.get('lr')!r}) to resume this checkpoint")
    want = {"betas": ADAM_BETAS, "eps": ADAM_EPS, "weight_decay": 0, "amsgrad": True, "maximize": False}
    for k, v in want.items():
        got = g.get(k, False if k == "maximize" else None)
        if (tuple(got) if isinstance(got, (list, tuple)) else got) != v:
            raise ValueError(f"checkpoint optimizer has {k}={got!r}; the training step runs Adam with {k}={v!r}")
    n = len(layout.names)
    if list(g.get("params", [])) != list(range(n)):
        raise ValueError(f"checkpoint optimizer covers {len(g.get('params', []))} parameters, the network has {n}")
    entries, steps = {}, set()
    for i, st in opt.get("state", {}).items():
        if not isinstance(i, int) or not 0 <= i < n:
            raise ValueError(f"checkpoint optimizer state has an entry for parameter {i!r}, the network has {n}")
        if layout.offsets[i] is None:
            raise ValueError(f"checkpoint optimizer state has an entry for '{layout.names[i]}', which the step does not train")
        absent = [k for k in STATE_KEYS if k not in st]
        if absent:
            raise ValueError(f"checkpoint optimizer state of '{layout.names[i]}' lacks {absent}")
        for k in MOMENTS:
            if not torch.is_tensor(st[k]) or tuple(st[k].shape) != tuple(layout.shapes[i]):
                raise ValueError(f"checkpoint optimizer state '{k}' of '{layout.names[i]}' has shape "
                                 f"{tuple(st[k].shape) if torch.is_tensor(st[k]) else None}, the parameter {tuple(layout.shapes[i])}")
        steps.add(float(st["step"]))
        entries[i] = st
    if len(steps) > 1:
        raise ValueError(f"checkpoint optimizer state has different step counts {sorted(steps)}; the training step keeps "
                         "a single one")
    step = steps.pop() if steps else 0.0
    if schedule is not None:
        if not (step >= 0 and step == int(step)):
            raise ValueError(f"checkpoint optimizer step {step!r} is not a whole number of steps")
        want = schedule.lr(int(step))
        if g.get("lr") != want:
            raise ValueError(f"checkpoint lr {g.get('lr')!r} at step {int(step)} is not the learning-rate schedule's {want!r} "
                             f"there: it was saved under a different schedule ({schedule})")
    return model, entries, step


def model_to_flat(layout: FlatLayout, model: Dict[str, torch.Tensor]) -> torch.Tensor:
    """The trained parameters of a (validated, un-prefixed) model dict as one host flat fp32 buffer, zero padding."""
    flat = torch.zeros(layout.numel, dtype=torch.float32)
    for name, v in zip(layout.names, views(layout, flat)):
        if v is not None:
            v.copy_(model[name])
    return flat


def optimizer_to_flat(layout: FlatLayout, entries: Optional[Dict[int, dict]]) -> List[torch.Tensor]:
    """exp_avg, exp_avg_sq, max_exp_avg_sq of (validated) state entries as host flat fp32 buffers.  A trained parameter
    without an entry gets zero moments: the reference writes none for parameters that never received a gradient, and
    Adam moves such a parameter by exactly nothing from zero moments."""
    flats = [torch.zeros(layout.numel, dtype=torch.float32) for _ in MOMENTS]
    for k, flat in zip(MOMENTS, flats):
        per = views(layout, flat)
        for i, st in (entries or {}).items():
            per[i].copy_(st[k])
    return flats


def save_checkpoint(path: str, train_step, conf, epoch: int, step: int) -> None:
    """Writes ``du.write_checkpoint``'s dict ``{'model', 'conf', 'optimizer', 'epoch', 'step'}`` for ``train_step``
    (``conf`` as given: the evaluator reads ``conf.model``), and ``ema`` after them when the step keeps a moving average
    of the weights, as OpenFold's checkpoints carry it.  The file is written next to ``path`` under a temporary name
    and renamed onto it, so an interrupted save leaves the previous checkpoint in place."""
    sd = train_step.state_dict()
    ckpt = {"model": sd["model"], "conf": conf, "optimizer": sd["optimizer"], "epoch": epoch, "step": step}
    if "ema" in sd:
        ckpt["ema"] = sd["ema"]
    d = os.path.dirname(os.path.abspath(path))
    fd, tmp = tempfile.mkstemp(dir=d, prefix=os.path.basename(path) + ".", suffix=".tmp")
    try:
        with os.fdopen(fd, "wb") as f:
            torch.save(ckpt, f, pickle_protocol=pickle.HIGHEST_PROTOCOL)
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.unlink(tmp)
        raise


def load_checkpoint(path: str, train_step) -> Tuple[int, int]:
    """Loads a checkpoint written by save_checkpoint or by the reference trainer into ``train_step`` in place and returns
    its (epoch, step).  Checkpoints are trusted input: ``conf`` is an arbitrary pickled object, so the file is read with
    ``weights_only=False`` as the reference does; never load a checkpoint from an untrusted source."""
    ckpt = torch.load(path, map_location="cpu", weights_only=False)
    train_step.load_state_dict(ckpt)
    return ckpt.get("epoch"), ckpt.get("step")
