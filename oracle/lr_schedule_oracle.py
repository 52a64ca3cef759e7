"""float64 restatement of AlphaFoldLRScheduler.get_lr (openfold/utils/lr_schedulers.py:64-82), the learning-rate schedule
the reference trainer imports (train_DFOLD_dynamics.py:56).  Python floats are IEEE binary64 and each operation below is
rounded on its own, in the reference's order, so the value equals the reference's bit for bit
(tests/golden/lr_schedule.pt); fp32 of it is what the device schedule kernel must produce.

TEST INFRASTRUCTURE ONLY: the package carries its own copy (train_step.AlphaFoldSchedule.lr) for checkpoints."""
import math

ALPHAFOLD_DEFAULTS = dict(base_lr=0.0, max_lr=0.001, warmup_no_steps=1000, start_decay_after_n_steps=50000,
                          decay_every_n_steps=50000, decay_factor=0.95)
TEST_AF2_DEFAULTS = dict(base_lr=0.0, max_lr=0.0001, warmup_no_steps=10, start_decay_after_n_steps=100,
                         decay_every_n_steps=10, decay_factor=0.95)


def alphafold_lr(step: int, base_lr: float, max_lr: float, warmup_no_steps: int, start_decay_after_n_steps: int,
                 decay_every_n_steps: int, decay_factor: float) -> float:
    """The lr at last_epoch = step: the lr of optimizer step step + 1 (the scheduler steps once in its constructor)."""
    assert isinstance(step, int) and step >= 0
    if step <= warmup_no_steps:                                         # linear warmup from base_lr
        frac = float(step) / float(warmup_no_steps)
        return float(base_lr) + frac * float(max_lr)
    if step > start_decay_after_n_steps:                                # step decay, first factor one step after the start
        e = (step - start_decay_after_n_steps) // decay_every_n_steps + 1
        return float(max_lr) * math.pow(float(decay_factor), float(e))
    return float(max_lr)                                                # plateau
