"""The learning-rate schedule of mortal/train.py: a linear warm-up from `init` to `peak` over `warm_up_steps`, then a half cosine
from `peak` down to `final` at `max_steps`, `final` afterwards. `offset` shifts the step count; with `epoch_size` > 0 the
(shifted) step count wraps every `epoch_size` steps. The optimizer's lr is 1, so the factor is the learning rate itself.

It keeps the attribute names of the reference's LinearWarmUpCosineAnnealingLR (init, peak, final, warm_up_steps, max_steps,
offset, epoch_size), so the `scheduler` entry of a state file loads in either trainer."""
from __future__ import annotations

import math

from torch.optim.lr_scheduler import LambdaLR


class LinearWarmUpCosineAnnealingLR(LambdaLR):
    def __init__(self, optimizer, *, peak, final, warm_up_steps, max_steps, init=1e-8, offset=0, epoch_size=0, **kwargs):
        if not peak >= final >= init >= 0:
            raise ValueError(f"need peak >= final >= init >= 0, got peak={peak}, final={final}, init={init}")
        if max_steps < warm_up_steps:
            raise ValueError(f"max_steps ({max_steps}) must be at least warm_up_steps ({warm_up_steps})")
        self.init = init
        self.peak = peak
        self.final = final
        self.warm_up_steps = warm_up_steps
        self.max_steps = max_steps
        self.offset = offset
        self.epoch_size = epoch_size
        super().__init__(optimizer=optimizer, lr_lambda=self.lr_at, **kwargs)

    def lr_at(self, step: int) -> float:
        """the learning rate after `step` scheduler steps"""
        step += self.offset
        if self.epoch_size > 0:
            step %= self.epoch_size
        if self.warm_up_steps > 0 and step < self.warm_up_steps:
            return self.init + (self.peak - self.init) / self.warm_up_steps * step  # the slope first: the same rounding as train.py
        if step >= self.max_steps:
            return self.final
        progress = (step - self.warm_up_steps) / (self.max_steps - self.warm_up_steps)
        return self.final + 0.5 * (self.peak - self.final) * (1 + math.cos(progress * math.pi))
