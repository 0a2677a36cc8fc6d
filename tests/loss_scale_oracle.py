"""CPU oracle (numpy, fp32) of the train_op with dynamic loss scaling (include/gaccum.h, gaccum_loss_scale_config).

Built on ``oracle_np.ReferenceTrainOp``: accumulate steps are unchanged; on an apply step the normalised gradient is
``c = ((1.0*a')/N) * (1/S)``, the window is skipped when an element of ``a'`` or (with clipping) the global norm is not
finite, and S follows TF 2's ``DynamicLossScale`` counted in windows.  Test infrastructure only.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

import oracle_np as onp

F32 = np.float32


def update_scale(scale: np.float32, good: int, overflow: bool, multiplier: float, growth_interval: int):
    """(S, good) after one window.  Overflow: S = max(1, S / multiplier), good = 0.  Applied: S grows by the
    multiplier (if the product is finite) once good + 1 reaches growth_interval, and good restarts at 0."""
    mult = F32(multiplier)
    if overflow:
        return max(F32(1.0), F32(scale / mult)), 0
    if good + 1 >= growth_interval:
        with np.errstate(over="ignore"):
            up = F32(scale * mult)
        return (up if np.isfinite(up) else scale), 0
    return scale, good + 1


class LossScaledReferenceTrainOp(onp.ReferenceTrainOp):
    """``ReferenceTrainOp`` whose producer feeds gradients of ``loss * S``.  ``scale``, ``good_windows``,
    ``skipped_windows`` and ``last_skipped`` mirror gaccum_loss_scale_state."""

    def __init__(self, *args, initial_scale: float = 2.0 ** 15, multiplier: float = 2.0, growth_interval: int = 2000,
                 **kw):
        super().__init__(*args, **kw)
        self.scale = F32(initial_scale)
        self.multiplier, self.growth_interval = multiplier, int(growth_interval)
        self.good_windows = 0
        self.skipped_windows = 0
        self.last_skipped = False

    def run(self, grads: Sequence[Optional[np.ndarray]]) -> onp.StepInfo:
        g = self.global_step
        hp = self.hp
        lr = self.lr(g)
        is_apply = (int(np.int32(np.int64(g))) % self.N) == 0
        for a, gr in zip(self.accum, grads):
            if gr is not None:
                np.add(a, np.asarray(gr, dtype=F32).reshape(a.shape), out=a, dtype=F32)
        info = onp.StepInfo(global_step=g, applied=is_apply, lr=lr)
        if is_apply:
            nf = F32(self.N)
            inv_s = F32(F32(1.0) / self.scale)
            with np.errstate(over="ignore", invalid="ignore"):
                normalized = [np.multiply(np.divide(np.multiply(F32(1.0), a, dtype=F32), nf, dtype=F32), inv_s, dtype=F32)
                              for a in self.accum]
                overflow = any(not np.all(np.isfinite(a)) for a in self.accum)
                clipping = bool(hp.clip_norm and hp.clip_norm > 0)
                if clipping:
                    gn = self._global_norm(normalized)
                    s = onp.clip_scale(gn, hp.clip_norm)
                    info.global_norm, info.clip_scale = gn, s
                    overflow = overflow or not np.isfinite(gn)
                if not overflow:
                    clipped = [np.multiply(n, s, dtype=F32) for n in normalized] if clipping else normalized
                    for i, c in enumerate(clipped):
                        if hp.variant == onp.VARIANT_ADAM_WEIGHT_DECAY:
                            p2, m2, v2 = onp.adam_weight_decay_update(
                                self.params[i], self.m[i], self.v[i], c, lr, hp.beta1, hp.beta2,
                                hp.epsilon, hp.weight_decay_rate, self.decay[i])
                        else:
                            p2, m2, v2 = onp.adam_update(
                                self.params[i], self.m[i], self.v[i], c, lr, hp.beta1, hp.beta2,
                                hp.epsilon, self.beta1_power, self.beta2_power)
                        self.params[i][...] = p2; self.m[i][...] = m2; self.v[i][...] = v2
                    if hp.variant == onp.VARIANT_ADAM:
                        self.beta1_power = F32(self.beta1_power * F32(hp.beta1))
                        self.beta2_power = F32(self.beta2_power * F32(hp.beta2))
            self.scale, self.good_windows = update_scale(self.scale, self.good_windows, overflow, self.multiplier,
                                                         self.growth_interval)
            self.skipped_windows += int(overflow)
            self.last_skipped = overflow
            for a in self.accum:
                a[...] = F32(0.0)
            self.reduced = None
        self.global_step = g + 1
        return info
