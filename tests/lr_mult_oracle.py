"""CPU oracle (numpy, fp32) of the train_op with per-tensor learning-rate multipliers (include/gaccum.h,
gaccum_plan_set_lr_multipliers).

Tensor t trains with ``lr_t = fp32(lr * mult[t])`` -- one correctly rounded fp32 multiply -- in place of the step's lr:
AdamWeightDecay ``p - lr_t*u``, Adam ``alpha_t = (lr_t*sqrt(1-b2^t)) / (1-b1^t)``, LAMB ``p - (r*lr_t)*u``.  Everything
else is the existing oracles' arithmetic, op for op: ``oracle_np.adam_weight_decay_update`` / ``adam_update`` and
``lamb_oracle.lamb_update`` per tensor, the window logic of ``ReferenceTrainOp``, the loss scaling of
``loss_scale_oracle`` (``initial_scale`` given) and LAMB's adaptation mask.  One class covers the three variants; with
every multiplier at 1 it computes what ``ReferenceTrainOp`` / ``LossScaledReferenceTrainOp`` / ``LambReferenceTrainOp``
compute, bit for bit (tests/test_lr_multipliers_host.py checks that).  ``reference_op`` is ``apply_matrix.reference_op``
with a table.  Test infrastructure only.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

import oracle_np as onp
from apply_matrix import LS_CFG, SCHED, LockStep, oracle_hparams
from lamb_oracle import adaptation_mask, lamb_update, reduced_ratios
from loss_scale_oracle import update_scale

F32 = np.float32
VARIANT_LAMB = 2


class LrMultReferenceTrainOp(onp.ReferenceTrainOp):
    """``ReferenceTrainOp`` with a per-tensor learning-rate multiplier ``lr_mult`` (default: 1 everywhere), any variant
    (hp.variant 0, 1 or 2), with or without loss scaling (``initial_scale``).  LAMB: ``adapt`` / ``adapt_exclude`` and
    ``ratios`` as in ``LambReferenceTrainOp``.  Loss scaling: ``scale`` / ``good_windows`` / ``skipped_windows`` /
    ``last_skipped`` as in ``LossScaledReferenceTrainOp``."""

    def __init__(self, params, names, hp, accum_n, *, lr_mult: Optional[Sequence[float]] = None,
                 adapt: Optional[Sequence[bool]] = None, adapt_exclude=None, initial_scale: Optional[float] = None,
                 multiplier: float = 2.0, growth_interval: int = 2000, **kw):
        super().__init__(params, names, hp, accum_n, **kw)
        T = len(self.params)
        self.lr_mult = [F32(1.0)] * T if lr_mult is None else [F32(m) for m in lr_mult]
        assert len(self.lr_mult) == T
        exclude = kw.get("exclude", onp.DEFAULT_EXCLUDE)
        self.adapt = list(adapt) if adapt is not None else \
            adaptation_mask(names, adapt_exclude if adapt_exclude is not None else exclude)
        self.ratios = [F32(1.0)] * T
        self.ls = initial_scale is not None
        self.scale = F32(initial_scale if self.ls else 1.0)
        self.multiplier, self.growth_interval = multiplier, int(growth_interval)
        self.good_windows = self.skipped_windows = 0
        self.last_skipped = False

    def lr_t(self, lr: np.float32, i: int) -> np.float32:
        return np.multiply(F32(lr), self.lr_mult[i], dtype=F32)

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
            with np.errstate(over="ignore", invalid="ignore"):
                c = [np.divide(np.multiply(F32(1.0), a, dtype=F32), nf, dtype=F32) for a in self.accum]
                overflow = False
                if self.ls:
                    inv_s = F32(F32(1.0) / self.scale)
                    c = [np.multiply(x, inv_s, dtype=F32) for x in c]
                    overflow = any(not np.all(np.isfinite(a)) for a in self.accum)
                if hp.clip_norm and hp.clip_norm > 0:
                    gn = self._global_norm(c)
                    s = onp.clip_scale(gn, hp.clip_norm)
                    info.global_norm, info.clip_scale = gn, s
                    overflow = overflow or (self.ls and not np.isfinite(gn))
                    if not overflow:
                        c = [np.multiply(x, s, dtype=F32) for x in c]
            if not overflow:
                ratios, self.window_pu = reduced_ratios(self)
                for i, ci in enumerate(c):
                    lr_t = self.lr_t(lr, i)
                    if hp.variant == VARIANT_LAMB:
                        p2, m2, v2, r = lamb_update(self.params[i], self.m[i], self.v[i], ci, lr_t, hp.beta1, hp.beta2,
                                                    hp.epsilon, hp.weight_decay_rate, self.decay[i], self.adapt[i],
                                                    self.beta1_power, self.beta2_power, ratios[i], self.window_pu)
                        self.ratios[i] = r
                    elif hp.variant == onp.VARIANT_ADAM_WEIGHT_DECAY:
                        p2, m2, v2 = onp.adam_weight_decay_update(self.params[i], self.m[i], self.v[i], ci, lr_t, hp.beta1,
                                                                  hp.beta2, hp.epsilon, hp.weight_decay_rate, self.decay[i])
                    else:
                        p2, m2, v2 = onp.adam_update(self.params[i], self.m[i], self.v[i], ci, lr_t, hp.beta1, hp.beta2,
                                                     hp.epsilon, self.beta1_power, self.beta2_power)
                    self.params[i][...] = p2; self.m[i][...] = m2; self.v[i][...] = v2
                if hp.variant != onp.VARIANT_ADAM_WEIGHT_DECAY:
                    self.beta1_power = F32(self.beta1_power * F32(hp.beta1))
                    self.beta2_power = F32(self.beta2_power * F32(hp.beta2))
            if self.ls:
                self.scale, self.good_windows = update_scale(self.scale, self.good_windows, overflow, self.multiplier,
                                                             self.growth_interval)
                self.skipped_windows += int(overflow)
                self.last_skipped = overflow
            for a in self.accum:
                a[...] = F32(0.0)
            self.reduced = None
        self.global_step = g + 1
        return info


def reference_op(variant: str, mode: str, params, names, N: int, lr_mult: Optional[Sequence[float]] = None,
                 adapt: Optional[Sequence[bool]] = None, ls_cfg=LS_CFG, sched=SCHED,
                 global_step: int = 0) -> LrMultReferenceTrainOp:
    """``apply_matrix.reference_op`` with a learning-rate table: the oracle of one dispatch key."""
    hp = oracle_hparams(variant, mode)
    params = [np.array(p, dtype=F32, copy=True) for p in params]
    lskw = dict(initial_scale=ls_cfg[0], multiplier=ls_cfg[1], growth_interval=ls_cfg[2]) if mode.startswith("ls_") else {}
    return LrMultReferenceTrainOp(params, names, hp, N, lr_mult=lr_mult, adapt=adapt, **lskw, **sched,
                                  global_step=global_step)


class LrMultLockStep(LockStep):
    """``LockStep`` whose train op has the learning-rate table ``lr_mult``, against ``LrMultReferenceTrainOp``.  The
    table goes to the plan before its first compute call (``Plan.set_lr_multipliers``), which is what the train ops'
    ``lr_multipliers`` argument does."""

    def __init__(self, man, variant: str, mode: str, *args, lr_mult: Sequence[float], **kw):
        super().__init__(man, variant, mode, *args, **kw)
        self.lr_mult = np.asarray(lr_mult, F32)
        self.op.plan.set_lr_multipliers(self.lr_mult)
        adapt = self.op.adapt if variant == "lamb" else None
        self.ref = reference_op(variant, mode, self.ref.params, [n for n, _ in man], self.N, lr_mult=self.lr_mult,
                                adapt=adapt, ls_cfg=self.ls_cfg, sched=self.sched, global_step=self.g0)
