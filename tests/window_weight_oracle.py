"""CPU oracle (numpy, fp32) of the train_op with per-window normalisation by the window's total weight (include/gaccum.h,
gaccum_plan_set_window_weight).

The producer adds each micro-batch's weight w_i into W with fp32 adds; the apply step computes ``c = a' / W`` -- one
correctly rounded fp32 division -- in place of ``(1.0*a') / N``, records ``last_weight = W`` and resets W to +0, applied
or skipped alike.  N still decides where a window ends.  Everything after the division is ``lr_mult_oracle``'s
arithmetic, op for op: the loss scaling, the clip, every variant's update and the learning-rate multipliers.  With
W = N (as fp32) it computes exactly what ``LrMultReferenceTrainOp`` computes, since (1.0*a')/N is a'/N
(tests/test_window_weight_host.py checks that).  Test infrastructure only.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

import oracle_np as onp
from apply_matrix import LS_CFG, SCHED, oracle_hparams
from lamb_oracle import lamb_update, reduced_ratios
from loss_scale_oracle import update_scale
from lr_mult_oracle import VARIANT_LAMB, LrMultLockStep, LrMultReferenceTrainOp

F32 = np.float32


class WindowWeightReferenceTrainOp(LrMultReferenceTrainOp):
    """``LrMultReferenceTrainOp`` whose apply step divides by the window's weight ``weight`` (W) instead of N.
    ``add_weight(w)`` is the producer's fp32 add; ``run(grads, weight=w)`` adds w and then steps.  ``last_weight`` is
    the W of the last apply step."""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.weight = F32(0.0)
        self.last_weight = F32(0.0)

    def add_weight(self, w) -> None:
        with np.errstate(over="ignore", invalid="ignore"):
            self.weight = np.add(self.weight, F32(w), dtype=F32)

    def run(self, grads: Sequence[Optional[np.ndarray]], weight=None) -> onp.StepInfo:
        if weight is not None:
            self.add_weight(weight)
        g = self.global_step
        hp = self.hp
        lr = self.lr(g)
        is_apply = (int(np.int32(np.int64(g))) % self.N) == 0
        for a, gr in zip(self.accum, grads):
            if gr is not None:
                np.add(a, np.asarray(gr, dtype=F32).reshape(a.shape), out=a, dtype=F32)
        info = onp.StepInfo(global_step=g, applied=is_apply, lr=lr)
        if is_apply:
            W = self.weight
            with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
                c = [np.divide(a, W, dtype=F32) for a in self.accum]          # a' / W, one rounding
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
                            p2, m2, v2 = onp.adam_weight_decay_update(self.params[i], self.m[i], self.v[i], ci, lr_t,
                                                                      hp.beta1, hp.beta2, hp.epsilon, hp.weight_decay_rate,
                                                                      self.decay[i])
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
            self.last_weight, self.weight = W, F32(0.0)
        self.global_step = g + 1
        return info


def reference_op(variant: str, mode: str, params, names, N: int, lr_mult: Optional[Sequence[float]] = None,
                 adapt: Optional[Sequence[bool]] = None, ls_cfg=LS_CFG, sched=SCHED,
                 global_step: int = 0) -> WindowWeightReferenceTrainOp:
    """``lr_mult_oracle.reference_op`` with the window weight: the oracle of one dispatch key."""
    hp = oracle_hparams(variant, mode)
    params = [np.array(p, dtype=F32, copy=True) for p in params]
    lskw = dict(initial_scale=ls_cfg[0], multiplier=ls_cfg[1], growth_interval=ls_cfg[2]) if mode.startswith("ls_") else {}
    return WindowWeightReferenceTrainOp(params, names, hp, N, lr_mult=lr_mult, adapt=adapt, **lskw, **sched,
                                      global_step=global_step)


class WindowWeightLockStep(LrMultLockStep):
    """``LrMultLockStep`` whose plan divides each window by W (``Plan.set_window_weight`` on a zeroed 16-byte block,
    before the first compute call -- what the train ops' ``window_weight=True`` does), against
    ``WindowWeightReferenceTrainOp``.  ``wstep(grads, w)`` adds w into the device W (an fp32 add on the stream) and into
    the oracle's, then steps both; ``check`` also compares W and last_weight exactly."""

    def __init__(self, man, variant: str, mode: str, *args, lr_mult: Optional[Sequence[float]] = None, **kw):
        T = len(man)
        super().__init__(man, variant, mode, *args, lr_mult=np.ones(T, F32) if lr_mult is None else lr_mult, **kw)
        torch = self.torch
        self.ww = torch.zeros(4, dtype=torch.float32, device="cuda")
        self.op.plan.set_window_weight(self.ww.data_ptr())
        adapt = self.op.adapt if variant == "lamb" else None
        self.ref = reference_op(variant, mode, self.ref.params, [n for n, _ in man], self.N, lr_mult=self.lr_mult,
                                adapt=adapt, ls_cfg=self.ls_cfg, sched=self.sched, global_step=self.g0)

    def wstep(self, grads, w) -> bool:
        self.ref.add_weight(w)
        with self.torch.no_grad():
            self.ww[0].add_(float(w))
        return self.step(grads)

    def check(self, info) -> None:
        super().check(info)
        got = self.ww[:2].cpu().numpy()
        assert got[0].tobytes() == F32(self.ref.weight).tobytes(), (got[0], self.ref.weight)
        assert got[1].tobytes() == F32(self.ref.last_weight).tobytes(), (got[1], self.ref.last_weight)
