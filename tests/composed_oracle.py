"""CPU oracle (numpy, fp32) of the train_op's apply step with every option the product has (include/gaccum.h).

``ComposedReferenceTrainOp`` is ``oracle_np.ReferenceTrainOp`` -- its accumulate, window predicate and schedule
unchanged -- with one ``run`` that adds, op for op:

* the variant (hp.variant): AdamWeightDecay and Adam as ``oracle_np`` computes them, or LAMB (GACCUM_LAMB):

      m = b1*m + omb1*c;  v = b2*v + omb2*c^2;  mh = m/(1-b1^t);  vh = v/(1-b2^t);  u = mh/(sqrt(vh)+eps) [+ wd*p]
      r = ||p|| / ||u||  (adapted tensors, both norms > 0; else 1);  p = p - (r*lr)*u

  with the norms summed in fp64 and rounded to fp32 once.  Adam's and LAMB's beta powers are TF1 Adam's running fp32
  products, advanced after every applied window;
* dynamic loss scaling (gaccum_loss_scale_config; ``initial_scale`` given): the producer feeds gradients of loss * S,
  c is multiplied by 1/S, a window is skipped when an element of a' or (with clipping) the global norm is not finite,
  and S follows TF 2's ``DynamicLossScale`` counted in windows;
* per-tensor learning-rate multipliers (gaccum_plan_set_lr_multipliers; ``lr_mult``): tensor t trains with
  ``lr_t = fp32(lr * mult[t])`` -- AdamWeightDecay ``p - lr_t*u``, Adam ``alpha_t = (lr_t*sqrt(1-b2^t)) / (1-b1^t)``,
  LAMB ``p - (r*lr_t)*u``;
* the window weight (gaccum_plan_set_window_weight; ``window_weight=True``): the producer adds each micro-batch's weight
  into W with fp32 adds, and the apply step computes ``c = a' / W`` -- one correctly rounded fp32 division -- in place of
  ``(1.0*a') / N``, records ``last_weight = W`` and resets W to +0, applied or skipped alike.  N still decides where a
  window ends.

An apply step is: c = a'/N or a'/W; c *= 1/S; gn and the clip scale s of c; skip or c *= s; every tensor's update at its
lr_t.  With every option at identity it computes what ``ReferenceTrainOp`` computes, bit for bit
(tests/test_lr_multipliers_host.py checks that against it and against the C oracle).  Test infrastructure only.
"""
from __future__ import annotations

import re
from typing import List, Optional, Sequence

import numpy as np

import oracle_np as onp

F32 = np.float32
VARIANT_LAMB = 2


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


def norm(x: np.ndarray) -> np.float32:
    """||x|| = sqrtf(fp32(sum x^2)), the sum in fp64."""
    x64 = np.asarray(x, np.float64).ravel()
    return np.sqrt(F32(float(np.dot(x64, x64)) if x64.size else 0.0), dtype=F32)


def trust_ratio(wn: np.float32, un: np.float32) -> np.float32:
    with np.errstate(divide="ignore", invalid="ignore"):
        return F32(wn / un) if (wn > 0 and un > 0) else F32(1.0)


def lamb_update(p, m, v, c, lr, beta1, beta2, eps, wd, use_decay, adapt, beta1_power, beta2_power, ratio=None,
                record=None):
    """One tensor.  Returns (p', m', v', r).  ``ratio``: r of an adapted tensor as a device reduced it, used in place
    of ``trust_ratio(norm(p), norm(u))``; ``record``: a list that (p, u) of an adapted tensor is appended to."""
    b1, b2 = F32(beta1), F32(beta2)
    omb1, omb2 = F32(1.0 - float(beta1)), F32(1.0 - float(beta2))
    next_m = np.add(np.multiply(b1, m, dtype=F32), np.multiply(omb1, c, dtype=F32), dtype=F32)
    next_v = np.add(np.multiply(b2, v, dtype=F32), np.multiply(omb2, np.square(c, dtype=F32), dtype=F32), dtype=F32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        mh = np.divide(next_m, F32(F32(1.0) - F32(beta1_power)), dtype=F32)
        vh = np.divide(next_v, F32(F32(1.0) - F32(beta2_power)), dtype=F32)
        u = np.divide(mh, np.add(np.sqrt(vh, dtype=F32), F32(eps), dtype=F32), dtype=F32)
        if use_decay:
            u = np.add(u, np.multiply(F32(wd), p, dtype=F32), dtype=F32)
        if adapt and record is not None:
            record.append((np.array(p, F32, copy=True), u))
        if not adapt:
            r = F32(1.0)
        else:
            r = trust_ratio(norm(p), norm(u)) if ratio is None else F32(ratio)
        next_p = np.subtract(p, np.multiply(F32(r * F32(lr)), u, dtype=F32), dtype=F32)
    return next_p, next_m, next_v, r


def reduced_ratios(op: onp.ReferenceTrainOp):
    """(per-tensor r to pass to ``lamb_update``, its ``record`` list) for the window ``op`` is applying: the device's r
    and a fresh list when ``op.reduced`` is set, else None for every tensor and no record."""
    T = len(op.params)
    if op.reduced is None or op.reduced.ratios is None:
        return [None] * T, None
    return list(op.reduced.ratios), []


def adaptation_mask(names: Sequence[str], exclude: Optional[Sequence[str]]) -> List[bool]:
    return [not any(re.search(r, onp.get_variable_name(n)) is not None for r in exclude or ()) for n in names]


class ComposedReferenceTrainOp(onp.ReferenceTrainOp):
    """``ReferenceTrainOp`` with every option of the apply step; each defaults to off.

    * LAMB (hp.variant 2): ``adapt_exclude`` defaults to ``exclude`` (TF-Addons); ``adapt`` overrides the mask.
      ``ratios`` holds the last applied window's trust ratios (1 for the other variants).
    * Loss scaling (``initial_scale`` given): ``scale``, ``good_windows``, ``skipped_windows`` and ``last_skipped``
      mirror gaccum_loss_scale_state.  Without it ``scale`` stays 1 and no window is skipped.
    * ``lr_mult``: one multiplier per tensor.  None leaves the step's lr as it is.
    * ``window_weight``: ``add_weight(w)`` is the producer's fp32 add into ``weight`` (W); ``run(grads, weight=w)`` adds
      w and then steps.  ``last_weight`` is the W of the last apply step.  An unweighted oracle refuses a weight, as an
      unweighted train op does.
    """

    def __init__(self, params, names, hp, accum_n, *, adapt: Optional[Sequence[bool]] = None, adapt_exclude=None,
                 initial_scale: Optional[float] = None, multiplier: float = 2.0, growth_interval: int = 2000,
                 lr_mult: Optional[Sequence[float]] = None, window_weight: bool = False, **kw):
        super().__init__(params, names, hp, accum_n, **kw)
        T = len(self.params)
        exclude = kw.get("exclude", onp.DEFAULT_EXCLUDE)
        self.adapt = list(adapt) if adapt is not None else \
            adaptation_mask(names, adapt_exclude if adapt_exclude is not None else exclude)
        self.ratios = [F32(1.0)] * T
        self.ls = initial_scale is not None
        self.scale = F32(initial_scale if self.ls else 1.0)
        self.multiplier, self.growth_interval = multiplier, int(growth_interval)
        self.good_windows = self.skipped_windows = 0
        self.last_skipped = False
        self.lr_mult = None if lr_mult is None else [F32(m) for m in lr_mult]
        assert self.lr_mult is None or len(self.lr_mult) == T
        self.window_weight = bool(window_weight)
        self.weight = self.last_weight = F32(0.0)

    def add_weight(self, w) -> None:
        if not self.window_weight:
            raise ValueError("a weight was given to an oracle without the window weight")
        with np.errstate(over="ignore", invalid="ignore"):
            self.weight = np.add(self.weight, F32(w), dtype=F32)

    def lr_t(self, lr: np.float32, i: int) -> np.float32:
        return F32(lr) if self.lr_mult is None else np.multiply(F32(lr), self.lr_mult[i], dtype=F32)

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
            with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
                if self.window_weight:
                    c = [np.divide(a, self.weight, dtype=F32) for a in self.accum]          # a' / W, one rounding
                else:
                    nf = F32(self.N)
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
                self._update(c, lr)
            if self.ls:
                self.scale, self.good_windows = update_scale(self.scale, self.good_windows, overflow, self.multiplier,
                                                             self.growth_interval)
                self.skipped_windows += int(overflow)
                self.last_skipped = overflow
            for a in self.accum:
                a[...] = F32(0.0)
            self.reduced = None
            if self.window_weight:
                self.last_weight, self.weight = self.weight, F32(0.0)
        self.global_step = g + 1
        return info

    def _update(self, c: Sequence[np.ndarray], lr: np.float32) -> None:
        """Every tensor's update from its c at its lr_t, then the beta powers (Adam and LAMB)."""
        hp = self.hp
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
