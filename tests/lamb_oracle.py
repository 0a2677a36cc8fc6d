"""CPU oracle (numpy, fp32) of the train_op with the LAMB optimizer (include/gaccum.h, GACCUM_LAMB).

Built on ``oracle_np.ReferenceTrainOp``: accumulate steps are unchanged; an apply step forms c exactly as the
AdamWeightDecay apply does (``/N``, ``*1/S`` under loss scaling, ``*clip_scale``), then per tensor

    m = b1*m + omb1*c;  v = b2*v + omb2*c^2;  mh = m/(1-b1^t);  vh = v/(1-b2^t);  u = mh/(sqrt(vh)+eps) [+ wd*p]
    r = ||p|| / ||u||  (adapted tensors, both norms > 0; else 1);  p = p - (r*lr)*u

with one numpy ufunc per op in fp32 and the norms summed in fp64, rounded to fp32 once.  The beta powers are TF1 Adam's
running fp32 products, advanced after every applied window.  Loss scaling (``initial_scale`` given) follows
``loss_scale_oracle``.  Test infrastructure only.
"""
from __future__ import annotations

import re
from typing import List, Optional, Sequence

import numpy as np

import oracle_np as onp
from loss_scale_oracle import update_scale

F32 = np.float32


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


class LambReferenceTrainOp(onp.ReferenceTrainOp):
    """``ReferenceTrainOp`` with LAMB.  ``adapt_exclude`` defaults to ``exclude`` (TF-Addons); ``adapt`` overrides the
    mask.  ``ratios`` holds the last applied window's trust ratios.  With ``initial_scale`` the producer feeds gradients
    of ``loss * S`` (gaccum_loss_scale_config) and ``scale`` / ``good_windows`` / ``skipped_windows`` / ``last_skipped``
    mirror the device block."""

    def __init__(self, params, names, hp, accum_n, *, adapt_exclude=None, adapt: Optional[Sequence[bool]] = None,
                 initial_scale: Optional[float] = None, multiplier: float = 2.0, growth_interval: int = 2000, **kw):
        super().__init__(params, names, hp, accum_n, **kw)
        exclude = kw.get("exclude", onp.DEFAULT_EXCLUDE)
        self.adapt = list(adapt) if adapt is not None else \
            adaptation_mask(names, adapt_exclude if adapt_exclude is not None else exclude)
        self.ratios = [F32(1.0)] * len(self.params)
        self.ls = initial_scale is not None
        self.scale = F32(initial_scale if self.ls else 1.0)
        self.multiplier, self.growth_interval = multiplier, int(growth_interval)
        self.good_windows = self.skipped_windows = 0
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
                    c = [np.multiply(x, s, dtype=F32) for x in c]
            if not overflow:
                ratios, self.window_pu = reduced_ratios(self)
                for i, ci in enumerate(c):
                    p2, m2, v2, r = lamb_update(self.params[i], self.m[i], self.v[i], ci, lr, hp.beta1, hp.beta2,
                                                hp.epsilon, hp.weight_decay_rate, self.decay[i], self.adapt[i],
                                                self.beta1_power, self.beta2_power, ratios[i], self.window_pu)
                    self.params[i][...] = p2; self.m[i][...] = m2; self.v[i][...] = v2
                    self.ratios[i] = r
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
