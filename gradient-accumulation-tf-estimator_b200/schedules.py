"""TF1's learning-rate schedules (``tf.compat.v1.train.*_decay``, TF 1.15 ``learning_rate_schedule.py``) restated in
numpy fp32: one correctly rounded fp32 op per TF op, in TF's op order, with TF's conversions (Python floats become fp32
constants, the step is cast to fp32 with round to nearest, Python arithmetic on Python floats stays in double).

Each schedule is a host ``lr_fn`` (``schedule(g)`` is the fp32 learning rate of the micro-step whose pre-increment
step is g, as a Python float) and produces the table a device-scheduled train op replays (``schedule.table(n)``: steps
0 .. n-1, np.float32; ``train_op.LrTable``).  Both evaluate the same vectorized numpy expression, so ``table(n)[g]`` is
``schedule(g)`` bit for bit.

``pow`` and ``cos`` are numpy's fp32 ``power`` and ``cos``; TF's CPU kernels reach the platform's libm (through
Eigen) for the same functions, so these values match TensorFlow's up to how those libraries round -- bit equality is
plausible, but not verified against TensorFlow.  The +, -, *, / and min are exact restatements.
"""
from __future__ import annotations

import math
from typing import Callable, Sequence

import numpy as np

F32 = np.float32


class Schedule:
    """A learning-rate schedule over int64 steps: ``fn`` maps an int64 array of steps to their fp32 learning rates."""

    def __init__(self, fn: Callable[[np.ndarray], np.ndarray]):
        self._fn = fn

    def values(self, steps) -> np.ndarray:
        steps = np.asarray(steps, dtype=np.int64)
        with np.errstate(all="ignore"):               # IEEE results propagate, as in TF
            return np.asarray(self._fn(steps), dtype=F32)

    def __call__(self, step: int) -> float:
        return float(self.values(np.array([int(step)]))[0])

    def table(self, num_steps: int) -> np.ndarray:
        """The learning rates of steps 0 .. num_steps - 1 (np.float32)."""
        n = int(num_steps)
        if n < 1:
            raise ValueError(f"a learning-rate table needs num_steps >= 1 (got {n})")
        return self.values(np.arange(n, dtype=np.int64))


def _step_f32(steps: np.ndarray) -> np.ndarray:
    """cast(global_step, float32): int64 -> fp32, round to nearest."""
    return steps.astype(F32)


def polynomial_decay(learning_rate: float, decay_steps: int, end_learning_rate: float = 0.0001, power: float = 1.0,
                     cycle: bool = False) -> Schedule:
    """tf.train.polynomial_decay (PolynomialDecay.__call__):
    ``(lr - end) * pow(1 - min(g, ds) / ds, power) + end``; with ``cycle``, ds is multiplied by ceil(g / ds) (1 at g = 0)
    instead of g being clamped."""
    lr0, end, pw, ds0 = F32(learning_rate), F32(end_learning_rate), F32(power), F32(decay_steps)

    def fn(steps):
        gs = _step_f32(steps)
        if cycle:
            mult = np.where(gs == F32(0), F32(1.0), np.ceil(gs / ds0))
            ds = ds0 * mult
        else:
            gs = np.minimum(gs, ds0)
            ds = ds0
        p = gs / ds
        return (lr0 - end) * np.power(F32(1) - p, pw) + end
    return Schedule(fn)


def cosine_decay(learning_rate: float, decay_steps: int, alpha: float = 0.0) -> Schedule:
    """tf.train.cosine_decay (CosineDecay.__call__):
    ``lr * ((1 - alpha) * 0.5 * (1 + cos(pi * min(g, ds) / ds)) + alpha)``, pi an fp32 constant and (1 - alpha) a Python
    double rounded to fp32 once."""
    lr0, ds, pi = F32(learning_rate), F32(decay_steps), F32(math.pi)
    one_minus_alpha, a = F32(1 - alpha), F32(alpha)

    def fn(steps):
        gs = np.minimum(_step_f32(steps), ds)
        frac = gs / ds
        cosine = F32(0.5) * (F32(1.0) + np.cos(pi * frac))
        return lr0 * (one_minus_alpha * cosine + a)
    return Schedule(fn)


def exponential_decay(learning_rate: float, decay_steps: int, decay_rate: float, staircase: bool = False) -> Schedule:
    """tf.train.exponential_decay (ExponentialDecay.__call__): ``lr * pow(rate, g / ds)``, the exponent floored with
    ``staircase``."""
    lr0, ds, rate = F32(learning_rate), F32(decay_steps), F32(decay_rate)

    def fn(steps):
        p = _step_f32(steps) / ds
        if staircase:
            p = np.floor(p)
        return lr0 * np.power(rate, p)
    return Schedule(fn)


def piecewise_constant(boundaries: Sequence[int], values: Sequence[float]) -> Schedule:
    """tf.train.piecewise_constant (PiecewiseConstantDecay.__call__): values[0] while g <= boundaries[0], values[i] while
    boundaries[i-1] < g <= boundaries[i], values[-1] once g > boundaries[-1].  Integer boundaries, compared with the
    int64 step; each value an fp32 constant."""
    b = np.asarray([int(x) for x in boundaries], dtype=np.int64)
    v = np.asarray([float(x) for x in values], dtype=np.float64).astype(F32)
    if len(v) != len(b) + 1:
        raise ValueError(f"piecewise_constant needs one more value than boundaries (got {len(b)} and {len(v)})")
    if np.any(np.diff(b) < 0):
        raise ValueError("piecewise_constant boundaries must be increasing")

    def fn(steps):
        return v[np.searchsorted(b, steps, side="left")]   # the number of boundaries < g
    return Schedule(fn)


def with_bert_warmup(schedule: Schedule, init_lr: float, num_warmup_steps: int) -> Schedule:
    """BERT's linear warm-up over ``schedule`` (reference optimization.py:40-54): with a warm-up,
    ``(1 - is_warmup) * lr + is_warmup * (init_lr * (int32(g) / int32(W)))``, is_warmup = int32(g) < int32(W) as fp32;
    without one (``num_warmup_steps`` 0 or None), ``schedule`` itself."""
    if not num_warmup_steps:
        return schedule
    w_i = np.int32(num_warmup_steps)
    w_f, lr0 = F32(w_i), F32(init_lr)

    def fn(steps):
        lr = schedule.values(steps)
        g_i = steps.astype(np.int32)                          # cast(global_step, int32): wraps
        pct = g_i.astype(F32) / w_f
        wlr = lr0 * pct
        is_w = (g_i < w_i).astype(F32)
        return (F32(1.0) - is_w) * lr + is_w * wlr
    return Schedule(fn)
