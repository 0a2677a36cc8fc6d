"""The per-tensor norms an apply step reports (gaccum.h, gaccum_plan_set_tensor_norms), computed from the kernel's own
inputs: the accumulator slab before the apply, the apply's gradients, the divisor (N, or a weighted plan's W), the loss
scale S, and the weights before and after the apply.

Every sum is taken in fp64 and rounded to fp32 once, then square-rooted in fp32: ||x|| = sqrtf(fp32(sum x^2)).  The
kernel's sums are those of fp32 per-thread partials added in fp64, so the two agree within a few fp32 ulps, not bit for
bit.  Test infrastructure only."""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

F32 = np.float32


def norm(x) -> F32:
    """sqrtf(fp32(sum x^2)), the sum in fp64.  inf -> inf, NaN -> NaN, no elements -> 0."""
    x = np.asarray(x, np.float64).reshape(-1)
    with np.errstate(over="ignore", invalid="ignore"):
        s = F32(np.sum(x * x)) if x.size else F32(0.0)
        return np.sqrt(s, dtype=F32)


def window_gradient(accum, grad, divisor: float, scale: Optional[float] = None) -> np.ndarray:
    """c of one tensor, as the apply forms it before any clip scale: a' = a + G in fp32 (a' = a without a gradient),
    c = a' / D in fp32 (D = N, or W), times 1/S under loss scaling (S a power of two: exact)."""
    a = np.asarray(accum, F32)
    with np.errstate(over="ignore", invalid="ignore"):
        if grad is not None:
            a = (a + np.asarray(grad, F32)).astype(F32)
        c = (a / F32(divisor)).astype(F32)
        if scale is not None:
            c = (c * (F32(1.0) / F32(scale))).astype(F32)
    return c


def expected_norms(accum: Sequence[np.ndarray], grads: Optional[Sequence[Optional[np.ndarray]]], divisor: float,
                   scale: Optional[float], before: Sequence[np.ndarray], after: Sequence[np.ndarray]) -> np.ndarray:
    """The (T, 3) np.float32 array one apply reports: gradient, weight (before the update) and update
    (||p_before - p_after||, the fp32 difference) norms of every tensor."""
    out = np.zeros((len(accum), 3), F32)
    for t, a in enumerate(accum):
        g = grads[t] if grads is not None else None
        out[t, 0] = norm(window_gradient(a, g, divisor, scale))
        out[t, 1] = norm(before[t])
        with np.errstate(over="ignore", invalid="ignore"):
            d = (np.asarray(before[t], F32) - np.asarray(after[t], F32)).astype(F32)
        out[t, 2] = norm(d)
    return out


def assert_close(got: np.ndarray, exp: np.ndarray, rtol: float = 1e-6, what: str = "") -> None:
    """Element-wise: finite values within rtol of the expected one (0 exactly where 0 is expected), inf where inf is
    expected, NaN where NaN is."""
    got = np.asarray(got, np.float64); exp = np.asarray(exp, np.float64)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    nan = np.isnan(exp)
    inf = np.isinf(exp)
    assert np.array_equal(np.isnan(got), nan), (what, np.argwhere(np.isnan(got) != nan))
    assert np.array_equal(np.isinf(got) & ~nan, inf), (what, np.argwhere((np.isinf(got) & ~nan) != inf))
    fin = ~(nan | inf)
    err = np.abs(got[fin] - exp[fin])
    bad = err > rtol * np.abs(exp[fin])
    assert not bad.any(), (what, [(tuple(i), got[tuple(i)], exp[tuple(i)]) for i in np.argwhere(fin)[bad][:8]])
