"""Exact sums of squares of fp32 arrays, their correctly rounded fp32 norms, and the error bound of the clip-apply's
global norm.  Test infrastructure only (numpy and Python ints; no torch).

* ``exact_sumsq(x)``: sum(x^2) over an fp32 array, exactly, as a ``Fraction`` (inf / NaN when an element is not finite).
* ``round_f32(e)``: e rounded to fp32 once, to nearest, ties to even; inf at or above FLT_MAX + half an ulp.
* ``ref_norm(e)``: sqrtf(round_f32(e)) -- what an exact accumulator rounded once to fp32 gives (include/gaccum.h).
* ``near_tie(e, rel)``: e lies within ``rel`` (relative) of a point where the fp32 rounding changes.
* ``clip_norm_bound(e, n)``: how far the clip-apply's global norm may lie from sqrt(e), derived below.

The clip-apply's global norm (gaccum_kernels.cuh ``norm_tile``, ``add_sq``, ``acc_add``, ``window_decision``).  Let
u = 2^-24 (fp32) and u' = 2^-53 (fp64), gamma_k(u) = k u / (1 - k u), and E = sum(c^2) exactly.

1. A thread adds the c^2 of its elements of one tile with ``fmaf(c, c, acc)`` from acc = 0: two float4 vectors and
   at most one of the < 4 tail elements (``walk_tile``), or 8 elements kThreads apart on the scalar path -- k <= 9
   fmas, each one rounding of an exact acc + c^2.  Recursive summation: |P - sum| <= gamma_9(u) * sum for normal
   results.  A result below 2^-126 is rounded with an absolute error of at most 2^-150 instead (half the subnormal
   spacing), at most once per element: n * 2^-150 over the whole model.
2. A warp adds its 32 partials (exact in fp64) in a butterfly of depth 5: each lane's total is off by at most
   gamma_5(u') of the warp's sum.
3. The accumulator adds the warp totals exactly (``acc_add``).
4. The exact total S is rounded to fp32 once: one more factor (1 + d), |d| <= u, or 2^-150 absolutely below 2^-126.
5. ``sqrtf``: gn = sqrt(S_f) (1 + d'), |d'| <= u.

So |S_f - E| <= D = (gamma_9(u) + gamma_5(u') + u + (gamma_9(u) + gamma_5(u')) u) E + (n + 1) 2^-150, and with
|sqrt(a) - sqrt(b)| = |a - b| / (sqrt(a) + sqrt(b)) <= sqrt(|a - b|),

    |gn - sqrt(E)| <= min(D / (sqrt(E) + sqrt(E - D)), sqrt(D)) + u sqrt(E + D).

Relative to sqrt(E), the first term is about (9u + u) / 2 and the second u: about 6u = 3.6e-7 in all.  Every warp
total is one fp32 sum of at most 9 elements per thread; nothing here depends on which thread holds which element.

LAMB's ||p|| and ||u|| (gaccum_lamb.cuh phase 2) form their per-thread partials in fp64 (``add_sq64``): the exact sum
is known to ~2^-49 before it is rounded to fp32 once, so away from an fp32 rounding boundary (``near_tie``) the
kernel's norm is ``ref_norm`` bit for bit.
"""
from __future__ import annotations

import math
from fractions import Fraction
from typing import Union

import numpy as np

F32 = np.float32
U32 = 2.0 ** -24                      # unit roundoff of fp32
U64 = 2.0 ** -53                      # ... of fp64
SCALE = 298                           # every square of an fp32 is an integer multiple of 2^-298 = (2^-149)^2
FLT_MAX = Fraction(int(np.finfo(F32).max))
OVERFLOW = FLT_MAX + 2 ** 103                       # FLT_MAX plus half its ulp (2^104): this and above round to inf
_CHUNK = 1 << 24                      # elements per bincount: 2^24 * (2^12)^2 < 2^53, exact in the fp64 weights

Exact = Union[Fraction, float]        # a Fraction, or inf / nan for a non-finite input


def exact_sumsq(x) -> Exact:
    """sum(x^2) over the fp32 array ``x``, exact.  +inf if an element is +-inf and none is NaN, NaN if one is NaN --
    the kernel's accumulator flags (``acc_add``: NaN wins); 0 for an empty array.

    Each element is k * 2^(e - 150), k < 2^24 and e its biased exponent field (1 for subnormals); k = kh * 2^12 + kl
    with kh, kl < 2^12, so k^2 = kh^2 2^24 + 2 kh kl 2^12 + kl^2 and the three pieces, each < 2^24, are summed per
    exponent with np.bincount in chunks small enough that the fp64 bin totals stay exact."""
    a = np.ascontiguousarray(np.asarray(x, dtype=F32)).reshape(-1)
    if a.size == 0:
        return Fraction(0)
    bits = a.view(np.uint32)
    total = 0                                                      # in units of 2^-298
    nonfinite = False
    for lo in range(0, a.size, _CHUNK):
        b = bits[lo:lo + _CHUNK]
        e = ((b >> 23) & 0xFF).astype(np.int64)
        if (e == 0xFF).any():
            if np.isnan(a[lo:lo + _CHUNK]).any():
                return float("nan")
            nonfinite = True
            continue
        k = (b & 0x7FFFFF).astype(np.int64) | ((e != 0).astype(np.int64) << 23)
        kh, kl = k >> 12, k & 0xFFF
        e = np.maximum(e, 1)
        hh = np.bincount(e, weights=(kh * kh).astype(np.float64), minlength=256)
        hl = np.bincount(e, weights=(kh * kl).astype(np.float64), minlength=256)
        ll = np.bincount(e, weights=(kl * kl).astype(np.float64), minlength=256)
        for ex in np.flatnonzero(hh + hl + ll):
            s = (int(hh[ex]) << 24) + (int(hl[ex]) << 13) + int(ll[ex])     # sum of k^2 at this exponent
            total += s << (2 * (int(ex) - 1))                              # (2^(ex - 150))^2 = 2^(2(ex-1)) 2^-298
    if nonfinite:
        return float("inf")
    return Fraction(total, 1 << SCALE)


def _finite(e: Exact) -> bool:
    return isinstance(e, Fraction)


def round_f32(e: Exact) -> np.float32:
    """The non-negative ``e`` rounded to fp32 once: to nearest, ties to even; inf from FLT_MAX + half an ulp up
    (that point is a tie, and the even neighbour is 2^128)."""
    if not _finite(e):
        return F32(e)
    assert e >= 0
    if e == 0:
        return F32(0.0)
    if e >= OVERFLOW:
        return F32(np.inf)
    # the fp32 spacing at e: 2^(max(exponent, -126) - 23)
    ex = e.numerator.bit_length() - e.denominator.bit_length()     # 2^ex <= e < 2^(ex+2)
    if Fraction(2) ** ex > e:
        ex -= 1
    elif Fraction(2) ** (ex + 1) <= e:
        ex += 1
    q = Fraction(2) ** (max(ex, -126) - 23)
    n, r = divmod(e / q, 1)
    n = int(n)
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n & 1):
        n += 1
    return F32(math.ldexp(float(n), max(ex, -126) - 23))          # n <= 2^24: exact in double and in fp32


def ref_norm(e: Exact) -> np.float32:
    """sqrtf(round_f32(e)): the norm an exact sum of squares gives when it is rounded to fp32 once."""
    return np.sqrt(round_f32(e), dtype=F32)


def _neighbours(v: np.float32):
    return np.nextafter(v, F32(0.0)), np.nextafter(v, F32(np.inf))


def near_tie(e: Exact, rel: float) -> bool:
    """True when the finite ``e`` lies within ``rel * e`` of a boundary between two fp32 roundings: the midpoint
    between round_f32(e) and either neighbour (or e itself is that close to the overflow point)."""
    if not _finite(e) or e == 0:
        return False
    v = round_f32(e)
    mids = []
    base = Fraction(float(FLT_MAX)) if np.isinf(v) else Fraction(float(v))
    for w in _neighbours(F32(base)):
        if np.isfinite(w):
            mids.append((base + Fraction(float(w))) / 2)
    mids.append(OVERFLOW)
    return any(abs(e - m) <= Fraction(rel) * e for m in mids)


def norm_candidates(e: Exact, rel: float):
    """``ref_norm(e)``, and next to a tie (``near_tie``) also the norm of the fp32 value on the tie's other side: the
    values a sum known to ``rel`` can round to."""
    out = {ref_norm(e).tobytes(): ref_norm(e)}
    if near_tie(e, rel):
        v = round_f32(e)
        for w in _neighbours(v if np.isfinite(v) else F32(np.finfo(F32).max)):
            out[np.sqrt(w, dtype=F32).tobytes()] = np.sqrt(w, dtype=F32)
        if np.isinf(v):
            out[np.sqrt(np.finfo(F32).max, dtype=F32).tobytes()] = np.sqrt(np.finfo(F32).max, dtype=F32)
    return list(out.values())


# ---- inputs that tell a sum rounded to fp32 once from one rounded to fp64 first ----------------------------------------
# c values, one per tile: the exact sum of squares is 2 + 2^-23 + 2^-90, which rounds to fp32 2 + 2^-22; through an fp64
# it becomes the tie 2 + 2^-23 first, and then 2 (ties to even).  sqrtf: 0x3fb504f4 once, 0x3fb504f3 twice.
TIE_C = (1.0, 1.0, 2.0 ** -12, 2.0 ** -12, 2.0 ** -45)
TIE_NORM_BITS = 0x3FB504F4


def overflow_c(above: bool):
    """c values k * 2^j (k < 2^12, so every square is exact in fp32), one per tile, whose exact sum of squares lies
    within 2^-63 (relative) below the fp32 overflow point -- it rounds to FLT_MAX once, to inf through an fp64 --
    or, ``above``, just past it."""
    rem = OVERFLOW - 2 ** 63
    out = []
    while rem >= 2 ** 63:
        j = max((int(rem).bit_length() - 24) // 2, 0)
        k = min(math.isqrt(int(rem) >> (2 * j)), 4095)
        out.append(float(k) * 2.0 ** j)
        rem -= (k << j) ** 2
    if above:
        out.append(2.0 ** 32)
    return out


def _gamma(k: int, u: float) -> float:
    return k * u / (1.0 - k * u)


def clip_norm_bound(e: Exact, n: int) -> float:
    """The largest |gn - sqrt(e)| the clip-apply's global norm may show over ``n`` elements whose exact sum of squares
    is ``e`` (module docstring).  Computed in fp64 with its own rounding far below the bound."""
    E = float(e)
    rel = _gamma(9, U32) + _gamma(5, U64)
    D = (rel + U32 + rel * U32) * E + (n + 1) * 2.0 ** -150
    first = min(D / (math.sqrt(E) + math.sqrt(max(E - D, 0.0))), math.sqrt(D)) if E > 0 else math.sqrt(D)
    return (first + U32 * math.sqrt(E + D)) * (1 + 1e-12)
