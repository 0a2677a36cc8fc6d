"""The exact-sum reference (tests/exact_norm_oracle.py) against fractions.Fraction, and a restatement of the kernels'
exact accumulator (gaccum_kernels.cuh acc_add / acc_value) showing which inputs tell a sum rounded to fp32 once from
one rounded to fp64 first.  CPU only."""
import math
import struct
from fractions import Fraction

import numpy as np
import pytest

import exact_norm_oracle as eno

F32 = np.float32
FMAX = F32(np.finfo(F32).max)


def _frac_sumsq(x) -> Fraction:
    return sum((Fraction(float(v)) ** 2 for v in np.asarray(x, F32).ravel()), Fraction(0))


def _round_f32_slow(e: Fraction) -> np.float32:
    """fp32 nearest to e by comparing the candidates around float(e); ties to the even significand."""
    if e >= eno.OVERFLOW:
        return F32(np.inf)
    c = F32(float(e)) if float(e) <= float(FMAX) else FMAX
    cands = [np.nextafter(c, F32(0)), c, np.nextafter(c, F32(np.inf))]
    cands = [x for x in cands if np.isfinite(x)]
    return min(cands, key=lambda x: (abs(Fraction(float(x)) - e), int(x.view(np.uint32)) & 1))


ADVERSARIAL = {
    "subnormals": np.array([1e-45, 2e-45, 1.1754942e-38, -1e-40, 0.0], F32),
    "flt_max": np.array([FMAX, -FMAX], F32),
    "mixed_range": np.array([FMAX, 1e-45, 1.0, 2.0 ** -70, -3.0], F32),
    "zeros": np.zeros(17, F32),
    "neg_zero": np.array([-0.0, 0.0], F32),
    "one": np.array([1.0], F32),
    "tie_c": np.array(eno.TIE_C, F32),
}


@pytest.mark.parametrize("name", sorted(ADVERSARIAL))
def test_exact_sumsq_is_the_fraction_sum(name):
    x = ADVERSARIAL[name]
    assert eno.exact_sumsq(x) == _frac_sumsq(x)


@pytest.mark.parametrize("seed", range(6))
def test_exact_sumsq_random(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 3000))
    x = (rng.normal(size=n) * np.exp2(rng.integers(-150, 60, n))).astype(F32)
    assert eno.exact_sumsq(x) == _frac_sumsq(x)


def test_exact_sumsq_chunks_and_nonfinite():
    big = np.full((1 << 24) + 5, F32(4095.0 + 4095.0 / 4096), F32)     # every k = 2^24 - 1: the largest pieces
    assert eno.exact_sumsq(big) == Fraction(float(big[0])) ** 2 * big.size
    assert eno.exact_sumsq(np.zeros(0, F32)) == 0
    assert eno.exact_sumsq(np.array([1.0, np.inf, -np.inf], F32)) == math.inf
    assert math.isnan(eno.exact_sumsq(np.array([np.inf, np.nan, 1.0], F32)))


ROUNDING = [Fraction(1) + Fraction(1, 2 ** 24), Fraction(1) + 3 * Fraction(1, 2 ** 24), Fraction(2 + 2 ** -23),
            Fraction(2) + Fraction(1, 2 ** 23) + Fraction(1, 2 ** 90), Fraction(1, 2 ** 150), 3 * Fraction(1, 2 ** 150),
            Fraction(1, 2 ** 151), Fraction(1, 2 ** 126) - Fraction(1, 2 ** 150), Fraction(float(FMAX)),
            eno.OVERFLOW - Fraction(1, 2 ** 40), eno.OVERFLOW, eno.OVERFLOW + 1, Fraction(10) ** 45, Fraction(0),
            Fraction(1, 3), Fraction(7, 10)]


@pytest.mark.parametrize("e", ROUNDING, ids=lambda e: f"{float(e):.9g}")
def test_round_f32_is_correct_rounding(e):
    got = eno.round_f32(e)
    want = _round_f32_slow(e) if e else F32(0.0)
    assert got.tobytes() == want.tobytes(), (float(e), got, want)


def test_round_f32_ties_and_overflow():
    assert eno.round_f32(Fraction(1) + Fraction(1, 2 ** 24)) == F32(1.0)                  # tie to even
    assert eno.round_f32(Fraction(1) + 3 * Fraction(1, 2 ** 24)) == F32(1 + 2 ** -22)     # tie to even, upwards
    assert eno.round_f32(3 * Fraction(1, 2 ** 150)) == F32(2.0 ** -148)                   # subnormal tie
    assert eno.round_f32(Fraction(1, 2 ** 150)) == F32(0.0)
    assert eno.round_f32(eno.OVERFLOW - Fraction(1, 2 ** 40)) == FMAX
    assert np.isinf(eno.round_f32(eno.OVERFLOW))                                          # the tie goes to 2^128
    assert np.isinf(eno.round_f32(math.inf)) and np.isnan(eno.round_f32(math.nan))


@pytest.mark.parametrize("seed", range(4))
def test_round_f32_random(seed):
    rng = np.random.default_rng(100 + seed)
    for _ in range(300):
        e = Fraction(int(rng.integers(1, 2 ** 62))) * Fraction(2) ** int(rng.integers(-220, 70))
        assert eno.round_f32(e).tobytes() == _round_f32_slow(e).tobytes(), float(e)


def test_ref_norm_and_near_tie():
    e = eno.exact_sumsq(np.array(eno.TIE_C, F32))
    assert e == Fraction(2) + Fraction(1, 2 ** 23) + Fraction(1, 2 ** 90)
    assert int(eno.ref_norm(e).view(np.uint32)) == eno.TIE_NORM_BITS
    assert eno.near_tie(e, 1e-12) and not eno.near_tie(e, 1e-30)
    assert not eno.near_tie(Fraction(2), 1e-9)
    cands = eno.norm_candidates(e, 1e-12)
    assert {int(c.view(np.uint32)) for c in cands} >= {0x3FB504F3, eno.TIE_NORM_BITS}


def test_clip_norm_bound_is_about_six_units():
    rel = eno.clip_norm_bound(Fraction(4), 10) / 2
    assert 5.9 * 2 ** -24 < rel < 6.1 * 2 ** -24                  # (9u + u) / 2 + u
    # below the normal range the absolute term dominates: n subnormal roundings of at most 2^-150
    assert eno.clip_norm_bound(Fraction(0), 4) >= math.sqrt(4 * 2.0 ** -150)


def test_overflow_inputs_straddle_the_threshold():
    lo = eno.exact_sumsq(np.array(eno.overflow_c(False), F32))
    hi = eno.exact_sumsq(np.array(eno.overflow_c(True), F32))
    assert eno.OVERFLOW - Fraction(2) ** 64 < lo < eno.OVERFLOW < hi < eno.OVERFLOW + Fraction(2) ** 64
    assert eno.round_f32(lo) == FMAX and np.isinf(eno.round_f32(hi))
    for c in eno.overflow_c(True):                      # each square is exact in fp32 and below FLT_MAX
        assert float(F32(c)) == c and Fraction(float(F32(F32(c) * F32(c))))  == Fraction(c) ** 2


# ---- the accumulator, restated -------------------------------------------------------------------------------------
KBINS = 68                             # gaccum_kernels.cuh kAccBins: digit i has weight 2^(32 i - 1074)


def acc_add(bins, w: float) -> None:
    """acc_add of the non-negative finite double w: its 53-bit significand, shifted to its exponent, into three digits."""
    x = struct.unpack("<Q", struct.pack("<d", w))[0]
    e, mant = (x >> 52) & 0x7FF, x & ((1 << 52) - 1)
    if e:
        mant |= 1 << 52
    if mant == 0:
        return
    pos = e - 1 if e else 0
    q, r = pos >> 5, pos & 31
    lo = (mant << r) & ((1 << 64) - 1)
    hi = mant >> (64 - r) if r else 0
    bins[q] += lo & 0xFFFFFFFF
    bins[q + 1] += lo >> 32
    bins[q + 2] += hi


def _digits(bins):
    out, carry = [], 0
    for b in bins:
        t = b + carry
        out.append(t & 0xFFFFFFFF)
        carry = t >> 32
    return out


def value_double_then_float(bins) -> np.float32:
    """The accumulator as the kernels read it before rounding once: the three leading digits combined into a double
    in two rounded steps, then the cast to fp32."""
    d = _digits(bins)
    top = max((i for i, v in enumerate(d) if v), default=-1)
    if top < 0:
        return F32(0.0)
    g = [d[i] if i >= 0 else 0 for i in (top - 2, top - 1, top)]
    m = (float(g[2]) * 4294967296.0 + float(g[1])) * 4294967296.0 + float(g[0])
    return F32(math.ldexp(m, 32 * (top - 2) - 1074))


def value_rounded_once(bins) -> np.float32:
    """acc_value as it is now: the leading 64 bits with a sticky bit for everything below, rounded to odd at 53 bits
    into a double, then to nearest fp32 -- one correct rounding of the exact sum (53 >= 24 + 2)."""
    d = _digits(bins)
    top = max((i for i, v in enumerate(d) if v), default=-1)
    if top < 0:
        return F32(0.0)
    g2, g1, g0 = (d[i] if i >= 0 else 0 for i in (top, top - 1, top - 2))
    sticky = any(d[i] for i in range(0, max(top - 2, 0)))
    lz = 32 - g2.bit_length()
    hi = (((g2 << 32) | g1) << lz) | ((g0 >> (32 - lz)) if lz else 0)
    sticky = sticky or ((g0 << lz) & 0xFFFFFFFF) != 0
    mant = (hi >> 11) | int(sticky or (hi & 0x7FF) != 0)      # round to odd at 53 bits
    return F32(math.ldexp(float(mant), 32 * (top - 1) - lz - 1074 + 11))


def _accumulate(squares):
    bins = [0] * KBINS
    for w in squares:
        acc_add(bins, w)
    return bins


def test_tie_inputs_tell_single_from_double_rounding():
    """The warp totals of TIE_C (one element per tile): double-then-float loses 2^-90 and rounds the tie 2 + 2^-23 to
    2; rounding once gives 2 + 2^-22, whose sqrtf is TIE_NORM_BITS."""
    sq = [c * c for c in eno.TIE_C]
    bins = _accumulate(sq)
    twice, once = value_double_then_float(bins), value_rounded_once(bins)
    assert twice == F32(2.0) and once == F32(2 + 2 ** -22)
    assert int(np.sqrt(twice, dtype=F32).view(np.uint32)) == 0x3FB504F3
    assert int(np.sqrt(once, dtype=F32).view(np.uint32)) == eno.TIE_NORM_BITS
    assert once == eno.round_f32(eno.exact_sumsq(np.array(eno.TIE_C, F32)))


def test_overflow_inputs_tell_single_from_double_rounding():
    lo = _accumulate([c * c for c in eno.overflow_c(False)])
    assert value_rounded_once(lo) == FMAX and np.isinf(value_double_then_float(lo))
    assert np.isinf(value_rounded_once(_accumulate([c * c for c in eno.overflow_c(True)])))


@pytest.mark.parametrize("seed", range(4))
def test_rounded_once_is_the_correctly_rounded_sum(seed):
    """Random warp totals over the whole fp32-square range, and near-ties: the restated acc_value is round_f32."""
    rng = np.random.default_rng(7 + seed)
    for _ in range(200):
        n = int(rng.integers(1, 12))
        base = float(rng.integers(1, 2 ** 24)) * 2.0 ** int(rng.integers(-170, 100))
        ws = [base] + [float(rng.integers(1, 2 ** 53)) * 2.0 ** int(rng.integers(-298, 60) - 53) for _ in range(n)]
        exact = sum((Fraction(w) for w in ws), Fraction(0))
        got = value_rounded_once(_accumulate(ws))
        assert got.tobytes() == eno.round_f32(exact).tobytes(), (ws, got, eno.round_f32(exact))
