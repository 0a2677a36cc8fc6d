"""The clipped and LAMB apply steps bit for bit against the oracle, and their norms against exact sums
(tests/exact_norm_oracle.py).

a. Every dispatch key that clips or runs LAMB (224 cases), in ``LockStep``'s injected mode: the oracle takes the
   kernel's global norm and trust ratios, so p, m, v, the master weights, the model copy, the EMA and the clip scale
   are compared bit for bit in every window, clipped ones included; gn is held to the exact sum of the window's c
   within the derived bound, and r to the ratio of the correctly rounded norms.  On the apply matrix's model, and
   with mixed window weights and learning-rate multipliers.
b. Known answers: c (and the first window's p) in {+-1, +-2, +-3} * 2^-j, so every partial sum in every order is exact:
   gn and the per-tensor gradient and weight norms must equal the norms of the exact sums bit for bit, and every
   element counts (one dropped or counted twice changes the integer sum, and sqrtf tells the two apart).  Unaligned
   views, tensors without a gradient, zero-element tensors, bf16 / fp16 gradients, loss scaling with a large S, the
   300-tensor CAP 1920 table, and a model large enough to have pool tiles (with and without EMA) and many LAMB CTA
   ranges; and one BERT-Large window whose gn is held to the exact sum at full size.
c. Single rounding of the exact sum: inputs whose sum of squares rounds differently once than through an fp64 first
   (exact_norm_oracle.TIE_C, overflow_c) in a clip-apply and a LAMB window.
"""
import math
import zlib

import numpy as np
import pytest

import exact_norm_oracle as eno
import oracle_np as onp
from apply_matrix import Case, LockStep, Schedule, matrix_cases

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

F32 = np.float32
MAN = [("a/kernel", (2 * 2048 + 777,)), ("a/bias", (5,)), ("one/kernel", (1,)), ("empty/kernel", (0,)),
       ("LayerNorm/gamma", (33,)), ("nograd/kernel", (64,)), ("t/kernel", (3, 1367))]
NOGRAD = (5,)
TINY = [(f"tiny{i}/{'bias' if i % 3 == 0 else 'kernel'}", (1 + i % 7,)) for i in range(300)]
STEPS = 10
INF_AT = (4, 0, 1000)
EMA = (0.9, True)
WEIGHTS = (3.0, 37.0, 1000.0, 5.0, 64.0, 11.0)
CYCLE = (0.37, 0.0, 2.5, 1.0)

CASES = [c for c in matrix_cases() if c.mode in ("clip", "ls_clip") or c.variant == "lamb"]


def _setup(case: Case):
    layout = "packed" if case.layout == "packed" else "table"
    dtype = case.layout.split("_")[-1] if layout == "table" else "fp32"
    return layout, dtype, (MAN + TINY if case.layout.startswith("t1920") else MAN)


def _gn_bits(op) -> int:
    return int(F32(op.stats()["global_norm"]).view(np.uint32))


# ---- a. bit for bit after clipping ------------------------------------------------------------------------------------
def test_case_count():
    assert len(CASES) == 224


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_clipped_and_lamb_windows_are_bit_exact(case: Case):
    layout, dtype, man = _setup(case)
    run = LockStep(man, case.variant, case.mode, layout, dtype, case.has_g, EMA if case.ema else None, N=3,
                   seed=zlib.crc32(case.id.encode()), nograd=NOGRAD, injected=True)
    ls = case.mode.startswith("ls_")
    run.run(STEPS, inf_at=INF_AT if ls else None)
    if ls:
        assert run.op.loss_scale_state()["skipped_windows"] == 1


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_weighted_windows_with_lr_multipliers_are_bit_exact(case: Case):
    layout, dtype, man = _setup(case)
    run = LockStep(man, case.variant, case.mode, layout, dtype, case.has_g, EMA if case.ema else None, N=3,
                   seed=zlib.crc32(case.id.encode()) ^ 3, nograd=NOGRAD, injected=True,
                   lr_mult=[CYCLE[i % len(CYCLE)] for i in range(len(man))], window_weight=True)
    ls = case.mode.startswith("ls_")
    for s in range(STEPS):
        run.wstep(run.grads(0.1, INF_AT[1:] if ls and s == INF_AT[0] else None), WEIGHTS[s % len(WEIGHTS)])
    if ls:
        assert run.op.loss_scale_state()["skipped_windows"] == 1


# ---- b. exactly representable known answers ---------------------------------------------------------------------------
def _units(rng, shape, j: int, kmax: int = 3) -> np.ndarray:
    """Elements in {+-1, ..., +-kmax} * 2^-j: none is zero, so every element position is a sentinel."""
    x = rng.integers(1, kmax + 1, size=shape) * rng.choice([-1, 1], size=shape)
    return (x * 2.0 ** -j).astype(F32)


def _known_answers(run: LockStep, steps: int, j: int, kmax: int = 3) -> None:
    """N = 1: every step is a window whose c is the unscaled gradient.  After each: gn and the tensor-norm gradient
    column are the norms of the exact sums, bit for bit; after the first, the weight column too (p still the units
    it started as)."""
    assert run.N == 1 and run.injected
    rng = np.random.default_rng(11)
    for s in range(steps):
        p0 = [x.copy() for x in run._weights()]
        grads = [None if i in run.nograd else _units(rng, shp, j, kmax) for i, (_, shp) in enumerate(run.man)]
        run.step(grads)
        st = run.op.stats()
        c = run.ref.window_c
        exact = [eno.exact_sumsq(x) for x in c]
        want = eno.ref_norm(sum(exact))
        assert F32(st["global_norm"]).tobytes() == want.tobytes(), (s, st["global_norm"], want)
        norms = run.op.tensor_norms()
        for i, (name, _) in enumerate(run.man):
            assert norms[i, 0].tobytes() == eno.ref_norm(exact[i]).tobytes(), (s, name, "gradient", norms[i, 0])
            if s == 0:
                w = eno.ref_norm(eno.exact_sumsq(p0[i]))
                assert norms[i, 1].tobytes() == w.tobytes(), (name, "weight", norms[i, 1], w)


def _init_units(man, j: int = 4):
    rng = np.random.default_rng(5)
    return {i: _units(rng, shp, j) for i, (_, shp) in enumerate(man)}


KNOWN = {
    # name: (variant, mode, layout, dtype, man, extra LockStep kwargs, j)
    "adamw_clip_fp32": ("adamw", "clip", "table", "fp32", MAN, {}, 0),
    "adam_clip_views": ("adam", "clip", "table", "fp32", MAN, dict(views={0: 1, 1: 3, 4: 2, 6: 1}), 2),
    "adamw_clip_packed": ("adamw", "clip", "packed", "fp32", MAN, {}, 1),
    "adamw_clip_bf16": ("adamw", "clip", "table", "bf16", MAN, {}, 3),
    "adam_clip_fp16": ("adam", "clip", "table", "fp16", MAN, {}, 5),
    "adamw_ls_clip_large_s": ("adamw", "ls_clip", "table", "fp32", MAN, dict(ls_cfg=(2.0 ** 40, 2.0, 2)), 3),
    "adam_ls_clip_bf16_large_s": ("adam", "ls_clip", "table", "bf16", MAN, dict(ls_cfg=(2.0 ** 24, 2.0, 1)), 0),
    "adamw_clip_cap1920": ("adamw", "clip", "table", "fp32", MAN + TINY, {}, 2),
    "lamb_clip_fp32": ("lamb", "clip", "table", "fp32", MAN, {}, 1),
    "lamb_ls_clip_cap1920_fp16": ("lamb", "ls_clip", "table", "fp16", MAN + TINY, {}, 4),
}


@pytest.mark.parametrize("name", sorted(KNOWN))
def test_known_answers(name):
    variant, mode, layout, dtype, man, kw, j = KNOWN[name]
    run = LockStep(man, variant, mode, layout, dtype, N=1, seed=3, nograd=NOGRAD, injected=True, tensor_norms=True,
                   init=_init_units(man), **kw)
    _known_answers(run, 3, j)


def _sched():
    return Schedule(torch.cuda.get_device_properties(0).multi_processor_count)


@pytest.mark.parametrize("variant, ema", [("adamw", False), ("adam", True), ("lamb", False)])
def test_known_answers_across_pool_and_lamb_ranges(variant, ema):
    """One tensor long enough that the clip-apply draws pool tiles past pool_lo (and LAMB splits it over every CTA), a
    short tensor after it, and a tail: every element is +-2^-j, so the sum is the element count and no tile on
    either side of pool_lo or a LAMB range end may be dropped or counted twice."""
    sch = _sched()
    nt = sch.STASH_TILES[ema] * sch.GROUPS * sch.sms + 5
    man = [("big/kernel", (nt * Schedule.TILE - 3,)), ("small/kernel", (2 * Schedule.TILE + 1,))]
    tiles = nt + 2 + 1
    assert sch.pool_lo(tiles, ema) < nt < tiles
    ranges = sch.lamb_ranges(tiles)
    assert len(ranges) == 3 * sch.sms and ranges[-1][1] == tiles
    run = LockStep(man, variant, "clip", N=1, seed=9, ema=EMA if ema else None, injected=True, tensor_norms=True,
                   init=_init_units(man))
    _known_answers(run, 2, 0, kmax=1)


def test_bert_large_window_norm_at_full_size():
    """One BERT-Large window (fp32, 335 M parameters): gn against the exact sum of squares of c = g / N."""
    import gaccum_b200 as g
    from gaccum_b200.train_op import GaccumTrainOp
    man = onp.bert_manifest(24, 1024)
    gen = torch.Generator(device="cuda").manual_seed(0)
    params = [torch.randn(s, device="cuda", generator=gen) * 0.02 for _, s in man]
    grads = [torch.randn(s, device="cuda", generator=gen) * 1e-3 for _, s in man]
    hp = g.HParams(0, 0, 0.9, 0.999, 1e-6, 0.01, 1.0)
    op = GaccumTrainOp(params, [n for n, _ in man], hp, 1, lambda s: 1e-4)
    assert op.run(grads)
    st = op.stats()
    e = sum((eno.exact_sumsq(x.cpu().numpy()) for x in grads), eno.Fraction(0))
    n = sum(x.numel() for x in grads)
    assert n > 330_000_000
    gn = F32(st["global_norm"])
    assert abs(float(gn) - math.sqrt(e)) <= eno.clip_norm_bound(e, n), (float(gn), math.sqrt(e))
    assert F32(st["clip_scale"]).tobytes() == onp.clip_scale(gn, 1.0).tobytes()


# ---- c. single rounding of the exact sum ------------------------------------------------------------------------------
def _one_per_tile(values):
    x = np.zeros(len(values) * Schedule.TILE, F32)
    x[::Schedule.TILE] = np.asarray(values, F32)
    return x


@pytest.mark.parametrize("variant, mode", [("adamw", "clip"), ("adam", "ls_clip")])
def test_global_norm_is_rounded_once(variant, mode):
    c = _one_per_tile(eno.TIE_C)
    run = LockStep([("x/kernel", c.shape)], variant, mode, N=1, seed=1, injected=True)
    run.step([c])
    gn = run.op.stats()
    assert int(F32(gn["global_norm"]).view(np.uint32)) == eno.TIE_NORM_BITS, hex(_gn_bits(run.op))
    assert F32(gn["clip_scale"]).tobytes() == onp.clip_scale(F32(gn["global_norm"]), 0.5).tobytes()


def test_lamb_weight_norm_is_rounded_once():
    p = _one_per_tile(eno.TIE_C)
    run = LockStep([("x/kernel", p.shape)], "lamb", "noclip", N=1, seed=2, injected=True, init={0: p})
    assert run.op.adapt[0]
    run.step(run.grads(0.1))
    (p0, u), = run.ref.window_pu
    wn = np.sqrt(eno.round_f32(eno.exact_sumsq(p0)), dtype=F32)
    assert int(wn.view(np.uint32)) == eno.TIE_NORM_BITS
    r = run.op.trust_ratios()[0]
    assert r.tobytes() == F32(wn / eno.ref_norm(eno.exact_sumsq(u))).tobytes(), (r, wn)


@pytest.mark.parametrize("mode", ["clip", "ls_clip"])
def test_sum_just_below_overflow_applies(mode):
    c = _one_per_tile(eno.overflow_c(False))
    run = LockStep([("x/kernel", c.shape)], "adamw", mode, N=1, seed=4, injected=True)
    assert run.step([c])
    gn = F32(run.op.stats()["global_norm"])
    assert gn == np.sqrt(np.finfo(F32).max, dtype=F32), hex(_gn_bits(run.op))
    if mode == "ls_clip":
        assert not run.op.loss_scale_state()["last_skipped"]


def test_sum_just_above_overflow_is_skipped():
    c = _one_per_tile(eno.overflow_c(True))
    run = LockStep([("x/kernel", c.shape)], "adamw", "ls_clip", N=1, seed=4, injected=True)
    run.step([c])
    assert np.isinf(run.op.stats()["global_norm"])
    st = run.op.loss_scale_state()
    assert st["last_skipped"] and st["skipped_windows"] == 1
