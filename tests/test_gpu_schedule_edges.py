"""The cooperative apply kernels at their schedule boundaries, against the composed oracle (tests/apply_matrix.py).

Shapes are derived from the GPU's SM count (``Schedule``), never hard-coded:
* clip-apply tile counts on both sides of 3*sms (the grid reaches its cap) and of kStashTiles*G for either stash depth
  (3 with an EMA, 4 without; from there on tiles are drawn from the ticket counters);
* pool paths: a leading tensor fills every stash and the awkward tiles follow it into the pool -- partial tiles, views
  that only the element or the 8-byte path can take, a tensor without a gradient, a zero-element tensor -- and the
  mirror image, with such tiles at a group's own positions b + j*G, j >= 1, between stashable ones;
* LAMB CTA ranges, with tensor boundaries on and one tile off CTA boundaries, a tensor across three or more CTAs,
  neighbours with alternating adaptation flags and the three cases of r = 1 (no adaptation, ||p|| = 0, ||u|| = 0);
* three launches on one plan, which alternate between the two counter sets, are bit-identical.

The pool-tile and LAMB cases run twice: reading the accumulators after every micro-step, and with the deferred reset
as training runs it (``LockStep(reset="deferred")``), where the clip-apply discards its pool tiles' a' lines and LAMB
its u lines from L2, and every first accumulate finds a poisoned slab.
"""
import itertools

import numpy as np
import pytest

from apply_matrix import LockStep, Schedule

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

T = Schedule.TILE


@pytest.fixture(scope="module")
def sched():
    return Schedule(torch.cuda.get_device_properties(0).multi_processor_count)


def _tile_counts(s: Schedule):
    G = s.clip_groups(3 * s.sms)
    out = []
    for base in (3 * s.sms, 3 * G, 4 * G):
        out += [base - 1, base, base + 1]
    return out


def _count_manifest(nt):
    """nt tiles: a body of full tiles, then a tensor of one full and one partial tile."""
    return [("body/kernel", ((nt - 2) * T,)), ("LayerNorm/beta", (T + 1001,))]


@pytest.mark.parametrize("k", range(9))
def test_clip_apply_tile_counts(sched, k):
    nt = _tile_counts(sched)[k]
    man = _count_manifest(nt)
    assert sum(-(-n // T) for _, (n,) in man) == nt
    for ema in (False, True):
        for dtype in ("fp32", "bf16"):
            run = LockStep(man, "adamw", "clip", dtype=dtype, ema=(0.9, True) if ema else None, N=2, seed=k)
            run.run(3)                                          # windows at steps 0 and 2
            assert run.clipped
    # loss-scaled, plain Adam with an EMA: the window applied at step 2 overflows in the last tile
    run = LockStep(man, "adam", "ls_clip", ema=(0.9, False), N=2, seed=100 + k)
    run.run(5, inf_at=(1, 1, T + 1000))
    assert run.op.loss_scale_state()["skipped_windows"] == 1


def _awkward(dtype):
    """(manifest entries, view offsets, no-grad names) of the tiles that cannot be stashed, each in its own tensor."""
    man = [(f"tail{n}/kernel", (n,)) for n in (1, 2, 3, 5, 6, 7, 12, 13, 14, 15)]   # len % 4 in 1..3, len % 8 in 4..7
    man += [("multi/bias", (2 * T + 13,)), ("nograd/kernel", (T,)), ("empty/kernel", (0,))]
    views = {}
    if dtype == "fp32":
        man += [("unal4/kernel", (2 * T + 5,))]                    # 4 bytes past an aligned address: element path
        views["unal4/kernel"] = 1
    else:
        man += [("unal8/kernel", (2 * T + 13,)), ("unal2/kernel", (T + 7,))]
        views["unal8/kernel"] = 4                                   # 8-byte aligned: the vector path
        views["unal2/kernel"] = 1                                   # 2-byte aligned: the element path
    return man, views, {"nograd/kernel"}


RESETS = ("materialized", "deferred")


def _lockstep(man, views, nograd, variant, mode, dtype, has_g, ema, seed, reset, N=2):
    names = [n for n, _ in man]
    return LockStep(man, variant, mode, dtype=dtype, has_g=has_g, ema=(0.9, True) if ema else None, N=N, seed=seed,
                    views={names.index(n): o for n, o in views.items()}, nograd=[names.index(n) for n in nograd],
                    reset=reset)


def _finish(run):
    if run.reset == "deferred":
        assert run.first_over_poison > 0
    run.finish()


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("ls", [False, True])
@pytest.mark.parametrize("ema", [False, True])
@pytest.mark.parametrize("has_g", [True, False])
def test_awkward_tiles_in_the_pool(sched, has_g, ema, ls, dtype):
    G = sched.clip_groups(3 * sched.sms)
    lead = Schedule.STASH_TILES[ema] * G                            # fills every group's stash
    aw, views, nograd = _awkward(dtype)
    man = [("lead/kernel", (lead * T,))] + aw
    assert sched.pool_lo(lead + 1, ema) == lead
    for reset in RESETS:
        run = _lockstep(man, views, nograd, "adamw", "ls_clip" if ls else "clip", dtype, has_g, ema, 3, reset)
        if ls:
            run.run(5, inf_at=(1, 8, 3))                            # an inf in a 13-element pool tile
            assert run.op.loss_scale_state()["skipped_windows"] == 1
        else:
            run.run(3)
        _finish(run)


def _mirror(G, ema, dtype):
    """Own tiles of group b are b + j*G.  j = 0: full aligned tiles; j = 1: one unstashable tile per group (partial,
    unaligned or gradient-less); j = 2 (and j = 3 without an EMA): full aligned tiles again; then pool tiles."""
    kinds = [13, 12, 2047, 1, 1000, 7, "view", "nograd"]
    man, views, nograd = [("own0/kernel", (G * T,))], {}, set()
    for b in range(G):
        kind = kinds[b % len(kinds)]
        name = f"j1_{b}/{'bias' if b % 5 == 0 else 'kernel'}"
        if kind == "view":
            views[name] = 1                                         # a full tile, 4 (fp32) or 2 (16-bit) bytes off
            man.append((name, (T,)))
        elif kind == "nograd":
            nograd.add(name)
            man.append((name, (T,)))
        else:
            man.append((name, (kind,)))
        if b == G // 2:
            man.append(("empty/kernel", (0,)))
    man.append(("own2/kernel", ((Schedule.STASH_TILES[ema] - 2) * G * T,)))
    man.append(("pool/kernel", (3 * T + 5,)))
    return man, views, nograd


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
@pytest.mark.parametrize("ema", [False, True])
@pytest.mark.parametrize("has_g", [True, False])
def test_unstashable_tiles_between_stashed_ones(sched, has_g, ema, dtype):
    G = sched.clip_groups(3 * sched.sms)
    man, views, nograd = _mirror(G, ema, dtype)
    ls = not has_g
    for reset in RESETS:
        run = _lockstep(man, views, nograd, "adamw", "ls_clip" if ls else "clip", dtype, has_g, ema, 4, reset)
        if ls:
            run.run(5, inf_at=(1, 2, 5))                            # an inf in own tile j = 1 of group 1
            assert run.op.loss_scale_state()["skipped_windows"] == 1
        else:
            run.run(3)
        _finish(run)


def _lamb_manifest(s: Schedule, nt: int):
    """nt tiles whose tensor boundaries fall on CTA boundaries and one tile before or after them; the first tensor
    spans at least three CTAs.  Then (no tiles) an adapted zero-element tensor; tensor 2 starts at zero (||p|| = 0 in
    the first window), tensor 3 has neither a gradient nor weight decay (u = 0, ||u|| = 0); the rest alternate between
    adapted and not."""
    starts = [lo for lo, _ in s.lamb_ranges(nt)]
    ends = [starts[3] + 1]
    k = 0
    for c in range(4, len(starts)):
        e = starts[c] + (0, 1, -1)[k % 3]
        if ends[-1] < e < nt:
            ends.append(e)
            k += 1
    ends.append(nt)
    tiles = np.diff([0] + ends)
    man = []
    for i, n in enumerate(tiles):
        numel = int(n) * T - (0, 1, T - 5)[i % 3]
        name = {0: "first/kernel", 1: "zero_w/kernel", 2: "zero_u/bias"}.get(i, f"t{i}/{'kernel' if i % 2 else 'noadapt'}")
        man.append((name, (numel,)))
    man.insert(1, ("empty/kernel", (0,)))
    return man


@pytest.mark.parametrize("which", range(4))
def test_lamb_cta_ranges(sched, which):
    nt = (3 * sched.sms - 1, 3 * sched.sms, 3 * sched.sms + 1, 6 * sched.sms + 1)[which]
    man = _lamb_manifest(sched, nt)
    assert sum(-(-n // T) for _, (n,) in man) == nt
    names = [n for n, _ in man]
    zw, zu, empty = names.index("zero_w/kernel"), names.index("zero_u/bias"), names.index("empty/kernel")
    for (dtype, mode), reset in itertools.product((("fp32", "clip"), ("bf16", "ls_clip")), RESETS):
        run = LockStep(man, "lamb", mode, dtype=dtype, N=2, seed=5 + which, zero=[zw], nograd=[zu],
                       adapt_exclude=("noadapt",), reset=reset)
        adapt = run.op.adapt
        assert adapt[zw] and adapt[zu] and adapt[empty]
        assert any(adapt[i] != adapt[i + 1] for i in range(4, len(man) - 1))
        window = 0
        for step in range(5 if mode == "ls_clip" else 3):
            inf = (0, 10) if mode == "ls_clip" and step == 1 else None
            w_zero = not run._weights()[zw].any()          # ||p|| = 0: until an apply with lr > 0 has moved it
            if run.step(run.grads(inf_at=inf)) and not run.skipped():
                assert w_zero or window > 0
                r = run.op.trust_ratios()
                for i in range(len(man)):
                    if not adapt[i] or i in (zu, empty) or (i == zw and w_zero):
                        assert r[i] == np.float32(1.0), (names[i], r[i])
                    else:
                        assert r[i] != np.float32(1.0), names[i]
                window += 1
        assert window == 2
        _finish(run)


@pytest.mark.parametrize("variant", ["adamw", "lamb"])
@pytest.mark.parametrize("ema", [False, True])
def test_three_launches_are_bit_identical(sched, variant, ema):
    """At nt = 4G + 1: three apply launches on one plan from the same state, alternating between the counter sets."""
    G = sched.clip_groups(3 * sched.sms)
    man = _count_manifest(4 * G + 1)
    run = LockStep(man, variant, "clip", ema=(0.9, False) if ema else None, N=1, seed=6)
    op = run.op
    gr = [torch.from_numpy(x).cuda() for x in run.grads()]
    slabs = [op.accum, op.m, op.v] + ([op.ema] if ema else [])
    saved = [t.clone() for t in slabs + list(op.params)]
    betas = (op.beta1_power, op.beta2_power)
    state0 = op.ema_state() if ema else None
    outs = []
    for _ in range(3):
        for t, s in zip(slabs + list(op.params), saved):
            t.copy_(s)
        op.beta1_power, op.beta2_power = betas
        if ema:
            op.plan.ema_init(op._ema_state.data_ptr(), state0["num_updates"], op._stream())
        op.apply_only(gr)
        torch.cuda.synchronize()
        got = [t.clone() for t in slabs + list(op.params)]
        extra = [np.array(list(op.stats().values()), np.float32)]
        if variant == "lamb":
            extra.append(op.trust_ratios())
        outs.append((got, extra))
    assert outs[0][1][0][3] < 1.0                                   # the window clipped
    for got, extra in outs[1:]:
        for x, y in zip(got, outs[0][0]):
            assert torch.equal(x.view(torch.int32), y.view(torch.int32))
        for x, y in zip(extra, outs[0][1]):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
