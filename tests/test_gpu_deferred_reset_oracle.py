"""The deferred reset of the accumulators (include/gaccum.h, gaccum_plan_set_deferred_reset) against the composed
oracle, where the suites that run it as training does (``LockStep(reset="deferred")``) cannot reach: what
``gaccum_accum_materialize`` may and may not touch, materialize captured in a CUDA graph, the mode turned off and on
between micro-steps, and one run with every feature on, a captured window replayed over a poisoned slab.

* Materialize touches no other state: the stats, loss-scaling, EMA, window-weight, schedule, norm and trust-ratio
  blocks, m, v, the master weights and the average are byte for byte the same around an ``op.accum`` read, with the
  plan's word set (right after an apply) and clear (mid-window).
* With the word clear it changes nothing: the raw slab, padding included, is bit-identical after a direct call.
* Captured right after a window's apply, it zero-fills the slab at every replay and leaves the padding alone.
* ``_set_deferred_reset`` off and on, right after an apply and mid-window, keeps training on the oracle.
* LAMB, loss scaling with a skipped window, bf16, EMA, lr multipliers, window weights, per-tensor norms and an
  ``LrTable`` device schedule: one window captured and replayed for 9 windows, the graph poisoning the slab after
  its apply.
"""
import gc
import itertools

import numpy as np
import pytest

from apply_matrix import Case, LockStep, poison_bits
from tensor_norms_oracle import assert_close, expected_norms
from test_gpu_device_schedule_matrix import MAN, NOGRAD, WEIGHTS, N, Scheduled, _capture, _fill
from test_gpu_lr_table import TableRun

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

F32 = np.float32


def _blocks(run):
    """Every device buffer of the op but the accumulators, and the blocks it keeps, as host bytes."""
    op = run.op
    torch.cuda.synchronize()
    out = {"stats": torch.from_numpy(np.array(list(op.stats().values()), F32)),
           "ratios": torch.from_numpy(op.trust_ratios()), "m": op.m, "v": op.v, "master": op.master, "ema": op.ema, "ema_state": op._ema_state, "ls": op._ls_state,
           "ww": run.ww, "sched": op._sched_state, "norms": op.tensor_norms_tensor}
    return {k: v.detach().cpu().contiguous().view(torch.uint8).clone() for k, v in out.items()}


def _raw_bits(run):
    torch.cuda.synchronize()
    return run.op._accum.view(torch.int32).cpu().clone()


def _all_features(seed):
    """LAMB, loss scaling, bf16, EMA; ``Scheduled`` adds lr multipliers, window weights, per-tensor norms and the
    device schedule."""
    return Scheduled(Case("lamb", "ls_clip", True, "t256_bf16", True), seed, reset="deferred")


def test_materialize_touches_no_other_state():
    run = _all_features(0xD1)
    assert run.micro() and run.poisoned                        # step 0 applied: the word is set
    for where in ("word set", "word clear"):
        before = _blocks(run)
        run.read_accum()                                       # op.accum: +0.0 right after the apply, else ref.accum
        after = _blocks(run)
        for k in before:
            assert torch.equal(before[k], after[k]), f"{where}: materialize changed {k}"
        assert not run.micro()                                 # a first accumulate, then mid-window
    while not run.micro():
        pass
    run.finish()


def test_materialize_with_the_word_clear_changes_nothing():
    run = _all_features(0xD2)
    run.micro(); run.micro()                                   # the apply at 0, the first accumulate at 1
    assert not run.poisoned
    before = _raw_bits(run)
    run.op.plan.accum_materialize(run.op._accum_ptr, run.op._stream())
    run.expected_materializes += 1
    assert torch.equal(before, _raw_bits(run)), "materialize wrote the slab with the word clear"
    for _ in range(2 * N):
        run.micro()
    run.finish()


@pytest.mark.parametrize("dtype", ["fp32", "bf16"])
def test_materialize_captured_after_an_apply(dtype):
    """A window's apply and an ``op.accum`` access captured in one graph (a device-scheduled graph starts at a window
    start), replayed at every window start with the window's accumulates launched eagerly in between: every replay
    leaves the slab's tensor elements at +0.0 and its padding untouched, and the run matches the oracle."""
    run = LockStep(MAN, "adamw", "clip", dtype=dtype, N=N, seed=0xD3, nograd=NOGRAD, device_schedule=True,
                   reset="deferred")
    for _ in range(N + 1):                                     # applies at 0 and 3: every kernel loads
        run.step(run.grads())
    run.read_accum()                                           # ... materialize's too
    while run.g_host % N:
        run.step(run.grads())
    op = run.op
    _, dev = run.inputs(run.grads())
    static = [None if t is None else torch.zeros_like(t) for t in dev]
    graph = torch.cuda.CUDAGraph()
    gc.collect()               # an earlier test's plan freed (cudaFree) during the capture would invalidate it
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        op.run(static)
        op.accum                                               # materializes: the word the apply just set
    run.expected_materializes += 1                             # the one call, made while capturing
    for _ in range(4):
        host, dev = run.inputs(run.grads())
        info = run.ref.run(host)
        _fill(static, dev)
        graph.replay()
        run.g_host += 1
        op._cursor.reset(run.g_host)                           # a one-launch graph leaves the host's step behind
        assert info.applied
        run.check(info)
        raw = _raw_bits(run).numpy()
        for o, (name, s) in zip(op.plan.offsets, MAN):
            assert not raw[o:o + int(np.prod(s))].any(), f"{name} is not +0.0 after the captured materialize"
        run.check_padding()
        for _ in range(N - 1):
            run.step(run.grads())                              # the word is clear: the slab holds real zeros
    run.finish()


TRANSITION_KEYS = list(itertools.product([("adamw", "clip"), ("adam", "ls_clip"), ("lamb", "clip")], ["fp32", "bf16"]))


@pytest.mark.parametrize("variant, mode, dtype", [(v, m, d) for (v, m), d in TRANSITION_KEYS],
                         ids=[f"{v}-{m}-{d}" for (v, m), d in TRANSITION_KEYS])
def test_mode_transitions_match_the_oracle(variant, mode, dtype):
    """N = 3 from step 0 (applies at 0, 3, 6, 9, 12).  Off right after the apply at 0 (a poisoned slab), on right after
    the apply at 3 (the stored zeros), off mid-window after 5, on mid-window after 7.  "sometimes/kernel" has a
    gradient on even steps only; under loss scaling the window that applies at 9 overflows and is skipped."""
    man = MAN + [("sometimes/kernel", (3, 700))]
    sometimes = len(man) - 1
    run = LockStep(man, variant, mode, dtype=dtype, N=N, seed=0xD4, nograd=NOGRAD, reset="deferred")
    switch = {0: "stored", 3: "deferred", 5: "stored", 7: "deferred"}
    for s in range(15):
        grads = run.grads(inf_at=(0, 17) if run.ls and s == 8 else None)
        if s % 2:
            grads[sometimes] = None
        run.step(grads)
        if s in switch:
            run.set_reset(switch[s])
    if run.ls:
        assert run.op.loss_scale_state()["skipped_windows"] == 1
    assert run.first_over_poison == 2                          # after the applies at 9 and 12
    run.finish()


def test_every_feature_with_a_captured_window_over_a_poisoned_slab():
    """LAMB, ls_clip, bf16, EMA, lr multipliers, window weights, per-tensor norms and an LrTable schedule.  An eager
    window, then the window that applies at 3 captured and replayed for 9 windows; the graph poisons the raw slab
    after its apply, with values changed between replays, and the apply of the sixth replay skips an overflowed window.
    After each replay (mid-window) everything ``check`` compares, the raw slab included, matches the composed oracle,
    and the norms of its apply match ``tensor_norms_oracle``."""
    table = [1e-3 * (1 + 0.1 * (i % 7)) for i in range(40)]
    run = TableRun(Case("lamb", "ls_clip", True, "t256_bf16", True), 0xD5, table, injected=False, reset="deferred")
    assert run.op.lr_table is not None and run.op.ema is not None and run.op.master is not None
    for _ in range(N):
        run.micro()
    assert run.first_over_poison == 1
    poison = torch.zeros(len(run.man), dtype=torch.int32, device="cuda")
    graph, static = _capture(run, N, weights=True, poison=poison)
    op = run.op
    for w in range(9):
        poison.copy_(torch.tensor([poison_bits(i, w + 1) for i in range(len(run.man))]))
        infos, w0 = [], run._weights()
        for j in range(N):
            s = run.step_no
            run.step_no += 1
            host, dev = run.inputs(run.grads(0.1, (0, 99) if w == 4 and j == 1 else None))
            weight = WEIGHTS[s % len(WEIGHTS)]
            run.ref.add_weight(weight)
            _fill(static[j], dev, weight)
            if j == 0:
                apply_in, S = ([a.copy() for a in run.ref.accum], host, F32(run.ref.weight)), F32(run.ref.scale)
            infos.append(run.ref.run(host))
        graph.replay()
        run.g_host += N
        assert infos[0].applied and run.skipped() == (w == 5)
        if not run.skipped():
            run.tracker.average(run._weights())                # check() averages on an applied step only
        run.check(infos[-1])
        acc, host0, W = apply_in
        assert_close(op.tensor_norms(), expected_norms(acc, host0, W, S, w0, run._weights()), what=f"norms, replay {w}")
    assert op.loss_scale_state()["skipped_windows"] == 1 and op.ema_state()["num_updates"] == 1 + 8
    assert run.materializes == 0
    run.finish()
