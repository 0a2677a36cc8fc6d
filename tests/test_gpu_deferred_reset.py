"""The deferred reset of the accumulators (gaccum.h, gaccum_plan_set_deferred_reset), which GaccumTrainOp turns on for
N >= 2: the apply leaves the accumulators logically zero instead of storing zeros, and the window's first accumulate
stores +0 + G (+0 where a tensor has no gradient).

Every case runs a deferred-reset op and a twin with the mode off side by side on the same inputs and compares them bit
for bit at every micro-step: parameters (and master weights), m, v, the stats block and the device state blocks, and
-- at the steps a case reads them -- the accumulators through ``accum`` and ``accum_view``.  Reading the accumulators
materializes a deferred reset, so the main loops read them only where no apply came since the last first accumulate,
leaving the first accumulate to store the zeros of tensors without a gradient itself.

Each case runs twice: once as above, and once with the deferred op's raw slab poisoned right after every apply
(``Pair(poison=True)``; never the twin's), so that a launch or a read that should have materialized first, or a first
accumulate that reads the slab, differs from the twin."""
import numpy as np
import pytest

from apply_matrix import poison_bits

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

# 2 x 2^21 elements: more tiles (2048 + tails) than the clip-apply's stash holds on an H100 (4 x 3 x 132), so pass 2
# also takes pool tiles; tails of 1-3 elements; a tensor that never has a gradient and one that skips some steps
MAN = [("bert/embeddings/word_embeddings", (2048, 2048)), ("layer/kernel", (3, 1367)), ("layer/bias", (777,)),
       ("LayerNorm/gamma", (5,)), ("one", (1,)), ("nograd/kernel", (130,)), ("sometimes/kernel", (64, 33))]
NOGRAD, SOMETIMES = 5, 6


def _bits(t):
    t = t.detach()
    if t.dtype in (torch.bfloat16, torch.float16):
        return t.contiguous().view(torch.int16)
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def _same(a, b, what):
    assert torch.equal(_bits(a), _bits(b)), what


def _stats_bits(op):
    return np.array(list(op.stats().values()), np.float32).view(np.uint32)


class Pair:
    """A deferred-reset GaccumTrainOp and its twin without the mode, built from the same parameters."""

    def __init__(self, N, hp=None, dtype=torch.float32, seed=0, poison=False, **kw):
        from gaccum_b200 import _lib
        from gaccum_b200.train_op import GaccumTrainOp
        self.N, self.dtype, self.poison, self.windows = N, dtype, poison, 0
        gen = torch.Generator(device="cuda").manual_seed(seed)
        init = [(torch.randn(s, device="cuda", generator=gen) * 0.02).to(dtype) for _, s in MAN]
        hp = hp if hp is not None else _lib.HParams.bert()
        kw.setdefault("global_step", 1)                  # step 1 starts a window
        kw["lr_fn"] = None if "device_schedule" in kw else (lambda s: 1e-3 * (1.0 + 0.01 * (s % 7)))
        names = [n for n, _ in MAN]
        self.op = GaccumTrainOp([p.clone() for p in init], names, hp, N, **kw)
        self.twin = GaccumTrainOp([p.clone() for p in init], names, hp, N, **kw)
        self.twin._set_deferred_reset(False)
        assert self.op._deferred and not self.twin._deferred
        self.gen = torch.Generator(device="cuda").manual_seed(seed + 1)
        self.i = 0

    def grads(self, scale=0.05, inf_at=None):
        out = []
        for t, (_, s) in enumerate(MAN):
            if t == NOGRAD or (t == SOMETIMES and self.i % 3 == 1):
                out.append(None)
                continue
            g = torch.randn(s, device="cuda", generator=self.gen) * scale
            if inf_at is not None and t == inf_at:
                g.view(-1)[7] = float("inf")
            out.append(g.to(self.dtype))
        return out

    def step(self, **kw):
        g = self.grads(**kw)
        a, b = self.op.run(g), self.twin.run(g)
        assert a == b
        self.i += 1
        if a:
            self.after_apply()
        return a

    def after_apply(self):
        """``poison``: the deferred op's raw accumulators, logically +0 until the window's first accumulate, get a
        value per tensor that no correct launch reads (``apply_matrix.POISON``)."""
        self.windows += 1
        if self.poison and _next_is_first(self):
            with torch.no_grad():
                for i in range(len(MAN)):
                    self.op._view(self.op._accum, i).view(torch.int32).fill_(poison_bits(i, self.windows))

    def check(self, what, accum=False):
        op, tw = self.op, self.twin
        torch.cuda.synchronize()
        for i in range(len(MAN)):
            _same(op.params[i], tw.params[i], f"{what}: param {i}")
        for name in ("m", "v", "master", "ema", "_ls_state", "_sched_state", "_ema_state", "_ww_state"):
            x, y = getattr(op, name, None), getattr(tw, name, None)
            if x is not None:
                _same(x, y, f"{what}: {name}")
        assert np.array_equal(_stats_bits(op), _stats_bits(tw)), what
        if accum:
            _same(op.accum, tw.accum, f"{what}: accum")
            for i in range(len(MAN)):
                _same(op.accum_view(i), tw.accum_view(i), f"{what}: accum_view {i}")
            assert np.array_equal(_stats_bits(op), _stats_bits(tw)), f"{what}: reading the accumulators changed the stats"

    def run_windows(self, windows, read_every_step=False, **kw):
        applies = 0
        for _ in range(windows * self.N):
            applied = self.step(**kw)
            applies += applied
            # the accumulators are read wherever doing so leaves the next first accumulate a deferred reset to do
            self.check(f"step {self.i}", accum=read_every_step or not _next_is_first(self))
        return applies


def _next_is_first(pair):
    from gaccum_b200 import _lib
    return _lib.is_first_accumulate(pair.op._step if pair.op._sched_state is None else pair.op._cursor.step, pair.N)


POISON = (False, True)


@pytest.mark.parametrize("N", [2, 3, 4, 8])
def test_clip_apply_matches_the_zero_storing_twin(N):
    for poison in POISON:
        p = Pair(N, seed=N, poison=poison)
        assert p.run_windows(3) == 3
        p.check("end", accum=True)


@pytest.mark.parametrize("read", [False, True])
def test_single_pass_apply_and_reads_right_after_an_apply(read):
    """AdamWeightDecay without clipping (apply_kernel); ``read``: the accumulators are also read right after every
    apply, which stores the zeros there and leaves the first accumulate none to store."""
    from gaccum_b200 import _lib
    hp = _lib.HParams.bert()
    hp.clip_norm = 0.0
    for poison in POISON:
        p = Pair(3, hp=hp, seed=11, poison=poison)
        p.run_windows(3, read_every_step=read)


def test_tf_adam_and_lamb():
    from gaccum_b200 import _lib
    hp = _lib.HParams.lamb()
    hp.clip_norm = 0.0
    for poison in POISON:
        Pair(4, hp=_lib.HParams.tf_adam(), seed=5, poison=poison).run_windows(2)
        Pair(3, hp=_lib.HParams.lamb(), seed=6, poison=poison).run_windows(3)
        Pair(2, hp=hp, seed=7, poison=poison).run_windows(3)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_16_bit_models(dtype):
    for poison in POISON:
        Pair(3, dtype=dtype, seed=8, poison=poison).run_windows(3)


@pytest.mark.parametrize("clip", [1.0, 0.0])
def test_loss_scale_skips(clip):
    """An overflowed window is skipped on the device: the accumulators are logically zero after it all the same."""
    from gaccum_b200 import _lib
    hp = _lib.HParams.bert()
    hp.clip_norm = clip
    for poison in POISON:
        p = Pair(3, hp=hp, seed=9, loss_scale=_lib.LossScaleConfig(2.0 ** 8, 2.0, 2), poison=poison)
        p.run_windows(1)
        p.step(); p.step(inf_at=0); p.step()             # the whole window is skipped
        assert p.op.loss_scale_state()["last_skipped"]
        p.check("skipped window")
        p.run_windows(2)
        assert p.op.loss_scale_state() == p.twin.loss_scale_state()


def test_ema_and_lamb_with_ema():
    from gaccum_b200 import _lib
    for poison in POISON:
        Pair(3, seed=12, ema=_lib.EmaConfig(0.99, True), poison=poison).run_windows(3)
        Pair(2, hp=_lib.HParams.lamb(), seed=13, ema=_lib.EmaConfig(0.9), poison=poison).run_windows(2)


def test_device_schedule_with_refused_launches():
    from gaccum_b200 import _lib
    cfg = _lib.ScheduleConfig(1e-3, 1000, 5)
    for poison in POISON:
        p = Pair(3, seed=14, device_schedule=cfg, poison=poison)
        p.run_windows(2)
        # right after an apply, an apply launched out of place (device at 7); then, mid-window, a first accumulate
        # launched one step late (device at 11)
        for extra, wrong in ((0, 9), (1, 10)):
            for _ in range(extra):
                p.step()
            g = p.op._cursor.step
            for op in (p.op, p.twin):
                args = _lib.StepArgs(wrong, 3, 0, 0.0, 0.0, 0.0, 0.0)
                op.plan.step(op._grad_table(p.grads()), op._param_ptrs, op._accum_ptr, op._m_ptr, op._v_ptr, args,
                             op._stream())
            torch.cuda.synchronize()
            assert p.op._read_schedule()["refused"] and p.twin._read_schedule()["refused"]
            p.check(f"refused launch at {wrong}, device at {g}", accum=True)
            for op in (p.op, p.twin):
                op.global_step = g                       # the documented recovery
            p.run_windows(1)
        p.check("end", accum=True)


def test_branches_alone_and_global_step_reassignment():
    for poison in POISON:
        p = Pair(3, seed=15, poison=poison)
        p.run_windows(1)                                 # an apply just ran: the accumulators are logically zero
        g = p.grads()
        for op in (p.op, p.twin):
            op.accumulate_only(g)
        p.check("accumulate_only after an apply", accum=True)
        p.run_windows(1)
        g = p.grads()
        for op in (p.op, p.twin):
            op.apply_only(g)                             # right after an apply
        p.after_apply()
        p.check("apply_only after an apply")
        p.run_windows(1)
        for op in (p.op, p.twin):
            op.apply_only(None)
        p.after_apply()
        p.run_windows(1)
        assert p.op.global_step == 13                    # right after the apply at 12
        # mid-window (reads the accumulators); unchanged, an apply; an apply after an apply; unchanged, a first
        # accumulate
        for g_new in (14, 15, 18, 19):
            for op in (p.op, p.twin):
                op.global_step = g_new
            p.step()
            p.check(f"global_step = {g_new}", accum=not _next_is_first(p))
        p.run_windows(2)


@pytest.mark.parametrize("where", ["mid_window", "after_apply"])
def test_checkpoint_round_trip(where):
    for poison in POISON:
        p = Pair(4, seed=16, poison=poison)
        p.run_windows(1)
        if where == "mid_window":
            p.step(); p.step()
        sd_a, sd_b = p.op.state_dict(), p.twin.state_dict()
        for k in sd_b:
            _same(sd_a[k], sd_b[k], f"state_dict {k}")
        # both restored into fresh ops whose slabs hold other values; the deferred one restores at a step right after
        # one of its own applies
        fresh = Pair(4, seed=17, poison=poison)
        fresh.run_windows(1)
        fresh.op.load_state_dict(sd_a)
        fresh.twin.load_state_dict(sd_b)
        fresh.gen, fresh.i, fresh.windows = p.gen, p.i, p.windows
        fresh.check("restored", accum=True)
        fresh.run_windows(2)
        assert fresh.op.global_step == fresh.twin.global_step


def test_data_parallel_driver_on_one_rank():
    from gaccum_b200.distributed import DataParallelTrainOp
    for poison in POISON:
        p = Pair(3, seed=18, poison=poison)
        dp, dt = DataParallelTrainOp(p.op, None), DataParallelTrainOp(p.twin, None)
        assert p.op._deferred                            # one rank: the driver delegates to the engine
        for _ in range(7):
            g = p.grads()
            a = dp.run(g)
            assert a == dt.run(g)
            p.i += 1
            if a:
                p.after_apply()
            p.check(f"dp step {p.i}", accum=not _next_is_first(p))
        sa, sb = dp.state_dict(), dt.state_dict()
        for k in sb:
            _same(sa[k], sb[k], f"dp state_dict {k}")


def test_a_plan_without_the_mode_stores_zeros_and_one_with_it_does_not():
    """The raw slabs right after an apply (the plan's own pointer, read without materializing): the zero-storing twin
    holds +0.0 everywhere; the deferred op, whose single-pass apply does not write the slab, still holds the window's
    sums.  Reading ``accum`` then stores the zeros."""
    from gaccum_b200 import _lib
    hp = _lib.HParams.bert()
    hp.clip_norm = 0.0
    p = Pair(2, hp=hp, seed=19)
    p.step()
    assert p.step()
    torch.cuda.synchronize()
    assert not bool(p.twin._accum.view(torch.int32).any())
    assert bool(p.op._accum.view(torch.int32).any())
    assert not bool(p.op.accum.view(torch.int32).any())
    assert not bool(p.op._accum.view(torch.int32).any())
    # the host-buffer session, which keeps its slabs to itself, refuses a plan with the mode
    with pytest.raises(_lib.GaccumError, match="deferred reset"):
        _lib.HostSession(p.op.plan)


def test_the_packed_entry_point_keeps_storing_zeros_on_a_deferred_plan():
    """gaccum_step_packed ignores the mode: its own slab (here beside the op's) gets the zeros from its applies."""
    from gaccum_b200 import _lib
    p = Pair(2, seed=20, poison=True)
    plan, n = p.op.plan, p.op.plan.padded_size
    slabs = [torch.zeros(n, device="cuda") for _ in range(4)]
    gslab = torch.randn(n, device="cuda", generator=p.gen) * 0.05
    stream = torch.cuda.current_stream().cuda_stream
    for g in (1, 2):                                     # accumulate, then apply
        plan.step_packed(gslab.data_ptr(), *(s.data_ptr() for s in slabs[:2]), slabs[2].data_ptr(), slabs[3].data_ptr(),
                         _lib.StepArgs(g, 2, 0, 1e-3, 0.9, 0.999, 0.0), -1, stream)
    torch.cuda.synchronize()
    assert bool(slabs[0].view(torch.int32).any()) and not bool(slabs[1].view(torch.int32).any())
    p.run_windows(2)
