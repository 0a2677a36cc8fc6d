"""Every apply-kernel instantiation against the composed oracle (tests/apply_matrix.py).

One case per dispatch key of gaccum_abi.cu: optimizer (AdamWeightDecay, Adam, LAMB) x mode (no clip, clip, loss scaling
without and with clip) x with gradients (``run``) or without (``accumulate_only`` + ``apply_only(None)``) x layout and
dtype (packed CAP 0 fp32; CAP 256 and 1920 in fp32, bf16, fp16) x EMA off / on -- 336 cases, which between them launch
each of the library's 120 apply instantiations (tests/test_kernel_inventory.py checks that mapping against the binary).

Each case trains a small model with tails, a multi-tile tensor, one element, a tensor without a gradient and a
zero-element tensor (CAP 1920: plus 300 tiny tensors) at N = 3 for ten micro-steps -- four applied windows.  Loss-scaled
cases put one inf into a gradient in the middle of the third window, which is skipped; S grows once before that.  The
train op and the oracle are compared after every micro-step (``LockStep.check``).

The 288 table-layout keys also run with the deferred reset as a training loop runs it (``reset="deferred"``: no
materialize, the raw accumulators poisoned after every apply, so every first accumulate finds a poisoned slab and a
tensor without a gradient); those with gradients also run with the mode off (``reset="stored"``: the applies store
+0.0).
"""
import zlib

import pytest

from apply_matrix import RESETS, Case, LockStep, matrix_cases

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

MAN = [("a/kernel", (2 * 2048 + 777,)), ("a/bias", (5,)), ("one/kernel", (1,)), ("empty/kernel", (0,)),
       ("LayerNorm/gamma", (33,)), ("nograd/kernel", (64,)), ("t/kernel", (3, 1367))]
NOGRAD = (5,)
TINY = [(f"tiny{i}/{'bias' if i % 3 == 0 else 'kernel'}", (1 + i % 7,)) for i in range(300)]
STEPS = 10                         # N = 3: windows applied at steps 0, 3, 6 and 9
INF_AT = (4, 0, 1000)              # loss-scaled: the window applied at step 6 overflows
EMA = (0.9, True)                  # num_updates mode: the first window averages with d = min(0.9, 1/10)


def _man(layout):
    return MAN + TINY if layout.startswith("t1920") else MAN


def reset_cases():
    """Every dispatch key with the accumulators read after every micro-step ("materialized"); every table-layout key
    (the packed entry point ignores the mode) with the deferred reset as training runs it; and, with the mode off,
    those with gradients (without, the applies launch the same kernels)."""
    return [pytest.param(c, r, id=c.id if r == "materialized" else f"{c.id}-{r}") for r in RESETS for c in matrix_cases()
            if r == "materialized" or (c.layout != "packed" and (r == "deferred" or c.has_g))]


@pytest.mark.parametrize("case, reset", reset_cases())
def test_apply_instantiation_matches_the_oracle(case: Case, reset):
    layout = "packed" if case.layout == "packed" else "table"
    dtype = case.layout.split("_")[-1] if layout == "table" else "fp32"
    run = LockStep(_man(case.layout), case.variant, case.mode, layout, dtype, case.has_g, EMA if case.ema else None,
                   N=3, seed=zlib.crc32(case.id.encode()), nograd=NOGRAD, reset=reset)
    assert run.cap == {"packed": 0, "table": 256 if case.layout.startswith("t256") else 1920}[layout]
    ls = case.mode.startswith("ls_")
    run.run(STEPS, inf_at=INF_AT if ls else None)
    if ls:
        st = run.op.loss_scale_state()
        assert st["skipped_windows"] == 1 and not st["last_skipped"] and st["scale"] == 16.0   # grew to 32, halved once
    if case.ema:
        assert run.op.ema_state()["num_updates"] == (3 if ls else 4)
    if reset == "deferred":
        assert run.first_over_poison == 3          # after the applies at steps 0, 3 and 6
    run.finish()


def test_reset_case_count():
    assert len(reset_cases()) == 336 + 288 + 144


@pytest.mark.parametrize("num_updates", [False, True])
@pytest.mark.parametrize("decay", [0.0, 1.0])
@pytest.mark.parametrize("kernel", ["apply", "clip_apply", "lamb"])
def test_ema_decay_edges(kernel, decay, num_updates):
    """decay 0 (the average is the weights), decay 1 (it never moves, unless num_updates caps d) on each apply kernel."""
    variant, mode = {"apply": ("adamw", "noclip"), "clip_apply": ("adamw", "clip"), "lamb": ("lamb", "clip")}[kernel]
    run = LockStep(MAN, variant, mode, ema=(decay, num_updates), N=2, seed=7, nograd=NOGRAD)
    start = [x.copy() for x in run.tracker.avg]
    run.run(5)
    if decay == 1.0 and not num_updates:
        for x, y in zip(run.tracker.avg, start):
            assert (x.view("u4") == y.view("u4")).all()
