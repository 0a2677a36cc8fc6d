"""Dynamic loss scaling without a GPU: the loss-scaled oracle's known answers, its S sequence against PyTorch's
``_amp_update_scale_``, its bit-identity with the unscaled oracle, and the C ABI's argument checks on a layout-only
plan."""
import ctypes as C

import numpy as np
import pytest

import oracle_np as onp
from composed_oracle import ComposedReferenceTrainOp, update_scale

MAN = [("a/kernel", (37, 5)), ("a/bias", (5,)), ("LayerNorm/gamma", (9,)), ("emb", (300,))]
F32 = np.float32


def _params(seed):
    rng = np.random.default_rng(seed)
    return [rng.normal(0, 0.05, s).astype(F32) for _, s in MAN]


def _grads(rng, sigma=0.1):
    return [rng.normal(0, sigma, s).astype(F32) for _, s in MAN]


def _hp(variant_b, clip):
    hp = onp.HParams.tf_adam() if variant_b else onp.HParams.bert()
    hp.clip_norm = clip
    return hp


def _ls_op(hp, N, **kw):
    return ComposedReferenceTrainOp(_params(1), [n for n, _ in MAN], hp, N, constant_lr=1e-3, **kw)


@pytest.mark.parametrize("bad", [np.inf, -np.inf, np.nan, "finite"])
@pytest.mark.parametrize("at", ["first", "middle", "last"])
def test_overflowed_window_leaves_state_and_backs_off(at, bad):
    N = 3
    op = _ls_op(_hp(True, 0.0), N, initial_scale=2.0 ** 10, growth_interval=100)
    rng = np.random.default_rng(3)
    for _ in range(N + 1):                      # two applied windows (g = 0 and g = 1..3), then the window under test
        op.run([x * op.scale for x in _grads(rng)])
    p0, m0, v0 = ([x.copy() for x in op.params], [x.copy() for x in op.m], [x.copy() for x in op.v])
    b0 = (op.beta1_power, op.beta2_power)
    assert (op.scale, op.good_windows) == (F32(2.0 ** 10), 2)
    k = {"first": 0, "middle": 1, "last": 2}[at]             # index in the window g = 4, 5, 6
    other = k + 1 if k < N - 1 else k - 1
    for j in range(N):
        gr = [x * op.scale for x in _grads(rng)]
        if bad == "finite":
            if j in (k, other):
                gr[3][7] = F32(3.0e38)          # finite gradients whose sum overflows fp32
        elif j == k:
            gr[3][5] = F32(bad)
        with np.errstate(over="ignore", invalid="ignore"):
            info = op.run(gr)
    assert info.applied and op.last_skipped
    for got, exp in zip(op.params + op.m + op.v, p0 + m0 + v0):
        assert np.array_equal(got.view(np.uint32), exp.view(np.uint32))
    assert all(not np.any(a.view(np.uint32)) for a in op.accum)
    assert (op.scale, op.good_windows, op.skipped_windows) == (F32(2.0 ** 9), 0, 1)
    assert (op.beta1_power, op.beta2_power) == b0


def test_scale_grows_after_growth_interval_and_is_bounded():
    op = _ls_op(_hp(False, 1.0), 1, initial_scale=4.0, growth_interval=3)
    rng = np.random.default_rng(4)
    seen = []
    for _ in range(7):
        op.run([x * op.scale for x in _grads(rng)])
        seen.append((float(op.scale), op.good_windows))
    assert seen == [(4, 1), (4, 2), (8, 0), (8, 1), (8, 2), (16, 0), (16, 1)]
    assert update_scale(F32(1.0), 5, True, 2.0, 10) == (F32(1.0), 0)              # floor at 1
    assert update_scale(F32(2.0), 5, True, 4.0, 10) == (F32(1.0), 0)
    assert update_scale(F32(2.0 ** 127), 0, False, 2.0, 1) == (F32(2.0 ** 127), 0)   # never past 2^127
    assert update_scale(F32(2.0 ** 120), 0, False, 2.0 ** 10, 1) == (F32(2.0 ** 120), 0)


def test_scale_sequence_matches_torch_amp_update_scale():
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(8)
    for interval in (1, 2, 5):
        s, good = F32(2.0 ** 40), 0
        ts = torch.tensor([2.0 ** 40], dtype=torch.float32)
        tracker = torch.zeros(1, dtype=torch.int32)
        for _ in range(200):
            inf = bool(rng.random() < 0.3) and s > 1.0     # patterns that stay above TF's floor, which torch lacks
            s, good = update_scale(s, good, inf, 2.0, interval)
            torch._amp_update_scale_(ts, tracker, torch.tensor([1.0 if inf else 0.0]), 2.0, 0.5, interval)
            assert s >= 1.0
            assert (float(s), good) == (float(ts[0]), int(tracker[0]))


@pytest.mark.parametrize("N", [1, 3, 4])
@pytest.mark.parametrize("clip", [0.0, 1.0, 1e-3])
@pytest.mark.parametrize("variant_b", [False, True])
def test_scaled_trajectory_is_bit_identical_to_unscaled(variant_b, clip, N):
    hp = _hp(variant_b, clip)
    ref = onp.ReferenceTrainOp(_params(1), [n for n, _ in MAN], hp, N, constant_lr=1e-3)
    ls = _ls_op(hp, N, initial_scale=2.0 ** 12, growth_interval=2)
    rng = np.random.default_rng(10 + N)
    scales = set()
    for _ in range(6 * N + 1):
        gr = _grads(rng)
        scales.add(float(ls.scale))
        a = ref.run(gr)
        b = ls.run([x * ls.scale for x in gr])
        assert (a.global_norm, a.clip_scale) == (b.global_norm, b.clip_scale)
    assert len(scales) > 1                               # the scale grew on the way
    for x, y in zip(ref.params + ref.m + ref.v + ref.accum, ls.params + ls.m + ls.v + ls.accum):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
    assert (ref.beta1_power, ref.beta2_power) == (ls.beta1_power, ls.beta2_power)


# ---- the C ABI on a layout-only plan ---------------------------------------------------------------------------
def _plan():
    import gaccum_b200 as g
    return g.Plan([10, 3000], None, g.HParams.bert(), device=-1)


def _set(plan, cfg, state=0x1000):
    from gaccum_b200 import _lib
    return _lib._load().gaccum_plan_set_loss_scale(plan._h, C.byref(cfg), state)


@pytest.mark.parametrize("cfg", [(3.0, 2.0, 10, 0), (0.5, 2.0, 10, 0), (2.0 ** 128, 2.0, 10, 0), (0.0, 2.0, 10, 0),
                                 (float("inf"), 2.0, 10, 0), (float("nan"), 2.0, 10, 0), (4.0, 1.0, 10, 0),
                                 (4.0, 3.0, 10, 0), (4.0, 2.0 ** 128, 10, 0), (4.0, 2.0, 0, 0), (4.0, 2.0, -1, 0),
                                 (4.0, 2.0, 10, 1)])
def test_bad_loss_scale_configs_are_rejected(cfg):
    from gaccum_b200 import _lib
    assert _set(_plan(), _lib.LossScaleConfig(*cfg)) == _lib.EINVAL


def test_good_configs_are_accepted_and_compute_still_needs_a_device():
    import gaccum_b200 as g
    from gaccum_b200 import _lib
    L = _lib._load()
    for cfg in ((1.0, 2.0, 1, 0), (2.0 ** 127, 2.0 ** 127, 2000, 0), (2.0 ** 24, 4.0, 7, 0)):
        plan = _plan()
        assert _set(plan, _lib.LossScaleConfig(*cfg)) == _lib.OK
        assert _set(plan, _lib.LossScaleConfig(*cfg), state=0) == _lib.EINVAL          # NULL state
        assert _set(plan, _lib.LossScaleConfig(*cfg), state=0x1004) == _lib.EINVAL     # not 16-byte aligned
        assert L.gaccum_loss_scale_init(plan._h, 0x1000, None) == _lib.ENODEVICE
        with pytest.raises(_lib.GaccumError) as e:
            plan.step_packed(0x1000, 0x1000, 0x1000, 0x1000, 0x1000, g.StepArgs(0, 1, 0, 1e-3, 0.9, 0.999, 0.0), 1)
        assert e.value.code == _lib.ENODEVICE
        # the compute call above counts: loss scaling can no longer be changed on this plan
        assert _set(plan, _lib.LossScaleConfig(*cfg)) == _lib.EINVAL
        assert "before the plan's first compute call" in L.gaccum_last_error().decode()


def test_loss_scale_init_needs_loss_scaling_on():
    from gaccum_b200 import _lib
    assert _lib._load().gaccum_loss_scale_init(_plan()._h, 0x1000, None) == _lib.EINVAL


def test_state_layout_matches_the_header():
    from gaccum_b200 import _lib
    assert C.sizeof(_lib.LossScaleState) == 32 and C.sizeof(_lib.LossScaleConfig) == 24
    assert [f for f, _ in _lib.LossScaleState._fields_] == ["scale", "good_windows", "skipped_windows", "last_skipped",
                                                           "beta1_power", "beta2_power", "reserved"]


def test_fused_data_parallel_and_host_train_ops_refuse_loss_scaling():
    torch = pytest.importorskip("torch")
    import gaccum_b200 as g
    from gaccum_b200.distributed import FusedDataParallelTrainOp
    from gaccum_b200.train_op import HostTrainOp
    p = [torch.zeros(4)]
    with pytest.raises(ValueError, match="loss scaling"):
        FusedDataParallelTrainOp(p, ["w"], g.HParams.bert(), 2, lambda s: 1e-3, loss_scale=g.LossScaleConfig())
    with pytest.raises(ValueError, match="loss scaling"):
        HostTrainOp(p, ["w"], g.HParams.bert(), 2, lambda s: 1e-3, loss_scale=g.LossScaleConfig())


def test_create_optimizer_reads_the_module_attribute():
    import inspect
    from gaccum_b200 import optimization
    assert optimization.loss_scale is None
    assert list(inspect.signature(optimization.create_optimizer).parameters) == \
        ["loss", "init_lr", "num_train_steps", "num_warmup_steps", "use_tpu"]
