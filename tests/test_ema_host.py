"""The exponential moving average without a GPU: the oracle's decay rule against known answers, the C ABI's setter
checks, its refusals and byte counts on layout-only plans, the Python front ends' refusals and the checkpoint names."""
import ctypes as C
import itertools

import numpy as np
import pytest

from ema_oracle import Ema, ema_coefficients, ema_update

F32 = np.float32


# ---- oracle known answers ------------------------------------------------------------------------------------------
def test_c_of_a_constant_decay_is_the_fp32_subtraction():
    d, c = ema_coefficients(0.9999, False, 12345)
    assert d == F32(0.9999) and c == F32(1.0) - F32(0.9999)
    # 1 - fp32(0.9999) is exact (Sterbenz) but fp32(0.9999) is not 0.9999: c is 1.66e-4 relatively off 1 - 0.9999
    assert float(c) == 1.0 - float(F32(0.9999))
    assert abs(float(c) - (1.0 - 0.9999)) / (1.0 - 0.9999) == pytest.approx(1.659e-4, rel=1e-3)


@pytest.mark.parametrize("n, expected_d", [(0, F32(1.0) / F32(10.0)), (1, F32(2.0) / F32(11.0)), (9, F32(10.0) / F32(19.0))])
def test_num_updates_warm_up(n, expected_d):
    d, c = ema_coefficients(0.9999, True, n)
    assert d == expected_d and c == F32(1.0) - expected_d
    assert d == F32(np.float32(1 + n) / np.float32(10 + n))
    # far from the start the warm-up bound exceeds the decay: d is the decay
    assert ema_coefficients(0.9, True, 10 ** 6)[0] == F32(0.9)


def test_counter_past_2_24_rounds_to_nearest():
    n = 2 ** 24 + 1
    assert F32(n) == F32(2 ** 24)                                         # the cast TF takes rounds
    d, _ = ema_coefficients(1.0, True, n)
    nf = F32(2 ** 24)
    assert d == np.divide(np.add(F32(1), nf, dtype=F32), np.add(F32(10), nf, dtype=F32), dtype=F32)
    assert d == ema_coefficients(1.0, True, 2 ** 24)[0]                  # n and n - 1 share one fp32 value
    assert F32(1) + nf == nf                                              # 1 + 2^24 rounds back to 2^24 (to even)


def test_update_is_three_rounded_ops_and_fixed_points():
    rng = np.random.default_rng(0)
    e, p = rng.normal(0, 1, 1000).astype(F32), rng.normal(0, 1, 1000).astype(F32)
    c = F32(0.1)
    got = ema_update(e, p, c)
    exp = [F32(F32(x) - F32(F32(F32(x) - F32(y)) * c)) for x, y in zip(e, p)]
    assert np.array_equal(got.view(np.uint32), np.array(exp, F32).view(np.uint32))
    assert np.array_equal(ema_update(p, p, c), p)                         # e == p stays
    assert np.array_equal(ema_update(e, p, F32(0.0)), e)                  # decay 1: the average never moves
    # decay 0: the average is p up to the rounding of e - (e - p), which TF's op order keeps
    np.testing.assert_allclose(ema_update(e, p, F32(1.0)), p, rtol=0, atol=4 * np.finfo(F32).eps)


def test_ema_state_advances_once_per_average():
    ema = Ema([np.zeros(3, F32)], 0.5, True)
    for k in range(3):
        ema.average([np.ones(3, F32)])
    assert ema.num_updates == 3 and ema.decay == ema_coefficients(0.5, True, 2)[0]
    # d_0 = 0.1, d_1 = 2/11, d_2 = 0.25: e = 1 - prod(d)
    np.testing.assert_allclose(ema.avg[0], 1.0 - 0.1 * (2 / 11) * 0.25, rtol=1e-6)


# ---- the C ABI on layout-only plans --------------------------------------------------------------------------------
def _L():
    from gaccum_b200 import _lib
    return _lib, _lib._load()


def _plan(variant=0):
    import gaccum_b200 as g
    hp = g.HParams(variant, 0, 0.9, 0.999, 1e-6, 0.01, 1.0)
    return g.Plan([1000, 37, 5], [True, False, True], hp, device=-1)


SLAB, STATE = 0x10000, 0x20000          # 16-byte aligned addresses: the setters only check and keep them


def _set_ema(plan, decay=0.9999, num_updates=0, reserved=0, slab=SLAB, state=STATE):
    lib, L = _L()
    cfg = lib.EmaConfig(decay, num_updates, reserved)
    return L.gaccum_plan_set_ema(plan._h, C.byref(cfg), slab, state)


def test_setter_validates_its_arguments():
    lib, L = _L()
    plan = _plan()
    for kw in (dict(decay=-0.1), dict(decay=1.5), dict(decay=float("nan")), dict(num_updates=2), dict(reserved=1),
               dict(slab=None), dict(slab=SLAB + 4), dict(state=None), dict(state=STATE + 8)):
        assert _set_ema(plan, **kw) == lib.EINVAL, kw
    assert L.gaccum_plan_set_ema(plan._h, None, SLAB, STATE) == lib.EINVAL
    for decay in (0.0, 1.0, 0.9999):
        assert _set_ema(plan, decay=decay) == 0
    assert _set_ema(plan, num_updates=1) == 0


def test_ema_init_checks():
    lib, L = _L()
    plan = _plan()
    assert L.gaccum_ema_init(plan._h, STATE, 0, None) == lib.EINVAL                  # no EMA on this plan
    assert _set_ema(plan) == 0
    assert L.gaccum_ema_init(plan._h, STATE + 4, 0, None) == lib.EINVAL
    assert L.gaccum_ema_init(plan._h, STATE + 16, 0, None) == lib.EINVAL            # not the block the apply reads
    assert "gaccum_plan_set_ema" in L.gaccum_last_error().decode()
    assert L.gaccum_ema_init(plan._h, None, 0, None) == lib.EINVAL
    assert L.gaccum_ema_init(plan._h, STATE, -1, None) == lib.EINVAL
    assert L.gaccum_ema_init(plan._h, STATE, 5, None) == lib.ENODEVICE              # layout-only plan


def test_setter_is_refused_after_a_compute_call():
    lib, L = _L()
    plan = _plan()
    args = lib.StepArgs(0, 1, 0, 1e-3, 0.9, 0.999, 0.0)
    assert L.gaccum_apply(plan._h, None, None, None, None, None, C.byref(args), None) != 0   # counts as a compute call
    assert _set_ema(plan) == lib.EINVAL
    assert "before the plan's first compute call" in lib._load().gaccum_last_error().decode()


@pytest.mark.parametrize("order", list(itertools.permutations(["ema", "dtype", "loss_scale", "adapt"])))
def test_setters_combine_in_any_order(order):
    lib, L = _L()
    plan = _plan(variant=2)
    calls = {
        "ema": lambda: _set_ema(plan),
        "dtype": lambda: L.gaccum_plan_set_param_dtype(plan._h, lib.DTYPE_BF16, 0x30000),
        "loss_scale": lambda: L.gaccum_plan_set_loss_scale(plan._h, C.byref(lib.LossScaleConfig()), 0x40000),
        "adapt": lambda: L.gaccum_plan_set_layer_adaptation(plan._h, C.cast((C.c_uint8 * 3)(1, 0, 1), C.c_void_p)),
    }
    for what in order:
        assert calls[what]() == 0, what
    assert plan.algorithmic_bytes(True) == 56 * plan.num_elements


@pytest.mark.parametrize("variant, plain, with_ema", [(0, 36, 44), (1, 36, 44), (2, 48, 56)])
@pytest.mark.parametrize("half", [False, True])
def test_algorithmic_bytes(variant, plain, with_ema, half):
    lib, L = _L()
    plan = _plan(variant)
    if half:
        assert L.gaccum_plan_set_param_dtype(plan._h, lib.DTYPE_F16, 0x30000) == 0
    P = plan.num_elements
    acc = plan.algorithmic_bytes(False)
    assert plan.algorithmic_bytes(True) == plain * P
    assert _set_ema(plan) == 0
    assert plan.algorithmic_bytes(True) == with_ema * P
    assert plan.algorithmic_bytes(False) == acc                                     # accumulate steps do not touch it


def test_data_parallel_and_host_session_refuse_an_ema_plan():
    lib, L = _L()
    plan = _plan()
    assert _set_ema(plan) == 0
    comm = lib.DpComm()
    comm.world = 2
    args = lib.StepArgs(0, 1, 0, 1e-3, 0.9, 0.999, 0.0)
    for fn in (L.gaccum_step_dp, L.gaccum_apply_dp):
        assert fn(plan._h, C.byref(comm), None, None, None, C.byref(args), 1, None) == lib.EINVAL
        assert "moving average" in L.gaccum_last_error().decode()
    h = C.c_void_p()
    assert L.gaccum_host_session_create(C.byref(h), plan._h) == lib.EINVAL
    assert "moving average" in L.gaccum_last_error().decode()


def test_python_front_ends_refuse_an_ema():
    import torch
    import gaccum_b200 as g
    from gaccum_b200.distributed import FusedDataParallelTrainOp
    from gaccum_b200.train_op import HostTrainOp
    with pytest.raises(ValueError, match="moving average"):
        HostTrainOp([torch.zeros(4)], ["w"], g.HParams.bert(), 2, lambda s: 1e-3, ema=g.EmaConfig(0.99))
    with pytest.raises(ValueError, match="moving average"):
        FusedDataParallelTrainOp([torch.zeros(4)], ["w"], g.HParams.bert(), 2, lambda s: 1e-3, ema=g.EmaConfig(0.99))


def test_exponential_moving_average_mirror():
    from gaccum_b200 import graph, optimization as opt
    import torch
    graph.reset_default_graph()
    v = graph.add_variable("bert/pooler/dense/kernel:0", torch.zeros(3))
    ema = opt.ExponentialMovingAverage(0.999, num_updates=True)
    cfg = ema.config()
    assert cfg.decay == 0.999 and cfg.num_updates == 1 and cfg.reserved == 0
    assert ema.average_name(v) == "bert/pooler/dense/kernel/ExponentialMovingAverage"
    assert ema.variables_to_restore() == {"bert/pooler/dense/kernel/ExponentialMovingAverage": v}
    with pytest.raises(ValueError):
        ema.average(v)
    assert opt.moving_average_decay is None


# ---- checkpoint names ----------------------------------------------------------------------------------------------
def test_tf_checkpoint_name_round_trip(tmp_path):
    import torch
    from gaccum_b200 import tf_checkpoint as tc
    names = ["a/kernel", "b/bias"]
    rng = np.random.default_rng(1)
    state = {"global_step": torch.tensor(7)}
    for n, s in zip(names, [(3, 4), (5,)]):
        for suffix in ("", "/adam_m", "/adam_v", "/accum_grad", "/ExponentialMovingAverage"):
            state[n + suffix] = torch.from_numpy(rng.normal(0, 1, s).astype(F32))
    state["ExponentialMovingAverage/num_updates"] = torch.tensor(3, dtype=torch.int64)
    ref = tc.to_reference_names(state, names, tc.ADAM_WEIGHT_DECAY)
    assert "a/kernel/ExponentialMovingAverage" in ref and int(ref["ExponentialMovingAverage/num_updates"]) == 3
    tc.write_bundle(str(tmp_path / "m.ckpt-7"), ref)
    back = tc.from_reference_names(tc.read_bundle(str(tmp_path / "m.ckpt-7")), names, tc.ADAM_WEIGHT_DECAY, ema=True)
    for k, x in state.items():
        assert np.array_equal(np.asarray(back[k]), x.numpy()), k
    # a checkpoint without averages: required in strict mode by a train op that keeps them, ignored otherwise
    plain = {k: v for k, v in ref.items() if "ExponentialMovingAverage" not in k}
    with pytest.raises(KeyError, match="ExponentialMovingAverage"):
        tc.from_reference_names(plain, names, tc.ADAM_WEIGHT_DECAY, ema=True)
    assert "ExponentialMovingAverage/num_updates" not in tc.from_reference_names(plain, names, tc.ADAM_WEIGHT_DECAY)
    assert "ExponentialMovingAverage/num_updates" not in tc.to_reference_names(
        {k: v for k, v in state.items() if "ExponentialMovingAverage" not in k}, names, tc.ADAM_WEIGHT_DECAY)
