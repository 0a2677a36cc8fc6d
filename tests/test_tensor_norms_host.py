"""Per-tensor norms without a GPU: the C setter's checks, the refusals of the Python front ends that do not support the
option, and the oracle's known answers.  The checks that need a device plan (the setter after a compute call, the
setters in every order, the C refusals and the byte counts of a plan with norms) are in tests/test_gpu_tensor_norms.py."""
import ctypes as C
import itertools

import numpy as np
import pytest

from tensor_norms_oracle import assert_close, expected_norms, norm, window_gradient

F32 = np.float32
BUF = 0x60000       # a 16-byte aligned address: a layout-only plan is refused before the pointer could be used


def _L():
    from gaccum_b200 import _lib
    return _lib, _lib._load()


def _plan(variant=0):
    import gaccum_b200 as g
    hp = g.HParams(variant, 0, 0.9, 0.999, 1e-6, 0.01, 1.0)
    return g.Plan([1000, 37, 5], [True, False, True], hp, device=-1)


# ---- the C ABI ---------------------------------------------------------------------------------------------------
def test_setter_refuses_a_null_plan():
    lib, L = _L()
    assert L.gaccum_plan_set_tensor_norms(None, BUF) == lib.EINVAL
    assert "plan is NULL" in L.gaccum_last_error().decode()


@pytest.mark.parametrize("bad", [None, BUF + 4, BUF + 8, BUF + 1])
def test_setter_refuses_null_and_misaligned_buffers(bad):
    lib, L = _L()
    assert L.gaccum_plan_set_tensor_norms(_plan()._h, bad) == lib.EINVAL
    assert "16-byte aligned" in L.gaccum_last_error().decode()


@pytest.mark.parametrize("variant", [0, 1, 2])
def test_setter_refuses_a_layout_only_plan(variant):
    lib, L = _L()
    assert L.gaccum_plan_set_tensor_norms(_plan(variant)._h, BUF) == lib.EINVAL
    assert "layout-only" in L.gaccum_last_error().decode()


@pytest.mark.parametrize("order", list(itertools.permutations(["ww", "lr_mult", "ema", "dtype", "loss_scale", "adapt"])))
def test_other_setters_in_any_order_leave_the_refusal_and_the_bytes(order):
    """Whatever the other setters did first, a layout-only plan still refuses the norms, and the byte count is the one
    the other settings give."""
    lib, L = _L()
    plan = _plan(variant=2)
    calls = {
        "ww": lambda: L.gaccum_plan_set_window_weight(plan._h, 0x50000),
        "lr_mult": lambda: L.gaccum_plan_set_lr_multipliers(plan._h, C.cast((C.c_float * 3)(0.5, 0.0, 2.0), C.c_void_p)),
        "ema": lambda: L.gaccum_plan_set_ema(plan._h, C.byref(lib.EmaConfig(0.999)), 0x10000, 0x20000),
        "dtype": lambda: L.gaccum_plan_set_param_dtype(plan._h, lib.DTYPE_BF16, 0x30000),
        "loss_scale": lambda: L.gaccum_plan_set_loss_scale(plan._h, C.byref(lib.LossScaleConfig()), 0x40000),
        "adapt": lambda: L.gaccum_plan_set_layer_adaptation(plan._h, C.cast((C.c_uint8 * 3)(1, 0, 1), C.c_void_p)),
    }
    for what in order:
        assert calls[what]() == 0, what
    assert L.gaccum_plan_set_tensor_norms(plan._h, BUF) == lib.EINVAL
    assert plan.algorithmic_bytes(True) == 56 * plan.num_elements
    assert plan.algorithmic_bytes(False) == 10 * plan.num_elements


def test_python_binding_raises():
    lib, _ = _L()
    with pytest.raises(lib.GaccumError):
        _plan().set_tensor_norms(BUF)


# ---- Python front ends that refuse the option (before touching a device) -----------------------------------------
def test_host_train_op_refuses_tensor_norms():
    import torch
    import gaccum_b200 as g
    from gaccum_b200.train_op import HostTrainOp
    with pytest.raises(ValueError, match="per-tensor norms"):
        HostTrainOp([torch.zeros(4)], ["w"], g.HParams.bert(), 2, lambda s: 1e-3, tensor_norms=True)


def test_fused_data_parallel_train_op_refuses_tensor_norms():
    import torch
    import gaccum_b200 as g
    from gaccum_b200.distributed import FusedDataParallelTrainOp
    with pytest.raises(ValueError, match="per-tensor norms"):
        FusedDataParallelTrainOp([torch.zeros(4)], ["w"], g.HParams.bert(), 2, lambda s: 1e-3, tensor_norms=True)


def test_optimization_forwards_the_option():
    import inspect
    from gaccum_b200 import optimization as opt
    assert opt.tensor_norms is False
    assert inspect.signature(opt.gradient_accumulation_train_op).parameters["tensor_norms"].default is False


# ---- the oracle's known answers ------------------------------------------------------------------------------------
def test_norm_of_a_hand_computed_tensor():
    assert norm(np.array([3.0, 4.0], F32)) == F32(5.0)
    assert norm(np.array([1.0, 2.0, 2.0], F32)) == F32(3.0)
    assert norm(np.array([], F32)) == F32(0.0)


def test_inf_and_nan_propagate():
    assert np.isposinf(norm(np.array([1.0, np.inf, 2.0], F32)))
    assert np.isposinf(norm(np.array([-np.inf], F32)))
    assert np.isnan(norm(np.array([1.0, np.nan], F32)))
    assert np.isnan(norm(np.array([np.inf, np.nan], F32)))


def test_sum_overflowing_fp32_reports_inf():
    # each square fits fp64; the fp64 sum rounded to fp32 does not
    assert np.isposinf(norm(np.array([3e19, 3e19], F32)))


def test_window_gradient_divides_then_unscales():
    a = np.array([6.0, -3.0], F32)
    g = np.array([2.0, 1.0], F32)
    assert np.array_equal(window_gradient(a, g, 4.0), np.array([2.0, -0.5], F32))
    assert np.array_equal(window_gradient(a, None, 3.0, scale=2.0), np.array([1.0, -0.5], F32))
    # W that is not a power of two: the correctly rounded fp32 quotient
    assert window_gradient(np.array([1.0], F32), None, 3.0)[0] == F32(1.0) / F32(3.0)


def test_expected_norms_of_a_small_model():
    accum = [np.array([6.0, 8.0], F32), np.array([], F32), np.array([1.0], F32)]
    grads = [np.array([0.0, 0.0], F32), None, np.array([1.0], F32)]
    before = [np.array([3.0, 4.0], F32), np.array([], F32), np.array([2.0], F32)]
    after = [np.array([3.0, 4.0], F32), np.array([], F32), np.array([1.5], F32)]   # tensor 0: multiplier 0
    got = expected_norms(accum, grads, 2.0, None, before, after)
    assert_close(got, np.array([[5.0, 5.0, 0.0], [0.0, 0.0, 0.0], [1.0, 2.0, 0.5]], F32))
    # a skipped window: the overflowed tensor's gradient is inf, the updates are 0
    accum[2] = np.array([np.inf], F32)
    got = expected_norms(accum, grads, 2.0, 4.0, before, before)
    assert np.isposinf(got[2, 0]) and got[0, 0] == F32(1.25) and not got[:, 2].any()


def test_assert_close_is_strict_about_classes():
    assert_close(np.array([1.0, np.inf, np.nan], F32), np.array([1.0 + 1e-7, np.inf, np.nan], F32))
    with pytest.raises(AssertionError):
        assert_close(np.array([np.inf], F32), np.array([np.nan], F32))
    with pytest.raises(AssertionError):
        assert_close(np.array([1.0], F32), np.array([1.00001], F32))
    with pytest.raises(AssertionError):
        assert_close(np.array([1e-30], F32), np.array([0.0], F32))
