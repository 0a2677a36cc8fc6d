"""The device schedule's host side (include/gaccum.h, gaccum_plan_set_device_schedule; no GPU needed).

The kernels evaluate create_optimizer's learning-rate schedule from the device counter (gaccum_kernels.cuh,
schedule_lr).  It is restated here op for op in numpy fp32 and compared bit for bit with the host schedule every
host-scheduled train op uses (``bert_learning_rate``, i.e. gaccum_learning_rate), over every step of the run and past
its end.  The ABI's validation and refusals need no device either.
"""
import ctypes as C

import numpy as np
import pytest

import gaccum_b200 as g
from gaccum_b200 import _lib as lib
from gaccum_b200.optimization import bert_learning_rate
from gaccum_b200.train_op import ScheduleLr

f32 = np.float32
BLOCK = 0x10000   # a 16-byte aligned address: the setter keeps it without dereferencing it


def kernel_lr(init_lr, T, W, step):
    """schedule_lr as the kernels evaluate it: every op one correctly rounded fp32 op, in TF's order."""
    lr0 = f32(init_lr)
    gs = f32(step)                       # int64 -> fp32, round to nearest
    ds = f32(T)
    if gs > ds:
        gs = ds
    with np.errstate(divide="ignore", invalid="ignore"):
        p = f32(gs / ds)
        lr = f32(lr0 * f32(f32(1.0) - p))
        if W != 0:
            gi, wi = np.int32(step), np.int32(W)
            pct = f32(f32(gi) / f32(wi))
            wlr = f32(lr0 * pct)
            isw = f32(1.0) if gi < wi else f32(0.0)
            lr = f32(f32(f32(f32(1.0) - isw) * lr) + f32(isw * wlr))
    return lr


@pytest.mark.parametrize("init_lr, T, W", [
    (2e-5, 2000, 200),       # BERT's 10 % warm-up
    (5e-5, 1000, 0),         # no warm-up
    (1e-2, 12, 3),
    (3e-4, 50, 50),          # warm-up == total
    (1e-3, 40, 64),          # warm-up longer than the run
    (1e-4, 1, 0),
    (0.1, 997, 13),          # lengths that are not powers of two
])
def test_kernel_schedule_matches_host_lr_fn_bitwise(init_lr, T, W):
    host = bert_learning_rate(init_lr, T, W)
    dev = ScheduleLr(lib.ScheduleConfig(init_lr, T, W))
    for step in range(T + 11):
        k = kernel_lr(init_lr, T, W, step)
        h = f32(host(step))
        assert k.view(np.uint32) == h.view(np.uint32), (step, k, h)
        assert f32(dev(step)).view(np.uint32) == h.view(np.uint32)


def test_block_layout():
    assert C.sizeof(lib.ScheduleState) == 48
    assert lib.ScheduleState.refused.offset == 44
    assert lib.ScheduleState.beta1_power.offset == 36
    assert C.sizeof(lib.ScheduleConfig) == 40


def _plan(variant=lib.ADAM_WEIGHT_DECAY):
    hp = lib.HParams(variant, 0, 0.9, 0.999, 1e-6, 0.01, 1.0)
    return lib.Plan([10, 20], [True, False], hp, device=-1)


def _set(plan, cfg, block=BLOCK):
    return lib._load().gaccum_plan_set_device_schedule(plan._h, C.byref(cfg), block)


def test_setter_validates_its_arguments():
    L = lib._load()
    plan = _plan()
    ok = lib.ScheduleConfig(1e-3, 100, 10)
    assert L.gaccum_plan_set_device_schedule(None, C.byref(ok), BLOCK) == lib.EINVAL
    assert L.gaccum_plan_set_device_schedule(plan._h, None, BLOCK) == lib.EINVAL
    assert _set(plan, ok, None) == lib.EINVAL
    assert _set(plan, ok, BLOCK + 4) == lib.EINVAL                  # not 16-byte aligned
    assert _set(plan, lib.ScheduleConfig(1e-3, 100, 10, end_lr=1e-5)) == lib.EINVAL
    assert b"end_lr must be 0" in L.gaccum_last_error()
    assert _set(plan, lib.ScheduleConfig(1e-3, 100, 10, power=2.0)) == lib.EINVAL
    assert _set(plan, lib.ScheduleConfig(1e-3, -1, 0)) == lib.EINVAL
    assert _set(plan, lib.ScheduleConfig(1e-3, 100, -5)) == lib.EINVAL
    assert _set(plan, lib.ScheduleConfig(float("nan"), 100, 5)) == lib.EINVAL
    assert _set(plan, ok) == lib.OK


def test_init_needs_the_plans_block_and_a_device():
    L = lib._load()
    plan = _plan()
    assert L.gaccum_schedule_init(plan._h, BLOCK, 0, 0.9, 0.999, None) == lib.EINVAL      # no schedule set
    assert _set(plan, lib.ScheduleConfig(1e-3, 100, 10)) == lib.OK
    assert L.gaccum_schedule_init(plan._h, BLOCK + 16, 0, 0.9, 0.999, None) == lib.EINVAL  # another block
    assert L.gaccum_schedule_init(plan._h, BLOCK, -1, 0.9, 0.999, None) == lib.EINVAL
    assert L.gaccum_schedule_init(plan._h, BLOCK, 0, 0.9, 0.999, None) == lib.ENODEVICE    # layout-only plan


@pytest.mark.parametrize("call", ["accumulate", "apply", "packed_forced", "host_session", "step_dp", "apply_dp"])
def test_paths_without_a_device_schedule_refuse_it(call):
    L = lib._load()
    plan = _plan()
    assert _set(plan, lib.ScheduleConfig(1e-3, 100, 10)) == lib.OK
    args = lib.StepArgs(3, 4, 0, 0.0, 0.0, 0.0, 0.0)
    grads = lib.Plan.ptr_array([BLOCK, BLOCK])
    comm = lib.DpComm()
    if call == "accumulate":
        rc = L.gaccum_accumulate(plan._h, grads, BLOCK, None)
    elif call == "apply":
        rc = L.gaccum_apply(plan._h, grads, grads, BLOCK, BLOCK, BLOCK, C.byref(args), None)
    elif call == "packed_forced":
        rc = L.gaccum_step_packed(plan._h, BLOCK, BLOCK, BLOCK, BLOCK, BLOCK, C.byref(args), 0, None)
    elif call == "host_session":
        h = C.c_void_p()
        rc = L.gaccum_host_session_create(C.byref(h), plan._h)
    elif call == "step_dp":
        rc = L.gaccum_step_dp(plan._h, C.byref(comm), grads, BLOCK, BLOCK, C.byref(args), 1, None)
    else:
        rc = L.gaccum_apply_dp(plan._h, C.byref(comm), grads, BLOCK, BLOCK, C.byref(args), 1, None)
    assert rc == lib.EINVAL
    msg = L.gaccum_last_error()
    assert b"device schedule" in msg or b"force_branch must be -1" in msg, msg


def test_setter_refused_after_the_first_compute_call():
    L = lib._load()
    plan = _plan()
    args = lib.StepArgs(0, 1, 0, 0.0, 0.0, 0.0, 0.0)
    grads = lib.Plan.ptr_array([BLOCK, BLOCK])
    # a layout-only plan fails the compute call, but the call still counts as the first one
    assert L.gaccum_step(plan._h, grads, grads, BLOCK, BLOCK, BLOCK, C.byref(args), None) == lib.ENODEVICE
    assert _set(plan, lib.ScheduleConfig(1e-3, 100, 10)) == lib.EINVAL
    assert b"before the plan's first compute call" in L.gaccum_last_error()


def test_header_documents_the_block():
    import os
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "gaccum.h")).read()
    assert "gaccum_plan_set_device_schedule" in hdr and "gaccum_schedule_init" in hdr
    assert g.version() == 200


# ---- the front end's kernel choice across the int32 wrap (train_op.ScheduleCursor) -------------------------------------
def _c_first_accumulate(step, n):
    """gaccum_abi.cu first_of_window, in C's arithmetic: (int32)g does not apply and (int32)((int32)g - 1) does."""
    def c_apply(x):
        x32 = int(np.int64(x).astype(np.int32))
        return x32 - int(x32 / n) * n == 0               # C's truncating %
    g32 = int(np.int64(step).astype(np.int32))
    return not c_apply(g32) and c_apply(g32 - 1)


def _oracle_applies(g0, n, steps):
    """The reference's predicate (oracle_np.ReferenceTrainOp.run) over ``steps`` micro-steps from g0."""
    return [int(np.int32(np.int64(g))) % n == 0 for g in range(g0, g0 + steps)]


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7])
@pytest.mark.parametrize("g0", [0, 2**31 - 20, 2**32 - 20, 3 * 2**31 - 20])
def test_eager_launches_choose_their_kernel_from_the_int32_step(n, g0):
    from gaccum_b200.train_op import ScheduleCursor
    cur = ScheduleCursor(n, lambda: pytest.fail("an eager op never reads the device counter"))
    cur.reset(g0)
    applies = _oracle_applies(g0, n, 40)
    for k in range(40):
        g = cur.launch(False)
        assert g == g0 + k                                 # StepArgs.global_step: the step the launch runs at
        apply, first = lib.is_apply_step(g, n), lib.is_first_accumulate(g, n)
        assert apply == applies[k]
        assert first == _c_first_accumulate(g, n)
        # a first accumulate follows an apply: the device's check, (int32)(g - 1) % N == 0
        if first:
            assert k == 0 or applies[k - 1]
        assert cur.advance() == apply


@pytest.mark.parametrize("n, applies_at", [
    (3, [2**31 - 5, 2**31 - 2, 2**31 + 2, 2**31 + 5]),     # the straddling window is 4 launches
    (5, [2**31 - 8, 2**31 - 3, 2**31 + 3, 2**31 + 8]),     # ... 6 launches
    (4, [2**31 - 8, 2**31 - 4, 2**31, 2**31 + 4]),         # a power of two: every window is N
])
def test_the_window_that_straddles_2_to_the_31(n, applies_at):
    from gaccum_b200.train_op import ScheduleCursor
    g0 = applies_at[0]
    cur = ScheduleCursor(n, lambda: None)
    cur.reset(g0)
    seen, firsts = [], []
    for _ in range(applies_at[-1] - g0 + 1):
        g = cur.launch(False)
        if lib.is_first_accumulate(g, n):
            firsts.append(g)
        if cur.advance():
            seen.append(g)
    assert seen == applies_at
    assert firsts == [a + 1 for a in applies_at[:-1]]


def test_first_eager_launch_after_a_capture_reads_the_device_counter_once():
    from gaccum_b200.train_op import ScheduleCursor
    reads = []
    device = {"g": None}

    def read():
        reads.append(device["g"])
        return device["g"]

    cur = ScheduleCursor(3, read)
    cur.reset(2**31 - 5)                                   # an apply step: a window start
    for _ in range(3):                                     # the captured window: nothing runs, nothing is read
        cur.launch(True)
        cur.advance()
    assert reads == []
    device["g"] = 2**31 + 1                                # two replays (the second refused at 2^31 + 1), then
    assert cur.launch(False) == 2**31 + 1                  # ... the first eager launch reads the counter
    assert not lib.is_apply_step(2**31 + 1, 3)
    cur.advance()
    assert cur.launch(False) == 2**31 + 2 and lib.is_apply_step(2**31 + 2, 3)
    cur.advance()
    assert reads == [2**31 + 1]                            # once


def test_capture_must_start_at_an_apply_step():
    from gaccum_b200.train_op import ScheduleCursor
    cur = ScheduleCursor(3, lambda: None)
    cur.reset(2**31 + 1)                                   # g mod 3 == 0, but int32(g) does not apply
    with pytest.raises(ValueError, match="must start at a window start"):
        cur.launch(True)
    assert cur.launch(False) == 2**31 + 1                  # the refused capture changed nothing
    cur.reset(2**31 + 2)
    assert cur.launch(True) == 2**31 + 2
