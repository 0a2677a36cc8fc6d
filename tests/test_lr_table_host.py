"""The learning-rate table's host side (include/gaccum.h, gaccum_plan_set_lr_table; no GPU needed) and the TF1
schedules that fill it (gaccum_b200/schedules.py).

* The setter's validation and the order of its refusals on a layout-only plan, in C and through ``Plan.set_lr_table``;
  ``LrTable``'s validation.
* ``schedules``: each schedule against its closed form in float64 and against PyTorch's ``torch.optim.lr_scheduler``
  (``PolynomialLR``, ``CosineAnnealingLR``, ``ExponentialLR``, ``StepLR``, ``MultiStepLR``) within a few fp32 ulps of
  the initial rate -- independent restatements, in the style of ``test_oracle_independent.py``; ``table(n)[g]`` equal to
  ``schedule(g)`` bit for bit.
* ``with_bert_warmup(polynomial_decay(power=1, end=0))`` bit-identical to ``gaccum_learning_rate`` (the formula the
  device schedule evaluates) at every step, across the end of warm-up and past ``num_train_steps``; ``create_optimizer``
  at its default module attributes bit-identical to that, and ``poly_power`` / ``end_learning_rate`` honoured.
"""
import ctypes as C
import math
import os

import numpy as np
import pytest

import gaccum_b200 as g
from gaccum_b200 import _lib as lib
from gaccum_b200 import schedules as S
from gaccum_b200.optimization import bert_learning_rate

F32 = np.float32
TABLE = 0x10000   # a 4-byte aligned address: the setter keeps it without dereferencing it
EPS = float(np.finfo(F32).eps)


def _plan():
    hp = lib.HParams(lib.ADAM_WEIGHT_DECAY, 0, 0.9, 0.999, 1e-6, 0.01, 1.0)
    return lib.Plan([10, 20], [True, False], hp, device=-1)


def _err():
    return lib._load().gaccum_last_error().decode()


# ---- the setter ----------------------------------------------------------------------------------------------------------
def test_setter_validates_its_arguments_in_order():
    L = lib._load()
    plan = _plan()
    assert L.gaccum_plan_set_lr_table(None, TABLE, 4) == lib.EINVAL and "plan is NULL" in _err()
    assert L.gaccum_plan_set_lr_table(plan._h, None, 4) == lib.EINVAL and "device_table is NULL" in _err()
    assert L.gaccum_plan_set_lr_table(plan._h, None, 0) == lib.EINVAL and "device_table is NULL" in _err()
    for n in (0, -1, -2**40):
        assert L.gaccum_plan_set_lr_table(plan._h, TABLE, n) == lib.EINVAL and "length must be >= 1" in _err()
    for off in (1, 2, 3):
        assert L.gaccum_plan_set_lr_table(plan._h, TABLE + off, 4) == lib.EINVAL and "4-byte aligned" in _err()
    # every argument valid: a layout-only plan has no launches to read a table
    assert L.gaccum_plan_set_lr_table(plan._h, TABLE, 4) == lib.EINVAL and "layout-only" in _err()
    assert L.gaccum_plan_set_lr_table(plan._h, TABLE + 4, 1) == lib.EINVAL and "layout-only" in _err()


def test_setter_on_a_layout_only_plan_combines_with_the_device_schedule_in_any_order():
    L = lib._load()
    for first in ("schedule", "table"):
        plan = _plan()
        cfg = lib.ScheduleConfig(1e-3, 100, 10)
        calls = {"schedule": lambda: L.gaccum_plan_set_device_schedule(plan._h, C.byref(cfg), TABLE),
                 "table": lambda: L.gaccum_plan_set_lr_table(plan._h, TABLE, 8)}
        order = ["schedule", "table"] if first == "schedule" else ["table", "schedule"]
        rcs = [calls[k]() for k in order]
        assert rcs == ([lib.OK, lib.EINVAL] if first == "schedule" else [lib.EINVAL, lib.OK])
        # the refused table left the plan as it was: the schedule's formula path still validates as before
        assert L.gaccum_plan_set_device_schedule(plan._h, C.byref(lib.ScheduleConfig(1e-3, 100, 10, power=0.5)),
                                                 TABLE) == lib.EINVAL


def test_after_the_first_compute_call_the_plan_is_refused_first_as_layout_only():
    L = lib._load()
    plan = _plan()
    args = lib.StepArgs(0, 1, 0, 0.0, 0.0, 0.0, 0.0)
    grads = lib.Plan.ptr_array([TABLE, TABLE])
    assert L.gaccum_step(plan._h, grads, grads, TABLE, TABLE, TABLE, C.byref(args), None) == lib.ENODEVICE
    assert L.gaccum_plan_set_lr_table(plan._h, TABLE, 4) == lib.EINVAL and "layout-only" in _err()


def test_python_setter_raises():
    plan = _plan()
    with pytest.raises(g.GaccumError, match="device_table is NULL"):
        plan.set_lr_table(0, 4)
    with pytest.raises(g.GaccumError, match="length must be >= 1"):
        plan.set_lr_table(TABLE, 0)
    with pytest.raises(g.GaccumError, match="4-byte aligned"):
        plan.set_lr_table(TABLE + 2, 4)
    with pytest.raises(g.GaccumError, match="layout-only"):
        plan.set_lr_table(TABLE, 4)


def test_algorithmic_bytes_of_a_layout_only_plan_are_unchanged_by_a_refused_table():
    a, b = _plan(), _plan()
    assert lib._load().gaccum_plan_set_lr_table(b._h, TABLE, 4) == lib.EINVAL
    for is_apply in (True, False):
        assert a.algorithmic_bytes(is_apply) == b.algorithmic_bytes(is_apply)


def test_header_documents_the_setter_and_the_version_stays():
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "gaccum.h")).read()
    assert "GACCUM_API int gaccum_plan_set_lr_table(gaccum_plan* plan, const float* device_table, int64_t length);" in hdr
    assert g.version() == 200
    assert C.sizeof(lib.ScheduleState) == 48 and C.sizeof(lib.ScheduleConfig) == 40


# ---- LrTable ----------------------------------------------------------------------------------------------------------
def test_lr_table_validates_and_rounds_once():
    from gaccum_b200.train_op import LrTable
    t = LrTable([1e-3, 0.0, 0.1])
    assert t.values.dtype == F32 and list(t.values) == [F32(1e-3), F32(0.0), F32(0.1)]
    assert not t.values.flags.writeable
    for bad in ([], [[1e-3]], [float("nan")], [1e-3, float("inf")], [-1e-9], [1e39], np.zeros((2, 2))):
        with pytest.raises(ValueError):
            LrTable(bad)
    sched = S.cosine_decay(1e-3, 10)
    assert LrTable((sched, 12)).values.tobytes() == sched.table(12).tobytes()
    assert list(LrTable((lambda s: 1e-3 * s, 3)).values) == [F32(0.0), F32(1e-3), F32(2e-3)]
    with pytest.raises(ValueError):
        LrTable((sched, 0))
    with pytest.raises(ValueError):
        LrTable((lambda s: -1.0, 2))


# ---- schedules: closed forms ------------------------------------------------------------------------------------------
def _close(ours, exact, lr0, ulps=4):
    """|ours - exact| within ``ulps`` fp32 ulps of the value plus ``ulps`` of the initial rate (a decayed value's own
    ulps are far finer than the rounding of the step fraction it came from)."""
    ours, exact = np.asarray(ours, np.float64), np.asarray(exact, np.float64)
    tol = ulps * EPS * (np.abs(exact) + abs(lr0))
    bad = np.abs(ours - exact) > tol
    assert not bad.any(), [(int(i), ours[i], exact[i]) for i in np.flatnonzero(bad)[:5]]


@pytest.mark.parametrize("power", [1.0, 0.5, 2.0, 3.0])
@pytest.mark.parametrize("end", [0.0, 1e-6])
@pytest.mark.parametrize("T", [1024, 1000, 7])
def test_polynomial_decay_closed_form(power, end, T):
    lr0 = 1e-3
    steps = np.arange(T + 20)
    exact = (lr0 - end) * (1 - np.minimum(steps, T) / T) ** power + end
    ours = S.polynomial_decay(lr0, T, end, power).table(T + 20)
    # the fraction g / T is rounded to fp32: near the end (1 - p) ** power carries that rounding, up to
    # power * (1 - p) ** (power - 1) * ulp(p) -- exact for T a power of two
    p = np.minimum(steps, T) / T
    with np.errstate(divide="ignore"):
        slack = np.where(p < 1, power * np.abs(1 - p) ** (power - 1), 0.0) * EPS * lr0 * (T & (T - 1) != 0)
    assert np.all(np.abs(ours.astype(np.float64) - exact) <= 4 * EPS * (exact + lr0) + slack)


def test_polynomial_decay_cycle_closed_form():
    lr0, T, end = 1e-3, 64, 1e-5
    ours = S.polynomial_decay(lr0, T, end, 1.0, cycle=True).table(5 * T)
    for gs in range(5 * T):
        ds = T * (1 if gs == 0 else math.ceil(gs / T))
        exact = (lr0 - end) * (1 - gs / ds) + end
        _close(ours[gs], exact, lr0)


@pytest.mark.parametrize("alpha", [0.0, 0.1])
@pytest.mark.parametrize("T", [1024, 1000])
def test_cosine_decay_closed_form(alpha, T):
    lr0 = 2e-4
    steps = np.arange(T + 10)
    exact = lr0 * ((1 - alpha) * 0.5 * (1 + np.cos(math.pi * np.minimum(steps, T) / T)) + alpha)
    _close(S.cosine_decay(lr0, T, alpha).table(T + 10), exact, lr0, ulps=8)


@pytest.mark.parametrize("staircase", [False, True])
def test_exponential_decay_closed_form(staircase):
    lr0, k, rate = 2.0 ** -10, 16, 1 - 2.0 ** -4              # exactly representable: only pow and * round
    steps = np.arange(2000)
    e = np.floor(steps / k) if staircase else steps / k
    _close(S.exponential_decay(lr0, k, rate, staircase).table(2000), lr0 * rate ** e, lr0, ulps=16)


def test_piecewise_constant_boundaries_are_inclusive_on_the_left_interval():
    s = S.piecewise_constant([10, 20, 30], [1.0, 0.5, 0.25, 0.125])
    want = [1.0] * 11 + [0.5] * 10 + [0.25] * 10 + [0.125] * 9        # g <= 10, 10 < g <= 20, ...
    assert list(s.table(40)) == want
    assert s(10**12) == 0.125
    assert S.piecewise_constant([], [0.3]).table(3).tolist() == [F32(0.3)] * 3
    with pytest.raises(ValueError):
        S.piecewise_constant([1, 2], [1.0])
    with pytest.raises(ValueError):
        S.piecewise_constant([5, 2], [1.0, 2.0, 3.0])


SCHEDULES = {
    "poly": lambda: S.polynomial_decay(1e-3, 100, 1e-5, 0.5),
    "poly_cycle": lambda: S.polynomial_decay(1e-3, 30, 0.0, 2.0, cycle=True),
    "cosine": lambda: S.cosine_decay(1e-3, 100, 0.05),
    "exp": lambda: S.exponential_decay(1e-3, 7, 0.9),
    "exp_stair": lambda: S.exponential_decay(1e-3, 7, 0.9, staircase=True),
    "piecewise": lambda: S.piecewise_constant([20, 50], [1e-3, 5e-4, 1e-4]),
    "warm_cosine": lambda: S.with_bert_warmup(S.cosine_decay(1e-3, 100), 1e-3, 10),
}


@pytest.mark.parametrize("name", sorted(SCHEDULES))
def test_table_entries_are_the_host_values_bit_for_bit(name):
    s = SCHEDULES[name]()
    tab = s.table(131)
    assert tab.dtype == F32 and tab.shape == (131,)
    for step in range(131):
        assert F32(s(step)).tobytes() == tab[step].tobytes(), step
    for step in (2**31 - 1, 2**31, 2**32 + 5):
        assert F32(s(step)).tobytes() == s.values([step])[0].tobytes()


# ---- schedules against torch.optim.lr_scheduler -----------------------------------------------------------------------
def _torch_lrs(make, steps, lr0):
    torch = pytest.importorskip("torch")
    opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=lr0)
    sch = make(opt)
    out = []
    for _ in range(steps):
        out.append(opt.param_groups[0]["lr"])
        opt.step()
        sch.step()
    return np.array(out)


@pytest.mark.parametrize("power", [1.0, 0.5, 2.0])
def test_polynomial_decay_against_torch_polynomial_lr(power):
    import torch
    lr0, T = 1e-3, 512
    ref = _torch_lrs(lambda o: torch.optim.lr_scheduler.PolynomialLR(o, total_iters=T, power=power), T + 8, lr0)
    _close(S.polynomial_decay(lr0, T, 0.0, power).table(T + 8), ref, lr0, ulps=8)


def test_cosine_decay_against_torch_cosine_annealing_lr():
    import torch
    lr0, T = 1e-3, 500
    ref = _torch_lrs(lambda o: torch.optim.lr_scheduler.CosineAnnealingLR(o, T_max=T), T + 1, lr0)
    _close(S.cosine_decay(lr0, T).table(T + 1), ref, lr0, ulps=8)


def test_exponential_decay_against_torch_exponential_and_step_lr():
    import torch
    lr0, gamma = 2.0 ** -9, 1 - 2.0 ** -6
    ref = _torch_lrs(lambda o: torch.optim.lr_scheduler.ExponentialLR(o, gamma=gamma), 1500, lr0)
    _close(S.exponential_decay(lr0, 1, gamma).table(1500), ref, lr0, ulps=16)
    ref = _torch_lrs(lambda o: torch.optim.lr_scheduler.StepLR(o, step_size=25, gamma=gamma), 1500, lr0)
    _close(S.exponential_decay(lr0, 25, gamma, staircase=True).table(1500), ref, lr0, ulps=16)


def test_piecewise_constant_against_torch_multi_step_lr():
    import torch
    lr0, gamma, milestones = 1e-3, 0.1, [30, 80, 120]
    ref = _torch_lrs(lambda o: torch.optim.lr_scheduler.MultiStepLR(o, milestones=milestones, gamma=gamma), 200, lr0)
    # MultiStepLR changes the rate at step m; TF's boundaries are inclusive on the left interval: m - 1
    s = S.piecewise_constant([m - 1 for m in milestones], [lr0 * gamma ** i for i in range(len(milestones) + 1)])
    _close(s.table(200), ref, lr0, ulps=1)


# ---- the reference's schedule -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("init_lr, T, W", [
    (2e-5, 2000, 200), (5e-5, 1000, 0), (1e-2, 12, 3), (3e-4, 50, 50), (1e-3, 40, 64), (1e-4, 1, 0), (0.1, 997, 13),
])
def test_bert_warmup_over_linear_decay_is_gaccum_learning_rate_bitwise(init_lr, T, W):
    s = S.with_bert_warmup(S.polynomial_decay(init_lr, T, 0.0, 1.0), init_lr, W)
    tab = s.table(T + 31)
    for step in range(T + 31):
        want = F32(g.learning_rate(init_lr, T, W, step))
        assert tab[step].tobytes() == want.tobytes(), (step, tab[step], want)
        assert F32(s(step)).tobytes() == want.tobytes()


def test_bert_warmup_past_the_int32_wrap_is_gaccum_learning_rate_bitwise():
    init_lr, T, W = 1e-3, 2**33, 2**20
    s = S.with_bert_warmup(S.polynomial_decay(init_lr, T, 0.0, 1.0), init_lr, W)
    for step in (0, 1, W - 1, W, W + 1, 2**31 - 1, 2**31, 2**31 + 1, 2**31 + W, 2**32 - 1, 2**32, 2**32 + W, T, T + 9):
        assert F32(s(step)).tobytes() == F32(g.learning_rate(init_lr, T, W, step)).tobytes(), step


def _create_optimizer_lr(monkeypatch, **attrs):
    """The learning_rate create_optimizer hands its optimizer (the train op itself needs a device)."""
    from gaccum_b200 import optimization as opt
    for k, v in attrs.items():
        monkeypatch.setattr(opt, k, v)
    seen = {}

    def capture(loss, optimizer, *a, **kw):
        seen["lr"] = optimizer.learning_rate
    monkeypatch.setattr(opt, "gradient_accumulation_train_op", capture)
    opt.create_optimizer(None, 2e-5, 1000, 100, False)
    return seen["lr"]


def test_create_optimizer_at_default_attributes_is_bit_identical(monkeypatch):
    from gaccum_b200 import optimization as opt
    assert (opt.poly_power, opt.end_learning_rate) == (1.0, 0.0)
    lr = _create_optimizer_lr(monkeypatch)
    ref = bert_learning_rate(2e-5, 1000, 100)
    for step in list(range(1200)) + [2**31 - 1, 2**31, 2**32 + 7]:
        assert F32(lr(step)).tobytes() == F32(ref(step)).tobytes(), step


def test_create_optimizer_reads_poly_power_and_end_learning_rate(monkeypatch):
    lr = _create_optimizer_lr(monkeypatch, poly_power=0.5, end_learning_rate=1e-6)
    want = S.with_bert_warmup(S.polynomial_decay(2e-5, 1000, 1e-6, 0.5), 2e-5, 100)
    for step in range(0, 1200, 7):
        assert F32(lr(step)).tobytes() == F32(want(step)).tobytes(), step
    assert lr(500) != bert_learning_rate(2e-5, 1000, 100)(500)
