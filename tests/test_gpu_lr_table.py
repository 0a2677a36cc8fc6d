"""The device schedule's learning-rate table (include/gaccum.h, gaccum_plan_set_lr_table) on the GPU.

a. Nothing else changes: at every dispatch key (336 cases), a table holding exactly gaccum_learning_rate(g) gives a run
   bit-identical to the formula's after every micro-step -- accumulators, p, m, v, master weights and model copy, the
   EMA and its state, the loss-scaling block, the window weight, the stats, trust ratios, per-tensor norms and the
   schedule block's step, beta powers and ``refused`` -- and each run matches the composed oracle (``LockStep``).
b. Cosine and power = 0.5 tables (with BERT's warm-up) against the composed oracle fed the same per-step lr, for
   AdamWeightDecay, Adam and LAMB with and without clipping and loss scaling; full-size BERT-Small LAMB with power 0.5.
c. One window captured as a CUDA graph and replayed for 31 windows (a loss-scaling skip among them, and past the table's
   end), bit-identical after every replay to eager launches of a host-scheduled op whose lr_fn reads the same table; an
   entry rewritten between replays takes effect at the next launch that reads it.
d. Table edges: g = L - 1, g = L and beyond, L = 1, and g past 2^31 with N a power of two -- clamped to a short table,
   and reading its own entry of a table longer than 2^31 entries.
e. Mid-window resume through ``state_dict`` with the table rebuilt; the setter and refusals on device plans.
"""
import contextlib
import ctypes as C
import types
import zlib

import numpy as np
import pytest

from apply_matrix import MODES, VARIANTS, Case, matrix_cases
from test_gpu_device_schedule_matrix import MAN, N, SCHED, STEPS, Scheduled, _assert_same, _buffers, _bytes, _capture
from test_gpu_device_schedule_matrix import _fill
from test_gpu_device_schedule_matrix import INF_AT, WEIGHTS, WRAP_MAN

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

F32 = np.float32


@contextlib.contextmanager
def _table_schedule(values):
    """LockStep builds its device-scheduled op with ``device_schedule=g._lib.ScheduleConfig(**sched)``: hand it an
    LrTable of ``values`` instead."""
    import gaccum_b200 as g
    from gaccum_b200.train_op import LrTable
    saved = g._lib.ScheduleConfig
    g._lib.ScheduleConfig = lambda **_: LrTable(values)
    try:
        yield
    finally:
        g._lib.ScheduleConfig = saved


class TableRun(Scheduled):
    """A ``Scheduled`` run whose lr comes from ``table``: with ``device_schedule`` the op gets ``LrTable(table)``, else
    a host-scheduled op's lr_fn reads it.  The oracle and ``check`` read the same table (``lr_at``)."""

    def __init__(self, case, seed, table, device_schedule=True, **kw):
        from gaccum_b200.train_op import LrTable
        self.table = np.array(LrTable(table).values)            # the host copy (writable)
        with _table_schedule(self.table) if device_schedule else contextlib.nullcontext():
            super().__init__(case, seed, device_schedule=device_schedule, **kw)
        g = self.g
        self.ref.lr = lambda s: self.lr_at(s)
        self.g = types.SimpleNamespace(is_apply_step=g.is_apply_step,
                                       learning_rate=lambda _lr, _t, _w, s: float(self.lr_at(s)))
        if not device_schedule:
            self.op.lr_fn = lambda s: float(self.lr_at(s))

    def lr_at(self, s) -> np.float32:
        return F32(self.table[min(int(s), len(self.table) - 1)])

    def set_entry(self, i: int, value: float) -> None:
        """Rewrite entry i on the host and, for a table op, on the device (stream-ordered)."""
        self.table[i] = F32(value)
        if self.op.lr_table is not None:
            self.op.lr_table[i] = float(F32(value))


def _state(run, sched=True):
    """``_buffers`` with the schedule block reduced to what both schedules keep: the step, the beta powers and
    ``refused`` (a table op's block holds a placeholder config's constants); without ``sched``, none of it."""
    out = _buffers(run)
    blk = out.pop("sched", None)
    if blk is not None and sched:
        out["sched"] = blk.view(torch.int32)[[0, 1, 9, 10, 11]].clone()
    return out


def _formula(sched=SCHED, length=STEPS):
    import gaccum_b200 as g
    return [g.learning_rate(sched["init_lr"], sched["num_train_steps"], sched["num_warmup_steps"], s)
            for s in range(length)]


# ---- a. nothing else changes -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", matrix_cases(), ids=lambda c: c.id)
def test_a_table_of_the_formula_changes_nothing(case: Case):
    seed = zlib.crc32(case.id.encode()) ^ 0x7B
    formula, table = Scheduled(case, seed), TableRun(case, seed, _formula())
    assert table.op.lr_table is not None and formula.op.lr_table is None
    applies = 0
    for s in range(STEPS):
        a = formula.micro()
        assert table.micro() == a
        applies += a
        _assert_same(_state(formula), _state(table), f"step {s}")
    assert applies == 5


# ---- b. other schedules against the oracle ------------------------------------------------------------------------------
def _shape_table(shape, length=STEPS + 1):
    from gaccum_b200 import schedules
    lr, T, W = SCHED["init_lr"], SCHED["num_train_steps"], SCHED["num_warmup_steps"]
    decay = schedules.cosine_decay(lr, T, 0.1) if shape == "cosine" else schedules.polynomial_decay(lr, T, 1e-4, 0.5)
    return schedules.with_bert_warmup(decay, lr, W).table(length)


ORACLE_KEYS = [(v, m, s) for v in VARIANTS for m in MODES for s in ("cosine", "poly_0.5")]


@pytest.mark.parametrize("variant, mode, shape", ORACLE_KEYS, ids=[f"{v}-{m}-{s}" for v, m, s in ORACLE_KEYS])
def test_schedule_tables_match_the_oracle(variant, mode, shape):
    tab = _shape_table(shape)
    assert len(set(tab.tolist())) > 8                      # the lr moves at every step but the clamped end
    case = Case(variant, mode, True, "t256_fp32", variant == "adam")
    run = TableRun(case, zlib.crc32(f"{variant}{mode}{shape}".encode()), tab)
    assert sum(run.micro() for _ in range(STEPS)) == 5     # check(): the oracle, the stats' lr, the block


def test_full_size_bert_small_lamb_power_one_half():
    import oracle_np as onp
    from gaccum_b200 import schedules
    man = onp.MANIFESTS["bert_small"]()
    tab = schedules.with_bert_warmup(schedules.polynomial_decay(1e-3, 6, 0.0, 0.5), 1e-3, 2).table(6)
    run = TableRun(Case("lamb", "clip", True, "t256_fp32", False), 0xB5, tab, man=man, n=2)
    assert sum(run.micro() for _ in range(7)) == 4


# ---- c. one window replayed for a whole run -----------------------------------------------------------------------------
REPLAY_KEYS = [("adamw", "ls_clip", "t256_fp32", False), ("lamb", "ls_clip", "packed", True),
               ("adam", "ls_noclip", "t256_bf16", False)]
WINDOWS = 31


@pytest.mark.parametrize("variant, mode, layout, ema", REPLAY_KEYS, ids=["-".join(map(str, k)) for k in REPLAY_KEYS])
def test_one_window_replayed_for_a_run_matches_eager_launches(variant, mode, layout, ema):
    from gaccum_b200 import schedules
    case = Case(variant, mode, True, layout, ema)
    seed = zlib.crc32(case.id.encode()) ^ 0x3C
    tab = schedules.with_bert_warmup(schedules.cosine_decay(1e-2, 60, 0.05), 1e-2, 6).table(70)
    eager, graphed = TableRun(case, seed, tab, device_schedule=False), TableRun(case, seed, tab)
    for _ in range(N):
        eager.micro()
        graphed.micro()
    _assert_same(_state(eager), _state(graphed, False), "eager window")
    graph, static = _capture(graphed, N, weights=True)
    for w in range(WINDOWS):
        if w == 12:                              # rewrite the next two windows' entries between replays
            for i in range(eager.g_host, eager.g_host + 2 * N):
                for r in (eager, graphed):
                    r.set_entry(i, 3e-3 + 1e-4 * i)
        for j in range(N):
            s = eager.step_no
            S = F32(eager.ref.scale) if eager.ls else F32(1.0)
            grads = eager.grads(0.1, INF_AT[1:] if eager.ls and s == INF_AT[0] else None)
            with np.errstate(over="ignore", invalid="ignore"):
                dev = [None if x is None else graphed._device(i, torch.from_numpy(x * S).to(graphed.dtype))
                       for i, x in enumerate(grads)]
            _fill(static[j], dev, WEIGHTS[s % len(WEIGHTS)])
            eager.step_no += 1
            eager.wstep(grads, WEIGHTS[s % len(WEIGHTS)])
        graph.replay()
        _assert_same(_state(eager), _state(graphed, False), f"replay {w}")
        if w == 12:
            assert F32(graphed.op.stats()["lr"]) == F32(3e-3 + 1e-4 * (eager.g_host - 1))   # the rewritten entry
    assert graphed.op.global_step == eager.g_host == N * (WINDOWS + 1) > len(tab)
    assert eager.op.loss_scale_state()["skipped_windows"] == 1
    assert graphed.op.lr_fn(10**6) == float(tab[-1])


# ---- d. table edges ---------------------------------------------------------------------------------------------------
EDGE_KEYS = [("adam", "clip", "t256_fp32"), ("lamb", "noclip", "packed"), ("adamw", "ls_clip", "t1920_bf16")]


@pytest.mark.parametrize("length, g0", [(1, 0), (7, 3), (9, 0)], ids=["L1", "L7_from_3", "L9"])
@pytest.mark.parametrize("variant, mode, layout", EDGE_KEYS, ids=["-".join(k) for k in EDGE_KEYS])
def test_table_edges(variant, mode, layout, length, g0):
    """Distinct entries: g = L - 1 reads the last one, g = L and beyond read it again."""
    vals = [1e-3 * (1 + 0.25 * i) for i in range(length)]
    run = TableRun(Case(variant, mode, True, layout, False), 7 * length + g0, vals, global_step=g0)
    lrs = []
    for _ in range(3 * N + 3):
        run.micro()
        lrs.append(F32(run.op.stats()["lr"]))
    assert lrs == [run.lr_at(g) for g in range(g0, g0 + 3 * N + 3)]
    assert lrs[-1] == F32(vals[-1])


@pytest.mark.parametrize("base", [2**31, 2**32])
def test_step_past_2_31_clamps_to_the_last_entry(base):
    vals = [1e-3, 2e-3, 5e-4]
    run = TableRun(Case("adamw", "clip", True, "t256_fp32", False), 31, vals, global_step=base - 8, n=4, man=WRAP_MAN)
    assert sum(run.micro() for _ in range(16)) == 4
    assert F32(run.op.stats()["lr"]) == F32(5e-4)


def test_step_past_2_31_reads_its_own_entry_of_a_longer_table():
    """A table of 2^31 + 64 entries (8 GB): the 64-bit index reads entry g itself across 2^31."""
    lo, length = 2**31 - 16, 2**31 + 64
    run = TableRun(Case("adam", "noclip", True, "t256_fp32", False), 41, [0.0], global_step=2**31 - 8, n=4,
                   man=WRAP_MAN)
    big = torch.zeros(length, dtype=torch.float32, device="cuda")
    near = (1e-3 * (1 + 0.01 * np.arange(length - lo))).astype(F32)
    big[lo:] = torch.from_numpy(near).cuda()
    run.op.plan.set_lr_table(big.data_ptr(), length)     # before the first compute call: replaces the one-entry table
    run.op.lr_table = big
    run.lr_at = lambda s: near[min(int(s), length - 1) - lo]
    lrs = []
    for _ in range(16):
        run.micro()
        lrs.append(F32(run.op.stats()["lr"]))
    assert lrs == [near[g - lo] for g in range(2**31 - 8, 2**31 + 8)]
    del run, big
    torch.cuda.empty_cache()


# ---- e. resume, setters and refusals ----------------------------------------------------------------------------------
def _op(params, table):
    import gaccum_b200 as g
    from gaccum_b200.train_op import GaccumTrainOp, LrTable
    names = [n for n, _ in MAN[:5]]
    return GaccumTrainOp([p.clone().cuda() for p in params], names, g.HParams.bert(), N, None,
                         device_schedule=LrTable(table))


def test_mid_window_resume_with_the_table_rebuilt():
    from gaccum_b200 import schedules
    rng = np.random.default_rng(5)
    params = [torch.from_numpy(rng.normal(0, 0.05, s).astype(F32)) for _, s in MAN[:5]]
    grads = [[torch.from_numpy(rng.normal(0, 0.1, s).astype(F32)).cuda() for _, s in MAN[:5]] for _ in range(14)]
    table = (schedules.polynomial_decay(1e-2, 12, 1e-4, 0.5), 14)

    def step(op, gr):
        return op.run(gr)

    whole, first = _op(params, table), _op(params, table)
    for s in range(4):                                       # 4: mid-window (N = 3)
        assert step(whole, grads[s]) == step(first, grads[s])
    sd = first.state_dict()
    assert not any("lr_table" in k or "learning_rate" in k for k in sd)     # configuration, not state
    del first
    resumed = _op([torch.zeros_like(p) for p in params], table)
    resumed.load_state_dict(sd)
    assert resumed.global_step == 4
    for s in range(4, 14):
        assert step(whole, grads[s]) == step(resumed, grads[s])
        a, b = whole.state_dict(), resumed.state_dict()
        assert a.keys() == b.keys()
        for k in a:
            assert torch.equal(_bytes(a[k].cpu()), _bytes(b[k].cpu())), (s, k)
        assert whole.stats() == resumed.stats()


def _device_plan(variant=0):
    import gaccum_b200 as g
    hp = g.HParams(variant, 0, 0.9, 0.999, 1e-6, 0.01, 1.0)
    return g.Plan([1000, 37, 5], [True, False, True], hp, device=0)


def _L():
    from gaccum_b200 import _lib
    return _lib, _lib._load()


def test_first_compute_call_without_a_device_schedule_fails_naming_it():
    lib, L = _L()
    plan = _device_plan()
    tab = torch.full((4,), 1e-3, device="cuda")
    plan.set_lr_table(tab.data_ptr(), 4)
    slab = torch.zeros(plan.padded_size, device="cuda")
    args = lib.StepArgs(1, 2, 0, 1e-3, 0.9, 0.999, 0.0)
    rc = L.gaccum_step_packed(plan._h, slab.data_ptr(), slab.data_ptr(), slab.data_ptr(), slab.data_ptr(),
                              slab.data_ptr(), C.byref(args), -1, None)
    assert rc == lib.EINVAL
    assert "needs a device schedule (gaccum_plan_set_device_schedule)" in L.gaccum_last_error().decode()
    torch.cuda.synchronize()
    assert not slab.any()                                    # nothing was launched
    assert L.gaccum_plan_set_lr_table(plan._h, tab.data_ptr(), 4) == lib.EINVAL       # the call counted as the first
    assert "before the plan's first compute call" in L.gaccum_last_error().decode()


@pytest.mark.parametrize("with_schedule", [False, True])
@pytest.mark.parametrize("call", ["accumulate", "apply", "host_session", "step_dp", "apply_dp"])
def test_entry_points_without_a_device_schedule_refuse_a_table_plan(call, with_schedule):
    lib, L = _L()
    plan = _device_plan()
    tab = torch.full((4,), 1e-3, device="cuda")
    blk = torch.zeros(6, dtype=torch.int64, device="cuda")
    plan.set_lr_table(tab.data_ptr(), 4)
    if with_schedule:
        plan.set_device_schedule(lib.ScheduleConfig(0.0, 0, 0), blk.data_ptr())
    slab = torch.zeros(plan.padded_size, device="cuda")
    p = slab.data_ptr()
    grads = lib.Plan.ptr_array([p, p, p])
    args = lib.StepArgs(3, 4, 0, 1e-3, 0.9, 0.999, 0.0)
    comm = lib.DpComm()
    if call == "accumulate":
        rc = L.gaccum_accumulate(plan._h, grads, p, None)
    elif call == "apply":
        rc = L.gaccum_apply(plan._h, grads, grads, p, p, p, C.byref(args), None)
    elif call == "host_session":
        h = C.c_void_p()
        rc = L.gaccum_host_session_create(C.byref(h), plan._h)
    elif call == "step_dp":
        rc = L.gaccum_step_dp(plan._h, C.byref(comm), grads, p, p, C.byref(args), 1, None)
    else:
        rc = L.gaccum_apply_dp(plan._h, C.byref(comm), grads, p, p, C.byref(args), 1, None)
    assert rc == lib.EINVAL
    msg = L.gaccum_last_error().decode()
    assert ("a device schedule" if with_schedule else "a learning-rate table (gaccum_plan_set_lr_table)") in msg, msg
    torch.cuda.synchronize()
    assert not slab.any()


OTHERS = ["schedule", "norms", "ww", "lr_mult", "ema", "dtype", "loss_scale", "adapt"]


@pytest.mark.parametrize("pos", range(len(OTHERS) + 1))
@pytest.mark.parametrize("reverse", [False, True])
def test_setters_combine_in_any_order(pos, reverse):
    lib, L = _L()
    plan = _device_plan(variant=2)
    tab = torch.full((4,), 1e-3, device="cuda")
    norms = torch.zeros(16, device="cuda")
    calls = {
        "table": lambda: L.gaccum_plan_set_lr_table(plan._h, tab.data_ptr(), 4),
        "schedule": lambda: L.gaccum_plan_set_device_schedule(plan._h, C.byref(lib.ScheduleConfig(1e-3, 10, 2)), 0x60000),
        "norms": lambda: L.gaccum_plan_set_tensor_norms(plan._h, norms.data_ptr()),
        "ww": lambda: L.gaccum_plan_set_window_weight(plan._h, 0x50000),
        "lr_mult": lambda: L.gaccum_plan_set_lr_multipliers(plan._h, C.cast((C.c_float * 3)(0.5, 0.0, 2.0), C.c_void_p)),
        "ema": lambda: L.gaccum_plan_set_ema(plan._h, C.byref(lib.EmaConfig(0.999)), 0x10000, 0x20000),
        "dtype": lambda: L.gaccum_plan_set_param_dtype(plan._h, lib.DTYPE_BF16, 0x30000),
        "loss_scale": lambda: L.gaccum_plan_set_loss_scale(plan._h, C.byref(lib.LossScaleConfig()), 0x40000),
        "adapt": lambda: L.gaccum_plan_set_layer_adaptation(plan._h, C.cast((C.c_uint8 * 3)(1, 0, 1), C.c_void_p)),
    }
    order = OTHERS[::-1] if reverse else list(OTHERS)
    order.insert(pos, "table")
    for what in order:
        before = [plan.algorithmic_bytes(a) for a in (True, False)]
        assert calls[what]() == 0, what
        if what == "table":
            assert [plan.algorithmic_bytes(a) for a in (True, False)] == before
    assert calls["table"]() == 0                              # set again before the first compute call: replaced


def test_front_ends_refuse_a_host_lr_fn_and_the_host_op_refuses_a_table():
    import gaccum_b200 as g
    from gaccum_b200.train_op import GaccumTrainOp, HostTrainOp, LrTable
    with pytest.raises(ValueError, match="lr_fn=None"):
        GaccumTrainOp([torch.ones(8, device="cuda")], ["w"], g.HParams.bert(), 2, lambda s: 1e-3,
                      device_schedule=LrTable([1e-3]))
    with pytest.raises(ValueError, match="device schedule"):
        HostTrainOp([torch.ones(8)], ["w"], g.HParams.bert(), 2, lambda s: 1e-3, device_schedule=LrTable([1e-3]))
