"""Per-tensor learning-rate multipliers without a GPU: the C setter's checks on layout-only plans, its combination with
the other setters, the refusals of the entry points that do not support it (C and Python), the byte counts, ELECTRA's
layer-wise table and the optimizers' key matching, and the oracle's identities (every option at identity = the reference
oracles; all ones = no table; a uniform m = the schedule times m)."""
import ctypes as C
import itertools
import math

import numpy as np
import pytest

import oracle_c
import oracle_np as onp
from apply_matrix import SCHED, oracle_hparams, reference_op
from composed_oracle import ComposedReferenceTrainOp

F32 = np.float32


def _L():
    from gaccum_b200 import _lib
    return _lib, _lib._load()


def _plan(variant=0):
    import gaccum_b200 as g
    hp = g.HParams(variant, 0, 0.9, 0.999, 1e-6, 0.01, 1.0)
    return g.Plan([1000, 37, 5], [True, False, True], hp, device=-1)


def _set(plan, values):
    lib, L = _L()
    if values is None:
        return L.gaccum_plan_set_lr_multipliers(plan._h, None)
    arr = (C.c_float * len(values))(*values)
    return L.gaccum_plan_set_lr_multipliers(plan._h, C.cast(arr, C.c_void_p))


# ---- the C ABI on layout-only plans --------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [None, [1.0, float("nan"), 1.0], [float("inf"), 1.0, 1.0], [1.0, 1.0, float("-inf")],
                                 [1.0, -0.5, 1.0], [-1e-30, 1.0, 1.0]])
def test_setter_refuses_bad_tables(bad):
    lib, L = _L()
    assert _set(_plan(), bad) == lib.EINVAL
    assert ("NULL" if bad is None else "finite and >= 0") in L.gaccum_last_error().decode()


@pytest.mark.parametrize("variant", [0, 1, 2])
def test_setter_accepts_finite_non_negative_values(variant):
    plan = _plan(variant)
    assert _set(plan, [0.0, 1.0, 3.4e38]) == 0
    assert _set(plan, [0.5, 1e-30, 2.0]) == 0                                         # may be called again before compute


def test_setter_is_refused_after_a_compute_call():
    lib, L = _L()
    plan = _plan()
    args = lib.StepArgs(0, 1, 0, 1e-3, 0.9, 0.999, 0.0)
    assert L.gaccum_apply(plan._h, None, None, None, None, None, C.byref(args), None) != 0   # counts as a compute call
    assert _set(plan, [1.0, 1.0, 1.0]) == lib.EINVAL
    assert "before the plan's first compute call" in L.gaccum_last_error().decode()


@pytest.mark.parametrize("order", list(itertools.permutations(["lr_mult", "ema", "dtype", "loss_scale", "adapt"])))
def test_setters_combine_in_any_order(order):
    lib, L = _L()
    plan = _plan(variant=2)
    calls = {
        "lr_mult": lambda: _set(plan, [0.5, 0.0, 2.0]),
        "ema": lambda: L.gaccum_plan_set_ema(plan._h, C.byref(lib.EmaConfig(0.999)), 0x10000, 0x20000),
        "dtype": lambda: L.gaccum_plan_set_param_dtype(plan._h, lib.DTYPE_BF16, 0x30000),
        "loss_scale": lambda: L.gaccum_plan_set_loss_scale(plan._h, C.byref(lib.LossScaleConfig()), 0x40000),
        "adapt": lambda: L.gaccum_plan_set_layer_adaptation(plan._h, C.cast((C.c_uint8 * 3)(1, 0, 1), C.c_void_p)),
    }
    for what in order:
        assert calls[what]() == 0, what
    assert plan.algorithmic_bytes(True) == 56 * plan.num_elements


@pytest.mark.parametrize("variant, apply_bytes", [(0, 36), (1, 36), (2, 48)])
def test_algorithmic_bytes_unchanged(variant, apply_bytes):
    plan = _plan(variant)
    acc = plan.algorithmic_bytes(False)
    assert _set(plan, [0.25, 1.0, 4.0]) == 0
    assert plan.algorithmic_bytes(True) == apply_bytes * plan.num_elements
    assert plan.algorithmic_bytes(False) == acc


def test_data_parallel_and_host_session_refuse_a_table():
    lib, L = _L()
    plan = _plan()
    assert _set(plan, [1.0, 1.0, 1.0]) == 0              # even a table of ones: the refusal is about the call
    comm = lib.DpComm()
    comm.world = 2
    args = lib.StepArgs(0, 1, 0, 1e-3, 0.9, 0.999, 0.0)
    for fn in (L.gaccum_step_dp, L.gaccum_apply_dp):
        assert fn(plan._h, C.byref(comm), None, None, None, C.byref(args), 1, None) == lib.EINVAL
        assert "learning-rate multipliers" in L.gaccum_last_error().decode()
    h = C.c_void_p()
    assert L.gaccum_host_session_create(C.byref(h), plan._h) == lib.EINVAL
    assert "learning-rate multipliers" in L.gaccum_last_error().decode()


# ---- Python ----------------------------------------------------------------------------------------------------------
def test_python_front_ends_refuse_a_table():
    import torch
    import gaccum_b200 as g
    from gaccum_b200.distributed import FusedDataParallelTrainOp
    from gaccum_b200.train_op import HostTrainOp
    with pytest.raises(ValueError, match="learning-rate multipliers"):
        HostTrainOp([torch.zeros(4)], ["w"], g.HParams.bert(), 2, lambda s: 1e-3, lr_multipliers=[1.0])
    with pytest.raises(ValueError, match="learning-rate multipliers"):
        FusedDataParallelTrainOp([torch.zeros(4)], ["w"], g.HParams.bert(), 2, lambda s: 1e-3, lr_multipliers=[1.0])


@pytest.mark.parametrize("bad", [[float("nan")], [float("inf")], [-1.0], [1e39], [1.0, 1.0]])
@pytest.mark.parametrize("cls", ["GaccumTrainOp", "PackedTrainOp"])
def test_train_ops_check_the_table_before_anything_else(cls, bad):
    import torch
    import gaccum_b200 as g
    from gaccum_b200 import train_op
    with pytest.raises(ValueError, match="learning-rate multiplier"):
        getattr(train_op, cls)([torch.zeros(4)], ["w"], g.HParams.bert(), 2, lambda s: 1e-3, lr_multipliers=bad)


def test_multiplier_array_rounds_to_fp32_once():
    from gaccum_b200 import _lib
    out = _lib.lr_multiplier_array([0.8 ** 14, 0.1, 0, 3.4028234663852886e38], 4)
    assert out.dtype == np.float32
    assert out.tolist() == [float(F32(0.8 ** 14)), float(F32(0.1)), 0.0, float(F32(3.4028234663852886e38))]


# ---- ELECTRA's table and the key matching --------------------------------------------------------------------------
def test_layerwise_multipliers_bert_base_known_answers():
    from gaccum_b200 import _lib
    from gaccum_b200 import optimization as opt
    table = opt.layerwise_lr_multipliers(0.8, 12)
    assert table["/embeddings/"] == 0.8 ** 14 and table["/embeddings_project/"] == 0.8 ** 14
    assert table["encoder/layer_0/"] == 0.8 ** 13 and table["encoder/layer_11/"] == 0.8 ** 2
    assert table["task_specific/"] == 1.0 and len(table) == 15
    names = [n for n, _ in onp.bert_manifest(12, 768)]
    mult = _lib.lr_multiplier_array(opt.lr_multipliers_for(names, table), len(names))
    by_name = dict(zip(names, mult))
    assert by_name["bert/embeddings/word_embeddings"] == F32(0.8 ** 14)
    assert by_name["bert/embeddings/LayerNorm/gamma"] == F32(0.8 ** 14)
    assert by_name["bert/encoder/layer_0/attention/self/query/kernel"] == F32(0.8 ** 13)
    assert by_name["bert/encoder/layer_1/output/dense/bias"] == F32(0.8 ** 12)       # not layer_10's or layer_11's
    assert by_name["bert/encoder/layer_10/output/dense/bias"] == F32(0.8 ** 3)
    assert by_name["bert/encoder/layer_11/output/LayerNorm/beta"] == F32(0.8 ** 2)
    for n in ("bert/pooler/dense/kernel", "bert/pooler/dense/bias", "output_weights", "output_bias"):
        assert by_name[n] == F32(1.0), n


def test_key_matching_rules():
    from gaccum_b200 import optimization as opt
    assert opt.lr_multipliers_for(["a/kernel:0", "b/kernel:0"], None) is None
    # no key matches: the scheduled lr (ELECTRA would raise)
    assert opt.lr_multipliers_for(["x/kernel:0", "task_specific/w:0"], {"task_specific/": 0.5}) == [1.0, 0.5]
    # two keys match: refused (ELECTRA would update the variable once per key)
    with pytest.raises(ValueError, match="more than one"):
        opt.lr_multipliers_for(["bert/encoder/layer_0/embeddings/x"], {"/embeddings/": 0.1, "encoder/layer_0/": 0.2})


def test_optimizers_take_the_dict():
    from gaccum_b200 import optimization as opt
    t = {"a/": 0.5}
    o = opt.AdamWeightDecayOptimizer(1e-3)                # the reference's signature: the table is an attribute
    assert o.lr_multipliers is None
    o.lr_multipliers = t
    assert o.lr_multipliers == t
    assert opt.LAMBOptimizer(1e-3, lr_multipliers=t).lr_multipliers == t
    assert opt.AdamOptimizer(1e-3, lr_multipliers=t).lr_multipliers == t
    assert opt.AdamOptimizer(1e-3).lr_multipliers is None


def test_number_of_layers_from_the_names(monkeypatch):
    import torch
    from gaccum_b200 import graph, optimization as opt
    assert opt._num_encoder_layers(["bert/encoder/layer_0/x", "bert/encoder/layer_11/y", "output_weights"]) == 12
    assert opt._num_encoder_layers(["electra/encoder/layer_3/attention/output/dense/kernel:0"]) == 4
    assert opt.layerwise_lr_decay is None
    graph.reset_default_graph()
    graph.add_variable("bert/pooler/dense/kernel:0", torch.zeros(3))
    monkeypatch.setattr(opt, "layerwise_lr_decay", 0.8)
    with pytest.raises(ValueError, match="encoder/layer_"):
        opt.create_optimizer(torch.zeros(()), 1e-4, 10, 1, False)


# ---- the oracle ------------------------------------------------------------------------------------------------------
MAN = [("a/kernel", (300,)), ("a/bias", (5,)), ("LayerNorm/gamma", (33,)), ("one/kernel", (1,)), ("t/kernel", (3, 71))]
VARIANTS = ("adamw", "adam", "lamb")
MODES = ("noclip", "clip", "ls_noclip", "ls_clip")


def _same_state(a, b):
    """a: the oracle with a table; b: the oracle it is compared with."""
    for what in ("params", "m", "v", "accum"):
        for x, y in zip(getattr(a, what), getattr(b, what)):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), what
    assert (F32(a.beta1_power), F32(a.beta2_power)) == (F32(b.beta1_power), F32(b.beta2_power))
    assert (a.scale, a.good_windows, a.skipped_windows, a.last_skipped) == \
        (b.scale, b.good_windows, b.skipped_windows, b.last_skipped)
    assert np.array_equal(np.array(a.ratios, F32), np.array(b.ratios, F32))


def _drive(a, b, N, seed, steps=10, m=1.0):
    """a: the oracle with a table, b: one fed fp32(lr * m) (m = 1: the schedule itself)."""
    rng = np.random.default_rng(seed)
    for s in range(steps):
        grads = [rng.normal(0, 0.1, sh).astype(F32) for _, sh in MAN]
        if s == 4 and a.ls:
            grads[0][7] = np.inf                            # one overflowed window under loss scaling
        ia, ib = a.run([g.copy() for g in grads]), b.run([g.copy() for g in grads])
        assert ia.applied == ib.applied and np.multiply(F32(ia.lr), F32(m), dtype=F32) == F32(ib.lr)
        for k in ("global_norm", "clip_scale"):
            x, y = F32(getattr(ia, k)), F32(getattr(ib, k))
            assert x.view(np.uint32) == y.view(np.uint32), k
        _same_state(a, b)


IDENTITY_KEYS = [(v, m) for v in ("adamw", "adam") for m in ("noclip", "clip")]


@pytest.mark.parametrize("g0", [0, 2**31 - 2], ids=["from_0", "from_2_31_minus_2"])
@pytest.mark.parametrize("variant, mode", IDENTITY_KEYS)
def test_oracle_at_identity_is_the_reference_oracle(variant, mode, g0):
    """Every option of the composed oracle at its identity -- a table of ones, a window weight that totals N in every
    window, loss scaling whose S stays 1 -- computes what oracle_np's and the C oracle's restatements of the reference
    compute, bit for bit, after every micro-step: with a tensor that never gets a gradient, one that misses some, a
    one-element tensor, and from two steps before global_step's int32 wrap (where a window is longer than N)."""
    N = 3
    rng = np.random.default_rng(6)
    params = [rng.normal(0, 0.05, s).astype(F32) for _, s in MAN]
    names = [n for n, _ in MAN]
    hp = oracle_hparams(variant, mode)
    a = ComposedReferenceTrainOp([p.copy() for p in params], names, hp, N, lr_mult=[1.0] * len(MAN),
                                 window_weight=True, initial_scale=1.0, growth_interval=2**30, **SCHED, global_step=g0)
    refs = [cls([p.copy() for p in params], names, hp, N, **SCHED, global_step=g0)
            for cls in (onp.ReferenceTrainOp, oracle_c.COracleTrainOp)]
    in_window = 0                                           # micro-steps of the open window so far
    for s in range(3 * N + 2):
        grads = [rng.normal(0, 0.1, sh).astype(F32) for _, sh in MAN]
        grads[1] = None
        if s % 3 == 2:
            grads[4] = None
        in_window += 1
        applies = int(np.int64(g0 + s).astype(np.int32)) % N == 0
        ia = a.run([None if x is None else x.copy() for x in grads], weight=N - in_window + 1 if applies else 1.0)
        if applies:
            in_window = 0
            assert a.last_weight == N and a.weight == 0
        for b in refs:
            ib = b.run(grads)
            assert (ia.global_step, ia.applied) == (ib.global_step, ib.applied) and ia.applied == applies
            for k in ("lr", "global_norm", "clip_scale"):
                assert F32(getattr(ia, k)).tobytes() == F32(getattr(ib, k)).tobytes(), (type(b).__name__, k)
            for what in ("params", "m", "v", "accum"):
                for i, (x, y) in enumerate(zip(getattr(a, what), getattr(b, what))):
                    assert x.tobytes() == y.tobytes(), (type(b).__name__, what, names[i])
            assert (F32(a.beta1_power), F32(a.beta2_power)) == (F32(b.beta1_power), F32(b.beta2_power))
    assert a.scale == 1.0 and a.skipped_windows == 0


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("variant", VARIANTS)
def test_oracle_with_ones_is_the_oracle_without(variant, mode):
    rng = np.random.default_rng(3)
    params = [rng.normal(0, 0.05, s).astype(F32) for _, s in MAN]
    names = [n for n, _ in MAN]
    _drive(reference_op(variant, mode, params, names, 3, lr_mult=[1.0] * len(MAN)),
           reference_op(variant, mode, params, names, 3), 3, 5)


@pytest.mark.parametrize("m", [0.0, 0.3, 2.5])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("variant", VARIANTS)
def test_uniform_multiplier_is_the_schedule_times_m(variant, mode, m):
    rng = np.random.default_rng(4)
    params = [rng.normal(0, 0.05, s).astype(F32) for _, s in MAN]
    names = [n for n, _ in MAN]
    ref = reference_op(variant, mode, params, names, 3)
    base = ref.lr
    ref.lr = lambda g: np.multiply(F32(base(g)), F32(m), dtype=F32)      # an lr_fn returning fp32(lr * m)
    _drive(reference_op(variant, mode, params, names, 3, lr_mult=[m] * len(MAN)), ref, 3, 6, m=m)


def test_oracle_multiplier_zero_freezes_the_weights_only():
    rng = np.random.default_rng(5)
    params = [rng.normal(0, 0.05, s).astype(F32) for _, s in MAN]
    names = [n for n, _ in MAN]
    for variant in VARIANTS:
        op = reference_op(variant, "clip", params, names, 2, lr_mult=[0.0, 1.0, 1.0, 0.5, 2.0])
        for _ in range(4):
            op.run([rng.normal(0, 0.1, s).astype(F32) for _, s in MAN])
        assert np.array_equal(op.params[0], params[0]) and not np.array_equal(op.params[4], params[4])
        assert np.any(op.m[0] != 0) and np.any(op.v[0] != 0)
        assert math.isfinite(float(op.params[3][0]))
