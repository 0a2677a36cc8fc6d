"""Per-tensor learning-rate multipliers on the GPU (include/gaccum.h, gaccum_plan_set_lr_multipliers).

* Every dispatch key (tests/apply_matrix.py: 336 cases, all 120 apply instantiations) with a table holding 0, 1, a value
  below 1 and one above 1, against the composed oracle (tests/composed_oracle.py) after every micro-step; loss-scaled
  cases go through one overflowed window.
* Oracle-free identities, bit for bit, for every variant x mode: a table of ones is a plan without the call; a uniform m
  is the run whose lr_fn returns fp32(lr * m) (stats.lr aside); a multiplier of 0 freezes that tensor's weights (and a
  16-bit model's copy) while its m and v advance.
* bf16 / fp16 against the upcast fp32 run with the same table; CUDA-graph capture and replay; a mid-window resume
  through state_dict; create_optimizer with layerwise_lr_decay against the oracle; the host session's refusal.
"""
import ctypes as C
import zlib

import numpy as np
import pytest

import oracle_np as onp
from apply_matrix import Case, LockStep, matrix_cases
from common import make_params, rel_err
from composed_oracle import ComposedReferenceTrainOp

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

F32 = np.float32
# the apply matrix's model: tails, a multi-tile tensor, one element, a zero-element tensor, a tensor without a gradient
MAN = [("a/kernel", (2 * 2048 + 777,)), ("a/bias", (5,)), ("one/kernel", (1,)), ("empty/kernel", (0,)),
       ("LayerNorm/gamma", (33,)), ("nograd/kernel", (64,)), ("t/kernel", (3, 1367))]
NOGRAD = (5,)
TINY = [(f"tiny{i}/{'bias' if i % 3 == 0 else 'kernel'}", (1 + i % 7,)) for i in range(300)]
STEPS = 10
INF_AT = (4, 0, 1000)
EMA = (0.9, True)
CYCLE = (0.37, 0.0, 2.5, 1.0)      # below 1, 0, above 1, 1


def _table(n):
    return [CYCLE[i % len(CYCLE)] for i in range(n)]


@pytest.mark.parametrize("case", matrix_cases(), ids=lambda c: c.id)
def test_apply_instantiation_with_a_table_matches_the_oracle(case: Case):
    layout = "packed" if case.layout == "packed" else "table"
    dtype = case.layout.split("_")[-1] if layout == "table" else "fp32"
    man = MAN + TINY if case.layout.startswith("t1920") else MAN
    run = LockStep(man, case.variant, case.mode, layout, dtype, case.has_g, EMA if case.ema else None, N=3,
                   seed=zlib.crc32(case.id.encode()), nograd=NOGRAD, lr_mult=_table(len(man)))
    ls = case.mode.startswith("ls_")
    run.run(STEPS, inf_at=INF_AT if ls else None)
    if ls:
        st = run.op.loss_scale_state()
        assert st["skipped_windows"] == 1 and not st["last_skipped"]


# ---- oracle-free identities -------------------------------------------------------------------------------------------
SMAN = [("a/kernel", (777,)), ("a/bias", (5,)), ("b/kernel", (3, 1367)), ("t/kernel", (2055,)), ("one", (1,)),
        ("LayerNorm/gamma", (33,)), ("nograd/kernel", (64,))]
SNOGRAD = 6
SCHED = dict(init_lr=1e-2, num_train_steps=40, num_warmup_steps=4)
MODES = ["noclip", "clip", "ls_noclip", "ls_clip"]
VARIANTS = ["adamw", "adam", "lamb"]


def _g():
    import gaccum_b200 as g
    return g


def _bits(t):
    return t.contiguous().view(torch.int32) if t.element_size() == 4 else t.contiguous().view(torch.int16)


def _same(x, y):
    return torch.equal(_bits(x), _bits(y))


def _lr(s):
    return _g().learning_rate(SCHED["init_lr"], SCHED["num_train_steps"], SCHED["num_warmup_steps"], s)


def _hp(variant, mode):
    g = _g()
    clip = 0.5 if mode in ("clip", "ls_clip") else 0.0
    if variant == "lamb":
        return g.HParams.lamb(clip_norm=clip)
    if variant == "adam":
        return g.HParams(g.ADAM, 0, 0.9, 0.999, 1e-8, 0.0, clip)
    return g.HParams(g.ADAM_WEIGHT_DECAY, 0, 0.9, 0.999, 1e-6, 0.01, clip)


def _params(seed, dtype=torch.float32):
    rng = np.random.default_rng(seed)
    ps = [rng.normal(0, 0.05, s).astype(F32) for _, s in SMAN]
    return ps if dtype == torch.float32 else [torch.from_numpy(p).to(dtype).float().numpy() for p in ps]


def _op(params, variant, mode, N, dtype=torch.float32, **kw):
    from gaccum_b200.train_op import GaccumTrainOp
    g = _g()
    ls = g.LossScaleConfig(16.0, 2.0, 2) if mode.startswith("ls_") else None
    return GaccumTrainOp([torch.from_numpy(p.copy()).cuda().to(dtype) for p in params], [n for n, _ in SMAN],
                         _hp(variant, mode), N, kw.pop("lr_fn", _lr), loss_scale=ls, **kw)


def _grads(rng, S=1.0, inf=False):
    out = [None if i == SNOGRAD else (rng.normal(0, 0.1, s) * S).astype(F32) for i, (_, s) in enumerate(SMAN)]
    if inf:
        out[0][3] = np.inf
    return out


def _cuda(grads, dtype=torch.float32):
    return [None if x is None else torch.from_numpy(x).cuda().to(dtype) for x in grads]


def _state(op):
    out = [op.accum, op.m, op.v] + list(op.params)
    if op.master is not None:
        out.append(op.master)
    if op._ls_state is not None:
        out.append(op._ls_state)
    return out


def _check_same(a, b, stats_lr=True):
    torch.cuda.synchronize()
    for i, (x, y) in enumerate(zip(_state(a), _state(b))):
        assert _same(x, y), i
    sa, sb = a.stats(), b.stats()
    if not stats_lr:
        sa.pop("lr"); sb.pop("lr")
    x, y = (np.array(list(s.values()), F32) for s in (sa, sb))
    assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
    if a.hp.variant == _g().LAMB:
        assert np.array_equal(a.trust_ratios(), b.trust_ratios())


def _drive(ops, mode, steps, seed, dtype=torch.float32, check=None):
    rng = np.random.default_rng(seed)
    for s in range(steps):
        S = float(ops[0].loss_scale_state()["scale"]) if mode.startswith("ls_") else 1.0
        gr = _cuda(_grads(rng, S, inf=mode.startswith("ls_") and s == 4), dtype)
        applied = [op.run(gr) for op in ops]
        assert len(set(applied)) == 1
        if check is not None:
            check(s, applied[0])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("variant", VARIANTS)
def test_table_of_ones_is_no_table(variant, mode):
    params = _params(1)
    a = _op(params, variant, mode, 3, lr_multipliers=[1.0] * len(SMAN))
    b = _op(params, variant, mode, 3)
    assert a.lr_multipliers.dtype == np.float32 and (a.lr_multipliers == 1).all() and not a.lr_multipliers.flags.writeable
    _drive([a, b], mode, 10, 2, check=lambda s, applied: _check_same(a, b))


@pytest.mark.parametrize("m", [0.3, 3.0])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("variant", VARIANTS)
def test_uniform_multiplier_is_a_scaled_schedule(variant, mode, m):
    params = _params(3)
    a = _op(params, variant, mode, 3, lr_multipliers=[m] * len(SMAN))
    b = _op(params, variant, mode, 3, lr_fn=lambda s: float(np.multiply(F32(_lr(s)), F32(m), dtype=F32)))

    def check(s, applied):
        _check_same(a, b, stats_lr=False)
        assert a.stats()["lr"] == _lr(s)                 # stats.lr stays the schedule's lr
    _drive([a, b], mode, 10, 4, check=check)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("variant", VARIANTS)
def test_multiplier_zero_freezes_weights_while_moments_advance(variant, mode, dtype):
    params = _params(5, dtype)
    mult = [0.0, 1.0, 0.0, 2.0, 0.5, 1.0, 0.0]
    op = _op(params, variant, mode, 2, dtype, lr_multipliers=mult)
    w0 = [(p.clone(), None if op.master is None else op.master_view(i).clone()) for i, p in enumerate(op.params)]
    _drive([op], mode, 7, 6, dtype)
    torch.cuda.synchronize()
    for i, mu in enumerate(mult):
        p0, m0 = w0[i]
        if mu == 0.0:
            assert _same(op.params[i], p0), i
            if m0 is not None:
                assert _same(op.master_view(i), m0), i
            if i != SNOGRAD:
                assert op.m_view(i).abs().sum() > 0 and op.v_view(i).abs().sum() > 0, i
        else:
            assert not torch.equal(op.params[i], p0), i


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("variant", VARIANTS)
def test_16_bit_model_is_the_upcast_fp32_run(variant, dtype):
    params = _params(7, dtype)                           # representable in the 16-bit dtype
    mult = _table(len(SMAN))
    h = _op(params, variant, "clip", 3, dtype, lr_multipliers=mult)
    f = _op(params, variant, "clip", 3, lr_multipliers=mult)
    rng = np.random.default_rng(8)
    for s in range(10):
        gr = _cuda(_grads(rng), dtype)
        assert h.run(gr) == f.run([None if x is None else x.float() for x in gr])
        torch.cuda.synchronize()
        for i in range(len(SMAN)):
            assert _same(h.master_view(i), f.params[i]), i
            assert _same(h.params[i], f.params[i].to(dtype)), i
        for x, y in ((h.m, f.m), (h.v, f.v), (h.accum, f.accum)):
            assert _same(x, y)


# Adam and LAMB take their beta powers from the step's arguments unless loss scaling keeps them on the device: a replayed
# graph reuses the captured arguments, so those two run loss-scaled here to be comparable with eager launches
@pytest.mark.parametrize("variant, mode", [("adamw", "noclip"), ("adamw", "clip"), ("adam", "ls_noclip"), ("lamb", "ls_clip")])
def test_graph_capture_and_replay(variant, mode):
    params = _params(9)
    mult = _table(len(SMAN))
    gr = _cuda(_grads(np.random.default_rng(10)))
    lr_fn = lambda s: 1e-2
    eager = _op(params, variant, mode, 1, lr_multipliers=mult, lr_fn=lr_fn)
    op = _op(params, variant, mode, 1, lr_multipliers=mult, lr_fn=lr_fn)
    for _ in range(3):
        eager.apply_only(gr)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        op.apply_only(gr)                                  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(stream)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        op.apply_only(gr)
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    for x, y in zip(_state(op), _state(eager)):
        assert _same(x, y)


@pytest.mark.parametrize("variant, mode", [("adamw", "clip"), ("adam", "noclip"), ("lamb", "ls_clip")])
def test_resume_mid_window_is_bit_identical(variant, mode):
    params = _params(11)
    mult = _table(len(SMAN))
    N = 4
    rng = np.random.default_rng(12)
    raw = [_grads(rng) for _ in range(3 * N)]
    full = _op(params, variant, mode, N, lr_multipliers=mult)
    first = _op(params, variant, mode, N, lr_multipliers=mult)
    second = _op(_params(99), variant, mode, N, lr_multipliers=mult)

    def feed(op, grads):
        S = float(op.loss_scale_state()["scale"]) if mode.startswith("ls_") else 1.0
        op.run(_cuda([None if x is None else (x * S).astype(F32) for x in grads]))
    for x in raw:
        feed(full, x)
    cut = N + 2
    for x in raw[:cut]:
        feed(first, x)
    sd = first.state_dict()
    assert not any("mult" in k for k in sd)              # configuration, not state
    second.load_state_dict(sd)
    for x in raw[cut:]:
        feed(second, x)
    torch.cuda.synchronize()
    for x, y in zip(_state(full), _state(second)):
        assert _same(x, y)


def test_create_optimizer_with_layerwise_lr_decay(monkeypatch):
    from gaccum_b200 import graph, optimization as opt
    monkeypatch.setattr(opt, "layerwise_lr_decay", 0.8)
    monkeypatch.setattr(opt, "gradient_accumulation_multiplier", 2)
    graph.reset_default_graph()
    man = onp.bert_manifest(3, 32, vocab=64, max_pos=16)
    params = make_params(man, np.random.default_rng(13))
    tv = [graph.add_variable(n, torch.from_numpy(p.copy()).cuda()) for (n, _), p in zip(man, params)]
    train_op = opt.create_optimizer(None, 1e-3, 50, 3, False)
    names = [n for n, _ in man]
    expect = [0.8 ** 5 if "/embeddings/" in n else
              next((0.8 ** (4 - i) for i in range(3) if f"encoder/layer_{i}/" in n), 1.0) for n in names]
    assert np.array_equal(train_op.engine.lr_multipliers, np.array(expect, F32))
    ref = ComposedReferenceTrainOp([p.copy() for p in params], names, onp.HParams.bert(), 2, lr_mult=expect,
                                   init_lr=1e-3, num_train_steps=50, num_warmup_steps=3)
    rng = np.random.default_rng(14)
    for _ in range(9):
        gr = [rng.normal(0, 0.1, s).astype(F32) for _, s in man]
        ref.run(gr)
        train_op.run_with_grads(_cuda(gr))
    torch.cuda.synchronize()
    for v, exp in zip(tv, ref.params):
        assert rel_err(v.tensor.cpu().numpy(), exp) <= 1e-5, v.name


def test_apply_gradients_takes_the_table():
    from gaccum_b200 import graph, optimization as opt
    graph.reset_default_graph()
    man = [("bert/embeddings/word_embeddings", (16, 8)), ("bert/encoder/layer_0/output/dense/kernel", (8, 8)),
           ("output_weights", (2, 8))]
    params = make_params(man, np.random.default_rng(15))
    tv = [graph.add_variable(n, torch.from_numpy(p.copy()).cuda()) for (n, _), p in zip(man, params)]
    table = {"/embeddings/": 0.25, "encoder/layer_0/": 0.5}
    o = opt.AdamWeightDecayOptimizer(1e-2, weight_decay_rate=0.01,
                                     exclude_from_weight_decay=["LayerNorm", "layer_norm", "bias"])
    o.lr_multipliers = table
    ref = ComposedReferenceTrainOp([p.copy() for p in params], [n for n, _ in man],
                                   onp.HParams(weight_decay_rate=0.01, clip_norm=0.0), 1, lr_mult=[0.25, 0.5, 1.0],
                                   constant_lr=1e-2)
    rng = np.random.default_rng(16)
    for _ in range(3):
        gr = [rng.normal(0, 0.1, s).astype(F32) for _, s in man]
        ref.run(gr)
        o.apply_gradients(list(zip(_cuda(gr), tv)))
    torch.cuda.synchronize()
    for v, exp in zip(tv, ref.params):
        assert np.array_equal(v.tensor.cpu().numpy().view(np.uint32), exp.view(np.uint32)), v.name


def test_host_session_step_refuses_a_table():
    g = _g()
    from gaccum_b200 import _lib
    L = _lib._load()
    plan = g.Plan([100, 7], [True, False], g.HParams.bert(), device=0)
    s = _lib.HostSession(plan)                             # created before the table: its step refuses the plan
    plan.set_lr_multipliers([0.5, 1.0])
    host = [torch.zeros(100), torch.zeros(7)]
    ptrs = g.Plan.ptr_array([t.data_ptr() for t in host])
    args = _lib.StepArgs(1, 2, 0, 1e-3, 0.9, 0.999, 0.0)
    assert L.gaccum_step_host(s._h, ptrs, None, C.byref(args), None) == _lib.EINVAL
    assert "learning-rate multipliers" in L.gaccum_last_error().decode()
    s.close()
