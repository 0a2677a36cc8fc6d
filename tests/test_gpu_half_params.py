"""bf16 / fp16 models with fp32 master weights on the GPU (gaccum_plan_set_param_dtype, GaccumTrainOp).

Widening a 16-bit number to fp32 is exact, so a 16-bit run is checked bit for bit against the REFERENCE RUN: the fp32
train op whose parameters start at the upcast model weights and which is fed the upcast gradients.
* master weights, m, v, the accumulators and the stats equal the reference run's p, m, v, accumulators and stats;
* after every step the model's tensors hold the master weights rounded to nearest-even (torch's ``.to(dtype)``);
across optimizer variants, clip 0 / 1.0 / 1e-3, N in {1, 3, 4}, tails, a 2055-element tile, a one-element tensor, and
model / gradient views that are 16-, only 8- or only 2-byte aligned (bulk copy + stash, vector and element paths).
"""
import numpy as np
import pytest

import oracle_c
import oracle_np as onp

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
MAN = [("a/kernel", (777,)), ("a/bias", (5,)), ("b/kernel", (3, 1367)), ("t/kernel", (2055,)), ("one", (1,)),
       ("LayerNorm/gamma", (33,))]
LR = 1e-3


def _g():
    import gaccum_b200 as g
    return g


def _hp(variant_b, clip):
    g = _g()
    hp = g.HParams.tf_adam() if variant_b else g.HParams.bert()
    hp.clip_norm = clip
    return hp


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _same(x, y):
    """Bit-equal, except that NaNs only have to sit at the same positions (conversions may canonicalise payloads)."""
    if x.dtype != y.dtype or x.shape != y.shape:
        return False
    nx, ny = torch.isnan(x), torch.isnan(y)
    if not torch.equal(nx, ny):
        return False
    return torch.equal(_bits(torch.where(nx, torch.zeros_like(x), x)), _bits(torch.where(ny, torch.zeros_like(y), y)))


def _carve(values, dtype, align):
    """Device copies of `values` (fp32 tensors) in `dtype`, each starting at an address that is 16-byte aligned, or
    8-byte but not 16-byte aligned, or 2-byte but not 4-byte aligned."""
    shift = {16: 0, 8: 4, 2: 1}[align]
    total = sum(v.numel() + 16 for v in values) + 16
    buf = torch.zeros(total, dtype=dtype, device="cuda")
    out, cur = [], 0
    for v in values:
        cur = (cur + 7) // 8 * 8 + shift
        t = buf[cur:cur + v.numel()].view(v.shape)
        t.copy_(v.to(dtype))
        assert t.data_ptr() % 16 == 2 * shift
        out.append(t)
        cur += v.numel()
    return out


def _params(man, seed):
    gen = torch.Generator().manual_seed(seed)
    return [torch.randn(s, generator=gen) * 0.05 for _, s in man]


def _pair(man, dtype, hp, N, align=16, ls=None, seed=1, global_step=0):
    """(16-bit op, its model tensors, the fp32 reference op)."""
    from gaccum_b200.train_op import GaccumTrainOp
    names = [n for n, _ in man]
    model = _carve(_params(man, seed), dtype, align)
    ref = GaccumTrainOp([p.float() for p in model], names, hp, N, lambda s: LR, global_step=global_step, loss_scale=ls)
    op = GaccumTrainOp(model, names, hp, N, lambda s: LR, global_step=global_step, loss_scale=ls)
    assert op.param_dtype == dtype and op.master is not None and ref.master is None
    return op, model, ref


def _check(op, model, ref, what):
    for i in range(len(model)):
        assert _same(op.master_view(i), ref.params[i]), f"master {i} {what}"
        assert _same(model[i], ref.params[i].to(model[i].dtype)), f"model copy {i} {what}"
    for x, y, n in ((op.m, ref.m, "m"), (op.v, ref.v, "v"), (op.accum, ref.accum, "accum")):
        assert _same(x, y), f"{n} {what}"


def _step(op, ref, grads32, dtype, align):
    gh = _carve(grads32, dtype, align)
    a = ref.run([x.float() for x in gh])
    b = op.run(gh)
    assert a == b
    if a:                                            # an overflowed window reports a NaN norm: compare bits
        st = lambda o: torch.tensor([float(x) for x in o.stats().values()], dtype=torch.float32)
        assert _same(st(op), st(ref))
    return a


# ---- bit-identity with the reference run ---------------------------------------------------------------------------
@pytest.mark.parametrize("align", [16, 8, 2])
@pytest.mark.parametrize("N", [1, 3, 4])
@pytest.mark.parametrize("clip", [0.0, 1.0, 1e-3])
@pytest.mark.parametrize("variant_b", [False, True])
@pytest.mark.parametrize("dtype", DTYPES)
def test_bit_identical_to_the_fp32_reference_run(dtype, variant_b, clip, N, align):
    op, model, ref = _pair(MAN, dtype, _hp(variant_b, clip), N, align)
    _check(op, model, ref, "at start")
    gen = torch.Generator().manual_seed(7)
    applies, scales = 0, set()
    for step in range(3 * N + 1):
        grads = [torch.randn(s, generator=gen) * 0.1 for _, s in MAN]
        if _step(op, ref, grads, dtype, align):
            applies += 1
            scales.add(op.stats()["clip_scale"])
        _check(op, model, ref, f"step {step}")
    assert applies >= 3
    if clip == 1e-3:
        assert scales != {1.0}


@pytest.mark.parametrize("dtype", DTYPES)
def test_apply_without_gradients_and_tensors_without_a_gradient(dtype):
    """apply_only(None) applies the accumulators as they are; a tensor without a gradient still gets its model copy."""
    op, model, ref = _pair(MAN, dtype, _hp(False, 1.0), 3)
    gen = torch.Generator().manual_seed(3)
    grads = [torch.randn(s, generator=gen) * 0.1 for _, s in MAN]
    with torch.no_grad():
        for x in model:
            x.zero_()                        # the apply must rewrite every model tensor
    gh = _carve(grads, dtype, 16)
    ref.accumulate_only([x.float() for x in gh])
    op.accumulate_only(gh)
    ref.apply_only(None)
    op.apply_only(None)
    _check(op, model, ref, "apply_only(None)")
    ref.global_step = op.global_step = 0
    sparse = [None if i % 2 else x for i, x in enumerate(_carve(grads, dtype, 16))]
    ref.run([None if x is None else x.float() for x in sparse])
    op.run(sparse)
    _check(op, model, ref, "tensors without a gradient")


# ---- the model copy: round to nearest-even, as torch's .to(dtype) ---------------------------------------------------
def _special_values():
    f = np.float32
    v = [0.0, -0.0, 1.0, -1.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11,
         1.0 + 2.0 ** -12, 65504.0, 65519.0, 65520.0, 65536.0, 1e5, -1e5, 3.3895e38, 3.4e38, -3.4e38,
         2.0 ** -14, 2.0 ** -20, 3e-6, 6e-8, 2.0 ** -25, 2.0 ** -25 * 1.5, 2.0 ** -26, 1e-30, 1e-40, -1e-40,
         2.0 ** -126, 2.0 ** -133, np.inf, -np.inf, np.nan]
    rng = np.random.default_rng(5)
    v += list(rng.standard_normal(200) * 10.0 ** rng.integers(-9, 9, 200))
    return torch.tensor(np.array(v, dtype=f))


@pytest.mark.parametrize("path", ["clip", "noclip"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_model_copy_rounds_to_nearest_even(dtype, path):
    """lr = 0 and no weight decay (tf_adam): the apply leaves the master weights as they are and stores their rounding."""
    from gaccum_b200.train_op import GaccumTrainOp
    vals = _special_values()
    n = vals.numel()
    man = [("x", (n,)), ("y", (n + 3,))]
    hp = _hp(True, 1.0 if path == "clip" else 0.0)
    for align in (16, 2):
        model = _carve([torch.zeros(n), torch.zeros(n + 3)], dtype, align)
        op = GaccumTrainOp(model, [m for m, _ in man], hp, 1, lambda s: 0.0)
        with torch.no_grad():
            op.master_view(0).copy_(vals)
            op.master_view(1)[3:].copy_(vals)
        op.run([torch.zeros_like(model[0]), torch.zeros_like(model[1])])
        torch.cuda.synchronize()
        assert _same(op.master_view(0).cpu(), vals)
        for i in range(2):
            assert _same(model[i], op.master_view(i).to(dtype)), (align, i)


# ---- first accumulate of a window: accum = +0 + float(G) ------------------------------------------------------------
@pytest.mark.parametrize("align", [16, 8, 2])
@pytest.mark.parametrize("dtype", DTYPES)
def test_first_accumulate_of_a_window_with_special_gradients(dtype, align):
    from gaccum_b200.train_op import GaccumTrainOp
    tiny = 2.0 ** -133 if dtype == torch.bfloat16 else 2.0 ** -24          # a subnormal of the dtype
    special = torch.tensor([0.0, -0.0, float("nan"), float("inf"), -float("inf"), tiny, -tiny, 3 * tiny, 1.5, -2.5])
    n = 2055
    g = torch.randn(n) * 0.1
    g[:special.numel()] = special
    g[-special.numel():] = special
    op = GaccumTrainOp(_carve([torch.zeros(n)], dtype, 16), ["w"], _hp(True, 0.0), 2, lambda s: LR)
    op.run(_carve([torch.randn(n)], dtype, 16))               # g = 0 applies
    with torch.no_grad():
        op.accum.fill_(0.0)                                    # what the apply leaves (and the precondition)
    gh = _carve([g], dtype, align)[0]
    assert not op.run([gh])                                    # g = 1: first accumulate of the window
    expect = torch.zeros(n, device="cuda") + gh.float()
    assert _same(op.accum_view(0), expect)
    assert not torch.signbit(op.accum_view(0)[1])              # -0 became +0


# ---- the 1920-entry pointer table -----------------------------------------------------------------------------------
@pytest.mark.parametrize("clip", [0.0, 1.0])
@pytest.mark.parametrize("dtype", DTYPES)
def test_more_than_256_tensors(dtype, clip):
    rng = np.random.default_rng(11)
    man = [(f"t{i}/kernel", (int(rng.integers(1, 70)),)) for i in range(300)] + [("big", (5000,))]
    op, model, ref = _pair(man, dtype, _hp(False, clip), 2, align=8)
    gen = torch.Generator().manual_seed(2)
    for step in range(5):
        _step(op, ref, [torch.randn(s, generator=gen) * 0.1 for _, s in man], dtype, 8)
        _check(op, model, ref, f"step {step}")


# ---- fp16 with loss scaling: overflowed windows ---------------------------------------------------------------------
BIG = 1700 * 2048 + 5      # more tiles than the clip kernel's stash holds (4 per group x 3 groups x 132 SMs): pool tiles


@pytest.mark.parametrize("bad", [float("inf"), float("nan")])
@pytest.mark.parametrize("where", ["stash", "pool"])
@pytest.mark.parametrize("at", ["first", "middle", "apply"])
@pytest.mark.parametrize("clip", [0.0, 1.0])
def test_fp16_loss_scaling_skips_overflowed_windows(clip, at, where, bad):
    g = _g()
    N = 3
    man = [("big", (BIG,)), ("b", (37,)), ("one", (1,))]
    ls = g.LossScaleConfig(2.0 ** 10, 2.0, 100)
    op, model, ref = _pair(man, torch.float16, _hp(clip == 0.0, clip), N, ls=ls)
    gen = torch.Generator().manual_seed(4)

    def grads():                                     # gradients of loss * S
        S = op.loss_scale_state()["scale"]
        return [torch.randn(s, generator=gen) * 1e-3 * S for _, s in man]

    for step in range(N + 1):                        # two applied windows: g = 0 and g = 1..3
        _step(op, ref, grads(), torch.float16, 16)
    _check(op, model, ref, "before the window")
    before = [t.clone() for t in [op.master, op.m, op.v] + model]
    S = op.loss_scale_state()["scale"]
    k = {"first": 0, "middle": 1, "apply": 2}[at]
    idx = 5 if where == "stash" else BIG - 3
    for j in range(N):
        gr = grads()
        if j == k:
            gr[0][idx] = bad
        _step(op, ref, gr, torch.float16, 16)
        _check(op, model, ref, f"micro-step {j} of the overflowed window")
    st = op.loss_scale_state()
    assert st["last_skipped"] and st["scale"] == S / 2 and st["skipped_windows"] == 1
    for x, y in zip([op.master, op.m, op.v] + model, before):
        assert _same(x, y)
    for step in range(2 * N):                        # later windows: still the reference run
        _step(op, ref, grads(), torch.float16, 16)
        _check(op, model, ref, f"after, step {step}")
    assert not op.loss_scale_state()["last_skipped"]


# ---- full-size BERT-Small in bf16 against the C oracle fed upcast gradients -----------------------------------------
def test_bert_small_full_size_bf16_against_the_oracle():
    g = _g()
    from gaccum_b200.train_op import GaccumTrainOp
    BERT = dict(init_lr=2e-5, num_train_steps=207900, num_warmup_steps=20790)
    man = onp.MANIFESTS["bert_small"]()
    names = [n for n, _ in man]
    rng = np.random.Generator(np.random.PCG64(19830610))
    model = [torch.from_numpy(rng.standard_normal(s, dtype=np.float32) * np.float32(0.02)).cuda().to(torch.bfloat16)
             for _, s in man]
    ref = oracle_c.COracleTrainOp([m.float().cpu().numpy() for m in model], names, onp.HParams.bert(), 4,
                                  global_step=100000, **BERT)
    lr_fn = lambda s: g.learning_rate(BERT["init_lr"], BERT["num_train_steps"], BERT["num_warmup_steps"], s)
    op = GaccumTrainOp(model, names, g.HParams.bert(), 4, lr_fn, global_step=100000)
    for s in range(5):
        grng = np.random.Generator(np.random.PCG64(1000 + s))
        gh = [torch.from_numpy(grng.standard_normal(sh, dtype=np.float32) * np.float32(1e-3)).cuda().to(torch.bfloat16)
              for _, sh in man]
        info = ref.run([x.float().cpu().numpy() for x in gh])
        assert op.run(gh) == info.applied
        if info.applied:
            st = op.stats()
            assert abs(st["global_norm"] - float(info.global_norm)) <= 2e-6 * float(info.global_norm)
            for i in range(len(man)):
                for got, exp in ((op.master_view(i).cpu().numpy(), ref.params[i]), (op.m_view(i).cpu().numpy(), ref.m[i]),
                                 (op.v_view(i).cpu().numpy(), ref.v[i])):
                    d = np.max(np.abs(got.astype(np.float64) - exp)) / max(np.max(np.abs(exp)), 1e-30)
                    assert d <= 1e-5, f"tensor {i} ({names[i]}) rel err {d} at step {s}"
                assert _same(model[i], op.master_view(i).to(torch.bfloat16))
        for i in range(len(man)):
            assert np.array_equal(op.accum_view(i).cpu().numpy(), ref.accum[i])


# ---- the drop-in API and checkpoints --------------------------------------------------------------------------------
def _module(dtype):
    torch.manual_seed(0)
    return torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.Tanh(), torch.nn.Linear(32, 4)).cuda().to(dtype)


@pytest.mark.parametrize("dtype,loss_scaled", [(torch.bfloat16, False), (torch.float16, True), (torch.bfloat16, True)])
def test_drop_in_api_on_a_16_bit_module(dtype, loss_scaled):
    g = _g()
    from gaccum_b200 import graph, optimization
    from gaccum_b200.train_op import GaccumTrainOp
    graph.reset_default_graph()
    net = _module(dtype)
    tvars = graph.register_module(net)
    x = torch.randn(8, 16, device="cuda", dtype=dtype)
    y = torch.randn(8, 4, device="cuda", dtype=dtype)
    loss = lambda: ((net(x) - y).float() ** 2).mean()
    ls = g.LossScaleConfig(2.0 ** 8, 2.0, 3) if loss_scaled else None
    opt = optimization.AdamWeightDecayOptimizer(1e-3, weight_decay_rate=0.01, exclude_from_weight_decay=["bias"])
    top = optimization.gradient_accumulation_train_op(loss, opt, 3, clip_norm=1.0, loss_scale=ls)
    eng = top.engine
    assert eng.param_dtype == dtype
    ref = GaccumTrainOp([v.tensor.float() for v in tvars], [v.name for v in tvars], opt._hparams(1.0), 3,
                        lambda s: 1e-3, exclude_from_weight_decay=["bias"], loss_scale=ls)
    for step in range(8):
        grads = top.gradients()
        assert all(gr.dtype == dtype for gr in grads)
        assert ref.run([gr.float() for gr in grads]) == top.run_with_grads(grads)
        for i, v in enumerate(tvars):
            assert _same(eng.master_view(i), ref.params[i]), step
            assert _same(v.tensor, ref.params[i].to(dtype)), step
        for a, b in ((eng.m, ref.m), (eng.v, ref.v), (eng.accum, ref.accum)):
            assert _same(a, b), step
    sd = top.state_dict()
    for i, n in enumerate(eng.names):
        assert sd[n].dtype == torch.float32 and _same(sd[n], eng.master_view(i))


@pytest.mark.parametrize("dtype", DTYPES)
def test_tf_checkpoint_mid_window_resumes_bit_identically(dtype, tmp_path):
    from gaccum_b200 import tf_checkpoint
    from gaccum_b200.train_op import GaccumTrainOp
    hp, N = _hp(False, 1.0), 3
    op, model, _ = _pair(MAN, dtype, hp, N)
    gen = torch.Generator().manual_seed(9)
    grads = [[torch.randn(s, generator=gen) * 0.1 for _, s in MAN] for _ in range(9)]
    for gr in grads[:5]:                                     # g = 0 applies, g = 1..3 a window, g = 4 mid-window
        op.run(_carve(gr, dtype, 16))
    tf_checkpoint.save(str(tmp_path), op)
    fresh_model = _carve([torch.zeros(s) for _, s in MAN], dtype, 16)
    fresh = GaccumTrainOp(fresh_model, [n for n, _ in MAN], hp, N, lambda s: LR)
    tf_checkpoint.restore(str(tmp_path), fresh)
    assert fresh.global_step == op.global_step == 5
    for i in range(len(MAN)):
        assert _same(fresh_model[i], model[i])
    for gr in grads[5:]:
        assert op.run(_carve(gr, dtype, 16)) == fresh.run(_carve(gr, dtype, 16))
        for a, b in ((op.master, fresh.master), (op.m, fresh.m), (op.v, fresh.v), (op.accum, fresh.accum)):
            assert _same(a, b)
        for a, b in zip(model, fresh_model):
            assert _same(a, b)


@pytest.mark.parametrize("dtype", DTYPES)
def test_fp32_and_16_bit_checkpoints_load_into_each_other(dtype):
    from gaccum_b200.train_op import GaccumTrainOp
    hp = _hp(True, 0.0)
    names = [n for n, _ in MAN]
    op32 = GaccumTrainOp([p.cuda() for p in _params(MAN, 3)], names, hp, 2, lambda s: LR)
    gen = torch.Generator().manual_seed(1)
    for _ in range(3):
        op32.run([torch.randn(s, generator=gen).cuda() * 0.1 for _, s in MAN])
    sd = op32.state_dict()
    model = _carve([torch.zeros(s) for _, s in MAN], dtype, 2)
    half = GaccumTrainOp(model, names, hp, 2, lambda s: LR)
    half.load_state_dict(sd)
    for i in range(len(MAN)):
        assert _same(half.master_view(i), op32.params[i])
        assert _same(model[i], op32.params[i].to(dtype))
    back = GaccumTrainOp([torch.zeros(s).cuda() for _, s in MAN], names, hp, 2, lambda s: LR)
    back.load_state_dict(half.state_dict())
    for i in range(len(MAN)):
        assert _same(back.params[i], op32.params[i])
    for a, b in ((back.m, op32.m), (back.v, op32.v), (back.accum, op32.accum)):
        assert _same(a, b)


# ---- Python refusals ------------------------------------------------------------------------------------------------
def test_python_refusals():
    g = _g()
    from gaccum_b200.distributed import DataParallelTrainOp
    from gaccum_b200.train_op import GaccumTrainOp, HostTrainOp, PackedTrainOp
    hp = g.HParams.bert()
    with pytest.raises(ValueError, match="mixed dtypes"):
        GaccumTrainOp([torch.zeros(4, device="cuda", dtype=torch.bfloat16), torch.zeros(4, device="cuda")], ["a", "b"],
                      hp, 2, lambda s: LR)
    for dt, other in ((torch.bfloat16, torch.float16), (torch.float16, torch.float32), (torch.bfloat16, torch.float32)):
        op = GaccumTrainOp([torch.zeros(4, device="cuda", dtype=dt)], ["a"], hp, 2, lambda s: LR)
        with pytest.raises(ValueError, match="gradients of a"):
            op.run([torch.zeros(4, device="cuda", dtype=other)])
        with pytest.raises(ValueError, match="multi-GPU"):
            DataParallelTrainOp(op)
        with pytest.raises(ValueError, match="does not support"):
            op.run_host([torch.zeros(4, dtype=dt)])
        with pytest.raises(ValueError, match="PackedTrainOp"):
            PackedTrainOp([torch.zeros(4, device="cuda", dtype=dt)], ["a"], hp, 2, lambda s: LR)
        with pytest.raises(ValueError, match="HostTrainOp"):
            HostTrainOp([torch.zeros(4, dtype=dt)], ["a"], hp, 2, lambda s: LR)
