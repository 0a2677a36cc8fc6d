"""The LAMB apply step on the GPU (include/gaccum.h, GACCUM_LAMB; csrc/gaccum_lamb.cuh).

* Trajectories against the numpy oracle (tests/composed_oracle.py): p within 1e-5; m / v as the AdamWeightDecay parity
  tests hold them (bit-exact without clipping); the accumulators +0; the trust ratios within 1e-6.
* Determinism: p and the ratios are bit-identical over repeated launches and CUDA-graph replays.
* Layout: one 30522 x 1024 tensor, 1920 tiny tensors, unaligned views, the packed entry point, full-size BERT-Small.
* bf16 / fp16 models are bit-identical to the upcast fp32 run; fp16 loss scaling skips overflowed windows exactly.
* Resume through state_dict and a TF-format checkpoint, and create_optimizer with optimizer_type = "lamb".
"""
import numpy as np
import pytest

import oracle_np as onp
from common import make_params, rel_err
from composed_oracle import ComposedReferenceTrainOp

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

# tails, a vector body with a 7-element tail (2055), several tiles, one element; decay and adaptation masks differ:
# weight decay skips LayerNorm and bias, layer adaptation skips LayerNorm only
MAN = [("a/kernel", (777,)), ("a/bias", (5,)), ("b/kernel", (3, 1367)), ("t/kernel", (2055,)), ("one", (1,)),
       ("LayerNorm/gamma", (33,)), ("nograd/kernel", (64,))]
NOGRAD = 6
ADAPT_EXCLUDE = ["LayerNorm"]
SCHED = dict(init_lr=1e-2, num_train_steps=40, num_warmup_steps=4)     # warm-up: lr(0) = 0


def _g():
    import gaccum_b200 as g
    return g


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(x, y):
    return torch.equal(_bits(x), _bits(y))


def _params(man, seed):
    rng = np.random.default_rng(seed)
    return [rng.normal(0, 0.05, s).astype(np.float32) for _, s in man]


def _lr(s):
    return _g().learning_rate(SCHED["init_lr"], SCHED["num_train_steps"], SCHED["num_warmup_steps"], s)


def _hp(clip, wd=0.01):
    return _g().HParams.lamb(weight_decay_rate=wd, clip_norm=clip), \
        onp.HParams(variant=2, beta1=0.9, beta2=0.999, epsilon=1e-6, weight_decay_rate=wd, clip_norm=clip)


def _op(man, params, hp, N, dtype=torch.float32, **kw):
    from gaccum_b200.train_op import GaccumTrainOp
    return GaccumTrainOp([torch.from_numpy(p.copy()).cuda().to(dtype) for p in params], [n for n, _ in man], hp, N,
                         kw.pop("lr_fn", _lr), exclude_from_layer_adaptation=kw.pop("adapt_exclude", ADAPT_EXCLUDE), **kw)


def _ref(man, params, hp, N, **kw):
    return ComposedReferenceTrainOp([p.copy() for p in params], [n for n, _ in man], hp, N,
                                    adapt_exclude=kw.pop("adapt_exclude", ADAPT_EXCLUDE), **SCHED, **kw)


def _grads(man, rng, sigma=0.1, nograd=NOGRAD):
    return [None if i == nograd else rng.normal(0, sigma, s).astype(np.float32) for i, (_, s) in enumerate(man)]


def _cuda(grads, dtype=torch.float32):
    return [None if x is None else torch.from_numpy(x).cuda().to(dtype) for x in grads]


def _check(op, ref, exact_mv, tol_mv=1e-5):
    for i in range(len(ref.params)):
        p = op.params[i].float().cpu().numpy()
        assert rel_err(p, ref.params[i]) <= 1e-5, i
        for got, exp in ((op.m_view(i), ref.m[i]), (op.v_view(i), ref.v[i])):
            got = got.cpu().numpy()
            if exact_mv:
                assert np.array_equal(got, exp), i
            else:
                # with clipping the clip scale may differ in its last bit (the AdamWeightDecay parity tests' standard)
                assert np.allclose(got, exp, rtol=tol_mv, atol=1e-8), i
        assert not np.any(op.accum_view(i).cpu().numpy().view(np.uint32)), i
    np.testing.assert_allclose(op.trust_ratios(), np.asarray(ref.ratios, np.float32), rtol=1e-6, atol=0)


@pytest.mark.parametrize("N", [1, 3, 4])
@pytest.mark.parametrize("clip", [0.0, 1.0])
def test_trajectory_matches_oracle(clip, N):
    hp, hpo = _hp(clip)
    params = _params(MAN, 1)
    op, ref = _op(MAN, params, hp, N), _ref(MAN, params, hpo, N)
    assert op.adapt == ref.adapt and op.adapt[0] and op.adapt[1] and not op.adapt[5]
    assert op.decay == ref.decay and op.decay[0] and not op.decay[1]
    rng = np.random.default_rng(10 + N)
    for step in range(4 * N + 1):
        gr = _grads(MAN, rng)
        a, b = op.run(_cuda(gr)), ref.run(gr)
        assert a == b.applied
        if a:
            st = op.stats()
            assert st["applied"] and st["lr"] == b.lr
            if clip:
                assert abs(st["global_norm"] - b.global_norm) <= 1e-6 * b.global_norm
    torch.cuda.synchronize()
    # p and the ratios differ in the last bits at most (exact vs fp64 norms); m and v do not depend on p
    _check(op, ref, exact_mv=clip == 0.0)
    assert np.float32(op.beta1_power) == ref.beta1_power and np.float32(op.beta2_power) == ref.beta2_power
    assert all(r != 1.0 for r, a in zip(op.trust_ratios(), op.adapt) if a)


def test_known_answers_one_element_and_no_adaptation():
    """One adapted element moves by exactly lr*|p| (r*|u| = |p|); without adaptation the update is bias-corrected AdamW."""
    g = _g()
    man = [("x", (1,)), ("LayerNorm/y", (300,))]
    params = [np.array([0.75], np.float32), _params(man, 3)[1]]
    hp, hpo = _hp(0.0, wd=0.0)
    op = _op(man, params, hp, 1, lr_fn=lambda s: 0.125)
    grads = [np.array([0.3], np.float32), np.random.default_rng(4).normal(0, 1, 300).astype(np.float32)]
    op.run(_cuda(grads))
    torch.cuda.synchronize()
    assert float(op.params[0][0]) == pytest.approx(0.75 - 0.125 * 0.75, rel=1e-6)
    assert op.trust_ratios()[1] == 1.0
    # fp64 closed form with the fp32 constants the op uses: omb = fp32(1 - beta), 1 - beta_power with beta_power = fp32(beta)
    c = grads[1].astype(np.float64)
    f = lambda x: float(np.float32(x))
    m, v = f(1 - 0.9) * c, f(1 - 0.999) * c * c
    u = (m / (1 - f(0.9))) / (np.sqrt(v / (1 - f(0.999))) + f(1e-6))
    np.testing.assert_allclose(op.params[1].cpu().numpy(), params[1] - 0.125 * u, rtol=1e-6, atol=1e-7)
    assert g.LAMB == 2


def test_repeated_launches_and_graph_replays_are_bit_identical():
    hp, _ = _hp(1.0)
    params = _params(MAN, 5)
    N = 3
    rng = np.random.default_rng(6)
    window = [_cuda(_grads(MAN, rng)) for _ in range(N)]
    ops = [_op(MAN, params, hp, N) for _ in range(3)]
    for op in ops:
        op.global_step = 1
        for gr in window[:-1]:
            op.run(gr)
    snap = [(op.accum.clone(), op.m.clone(), op.v.clone()) for op in ops]
    b1, b2 = ops[0].beta1_power, ops[0].beta2_power
    for op in ops[:2]:
        op.apply_only(window[-1])
    torch.cuda.synchronize()
    p_ref, r_ref = [p.clone() for p in ops[0].params], ops[0].trust_ratios()
    assert all(_same(x, y) for x, y in zip(p_ref, ops[1].params)) and np.array_equal(r_ref, ops[1].trust_ratios())
    # ops[2]: capture the apply once, replay it from the same state three times
    op = ops[2]
    p0 = [p.clone() for p in op.params]
    gr = [None if x is None else x.clone() for x in window[-1]]
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        op.apply_only(gr)                        # warm-up outside the capture (kernel attributes, occupancy)
    torch.cuda.current_stream().wait_stream(stream)
    graph = torch.cuda.CUDAGraph()
    op.beta1_power, op.beta2_power = b1, b2
    with torch.cuda.graph(graph):
        op.apply_only(gr)
    for _ in range(3):
        for p, x in zip(op.params, p0):
            p.copy_(x)
        op.accum.copy_(snap[2][0]); op.m.copy_(snap[2][1]); op.v.copy_(snap[2][2])
        graph.replay()
        torch.cuda.synchronize()
        assert all(_same(x, y) for x, y in zip(p_ref, op.params))
        assert np.array_equal(r_ref, op.trust_ratios())
        assert not torch.any(op.accum)


def _one_apply(man, params, grads, clip=1.0, N=1):
    hp, hpo = _hp(clip)
    op, ref = _op(man, params, hp, N), _ref(man, params, hpo, N)
    for gr in grads:
        op.run(_cuda(gr))
        ref.run(gr)
    torch.cuda.synchronize()
    return op, ref


def test_one_large_tensor_spread_over_every_cta():
    man = [("bert/embeddings/word_embeddings", (30522, 1024)), ("LayerNorm/beta", (1024,))]
    rng = np.random.default_rng(7)
    params = [rng.normal(0, 0.02, s).astype(np.float32) for _, s in man]
    op, ref = _one_apply(man, params, [[rng.normal(0, 1e-3, s).astype(np.float32) for _, s in man]])
    assert op.plan.num_tiles > 15000
    _check(op, ref, exact_mv=False)


def test_1920_tiny_tensors():
    rng = np.random.default_rng(8)
    man = [(f"t{i}/{'bias' if i % 3 == 0 else 'kernel'}", (1 + i % 7,)) for i in range(1920)]
    params = [rng.normal(0, 0.1, s).astype(np.float32) for _, s in man]
    # without clipping m and v are bit-exact, so the ratios of these few-element tensors -- whose u can cancel -- differ
    # from the oracle's only through the rounding of the norms
    op, ref = _one_apply(man, params, [[rng.normal(0, 0.1, s).astype(np.float32) for _, s in man] for _ in range(3)],
                         clip=0.0, N=2)
    _check(op, ref, exact_mv=True)


def test_unaligned_views_match_aligned_tensors():
    from gaccum_b200.train_op import GaccumTrainOp
    hp, _ = _hp(1.0)
    params = _params(MAN, 9)
    names = [n for n, _ in MAN]
    buf = torch.zeros(sum(p.size for p in params) + 8, device="cuda")
    views, o = [], 1                                    # 4 bytes past an aligned address: the scalar paths
    for p in params:
        views.append(buf[o:o + p.size].view(p.shape)); views[-1].copy_(torch.from_numpy(p)); o += p.size
    a = _op(MAN, params, hp, 2)
    b = GaccumTrainOp(views, names, hp, 2, _lr, exclude_from_layer_adaptation=ADAPT_EXCLUDE)
    rng = np.random.default_rng(11)
    gbuf = torch.zeros_like(buf)
    for _ in range(5):
        gr = _cuda(_grads(MAN, rng))
        gv, o = [], 3
        for x, p in zip(gr, params):
            if x is None:
                gv.append(None)
            else:
                gv.append(gbuf[o:o + p.size].view(p.shape)); gv[-1].copy_(x)
            o += p.size
        a.run(gr); b.run(gv)
    torch.cuda.synchronize()
    assert all(_same(x, y) for x, y in zip(a.params, b.params))
    assert np.array_equal(a.trust_ratios(), b.trust_ratios())


@pytest.mark.parametrize("ls", [False, True])
@pytest.mark.parametrize("clip", [0.0, 1.0])
def test_packed_matches_scattered_bit_for_bit(clip, ls):
    g = _g()
    from gaccum_b200.train_op import PackedTrainOp
    hp, _ = _hp(clip)
    params = _params(MAN, 12)
    names = [n for n, _ in MAN]
    cfg = (lambda: g.LossScaleConfig(2.0 ** 8, 2.0, 3)) if ls else (lambda: None)
    a = _op(MAN, params, hp, 3, loss_scale=cfg())
    b = PackedTrainOp([torch.from_numpy(p.copy()).cuda() for p in params], names, hp, 3, _lr, loss_scale=cfg(),
                      exclude_from_layer_adaptation=ADAPT_EXCLUDE)
    rng = np.random.default_rng(13)
    for _ in range(10):
        gr = _grads(MAN, rng, nograd=-1)
        S = a.loss_scale_state()["scale"] if ls else 1.0
        scaled = [x * np.float32(S) for x in gr]
        for p, x in zip(b.params, scaled):
            p.grad.add_(torch.from_numpy(x).cuda())
        assert a.run(_cuda(scaled)) == b.step()
    torch.cuda.synchronize()
    for i, p in enumerate(a.params):
        assert _same(p, b.params[i]), i
    assert _same(a.m, b.m) and _same(a.v, b.v)
    assert np.array_equal(a.trust_ratios(), b.trust_ratios())


def test_fullsize_bert_small_window():
    man = onp.MANIFESTS["bert_small"]()
    rng = np.random.default_rng(14)
    params = make_params(man, rng)
    grads = [[rng.normal(0, 1e-3, s).astype(np.float32) for _, s in man] for _ in range(4)]
    hp, hpo = _hp(1.0)
    op = _op(man, params, hp, 4, adapt_exclude=None, global_step=1)
    ref = ComposedReferenceTrainOp([p.copy() for p in params], [n for n, _ in man], hpo, 4, global_step=1, **SCHED)
    for gr in grads:
        op.run(_cuda(gr)); ref.run(gr)
    torch.cuda.synchronize()
    assert op.adapt == ref.adapt
    _check(op, ref, exact_mv=False)


@pytest.mark.parametrize("ls", [False, True])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_half_models_are_bit_identical_to_upcast_fp32(dtype, ls):
    g = _g()
    hp, _ = _hp(1.0)
    rng = np.random.default_rng(15)
    params = [torch.from_numpy(p).to(dtype).float().numpy() for p in _params(MAN, 16)]   # representable in dtype
    cfg = (lambda: g.LossScaleConfig(2.0 ** 4, 2.0, 2)) if ls else (lambda: None)
    h, f = _op(MAN, params, hp, 3, dtype=dtype, loss_scale=cfg()), _op(MAN, params, hp, 3, loss_scale=cfg())
    for _ in range(10):
        gr = [None if x is None else torch.from_numpy(x).cuda().to(dtype) for x in _grads(MAN, rng)]
        S = h.loss_scale if ls else 1.0
        gh = [None if x is None else (x * S).to(dtype) for x in gr]
        assert h.run(gh) == f.run([None if x is None else x.float() for x in gh])
    torch.cuda.synchronize()
    for i in range(len(MAN)):
        assert _same(h.master_view(i), f.params[i]), i
        assert torch.equal(h.params[i], f.params[i].to(dtype)), i              # the model copy, rounded to nearest-even
    assert _same(h.m, f.m) and _same(h.v, f.v)
    assert np.array_equal(h.trust_ratios(), f.trust_ratios())


@pytest.mark.parametrize("where", ["first_tile", "last_tile_of_largest"])
def test_fp16_overflowed_window_is_skipped_exactly(where):
    g = _g()
    hp, hpo = _hp(1.0)
    man = [("big/kernel", (40000,)), ("a/bias", (5,)), ("c/kernel", (2055,))]
    params = [torch.from_numpy(p).half().float().numpy() for p in _params(man, 17)]
    N = 3
    op = _op(man, params, hp, N, dtype=torch.float16, loss_scale=g.LossScaleConfig(2.0 ** 10, 2.0, 100))
    un = _op(man, params, hp, N, dtype=torch.float16)
    rng = np.random.default_rng(18)
    mk = lambda: [torch.from_numpy(rng.normal(0, 0.05, s).astype(np.float32)).cuda().half() for _, s in man]
    for _ in range(N + 1):                                 # two applied windows
        gr = mk()
        S = op.loss_scale_state()["scale"]
        op.run([(x.float() * S).half() for x in gr]); un.run(gr)
    for x, y in zip(op.params, un.params):                 # a window that does not overflow matches the unscaled run
        assert torch.equal(x, y)
    assert _same(op.master, un.master) and _same(op.m, un.m) and _same(op.v, un.v)
    torch.cuda.synchronize()
    before = [t.clone() for t in (op.master, op.m, op.v)] + [p.clone() for p in op.params]
    sd0 = op.state_dict()
    r0 = op.trust_ratios()
    for j in range(N):
        gr = [(x.float() * op.loss_scale_state()["scale"]).half() for x in mk()]
        if j == 1:
            if where == "first_tile":
                gr[0][0] = float("inf")
            else:
                gr[0][-1] = float("inf")                    # the last tile of the largest tensor
        op.run(gr)
    torch.cuda.synchronize()
    st = op.loss_scale_state()
    assert st["last_skipped"] and st["skipped_windows"] == 1 and st["scale"] == 2.0 ** 9
    after = [op.master, op.m, op.v] + list(op.params)
    assert all(_same(x, y) if x.dtype == torch.float32 else torch.equal(x, y) for x, y in zip(before, after))
    assert not torch.any(op.accum)
    sd1 = op.state_dict()
    assert float(sd1["beta1_power"]) == float(sd0["beta1_power"]) and float(sd1["beta2_power"]) == float(sd0["beta2_power"])
    assert np.array_equal(r0, op.trust_ratios())


@pytest.mark.parametrize("via", ["state_dict", "tf_checkpoint"])
def test_resume_mid_window_is_bit_identical(via, tmp_path):
    from gaccum_b200 import tf_checkpoint
    hp, _ = _hp(1.0)
    params = _params(MAN, 19)
    N = 4
    rng = np.random.default_rng(20)
    stream = [_cuda(_grads(MAN, rng)) for _ in range(3 * N)]
    full = _op(MAN, params, hp, N)
    for gr in stream:
        full.run(gr)
    first = _op(MAN, params, hp, N)
    cut = N + 2                                            # mid-window
    for gr in stream[:cut]:
        first.run(gr)
    second = _op(MAN, _params(MAN, 99), hp, N)
    if via == "state_dict":
        second.load_state_dict(first.state_dict())
    else:
        prefix = tf_checkpoint.save(str(tmp_path), first)
        keys = tf_checkpoint.read_bundle(prefix)
        assert "a/kernel/lamb_m" in keys and "a/kernel/lamb_v" in keys and "beta1_power" in keys
        tf_checkpoint.restore(str(tmp_path), second)
    for gr in stream[cut:]:
        second.run(gr)
    torch.cuda.synchronize()
    for x, y in zip(full.params, second.params):
        assert _same(x, y)
    assert _same(full.m, second.m) and _same(full.v, second.v) and _same(full.accum, second.accum)
    assert np.array_equal(full.trust_ratios(), second.trust_ratios())


def test_create_optimizer_with_optimizer_type_lamb(monkeypatch):
    from gaccum_b200 import graph, optimization as opt
    monkeypatch.setattr(opt, "optimizer_type", "lamb")
    monkeypatch.setattr(opt, "gradient_accumulation_multiplier", 2)
    graph.reset_default_graph()
    man = [("bert/encoder/layer_0/output/dense/kernel", (64, 32)), ("bert/encoder/layer_0/output/dense/bias", (32,)),
           ("bert/encoder/layer_0/output/LayerNorm/gamma", (32,))]
    params = make_params(man, np.random.default_rng(21))
    tv = [graph.add_variable(n, torch.from_numpy(p.copy()).cuda()) for (n, _), p in zip(man, params)]
    train_op = opt.create_optimizer(None, 1e-3, 50, 3, False)
    assert isinstance(train_op.optimizer, opt.LAMBOptimizer)
    ref = ComposedReferenceTrainOp([p.copy() for p in params], [n for n, _ in man], onp.HParams(variant=2), 2,
                                   init_lr=1e-3, num_train_steps=50, num_warmup_steps=3)
    assert train_op.engine.adapt == ref.adapt == [True, False, False]
    rng = np.random.default_rng(22)
    for _ in range(9):
        gr = [rng.normal(0, 0.1, s).astype(np.float32) for _, s in man]
        ref.run(gr)
        train_op.run_with_grads(_cuda(gr))
    torch.cuda.synchronize()
    for v, exp in zip(tv, ref.params):
        assert rel_err(v.tensor.cpu().numpy(), exp) <= 1e-5
    np.testing.assert_allclose(train_op.engine.trust_ratios(), np.asarray(ref.ratios, np.float32), rtol=1e-6)
