"""The exponential moving average of the weights on the GPU (include/gaccum.h, gaccum_plan_set_ema).

* Training is unchanged: p, m, v, accumulators, stats, trust ratios, the loss-scaling block and the 16-bit model copy
  are bit-identical to the same run without an EMA (every variant, clip 0 / 1 / 1e-3, N 1 / 3 / 4, fp32 / bf16 / fp16).
* The average is bit-identical to the oracle (tests/ema_oracle.py) fed the kernel's own weights after every applied
  window, and within 1e-5 of the oracle's whole trajectory; both decay modes.
* Loss scaling: an overflowed window leaves the average and n unchanged, bit for bit.
* Layouts: the packed entry point, unaligned views, tails, 1920 tensors, one 30522 x 1024 tensor, tensors without a
  gradient.  Launches and CUDA-graph replays are reproducible; a replay advances n.
* Resume through state_dict and a TF-format checkpoint, averaged_weights(), create_optimizer, full-size BERT-Small.
"""
import numpy as np
import pytest

import oracle_c
import oracle_np as onp
from common import make_params, rel_err
from composed_oracle import ComposedReferenceTrainOp
from ema_oracle import Ema, EmaReferenceTrainOp, ema_coefficients

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

# tails, a vector body with a 7-element tail (2055), several tiles, one element, a tensor without a gradient
MAN = [("a/kernel", (777,)), ("a/bias", (5,)), ("b/kernel", (3, 1367)), ("t/kernel", (2055,)), ("one", (1,)),
       ("LayerNorm/gamma", (33,)), ("nograd/kernel", (64,))]
NOGRAD = 6
SCHED = dict(init_lr=1e-2, num_train_steps=40, num_warmup_steps=4)
DECAY = 0.9


def _g():
    import gaccum_b200 as g
    return g


def _bits(t):
    return t.contiguous().view(torch.int32) if t.element_size() == 4 else t.contiguous().view(torch.int16)


def _same(x, y):
    return torch.equal(_bits(x), _bits(y))


def _params(man, seed, dtype=torch.float32):
    rng = np.random.default_rng(seed)
    ps = [rng.normal(0, 0.05, s).astype(np.float32) for _, s in man]
    return ps if dtype == torch.float32 else [torch.from_numpy(p).to(dtype).float().numpy() for p in ps]


def _lr(s):
    return _g().learning_rate(SCHED["init_lr"], SCHED["num_train_steps"], SCHED["num_warmup_steps"], s)


def _hp(variant, clip):
    g = _g()
    if variant == "lamb":
        return g.HParams.lamb(clip_norm=clip)
    if variant == "adam":
        return g.HParams(g.ADAM, 0, 0.9, 0.999, 1e-8, 0.0, clip)
    return g.HParams(g.ADAM_WEIGHT_DECAY, 0, 0.9, 0.999, 1e-6, 0.01, clip)


def _op(man, params, hp, N, dtype=torch.float32, ema=None, **kw):
    from gaccum_b200.train_op import GaccumTrainOp
    return GaccumTrainOp([torch.from_numpy(p.copy()).cuda().to(dtype) for p in params], [n for n, _ in man], hp, N,
                         kw.pop("lr_fn", _lr), ema=ema, **kw)


def _grads(man, rng, sigma=0.1, nograd=NOGRAD):
    return [None if i == nograd else rng.normal(0, sigma, s).astype(np.float32) for i, (_, s) in enumerate(man)]


def _cuda(grads, dtype=torch.float32):
    return [None if x is None else torch.from_numpy(x).cuda().to(dtype) for x in grads]


def _weights(op, i):
    return op.params[i] if op.master is None else op.master_view(i)


def _tracker(op, decay, num_updates):
    """The oracle's average, started where the op starts it: at the fp32 weights."""
    return Ema([_weights(op, i).float().cpu().numpy() for i in range(len(op.params))], decay, num_updates)


def _check_ema(op, tr):
    torch.cuda.synchronize()
    for i, e in enumerate(tr.avg):
        assert np.array_equal(op.ema_view(i).cpu().numpy().view(np.uint32), e.view(np.uint32)), i
    st = op.ema_state()
    assert st["num_updates"] == tr.num_updates and np.float32(st["decay"]) == tr.decay


def _training_state(op):
    out = [op.accum, op.m, op.v] + [p for p in op.params]
    if op.master is not None:
        out.append(op.master)
    if op._ls_state is not None:
        out.append(op._ls_state)
    return out


def _check_same_training(a, b):
    torch.cuda.synchronize()
    for x, y in zip(_training_state(a), _training_state(b)):
        assert _same(x, y)
    sa, sb = (np.array(list(x.stats().values()), np.float32) for x in (a, b))
    assert np.array_equal(sa.view(np.uint32), sb.view(np.uint32))     # an overflowed window's clip scale is NaN in both
    if a.hp.variant == _g().LAMB:
        assert np.array_equal(a.trust_ratios(), b.trust_ratios())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("N", [1, 3, 4])
@pytest.mark.parametrize("clip", [0.0, 1.0, 1e-3])
@pytest.mark.parametrize("variant", ["adamw", "adam", "lamb"])
def test_training_unchanged_and_ema_bit_exact(variant, clip, N, dtype):
    g = _g()
    hp = _hp(variant, clip)
    num_updates = N != 3                                   # both decay modes over the grid
    params = _params(MAN, 1, dtype)
    e = _op(MAN, params, hp, N, dtype, ema=g.EmaConfig(DECAY, num_updates))
    p = _op(MAN, params, hp, N, dtype)
    tr = _tracker(e, DECAY, num_updates)
    rng = np.random.default_rng(10 + N)
    for step in range(3 * N + 1):
        gr = _cuda(_grads(MAN, rng), dtype)
        applied = e.run(gr)
        assert applied == p.run(gr)
        _check_same_training(e, p)
        if applied:
            tr.average([_weights(e, i).cpu().numpy() for i in range(len(MAN))])
        _check_ema(e, tr)
    assert tr.num_updates == 4                             # windows applied at steps 0, N, 2N and 3N


@pytest.mark.parametrize("num_updates", [False, True])
@pytest.mark.parametrize("variant", ["adamw", "adam", "lamb"])
def test_ema_follows_the_oracle_trajectory(variant, num_updates):
    g = _g()
    clip = 0.0 if variant == "adam" else 1.0
    hp = _hp(variant, clip)
    N = 3
    params = _params(MAN, 2)
    names = [n for n, _ in MAN]
    if variant == "lamb":
        ref = ComposedReferenceTrainOp([x.copy() for x in params], names, onp.HParams(variant=2, clip_norm=clip), N,
                                       **SCHED)
    else:
        hpo = onp.HParams.bert() if variant == "adamw" else onp.HParams.tf_adam()
        ref = onp.ReferenceTrainOp([x.copy() for x in params], names, hpo, N, **SCHED)
    ref = EmaReferenceTrainOp(ref, DECAY, num_updates)
    op = _op(MAN, params, hp, N, ema=g.EmaConfig(DECAY, num_updates))
    rng = np.random.default_rng(3)
    for _ in range(4 * N + 1):
        gr = _grads(MAN, rng)
        assert op.run(_cuda(gr)) == ref.run(gr).applied
    torch.cuda.synchronize()
    for i, exp in enumerate(ref.ema.avg):
        assert rel_err(op.ema_view(i).cpu().numpy(), exp) <= 1e-5, i
    assert op.ema_state()["num_updates"] == ref.ema.num_updates == 5
    assert np.float32(op.ema_state()["decay"]) == ref.ema.decay


def test_counter_past_2_24_rounds_like_tf():
    """n = 2^24 + 1: fp32(n) rounds to 2^24, and the kernel's d is the oracle's."""
    g = _g()
    op = _op(MAN, _params(MAN, 4), _hp("adamw", 1.0), 1, ema=g.EmaConfig(0.99999999, True), lr_fn=lambda s: 1e-2)
    n0 = 2 ** 24 + 1
    op.plan.ema_init(op._ema_state.data_ptr(), n0, op._stream())
    tr = _tracker(op, 0.99999999, True)
    tr.num_updates = n0
    op.run(_cuda(_grads(MAN, np.random.default_rng(5))))
    tr.average([p.cpu().numpy() for p in op.params])
    _check_ema(op, tr)
    assert tr.decay == ema_coefficients(0.99999999, True, 2 ** 24)[0]


@pytest.mark.parametrize("where", ["first_tile", "last_tile"])
@pytest.mark.parametrize("variant", ["adamw", "lamb"])
def test_fp16_overflowed_window_leaves_the_average(variant, where):
    """The model's first tile is in a CTA's stash (clip-apply) and in LAMB's first CTA; its last tile -- the 7-element
    tail of the last tensor -- is in the pool (clip-apply, behind a 3 M-element tensor) and in LAMB's last CTA."""
    g = _g()
    hp = _hp(variant, 1.0)
    man = [("big/kernel", (3 * 2 ** 20,)), ("a/bias", (5,)), ("c/kernel", (2055,))]
    params = _params(man, 6, torch.float16)
    N = 2
    cfg = lambda: g.LossScaleConfig(2.0 ** 10, 2.0, 100)
    e = _op(man, params, hp, N, torch.float16, ema=g.EmaConfig(DECAY, True), loss_scale=cfg())
    p = _op(man, params, hp, N, torch.float16, loss_scale=cfg())
    rng = np.random.default_rng(7)
    mk = lambda: [torch.from_numpy(rng.normal(0, 0.05, s).astype(np.float32)).cuda() for _, s in man]
    for j in range(3 * N):                                  # windows applied at steps 0, N and 2N
        S = e.loss_scale_state()["scale"]
        gr = [(x * S).half() for x in mk()]
        if j == 2 * N - 1:                                  # the window that applies at step 2N overflows
            if where == "first_tile":
                gr[0][0] = float("inf")
            else:
                gr[-1][-1] = float("inf")
        if j == 2 * N:
            torch.cuda.synchronize()
            before = (e.ema.clone(), e.ema_state())
        e.run(gr); p.run(gr)
        _check_same_training(e, p)
        if j == 2 * N:
            assert e.loss_scale_state()["last_skipped"]
            assert _same(before[0], e.ema) and e.ema_state() == before[1]
    assert e.ema_state()["num_updates"] == 2


def _packed_grads(op, gr):
    for p, x in zip(op.params, gr):
        if x is not None:
            p.grad.add_(x)


@pytest.mark.parametrize("ls", [False, True])
@pytest.mark.parametrize("variant", ["adamw", "lamb"])
def test_packed_matches_scattered_bit_for_bit(variant, ls):
    g = _g()
    from gaccum_b200.train_op import PackedTrainOp
    hp = _hp(variant, 1.0)
    params = _params(MAN, 8)
    cfg = (lambda: g.LossScaleConfig(2.0 ** 8, 2.0, 3)) if ls else (lambda: None)
    a = _op(MAN, params, hp, 3, ema=g.EmaConfig(DECAY), loss_scale=cfg())
    b = PackedTrainOp([torch.from_numpy(x.copy()).cuda() for x in params], [n for n, _ in MAN], hp, 3, _lr,
                      loss_scale=cfg(), ema=g.EmaConfig(DECAY))
    rng = np.random.default_rng(9)
    for _ in range(10):
        S = a.loss_scale_state()["scale"] if ls else 1.0
        gr = [None if x is None else torch.from_numpy(x * np.float32(S)).cuda() for x in _grads(MAN, rng)]
        _packed_grads(b, gr)
        assert a.run(gr) == b.step()
    torch.cuda.synchronize()
    for i in range(len(MAN)):
        assert _same(a.ema_view(i), b.ema_view(i)), i
        assert _same(a.params[i], b.params[i]), i
    assert a.ema_state() == b.ema_state() and a.ema_state()["num_updates"] == 4


@pytest.mark.parametrize("variant", ["adamw", "lamb"])
def test_unaligned_views_1920_tensors_and_a_30522x1024_tensor(variant):
    """Each layout against the oracle fed the kernel's own weights."""
    g = _g()
    from gaccum_b200.train_op import GaccumTrainOp
    rng = np.random.default_rng(11)

    def run(man, op, num_updates):
        tr = _tracker(op, DECAY, num_updates)
        for _ in range(3):
            gr = _cuda([rng.normal(0, 1e-2, s).astype(np.float32) for _, s in man])
            if op.run(gr):
                tr.average([p.cpu().numpy() for p in op.params])
        _check_ema(op, tr)
        assert tr.num_updates >= 2

    # unaligned views: 4 bytes past an aligned address, the scalar paths
    params = _params(MAN, 12)
    buf = torch.zeros(sum(x.size for x in params) + 8, device="cuda")
    views, o = [], 1
    for x in params:
        views.append(buf[o:o + x.size].view(x.shape)); views[-1].copy_(torch.from_numpy(x)); o += x.size
    run(MAN, GaccumTrainOp(views, [n for n, _ in MAN], _hp(variant, 1.0), 2, _lr, ema=g.EmaConfig(DECAY, True)), True)
    man = [(f"t{i}/{'bias' if i % 3 == 0 else 'kernel'}", (1 + i % 7,)) for i in range(1920)]
    run(man, _op(man, _params(man, 13), _hp(variant, 0.0), 2, ema=g.EmaConfig(DECAY)), False)
    man = [("bert/embeddings/word_embeddings", (30522, 1024)), ("LayerNorm/beta", (1024,))]
    run(man, _op(man, _params(man, 14), _hp(variant, 1.0), 1, ema=g.EmaConfig(DECAY, True)), True)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("clip", [0.0, 1.0])
def test_repeated_launches_and_graph_replays(clip):
    """clip 0: apply_kernel, whose last CTA advances n and resets the launch's CTA counter; clip 1: apply_clip_kernel."""
    g = _g()
    hp = _hp("adamw", clip)
    params = _params(MAN, 15)
    rng = np.random.default_rng(16)
    gr = _cuda(_grads(MAN, rng))
    ops = [_op(MAN, params, hp, 1, ema=g.EmaConfig(DECAY, True), lr_fn=lambda s: 1e-2) for _ in range(3)]
    for op in ops[:2]:
        for _ in range(3):
            op.apply_only(gr)
    torch.cuda.synchronize()
    assert _same(ops[0].ema, ops[1].ema) and ops[0].ema_state() == ops[1].ema_state()
    # ops[2]: capture one apply and replay it: every replay averages once more and advances n
    op = ops[2]
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        op.apply_only(gr)                                  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(stream)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        op.apply_only(gr)
    torch.cuda.synchronize()
    assert op.ema_state()["num_updates"] == 1              # capturing launched nothing
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    assert op.ema_state()["num_updates"] == 3
    # the replays computed what the eager launches did
    assert _same(op.ema, ops[0].ema) and op.ema_state() == ops[0].ema_state()
    # an eager launch after the replays still advances n once (the CTA counter was left at 0)
    op.apply_only(gr)
    ops[0].apply_only(gr)
    torch.cuda.synchronize()
    assert op.ema_state()["num_updates"] == 4
    assert _same(op.ema, ops[0].ema) and op.ema_state() == ops[0].ema_state()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("via", ["state_dict", "tf_checkpoint"])
def test_resume_mid_window_is_bit_identical(via, dtype, tmp_path):
    from gaccum_b200 import tf_checkpoint
    g = _g()
    hp = _hp("adamw", 1.0)
    params = _params(MAN, 17, dtype)
    N = 4
    rng = np.random.default_rng(18)
    stream = [_cuda(_grads(MAN, rng), dtype) for _ in range(3 * N)]
    cfg = lambda: g.EmaConfig(DECAY, True)
    full = _op(MAN, params, hp, N, dtype, ema=cfg())
    for gr in stream:
        full.run(gr)
    first = _op(MAN, params, hp, N, dtype, ema=cfg())
    cut = N + 2
    for gr in stream[:cut]:
        first.run(gr)
    second = _op(MAN, _params(MAN, 99, dtype), hp, N, dtype, ema=cfg())
    if via == "state_dict":
        sd = first.state_dict()
        assert "a/kernel/ExponentialMovingAverage" in sd and int(sd["ExponentialMovingAverage/num_updates"]) == 2
        second.load_state_dict(sd)
    else:
        prefix = tf_checkpoint.save(str(tmp_path), first)
        keys = tf_checkpoint.read_bundle(prefix)
        assert "a/kernel/ExponentialMovingAverage" in keys and "ExponentialMovingAverage/num_updates" in keys
        tf_checkpoint.restore(str(tmp_path), second)
    for gr in stream[cut:]:
        second.run(gr)
    torch.cuda.synchronize()
    assert _same(full.ema, second.ema) and full.ema_state() == second.ema_state()
    for x, y in zip(full.params, second.params):
        assert _same(x, y)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_averaged_weights_swaps_in_and_restores(dtype):
    g = _g()
    op = _op(MAN, _params(MAN, 19, dtype), _hp("adamw", 1.0), 2, dtype, ema=g.EmaConfig(DECAY))
    rng = np.random.default_rng(20)
    for _ in range(5):
        op.run(_cuda(_grads(MAN, rng), dtype))
    torch.cuda.synchronize()
    saved = [p.clone() for p in op.params]
    with op.averaged_weights():
        for i, p in enumerate(op.params):
            assert torch.equal(p, op.ema_view(i).to(dtype)), i      # rounded to nearest-even on a 16-bit model
        assert not all(torch.equal(p, s) for p, s in zip(op.params, saved))
    for p, s in zip(op.params, saved):
        assert _same(p, s)


def test_create_optimizer_with_moving_average_decay(monkeypatch):
    from gaccum_b200 import graph, optimization as opt
    monkeypatch.setattr(opt, "moving_average_decay", 0.99)
    monkeypatch.setattr(opt, "gradient_accumulation_multiplier", 2)
    graph.reset_default_graph()
    man = [("bert/encoder/layer_0/output/dense/kernel", (64, 32)), ("bert/encoder/layer_0/output/dense/bias", (32,))]
    params = make_params(man, np.random.default_rng(21))
    tv = [graph.add_variable(n, torch.from_numpy(p.copy()).cuda()) for (n, _), p in zip(man, params)]
    train_op = opt.create_optimizer(None, 1e-3, 50, 3, False)
    assert isinstance(train_op.ema, opt.ExponentialMovingAverage)
    ref = EmaReferenceTrainOp(onp.ReferenceTrainOp([p.copy() for p in params], [n for n, _ in man], onp.HParams.bert(), 2,
                                                   init_lr=1e-3, num_train_steps=50, num_warmup_steps=3), 0.99)
    rng = np.random.default_rng(22)
    for _ in range(9):
        gr = [rng.normal(0, 0.1, s).astype(np.float32) for _, s in man]
        ref.run(gr)
        train_op.run_with_grads(_cuda(gr))
    torch.cuda.synchronize()
    for v, exp in zip(tv, ref.ema.avg):
        assert rel_err(train_op.ema.average(v).cpu().numpy(), exp) <= 1e-5
    restore = train_op.ema.variables_to_restore()
    assert set(restore) == {n + "/ExponentialMovingAverage" for n, _ in man}


def test_fullsize_bert_small_against_the_c_oracle():
    """The C oracle's parameters after every applied window, with the EMA oracle on top."""
    g = _g()
    man = onp.MANIFESTS["bert_small"]()
    rng = np.random.default_rng(23)
    params = make_params(man, rng)
    names = [n for n, _ in man]
    N = 4
    op = _op(man, params, g.HParams.bert(), N, ema=g.EmaConfig(0.999, True), global_step=1)
    ref = EmaReferenceTrainOp(oracle_c.COracleTrainOp([p.copy() for p in params], names, onp.HParams.bert(), N,
                                                      global_step=1, **SCHED), 0.999, True)
    for _ in range(2 * N):
        gr = [rng.normal(0, 1e-3, s).astype(np.float32) for _, s in man]
        assert op.run(_cuda(gr)) == ref.run(gr).applied
    torch.cuda.synchronize()
    assert op.ema_state()["num_updates"] == ref.ema.num_updates == 2
    for i, exp in enumerate(ref.ema.avg):
        assert rel_err(op.ema_view(i).cpu().numpy(), exp) <= 1e-5, names[i]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("via", ["state_dict", "tf_checkpoint"])
def test_non_strict_parameters_only_restore_restarts_the_average(via, dtype, tmp_path):
    """A pre-trained (parameters-only) checkpoint loaded with strict=False: the average starts at the restored fp32
    weights and n at 0, as TF creates a shadow variable from its variable's restored value."""
    from gaccum_b200 import tf_checkpoint
    g = _g()
    hp = _hp("adamw", 1.0)
    N = 2
    op = _op(MAN, _params(MAN, 24, dtype), hp, N, dtype, ema=g.EmaConfig(DECAY, True))
    rng = np.random.default_rng(25)
    for _ in range(3):                                     # an average and n away from their initial values
        op.run(_cuda(_grads(MAN, rng), dtype))
    pre = {n: torch.from_numpy(x) for (n, _), x in zip(MAN, _params(MAN, 26, dtype))}
    if via == "state_dict":
        op.load_state_dict(dict(pre, global_step=torch.tensor(0)), strict=False)
    else:
        tf_checkpoint.write_bundle(str(tmp_path / "model.ckpt-0"), {n: x.numpy() for n, x in pre.items()})
        tf_checkpoint.write_checkpoint_state(str(tmp_path), "model.ckpt-0")
        tf_checkpoint.restore(str(tmp_path), op, strict=False)
    torch.cuda.synchronize()
    for i, (n, _) in enumerate(MAN):
        assert _same(_weights(op, i), pre[n].cuda()), n
        assert _same(op.ema_view(i), _weights(op, i)), n
    assert op.ema_state()["num_updates"] == 0
    tr = _tracker(op, DECAY, True)
    for _ in range(2 * N):
        if op.run(_cuda(_grads(MAN, rng), dtype)):
            tr.average([_weights(op, i).cpu().numpy() for i in range(len(MAN))])
    _check_ema(op, tr)
