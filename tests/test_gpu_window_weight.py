"""Per-window normalisation by the window's total weight on the GPU (include/gaccum.h, gaccum_plan_set_window_weight).

* Every dispatch key (tests/apply_matrix.py: 336 cases, all 120 apply instantiations): a weight of 1 per micro-step is
  the unweighted run bit for bit (p, m, v, accumulators, stats, EMA, trust ratios, loss-scaling block), and mixed
  integer weights whose totals are not powers of two, with learning-rate multipliers on, match the composed oracle
  (tests/composed_oracle.py) after every micro-step.
* A uniform power-of-two weight k with gradients scaled by k is the unweighted run, bit for bit.
* The property the feature exists for: one weighted window over micro-batches with different numbers of valid tokens is
  one step on the concatenated batch with a per-token-mean loss; the unweighted window is not.
* CUDA-graph capture of whole windows (the producer's W += count included), mid-window resume through state_dict and a
  TF-format checkpoint, overflowed and W = 0 windows under loss scaling, and bf16 / fp16 against the upcast fp32 run.
"""
import zlib

import numpy as np
import pytest

from apply_matrix import Case, LockStep, matrix_cases

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
N = 3
WEIGHTS = (3.0, 37.0, 1000.0, 5.0, 64.0, 11.0)      # window totals 1040, 80, ...: not powers of two
CYCLE = (0.37, 0.0, 2.5, 1.0)


def _setup(case: Case):
    layout = "packed" if case.layout == "packed" else "table"
    dtype = case.layout.split("_")[-1] if layout == "table" else "fp32"
    man = MAN + TINY if case.layout.startswith("t1920") else MAN
    return layout, dtype, man


def _bits(t):
    return t.contiguous().view(torch.int32) if t.element_size() == 4 else t.contiguous().view(torch.int16)


def _device_state(op):
    out = [op.accum, op.m, op.v] + [p for p in op.params]
    for name in ("master", "ema", "_ls_state", "_ema_state"):
        x = getattr(op, name, None)
        if x is not None:
            out.append(x)
    if getattr(op, "param_slab", None) is not None:
        out.append(op.param_slab)
    return out


def _assert_same_state(a, b):
    torch.cuda.synchronize()
    for i, (x, y) in enumerate(zip(_device_state(a), _device_state(b))):
        assert torch.equal(_bits(x), _bits(y)), i
    sa, sb = (np.array(list(o.stats().values()), F32) for o in (a, b))
    assert np.array_equal(sa.view(np.uint32), sb.view(np.uint32))
    if a.hp.variant == 2:
        assert np.array_equal(a.trust_ratios().view(np.uint32), b.trust_ratios().view(np.uint32))


@pytest.mark.parametrize("case", matrix_cases(), ids=lambda c: c.id)
def test_weights_of_one_are_the_unweighted_run(case: Case):
    layout, dtype, man = _setup(case)
    seed = zlib.crc32(case.id.encode())
    kw = dict(N=N, seed=seed, nograd=NOGRAD, lr_mult=np.ones(len(man), F32))
    ema = EMA if case.ema else None
    a = LockStep(man, case.variant, case.mode, layout, dtype, case.has_g, ema, window_weight=True, **kw)
    b = LockStep(man, case.variant, case.mode, layout, dtype, case.has_g, ema, **kw)
    ls = case.mode.startswith("ls_")
    for s in range(STEPS):
        gr = a.grads(0.1, INF_AT[1:] if ls and s == INF_AT[0] else None)
        b.grads(0.1)                                       # keep the two generators in step
        # the one-micro-batch window at step 0 is divided by N unweighted: a weighted plan divides it by its W
        a.wstep(gr, float(N) if s == 0 else 1.0)
        b.step(gr)
        _assert_same_state(a.op, b.op)
    if ls:
        assert a.op.loss_scale_state()["skipped_windows"] == 1


@pytest.mark.parametrize("case", matrix_cases(), ids=lambda c: c.id)
def test_mixed_weights_match_the_oracle(case: Case):
    layout, dtype, man = _setup(case)
    run = LockStep(man, case.variant, case.mode, layout, dtype, case.has_g, EMA if case.ema else None, N=N,
                   seed=zlib.crc32(case.id.encode()) ^ 1, nograd=NOGRAD,
                   lr_mult=[CYCLE[i % len(CYCLE)] for i in range(len(man))], window_weight=True)
    ls = case.mode.startswith("ls_")
    for s in range(STEPS):
        run.wstep(run.grads(0.1, INF_AT[1:] if ls and s == INF_AT[0] else None), WEIGHTS[s % len(WEIGHTS)])
    if ls:
        assert run.op.loss_scale_state()["skipped_windows"] == 1


# ---- the train ops ---------------------------------------------------------------------------------------------------
SMAN = [("a/kernel", (777,)), ("a/bias", (5,)), ("b/kernel", (3, 1367)), ("t/kernel", (2055,)), ("one", (1,)),
        ("LayerNorm/gamma", (33,))]
MODES = ["noclip", "clip", "ls_noclip", "ls_clip"]
VARIANTS = ["adamw", "adam", "lamb"]


def _g():
    import gaccum_b200 as g
    return g


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


def _op(params, variant, mode, n, dtype=torch.float32, **kw):
    from gaccum_b200.train_op import GaccumTrainOp
    g = _g()
    ls = g.LossScaleConfig(16.0, 2.0, 2) if mode.startswith("ls_") else None
    lr_fn = kw.pop("lr_fn", lambda s: g.learning_rate(1e-2, 40, 4, s))
    return GaccumTrainOp([torch.from_numpy(p.copy()).cuda().to(dtype) for p in params], [n_ for n_, _ in SMAN],
                         _hp(variant, mode), n, lr_fn, loss_scale=ls, **kw)


def _grads(rng, k=1.0):
    return [(rng.normal(0, 0.1, s) * k).astype(F32) for _, s in SMAN]


def _cuda(grads, dtype=torch.float32):
    return [torch.from_numpy(x).cuda().to(dtype) for x in grads]


def _scale(op):
    return float(op.loss_scale_state()["scale"]) if op._ls_state is not None else 1.0


@pytest.mark.parametrize("k", [4.0, 0.125])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("variant", VARIANTS)
def test_uniform_power_of_two_weight_with_scaled_gradients_is_unweighted(variant, mode, k):
    params = _params(1)
    a = _op(params, variant, mode, N, window_weight=True)
    b = _op(params, variant, mode, N)
    rng = np.random.default_rng(2)
    for s in range(10):
        x = _grads(rng)
        Sa, Sb = _scale(a), _scale(b)
        a.run(_cuda([(g_ * F32(k) * F32(Sa)).astype(F32) for g_ in x]), weight=k * (N if s == 0 else 1))
        b.run(_cuda([(g_ * F32(Sb)).astype(F32) for g_ in x]))
        torch.cuda.synchronize()
        for i, (p, q) in enumerate(zip(a.params, b.params)):
            assert torch.equal(_bits(p), _bits(q)), (s, i)
        assert torch.equal(_bits(a.m), _bits(b.m)) and torch.equal(_bits(a.v), _bits(b.v))
    st = a.window_weight_state()
    assert st["weight"] == 0.0 and st["last_weight"] == k * N


def test_weighted_window_is_the_per_token_mean_of_the_concatenated_batch():
    """A masked-token linear model: N micro-batches with different numbers of valid tokens.  One weighted window
    (summed losses, weights = token counts) must be one N = 1 step on the concatenated batch with a per-token-mean loss;
    the unweighted window (per-micro-batch means, divided by N) differs."""
    g = _g()
    from gaccum_b200.train_op import GaccumTrainOp
    torch.manual_seed(0)
    D, V, Nw = 16, 11, 4
    counts = [3, 17, 1, 9]
    batches = [(torch.randn(c, D, device="cuda"), torch.randint(0, V, (c,), device="cuda")) for c in counts]
    w0 = torch.randn(D, V, device="cuda") * 0.1
    # a large epsilon keeps the first update close to linear in c (with 1e-6 it is nearly sign(c), whatever the scaling)
    hp = g.HParams(g.ADAM_WEIGHT_DECAY, 0, 0.9, 0.999, 1.0, 0.0, 0.0)

    def make(n, **kw):
        w = w0.clone().requires_grad_(True)
        return w, GaccumTrainOp([w], ["w/kernel"], hp, n, lambda s: 1e-2, global_step=1 if n > 1 else 0, **kw)

    def loss(w, x, y, reduction):
        return torch.nn.functional.cross_entropy(x @ w, y, reduction=reduction)

    ww, weighted = make(Nw, window_weight=True)
    wu, unweighted = make(Nw)
    wc, concat = make(1)
    # a window that starts after step 0 ends at global_step 4
    for x, y in batches:
        gw, = torch.autograd.grad(loss(ww, x, y, "sum"), [ww])
        weighted.run([gw], weight=torch.tensor(float(x.shape[0]), device="cuda"))
        gu, = torch.autograd.grad(loss(wu, x, y, "mean"), [wu])
        unweighted.run([gu])
    X = torch.cat([x for x, _ in batches]); Y = torch.cat([y for _, y in batches])
    gc, = torch.autograd.grad(loss(wc, X, Y, "mean"), [wc])
    concat.run([gc])
    torch.cuda.synchronize()
    assert weighted.last_applied and concat.last_applied
    d_w, d_c, d_u = (p.detach() - w0 for p in (ww, wc, wu))
    assert float((d_w - d_c).abs().max() / d_c.abs().max()) <= 1e-5
    assert float((d_u - d_c).abs().max() / d_c.abs().max()) > 1e-3
    assert weighted.window_weight_state() == {"weight": 0.0, "last_weight": float(sum(counts))}


@pytest.mark.parametrize("variant, mode", [("adamw", "noclip"), ("adamw", "clip"), ("adam", "ls_noclip"), ("lamb", "ls_clip")])
def test_graph_capture_of_whole_windows(variant, mode):
    params = _params(3)
    rng = np.random.default_rng(4)
    gr = [_cuda(_grads(rng)) for _ in range(N)]
    counts = [torch.tensor(c, dtype=torch.float32, device="cuda") for c in (3.0, 37.0, 1000.0)]
    lr_fn = lambda s: 1e-2
    eager = _op(params, variant, mode, N, window_weight=True, lr_fn=lr_fn, global_step=1)
    op = _op(params, variant, mode, N, window_weight=True, lr_fn=lr_fn, global_step=1)

    def window(o):
        # the window's steps are replayed as they were captured: global steps 1, 2, 3 (the last applies)
        o.global_step = 1
        for j in range(N):
            o.window_weight += counts[j]
            o.run_bound(o.bind(gr[j]))
    for _ in range(3):
        window(eager)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        window(op)                                          # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(stream)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        window(op)
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    for x, y in zip(_device_state(op), _device_state(eager)):
        assert torch.equal(_bits(x), _bits(y))
    assert op.window_weight_state() == {"weight": 0.0, "last_weight": 1040.0}


@pytest.mark.parametrize("via", ["state_dict", "tf_checkpoint"])
@pytest.mark.parametrize("variant, mode", [("adamw", "clip"), ("adam", "noclip"), ("lamb", "ls_clip")])
def test_resume_mid_window_is_bit_identical(variant, mode, via):
    from gaccum_b200 import tf_checkpoint as tfc
    params = _params(5)
    n = 4
    rng = np.random.default_rng(6)
    raw = [_grads(rng) for _ in range(3 * n)]
    ws = [WEIGHTS[i % len(WEIGHTS)] for i in range(3 * n)]
    full = _op(params, variant, mode, n, window_weight=True)
    first = _op(params, variant, mode, n, window_weight=True)
    second = _op(_params(99), variant, mode, n, window_weight=True)

    def feed(op, x, w):
        S = _scale(op)
        op.run(_cuda([(g_ * F32(S)).astype(F32) for g_ in x]), weight=w)
    for x, w in zip(raw, ws):
        feed(full, x, w)
    cut = n + 2
    for x, w in zip(raw[:cut], ws[:cut]):
        feed(first, x, w)
    sd = first.state_dict()
    key = "gradient_accumulation/window_weight"
    assert float(sd[key]) == sum(ws[n + 1:cut])          # the apply at global step n reset W
    if via == "tf_checkpoint":
        v = first.hp.variant
        ref = tfc.to_reference_names(sd, first.names, v)
        assert ref[key].dtype == np.float32 and ref[key].shape == ()
        back = tfc.from_reference_names(ref, first.names, v, window_weight=True)
        # the loss-scaling block has no reference name: it comes from the state_dict, everything else from the mapping
        sd = {**{k: t for k, t in sd.items() if k != key}, **{k: torch.as_tensor(np.asarray(a)) for k, a in back.items()}}
    second.load_state_dict(sd)
    for x, w in zip(raw[cut:], ws[cut:]):
        feed(second, x, w)
    torch.cuda.synchronize()
    for x, y in zip(_device_state(full), _device_state(second)):
        assert torch.equal(_bits(x), _bits(y))
    assert second.window_weight_state() == full.window_weight_state()


@pytest.mark.parametrize("variant", VARIANTS)
def test_overflowed_and_zero_weight_windows_are_skipped_and_reset(variant):
    params = _params(7)
    op = _op(params, variant, "ls_clip", 2, window_weight=True, global_step=1)
    rng = np.random.default_rng(8)
    x = _grads(rng)
    x[0][3] = np.inf
    op.run(_cuda(x), weight=5.0)                         # global step 1: accumulate
    p0 = [p.clone() for p in op.params]
    op.run(_cuda(_grads(rng)), weight=7.0)               # applies: the window overflowed
    st = op.loss_scale_state()
    assert st["last_skipped"] and op.window_weight_state() == {"weight": 0.0, "last_weight": 12.0}
    op.run(_cuda(_grads(rng)), weight=0.0)
    op.run(_cuda(_grads(rng)), weight=0.0)               # W = 0: infinite c, non-finite norm, skipped
    torch.cuda.synchronize()
    assert op.loss_scale_state()["last_skipped"] and op.loss_scale_state()["skipped_windows"] == 2
    assert op.window_weight_state() == {"weight": 0.0, "last_weight": 0.0}
    for p, q in zip(op.params, p0):
        assert torch.equal(_bits(p), _bits(q))
    assert float(op.accum.abs().sum()) == 0.0


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("variant", VARIANTS)
def test_16_bit_model_is_the_upcast_fp32_run(variant, dtype):
    params = _params(9, dtype)
    h = _op(params, variant, "clip", N, dtype, window_weight=True)
    f = _op(params, variant, "clip", N, window_weight=True)
    rng = np.random.default_rng(10)
    for s in range(10):
        gr = _cuda(_grads(rng), dtype)
        w = WEIGHTS[s % len(WEIGHTS)]
        assert h.run(gr, weight=w) == f.run([x.float() for x in gr], weight=w)
        torch.cuda.synchronize()
        for i in range(len(SMAN)):
            assert torch.equal(_bits(h.master_view(i)), _bits(f.params[i])), i
            assert torch.equal(_bits(h.params[i]), _bits(f.params[i].to(dtype))), i
        for x, y in ((h.m, f.m), (h.v, f.v), (h.accum, f.accum)):
            assert torch.equal(_bits(x), _bits(y))


def test_packed_train_op_takes_the_weight():
    from gaccum_b200.train_op import PackedTrainOp
    g = _g()
    params = [torch.from_numpy(p.copy()).cuda() for p in _params(11)]
    op = PackedTrainOp(params, [n for n, _ in SMAN], _hp("adamw", "clip"), 2, lambda s: 1e-2, window_weight=True,
                       global_step=1)
    rng = np.random.default_rng(12)
    for w in (3.0, 37.0):
        for p, x in zip(op.params, _cuda(_grads(rng))):
            p.grad.add_(x)
        op.step(weight=w)
    assert op.window_weight_state() == {"weight": 0.0, "last_weight": 40.0}
    with pytest.raises(ValueError, match="weight"):
        op.step()


# ---- power-of-two window totals: the exact multiply by 1/W ------------------------------------------------------------
# (weight per micro-step, gradient sigma), N = 2: windows of W = 4 (step 0), 64, 2^-126 (the smallest normal power of two,
# as two subnormal weights), 2^127 (the largest) and 1
POW2_STEPS = [(4.0, 0.1), (32.0, 0.1), (32.0, 0.1), (2.0 ** -127, 1e-30), (2.0 ** -127, 1e-30),
              (2.0 ** 126, 0.1), (2.0 ** 126, 0.1), (0.5, 0.1), (0.5, 0.1)]


@pytest.mark.parametrize("variant, mode, layout", [("adamw", "noclip", "table"), ("adamw", "clip", "table"),
                                                   ("adamw", "clip", "packed"), ("adam", "ls_clip", "table"),
                                                   ("lamb", "clip", "table")])
def test_power_of_two_window_totals_match_the_oracle(variant, mode, layout):
    run = LockStep(MAN, variant, mode, layout, "fp32", True, None, N=2, seed=77, nograd=NOGRAD,
                   lr_mult=np.ones(len(MAN), F32), window_weight=True)
    lasts = []
    for w, sigma in POW2_STEPS:
        run.wstep(run.grads(sigma), w)                     # W and last_weight compared bit for bit after every step
        lasts.append(float(run.ref.last_weight))
    assert [lasts[i] for i in (0, 2, 4, 6, 8)] == [4.0, 64.0, 2.0 ** -126, 2.0 ** 127, 1.0]


# ---- full size ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["adamw", "lamb"])
def test_bert_small_full_size_with_mixed_weights_matches_the_oracle(variant):
    """BERT-Small's 73 tensors (28.8 M parameters: the clip-apply's ticket pool and stash and LAMB's CTA ranges at
    their real sizes) with clipping, mixed weights whose window totals are not powers of two, against the oracle
    after every apply."""
    import oracle_np as onp
    from apply_matrix import SCHED, oracle_hparams, reference_op, rel_err
    from gaccum_b200.train_op import GaccumTrainOp
    g = _g()
    man = onp.MANIFESTS["bert_small"]()
    names = [n for n, _ in man]
    rng = np.random.default_rng(13)
    params = [(rng.standard_normal(s, dtype=np.float32) * F32(0.02)) for _, s in man]
    hpo = oracle_hparams(variant, "clip")
    hp = g.HParams(hpo.variant, 0, hpo.beta1, hpo.beta2, hpo.epsilon, hpo.weight_decay_rate, hpo.clip_norm)
    lr_fn = lambda s: g.learning_rate(SCHED["init_lr"], SCHED["num_train_steps"], SCHED["num_warmup_steps"], s)
    n = 4
    op = GaccumTrainOp([torch.from_numpy(p.copy()).cuda() for p in params], names, hp, n, lr_fn, window_weight=True)
    ref = reference_op(variant, "clip", params, names, n, adapt=op.adapt if variant == "lamb" else None,
                       window_weight=True)
    weights = (37.0, 5.0, 1000.0, 3.0, 11.0, 64.0, 7.0, 250.0, 19.0)
    for s, w in enumerate(weights):
        grads = [(rng.standard_normal(sh, dtype=np.float32) * F32(1e-3)) for _, sh in man]
        info = ref.run(grads, weight=w)
        assert op.run([torch.from_numpy(x).cuda() for x in grads], weight=w) == info.applied
        torch.cuda.synchronize()
        st = op.window_weight_state()
        assert st["weight"] == float(ref.weight) and st["last_weight"] == float(ref.last_weight)
        for i in range(len(man)):
            assert np.array_equal(op.accum_view(i).cpu().numpy(), ref.accum[i]), i
        if info.applied:
            for i in range(len(man)):
                assert rel_err(op.params[i].cpu().numpy(), ref.params[i]) <= 1e-5, i
                assert rel_err(op.m_view(i).cpu().numpy(), ref.m[i]) <= 1e-5, i
                assert rel_err(op.v_view(i).cpu().numpy(), ref.v[i]) <= 1e-5, i
    assert float(ref.last_weight) == 64.0 + 7.0 + 250.0 + 19.0        # the window of steps 5-8


# ---- TensorFlow-format checkpoint on disk --------------------------------------------------------------------------
@pytest.mark.parametrize("variant, mode", [("adamw", "clip"), ("adam", "noclip")])
def test_resume_mid_window_through_a_checkpoint_bundle(variant, mode, tmp_path):
    from gaccum_b200 import tf_checkpoint as tfc
    params = _params(15)
    n = 4
    rng = np.random.default_rng(16)
    raw = [_grads(rng) for _ in range(3 * n)]
    ws = [WEIGHTS[i % len(WEIGHTS)] for i in range(3 * n)]
    full = _op(params, variant, mode, n, window_weight=True)
    first = _op(params, variant, mode, n, window_weight=True)
    second = _op(_params(98), variant, mode, n, window_weight=True)
    for x, w in zip(raw, ws):
        full.run(_cuda(x), weight=w)
    cut = n + 3
    for x, w in zip(raw[:cut], ws[:cut]):
        first.run(_cuda(x), weight=w)
    prefix = tfc.save(str(tmp_path), first)
    bundle = tfc.read_bundle(prefix)
    key = "gradient_accumulation/window_weight"
    assert np.asarray(bundle[key]).dtype == np.float32 and float(bundle[key]) == sum(ws[n + 1:cut])
    assert tfc.restore(str(tmp_path), second) == prefix
    assert second.window_weight_state()["weight"] == sum(ws[n + 1:cut])
    for x, w in zip(raw[cut:], ws[cut:]):
        second.run(_cuda(x), weight=w)
    torch.cuda.synchronize()
    for x, y in zip(_device_state(full), _device_state(second)):
        assert torch.equal(_bits(x), _bits(y))
