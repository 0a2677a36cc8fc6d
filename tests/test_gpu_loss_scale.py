"""Dynamic loss scaling on the GPU (include/gaccum.h, gaccum_plan_set_loss_scale).

* With finite gradients and S a power of two, a loss-scaled run fed S * g is bit-identical to the run without loss
  scaling fed g: p, m, v, the accumulators, gn and the clip scale, growth events included.
* A window in which a gradient overflows -- at its first micro-step, a middle one or the apply step; in a stashed or a
  pool tile of the clip kernel, a vector body, a scalar tail or an unaligned view -- leaves p, m and v unchanged bit for
  bit, zeroes the accumulators and backs S off; later windows match the numpy oracle (tests/composed_oracle.py).
"""
import os
import socket
import sys

import numpy as np
import pytest

import oracle_np as onp
from composed_oracle import ComposedReferenceTrainOp

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# tails (< 4 elements), a tile with a vector body and a 3-element tail (2055 = 2048 + 7), several tiles, one element
MAN = [("a/kernel", (777,)), ("a/bias", (5,)), ("b/kernel", (3, 1367)), ("t/kernel", (2055,)), ("one", (1,)),
       ("LayerNorm/gamma", (33,))]
LR = 1e-3


def _g():
    import gaccum_b200 as g
    return g


def _hp(variant_b, clip):
    g = _g()
    hp_g = g.HParams.tf_adam() if variant_b else g.HParams.bert()
    hp_o = onp.HParams.tf_adam() if variant_b else onp.HParams.bert()
    hp_g.clip_norm = clip
    hp_o.clip_norm = clip
    return hp_g, hp_o


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(x, y):
    return torch.equal(_bits(x), _bits(y))


def _params(man, seed):
    rng = np.random.default_rng(seed)
    return [rng.normal(0, 0.05, s).astype(np.float32) for _, s in man]


def _gaccum_op(man, params, hp, N, ls=None, global_step=0):
    from gaccum_b200.train_op import GaccumTrainOp
    return GaccumTrainOp([torch.from_numpy(p.copy()).cuda() for p in params], [n for n, _ in man], hp, N, lambda s: LR,
                         global_step=global_step, loss_scale=ls)


def _state(op):
    return op.loss_scale_state()


# ---- bit-identity with the run without loss scaling ---------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 3, 4])
@pytest.mark.parametrize("clip", [0.0, 1.0, 1e-3])
@pytest.mark.parametrize("variant_b", [False, True])
def test_scaled_run_is_bit_identical_to_unscaled(variant_b, clip, N):
    g = _g()
    hp, _ = _hp(variant_b, clip)
    params = _params(MAN, 1)
    off = _gaccum_op(MAN, params, hp, N)
    on = _gaccum_op(MAN, params, hp, N, g.LossScaleConfig(2.0 ** 12, 2.0, 2))
    gen = torch.Generator(device="cuda").manual_seed(7)
    scales = set()
    for step in range(6 * N + 1):
        grads = [torch.randn(s, device="cuda", generator=gen) * 0.1 for _, s in MAN]
        S = _state(on)["scale"]
        scales.add(S)
        a = off.run(grads)
        b = on.run([x * on.loss_scale for x in grads])
        assert a == b
        if a:
            assert off.stats() == on.stats()
        for x, y in zip(off.params + [off.m, off.v, off.accum * S], on.params + [on.m, on.v, on.accum]):
            assert _same(x, y), step                   # the accumulators hold S * sum(g): exact, S is a power of two
    assert len(scales) > 2
    st = on.state_dict()
    if variant_b:
        assert float(st["beta1_power"]) == np.float32(off.beta1_power)
        assert float(st["beta2_power"]) == np.float32(off.beta2_power)


@pytest.mark.parametrize("N", [1, 3, 4])
@pytest.mark.parametrize("clip", [0.0, 1.0])
@pytest.mark.parametrize("variant_b", [False, True])
def test_packed_scaled_run_is_bit_identical_to_unscaled(variant_b, clip, N):
    g = _g()
    from gaccum_b200.train_op import PackedTrainOp
    hp, _ = _hp(variant_b, clip)
    params = _params(MAN, 2)
    names = [n for n, _ in MAN]
    mk = lambda ls: PackedTrainOp([torch.from_numpy(p.copy()).cuda() for p in params], names, hp, N, lambda s: LR,
                                  loss_scale=ls)
    off, on = mk(None), mk(g.LossScaleConfig(2.0 ** 10, 4.0, 1))
    gen = torch.Generator(device="cuda").manual_seed(8)
    for step in range(4 * N + 1):
        grads = [torch.randn(s, device="cuda", generator=gen) * 0.1 for _, s in MAN]
        S = _state(on)["scale"]
        for p_off, p_on, x in zip(off.params, on.params, grads):   # what AccumulateGrad does: grad += new_grad
            p_off.grad.add_(x)
            p_on.grad.add_(x * on.loss_scale)
        assert off.step() == on.step()
        for x, y in ((off.param_slab, on.param_slab), (off.m, on.m), (off.v, on.v), (off.accum * S, on.accum)):
            assert _same(x, y), step
    assert _state(on)["scale"] > 2.0 ** 10


@pytest.mark.parametrize("variant_b", [False, True])
def test_full_size_bert_small_is_bit_identical_to_unscaled(variant_b):
    g = _g()
    man = onp.MANIFESTS["bert_small"]()
    hp, _ = _hp(variant_b, 0.0 if variant_b else 1.0)
    gen = torch.Generator(device="cuda").manual_seed(1)
    init = [torch.randn(s, device="cuda", generator=gen) * 0.02 for _, s in man]
    from gaccum_b200.train_op import GaccumTrainOp
    mk = lambda ls: GaccumTrainOp([p.clone() for p in init], [n for n, _ in man], hp, 2, lambda s: 1e-4, loss_scale=ls)
    off, on = mk(None), mk(g.LossScaleConfig(2.0 ** 14, 2.0, 2))
    grads = [torch.empty(s, device="cuda") for _, s in man]
    for step in range(9):
        for x in grads:
            x.normal_(0.0, 1e-3, generator=gen)
        off.run(grads)
        on.run([x * on.loss_scale for x in grads])
    torch.cuda.synchronize()
    assert off.stats() == on.stats()
    for x, y in zip(off.params + [off.m, off.v, off.accum], on.params + [on.m, on.v, on.accum]):
        assert _same(x, y)
    assert _state(on) == {"scale": 2.0 ** 16, "good_windows": 1, "skipped_windows": 0, "last_skipped": False}


# ---- overflow injection -------------------------------------------------------------------------------------------
# More than 4 stash tiles x 3 groups x 132 CTAs = 1584 tiles, so that the clip kernel has pool tiles: "emb" tile 0 is a
# stashed tile, tile 1700 a pool tile.  "t" has a 7-element tile (vector body + 3-element tail); "u" gets its gradient
# as a view 4 bytes past a 16-byte boundary (scalar path).
BIG = [("emb", (3_500_000,)), ("t/kernel", (2055,)), ("u/kernel", (1000,)), ("LayerNorm/gamma", (5,))]
WHERE = {"stash": (0, 100), "pool": (0, 1700 * 2048 + 9), "vector": (1, 2048 + 1), "tail": (1, 2048 + 5),
         "unaligned": (2, 513)}


def _device_grads(grads, ubuf):
    out = []
    for i, x in enumerate(grads):
        if i == 2:
            v = ubuf[1:1 + x.size]
            v.copy_(torch.from_numpy(x))
            out.append(v)
        else:
            out.append(torch.from_numpy(x).cuda())
    return out


@pytest.mark.parametrize("where", list(WHERE))
@pytest.mark.parametrize("when", ["first", "middle", "apply"])
@pytest.mark.parametrize("kind", ["inf", "-inf", "nan", "finite"])
def test_overflowed_window_is_skipped(kind, when, where):
    g = _g()
    N = 3
    hp, hp_o = _hp(False, 1.0)
    params = _params(BIG, 3)
    cfg = dict(initial_scale=2.0 ** 10, multiplier=2.0, growth_interval=1000)
    op = _gaccum_op(BIG, params, hp, N, g.LossScaleConfig(cfg["initial_scale"], cfg["multiplier"], cfg["growth_interval"]))
    ref = ComposedReferenceTrainOp([p.copy() for p in params], [n for n, _ in BIG], hp_o, N, constant_lr=LR, **cfg)
    ubuf = torch.zeros(1100, device="cuda")
    rng = np.random.default_rng(4)
    t_i, e_i = WHERE[where]
    k = {"first": 0, "middle": 1, "apply": 2}[when]
    val = {"inf": np.inf, "-inf": -np.inf, "nan": np.nan, "finite": 3.0e38}[kind]
    snap = None
    for step in range(3 * N + 1):               # windows g = 0 | 1, 2, 3 (injected) | 4, 5, 6 | 7, 8, 9
        scale = np.float32(ref.scale)
        grads = [(rng.normal(0, 1e-5, s) * scale).astype(np.float32) for _, s in BIG]
        j = step - 1
        if 0 <= j < N and (j == k or (kind == "finite" and j == (k - 1 if k else 1))):
            grads[t_i].reshape(-1)[e_i] = np.float32(val)
        if step == 1:
            torch.cuda.synchronize()
            snap = [t.clone() for t in op.params + [op.m, op.v]]
        with np.errstate(over="ignore", invalid="ignore"):
            info = ref.run(grads)
        assert op.run(_device_grads(grads, ubuf)) == info.applied
        if step == N:
            torch.cuda.synchronize()
            assert ref.last_skipped
            for x, y in zip(snap, op.params + [op.m, op.v]):
                assert _same(x, y)
            assert not bool(_bits(op.accum).any())
            assert _state(op) == {"scale": 2.0 ** 9, "good_windows": 0, "skipped_windows": 1, "last_skipped": True}
    torch.cuda.synchronize()
    assert _state(op) == {"scale": 2.0 ** 9, "good_windows": 2, "skipped_windows": 1, "last_skipped": False}
    for i in range(len(BIG)):
        for got, exp in ((op.params[i], ref.params[i]), (op.m_view(i), ref.m[i]), (op.v_view(i), ref.v[i]),
                         (op.accum_view(i), ref.accum[i])):
            assert np.array_equal(got.cpu().numpy().view(np.uint32), exp.view(np.uint32))


@pytest.mark.parametrize("variant_b", [False, True])
def test_squared_sum_overflow_skips_only_with_clipping(variant_b):
    """Finite elements whose squares overflow fp32: a non-finite norm skips the window with clipping on; with clipping
    off every element is finite, so the window is applied and matches the oracle."""
    g = _g()
    for clip, skipped in ((1.0, True), (0.0, False)):
        hp, hp_o = _hp(variant_b, clip)
        params = _params(MAN, 5)
        op = _gaccum_op(MAN, params, hp, 1, g.LossScaleConfig(1.0, 2.0, 100))
        ref = ComposedReferenceTrainOp([p.copy() for p in params], [n for n, _ in MAN], hp_o, 1, constant_lr=LR,
                                       initial_scale=1.0, multiplier=2.0, growth_interval=100)
        rng = np.random.default_rng(6)
        for step in range(2):                    # (with clipping off, v = inf afterwards: later steps would make NaNs)
            grads = [rng.normal(0, 0.1, s).astype(np.float32) for _, s in MAN]
            if step == 1:
                grads[2].reshape(-1)[:4] = np.float32(2e19)
            with np.errstate(over="ignore", invalid="ignore"):
                ref.run(grads)
            op.run([torch.from_numpy(x).cuda() for x in grads])
            if step == 1:
                assert _state(op)["last_skipped"] == skipped == ref.last_skipped
        for i in range(len(MAN)):
            for got, exp in ((op.params[i], ref.params[i]), (op.m_view(i), ref.m[i]), (op.v_view(i), ref.v[i])):
                got = got.cpu().numpy()
                if clip > 0:                     # gn is accumulated differently: clip scales agree to ~1 ulp
                    d = np.max(np.abs(got.astype(np.float64) - exp)) / max(float(np.max(np.abs(exp))), 1e-30)
                    assert d <= 1e-5
                else:
                    assert np.array_equal(got.view(np.uint32), exp.view(np.uint32))


@pytest.mark.parametrize("seed", range(6))
def test_random_trajectories_with_overflows_match_the_oracle(seed):
    g = _g()
    rng = np.random.default_rng(900 + seed)
    variant_b = bool(seed % 2)
    clip = 1.0 if seed % 3 else 0.0
    N = int(rng.integers(1, 5))
    hp, hp_o = _hp(variant_b, clip)
    params = _params(MAN, seed)
    cfg = dict(initial_scale=2.0 ** int(rng.integers(0, 20)), multiplier=2.0 ** int(rng.integers(1, 3)),
               growth_interval=int(rng.integers(1, 4)))
    op = _gaccum_op(MAN, params, hp, N, g.LossScaleConfig(cfg["initial_scale"], cfg["multiplier"], cfg["growth_interval"]))
    ref = ComposedReferenceTrainOp([p.copy() for p in params], [n for n, _ in MAN], hp_o, N, constant_lr=LR, **cfg)
    for step in range(8 * N + 2):
        # small gradients: gn < 1, so the clip scale is exactly 1 on both sides and every value compares bit for bit
        grads = [(rng.normal(0, 1e-5, s) * np.float32(ref.scale)).astype(np.float32) for _, s in MAN]
        if rng.random() < 0.15:
            t = int(rng.integers(0, len(MAN)))
            grads[t].reshape(-1)[int(rng.integers(0, grads[t].size))] = rng.choice([np.inf, -np.inf, np.nan])
        with np.errstate(over="ignore", invalid="ignore"):
            info = ref.run(grads)
        assert op.run([torch.from_numpy(x).cuda() for x in grads]) == info.applied
        st = _state(op)
        assert (st["scale"], st["good_windows"], st["skipped_windows"]) == \
            (float(ref.scale), ref.good_windows, ref.skipped_windows), step
        for i in range(len(MAN)):
            for got, exp in ((op.params[i], ref.params[i]), (op.m_view(i), ref.m[i]), (op.v_view(i), ref.v[i]),
                             (op.accum_view(i), ref.accum[i])):
                # mid-window accumulators may hold NaNs: the GPU's add returns the canonical NaN, numpy keeps the payload
                got = got.cpu().numpy().ravel()
                exp = exp.ravel()
                nan = np.isnan(exp)
                assert np.array_equal(np.isnan(got), nan), (step, i)
                assert np.array_equal(got[~nan].view(np.uint32), exp[~nan].view(np.uint32)), (step, i)
    if variant_b:
        sd = op.state_dict()
        assert float(sd["beta1_power"]) == ref.beta1_power and float(sd["beta2_power"]) == ref.beta2_power


# ---- CUDA graphs, checkpoints, the training front end ---------------------------------------------------------------
def test_graph_captured_window_replays_through_overflow_backoff_and_growth():
    """A whole window -- the producer scaling its gradients by op.loss_scale on the device, N - 1 accumulates and the
    apply -- captured once and replayed: S backs off on an overflowed window and grows again with no host sync."""
    g = _g()
    N = 2
    hp, _ = _hp(True, 0.0)
    params = _params(MAN, 9)
    cfg = g.LossScaleConfig(2.0 ** 8, 2.0, 2)
    eager = _gaccum_op(MAN, params, hp, N, cfg, global_step=1)
    graphed = _gaccum_op(MAN, params, hp, N, cfg, global_step=1)
    src = [[torch.zeros(s, device="cuda") for _, s in MAN] for _ in range(N)]
    bufs = [[torch.zeros(s, device="cuda") for _, s in MAN] for _ in range(N)]
    tables = [graphed.bind(b) for b in bufs]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    cg = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        for k in range(N):                                  # warm-up outside capture, then reset the state
            graphed.run_bound(tables[k], side.cuda_stream)
        graphed.load_state_dict(eager.state_dict())
        torch.cuda.synchronize()
        with torch.cuda.graph(cg, stream=side):
            for k in range(N):
                for b, x in zip(bufs[k], src[k]):
                    torch.mul(x, graphed.loss_scale, out=b)
                graphed.run_bound(tables[k], side.cuda_stream)
    rng = np.random.default_rng(10)
    scales = []
    for w in range(6):
        host = [[rng.normal(0, 0.1, s).astype(np.float32) for _, s in MAN] for _ in range(N)]
        if w == 1:
            host[0][3].reshape(-1)[17] = np.inf
        for k in range(N):
            for x, h in zip(src[k], host[k]):
                x.copy_(torch.from_numpy(h))
        cg.replay()
        eager.global_step = 1
        for k in range(N):
            eager.run([torch.from_numpy(h).cuda() * eager.loss_scale for h in host[k]])
        torch.cuda.synchronize()
        scales.append(_state(graphed)["scale"])
        assert _state(graphed) == _state(eager)
        for x, y in zip(eager.params + [eager.m, eager.v, eager.accum], graphed.params + [graphed.m, graphed.v, graphed.accum]):
            assert _same(x, y)
    assert scales == [2.0 ** 8, 2.0 ** 7, 2.0 ** 7, 2.0 ** 8, 2.0 ** 8, 2.0 ** 9]


@pytest.mark.parametrize("variant_b", [False, True])
def test_state_dict_round_trip_mid_window_continues_bit_identically(variant_b):
    g = _g()
    N = 3
    hp, _ = _hp(variant_b, 1.0)
    params = _params(MAN, 11)
    cfg = g.LossScaleConfig(2.0 ** 6, 2.0, 2)
    a = _gaccum_op(MAN, params, hp, N, cfg)
    gen = torch.Generator(device="cuda").manual_seed(3)
    grads = [[torch.randn(s, device="cuda", generator=gen) * 0.1 for _, s in MAN] for _ in range(5 * N)]
    for step in range(3 * N + 2):                       # stops mid-window: g = 3N + 1 starts a window
        gr = grads[step]
        if step == N:
            gr = [x.clone() for x in gr]; gr[0][0] = float("nan")
        a.run([x * a.loss_scale for x in gr])
    sd = a.state_dict()
    assert float(sd["loss_scale/current_loss_scale"]) == _state(a)["scale"]
    assert int(sd["loss_scale/good_steps"]) == _state(a)["good_windows"]
    b = _gaccum_op(MAN, params, hp, N, g.LossScaleConfig(2.0 ** 20, 2.0, 2))
    b.load_state_dict(sd)
    for step in range(3 * N + 2, 5 * N):
        a.run([x * a.loss_scale for x in grads[step]])
        b.run([x * b.loss_scale for x in grads[step]])
    torch.cuda.synchronize()
    for x, y in zip(a.params + [a.m, a.v, a.accum], b.params + [b.m, b.v, b.accum]):
        assert _same(x, y)
    sa, sb = a.state_dict(), b.state_dict()
    for key in ("loss_scale/current_loss_scale", "loss_scale/good_steps") + (("beta1_power", "beta2_power") if variant_b else ()):
        assert torch.equal(sa[key], sb[key]), key
    bad = dict(sd)
    bad["loss_scale/current_loss_scale"] = torch.tensor(3.0)
    with pytest.raises(ValueError):
        b.load_state_dict(bad)


def test_autocast_fp16_training_backs_off_then_learns():
    """A small model under torch.autocast(float16) through gradient_accumulation_train_op, starting at S = 2^24: the
    first windows overflow and back off, then the loss falls; no parameter is ever non-finite."""
    g = _g()
    from gaccum_b200 import graph
    from gaccum_b200.optimization import AdamOptimizer, gradient_accumulation_train_op
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(32, 64), torch.nn.ReLU(), torch.nn.Linear(64, 1)).cuda()
    tvars = [graph.Variable(n, p) for n, p in model.named_parameters()]
    X = torch.randn(512, 32, device="cuda")
    y = X[:, :1] * 0.5 - X[:, 1:2] * 0.25
    it = iter(range(10 ** 9))

    def loss_fn():
        i = next(it) % 8
        with torch.autocast("cuda", dtype=torch.float16):
            out = model(X[i * 64:(i + 1) * 64])
        return torch.nn.functional.mse_loss(out.float(), y[i * 64:(i + 1) * 64])

    op = gradient_accumulation_train_op(loss_fn, AdamOptimizer(1e-2), 4, tvars=tvars, global_step=graph.GlobalStep(0),
                                        loss_scale=g.LossScaleConfig(2.0 ** 24, 2.0, 5))
    losses = []
    for step in range(400):
        losses.append(float(op.run()))
        if step % 4 == 3:
            assert all(bool(torch.isfinite(p).all()) for p in model.parameters())
    st = op.engine.loss_scale_state()
    assert st["skipped_windows"] >= 1 and st["scale"] < 2.0 ** 24
    assert np.mean(losses[-40:]) < 0.5 * np.mean(losses[:40])


def _dp_worker(rank, world, port, outdir):
    for p in (ROOT, os.path.join(ROOT, "oracle")):
        sys.path.insert(0, p)
    import torch.distributed as dist
    import gaccum_b200 as g
    from gaccum_b200.distributed import DataParallelTrainOp
    from gaccum_b200.train_op import GaccumTrainOp
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world,
                            device_id=torch.device("cuda", rank))
    rng = np.random.default_rng(5)
    params = [torch.from_numpy(rng.normal(0, 0.02, s).astype(np.float32)).cuda() for _, s in MAN]
    op = GaccumTrainOp(params, [n for n, _ in MAN], g.HParams.tf_adam(), 2, lambda s: 1e-2,
                       loss_scale=g.LossScaleConfig(2.0 ** 8, 2.0, 2))
    dp = DataParallelTrainOp(op, None)
    snaps = []
    for s in range(7):
        r = np.random.default_rng(100 * rank + s)
        grads = [torch.from_numpy(r.normal(0, 0.1, sh).astype(np.float32)).cuda() * op.loss_scale for _, sh in MAN]
        if rank == 1 and s == 3:
            grads[1][2] = float("inf")              # only this rank overflows, in the window that applies at s = 4
        dp.run(grads)
        torch.cuda.synchronize()
        snaps.append(op.loss_scale_state()["last_skipped"])
    np.savez(os.path.join(outdir, f"ls_rank{rank}.npz"), *[p.cpu().numpy() for p in params], m=op.m.cpu().numpy(),
             v=op.v.cpu().numpy(), skipped=np.array(snaps), scale=op.loss_scale_state()["scale"],
             b1=float(op.state_dict()["beta1_power"]))
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_allreduce_data_parallel_skips_on_every_rank(tmp_path):
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]
    mp.spawn(_dp_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = np.load(tmp_path / "ls_rank0.npz"), np.load(tmp_path / "ls_rank1.npz")
    for k in r0.files:
        assert np.array_equal(r0[k], r1[k]), f"replicas differ in {k}"
    assert list(r0["skipped"]) == [False, False, False, False, True, True, False]


def test_device_paths_that_refuse_loss_scaling():
    """gaccum_step_dp / gaccum_apply_dp and the host-buffer session refuse a loss-scaled plan."""
    g = _g()
    from gaccum_b200 import _lib
    plan = g.Plan([100], None, g.HParams.bert(), device=0)
    state = torch.zeros(8, device="cuda")
    plan.set_loss_scale(g.LossScaleConfig(), state.data_ptr())
    with pytest.raises(_lib.GaccumError, match="loss scaling"):
        _lib.HostSession(plan)
    comm = _lib.DpComm()
    slab = torch.zeros(128, device="cuda")
    with pytest.raises(_lib.GaccumError, match="loss scaling"):
        plan.apply_dp(comm, None, slab.data_ptr(), slab.data_ptr(), g.StepArgs(0, 1, 0, 1e-3, 0.9, 0.999, 0.0), 1)
    with pytest.raises(_lib.GaccumError, match="loss scaling"):
        plan.step_dp(comm, None, slab.data_ptr(), slab.data_ptr(), g.StepArgs(0, 1, 0, 1e-3, 0.9, 0.999, 0.0), 1)
