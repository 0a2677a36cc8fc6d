"""Per-tensor norms of the apply step on the GPU (gaccum.h, gaccum_plan_set_tensor_norms).

* every dispatch key: a train op with norms in lock-step with the same op without; everything else bit-identical, the
  norms against the oracle fed the kernel's own accumulators and weights, and with clipping sum_t gradient_t^2 against
  the global norm;
* skipped windows (loss scaling), overflow in the model's first and last tile;
* position independence: one tensor's norms bit for bit whether it comes first or behind a filler that puts its tiles
  across the clip-apply's stash/pool boundary and LAMB CTA boundaries;
* replays: repeated launches from one state, and a CUDA graph of whole windows with the device schedule and a window
  weight, bit for bit against the eager run;
* shapes and layouts, BERT-Small at full size, the C ABI on device plans, and the drop-in API."""
import ctypes as C
import zlib

import numpy as np
import pytest

from apply_matrix import LAYOUTS, Case, Schedule, matrix_cases
from tensor_norms_oracle import assert_close, expected_norms, norm

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

F32 = np.float32
MAN = [("a/kernel", (2 * 2048 + 777,)), ("a/bias", (5,)), ("one/kernel", (1,)), ("empty/kernel", (0,)),
       ("LayerNorm/gamma", (33,)), ("nograd/kernel", (64,)), ("t/kernel", (3, 1367))]
NOGRAD = (5,)
TINY = [(f"tiny{i}/{'bias' if i % 3 == 0 else 'kernel'}", (1 + i % 7,)) for i in range(300)]
N = 3
STEPS = 10                 # applies at steps 0, 3, 6 and 9
INF_AT = (4, 0, 1000)      # loss-scaled runs: the window that applies at step 6 overflows and is skipped
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}


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


def _bits(t):
    return t.contiguous().view(torch.int32) if t.element_size() == 4 else t.contiguous().view(torch.int16)


def _device_state(op):
    out = [op.accum, op.m, op.v] + [p for p in op.params]
    for name in ("master", "ema", "_ls_state", "_ema_state", "_ww_state", "_sched_state", "param_slab"):
        x = getattr(op, name, None)
        if x is not None:
            out.append(x)
    return out


def _assert_same_state(a, b):
    torch.cuda.synchronize()
    for i, (x, y) in enumerate(zip(_device_state(a), _device_state(b))):
        assert torch.equal(_bits(x), _bits(y)), i
    sa, sb = (np.array(list(o.stats().values()), F32) for o in (a, b))
    assert np.array_equal(sa.view(np.uint32), sb.view(np.uint32))
    if a.hp.variant == 2:
        assert np.array_equal(a.trust_ratios().view(np.uint32), b.trust_ratios().view(np.uint32))


class Pair:
    """One dispatch key's train op twice, with and without norms, stepped with the same gradients."""

    def __init__(self, case: Case, man, seed: int, nograd=NOGRAD):
        g = _g()
        from gaccum_b200.train_op import GaccumTrainOp, PackedTrainOp
        self.case, self.man, self.nograd = case, man, set(nograd)
        self.packed = case.layout == "packed"
        self.dtype = DTYPES[LAYOUTS[case.layout][2]]
        self.ls = case.mode.startswith("ls_")
        self.rng = np.random.default_rng(seed)
        names = [n for n, _ in man]
        params = [torch.from_numpy(self.rng.normal(0, 0.05, s).astype(F32)).to(self.dtype) for _, s in man]
        kw = dict(loss_scale=g.LossScaleConfig(16.0, 2.0, 2) if self.ls else None,
                  ema=g.EmaConfig(0.9, True) if case.ema else None)
        lr_fn = lambda s: g.learning_rate(1e-2, 40, 4, s)
        cls = PackedTrainOp if self.packed else GaccumTrainOp
        self.ops = [cls([p.clone().cuda() for p in params], names, _hp(case.variant, case.mode), N, lr_fn,
                        tensor_norms=on, **kw) for on in (False, True)]
        self.gslab = [torch.zeros_like(o.accum) for o in self.ops] if self.packed and case.has_g else None
        self.applies = 0

    def _slab(self, op, slab):
        host = slab.cpu().numpy()
        return [host[o:o + int(np.prod(s))].reshape(s).copy() for o, (_, s) in zip(op.plan.offsets, self.man)]

    def weights(self, op):
        if getattr(op, "master", None) is not None:
            return self._slab(op, op.master)
        if self.packed:
            return self._slab(op, op.param_slab)
        return [p.detach().float().cpu().numpy().copy() for p in op.params]

    def step(self, s: int) -> None:
        g = _g()
        x = [None if i in self.nograd else self.rng.normal(0, 0.1, sh).astype(F32) for i, (_, sh) in enumerate(self.man)]
        if self.ls and s == INF_AT[0]:
            x[INF_AT[1]].reshape(-1)[INF_AT[2]] = np.inf
        op_n = self.ops[1]
        S = float(op_n.loss_scale_state()["scale"]) if self.ls else 1.0
        dev = []
        with np.errstate(over="ignore", invalid="ignore"):
            for xi in x:
                dev.append(None if xi is None else torch.from_numpy(xi * F32(S)).to(self.dtype).cuda())
        host = [None if t is None else t.float().cpu().numpy() for t in dev]
        gstep = op_n.global_step
        applied = g.is_apply_step(gstep, N)
        snap = None
        for k, op in enumerate(self.ops):
            if self.packed:
                if self.case.has_g:
                    gs = self.gslab[k]
                    gs.zero_()
                    for i, t in enumerate(dev):
                        if t is not None:
                            op._view(gs, i).copy_(t)
                    if k == 1 and applied:
                        snap = (self._slab(op, op.accum), host, self.weights(op))
                    op.plan.step_packed(gs.data_ptr(), op.param_slab.data_ptr(), op.accum.data_ptr(), op.m.data_ptr(),
                                        op.v.data_ptr(), op._step_args(gstep, op.lr_fn(gstep)), -1, op._stream())
                    if applied:
                        op._advance_beta_powers()
                    op.global_step = gstep + 1
                else:
                    for p, t in zip(op.params, dev):
                        if t is not None:
                            p.grad.add_(t)
                    if k == 1 and applied:
                        snap = (self._slab(op, op.accum), None, self.weights(op))
                    assert op.step() == applied
            elif self.case.has_g:
                if k == 1 and applied:
                    snap = (self._slab(op, op.accum), host, self.weights(op))
                assert op.run(dev) == applied
            else:
                op.accumulate_only(dev)
                if applied:
                    if k == 1:
                        snap = (self._slab(op, op.accum), None, self.weights(op))
                    op.apply_only(None)
                op.global_step = gstep + 1
        _assert_same_state(*self.ops)
        if applied:
            self.applies += 1
            accum, grads, before = snap
            exp = expected_norms(accum, grads, N, S if self.ls else None, before, self.weights(op_n))
            got = op_n.tensor_norms()
            assert_close(got, exp, what=f"step {s}")
            if self.case.mode in ("clip", "ls_clip"):
                gn = op_n.stats()["global_norm"]
                if np.isfinite(gn) and gn > 0:
                    tot = float(np.sum(got[:, 0].astype(np.float64) ** 2))
                    assert abs(tot - gn * gn) <= 1e-6 * gn * gn, (tot, gn * gn)
            if self.ls and s == 6:
                assert op_n.loss_scale_state()["last_skipped"]
                assert np.isposinf(got[INF_AT[1], 0]) and not got[:, 2].any()


def _man(case: Case):
    return MAN + TINY if case.layout.startswith("t1920") else MAN


@pytest.mark.parametrize("case", matrix_cases(), ids=lambda c: c.id)
def test_every_dispatch_key_matches_the_oracle_and_changes_nothing_else(case: Case):
    pair = Pair(case, _man(case), zlib.crc32(case.id.encode()))
    for s in range(STEPS):
        pair.step(s)
    assert pair.applies == 4


def test_norms_are_zero_before_the_first_apply_and_readable_without_a_sync():
    g = _g()
    from gaccum_b200.train_op import GaccumTrainOp
    op = GaccumTrainOp([torch.ones(10, device="cuda")], ["w"], g.HParams.bert(), 2, lambda s: 1e-3, tensor_norms=True,
                       global_step=1)
    assert not op.tensor_norms().any()
    op.run([torch.ones(10, device="cuda")])                   # an accumulate step writes nothing
    assert not op.tensor_norms().any()
    t = op.tensor_norms_tensor
    assert t.shape == (1, 3) and t.dtype == torch.float32 and t.is_cuda
    op.run([torch.ones(10, device="cuda")])
    assert np.array_equal(op.tensor_norms(), t.cpu().numpy())
    assert op.tensor_norms()[0, 0] == np.sqrt(F32(10.0), dtype=F32)
    plain = GaccumTrainOp([torch.ones(10, device="cuda")], ["w"], g.HParams.bert(), 2, lambda s: 1e-3)
    with pytest.raises(ValueError):
        plain.tensor_norms()
    with pytest.raises(ValueError):
        plain.tensor_norms_tensor


# ---- skipped windows: overflow in the first tile and in the last tile ----------------------------------------------
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("variant, mode", [("adamw", "ls_clip"), ("adam", "ls_noclip"), ("lamb", "ls_clip"),
                                           ("lamb", "ls_noclip")])
def test_skipped_window_reports_the_overflowed_tensor(variant, mode, where):
    """fp16 model, loss-scaled: one gradient element overflows fp16 in the model's first tile (a stashed tile; LAMB's
    first CTA) or its last (a pool tile; LAMB's last CTA)."""
    g = _g()
    from gaccum_b200.train_op import GaccumTrainOp
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    nt = Schedule.STASH_TILES[False] * Schedule(sms).clip_groups(10 ** 6) + 40     # every stash slot filled, then a pool
    man = [("first/kernel", (2048,)), ("mid/kernel", ((nt - 2) * 2048,)), ("last/kernel", (1000,))]
    rng = np.random.default_rng(7)
    params = [torch.from_numpy(rng.normal(0, 0.05, s).astype(F32)).half().cuda() for _, s in man]
    op = GaccumTrainOp(params, [n for n, _ in man], _hp(variant, mode), 1, lambda s: 1e-2,
                       loss_scale=g.LossScaleConfig(16.0, 2.0, 2), tensor_norms=True)
    op.run([torch.from_numpy(rng.normal(0, 0.1, s).astype(F32)).half().cuda() for _, s in man])   # one applied window
    before = [op.master_view(i).cpu().numpy().copy() for i in range(3)]
    gr = [torch.from_numpy(rng.normal(0, 0.1, s).astype(F32)).half().cuda() for _, s in man]
    bad = 0 if where == "first" else 2
    gr[bad].view(-1)[7] = float("inf")
    op.run(gr)
    torch.cuda.synchronize()
    assert op.loss_scale_state()["last_skipped"]
    got = op.tensor_norms()
    assert np.isinf(got[bad, 0]) or np.isnan(got[bad, 0])
    assert all(np.isfinite(got[i, 0]) and got[i, 0] > 0 for i in range(3) if i != bad)
    assert not got[:, 2].any()
    assert_close(got[:, 1], np.array([norm(b) for b in before], F32))
    for i in range(3):
        assert np.array_equal(op.master_view(i).cpu().numpy(), before[i])


# ---- position independence --------------------------------------------------------------------------------------------
POS_CASES = [("adamw", "clip", False), ("adamw", "clip", True), ("adam", "ls_noclip", False), ("lamb", "clip", False),
             ("lamb", "noclip", False), ("adamw", "noclip", False)]


@pytest.mark.parametrize("variant, mode, ema", POS_CASES)
def test_tensor_norms_do_not_depend_on_the_tensor_position(variant, mode, ema):
    g = _g()
    from gaccum_b200.train_op import GaccumTrainOp
    sched = Schedule(torch.cuda.get_device_properties(0).multi_processor_count)
    x_tiles = 8
    # behind the filler, the tensor's tiles start 3 before the clip-apply's first pool tile (a group's own tiles before
    # it, pool tiles after it); with ~4 tiles per LAMB CTA they also cross LAMB CTA boundaries
    f_tiles = sched.pool_lo(10 ** 6, ema) - 3
    nt = f_tiles + x_tiles
    assert sched.pool_lo(nt, ema) == f_tiles + 3
    if variant == "lamb":
        ranges = sched.lamb_ranges(nt)
        assert sum(1 for lo, hi in ranges if f_tiles < lo < nt) >= 1
    x_shape, f_shape = (x_tiles * 2048 - 100,), (f_tiles * 2048,)
    rng = np.random.default_rng(11)
    x0, f0 = rng.normal(0, 0.05, x_shape).astype(F32), rng.normal(0, 0.05, f_shape).astype(F32)
    xg = [rng.normal(0, 0.1, x_shape).astype(F32) for _ in range(2)]
    fg = [rng.normal(0, 0.1, f_shape).astype(F32) for _ in range(2)]
    ls = g.LossScaleConfig(16.0, 2.0, 2) if mode.startswith("ls_") else None
    emac = g.EmaConfig(0.9, True) if ema else None
    rows = []
    for order in ((0, 1), (1, 0)):
        data = [(("x/kernel", x0), xg), (("filler/kernel", f0), fg)]
        data = [data[i] for i in order]
        op = GaccumTrainOp([torch.from_numpy(p).cuda() for (_, p), _ in data], [n for (n, _), _ in data],
                           _hp(variant, mode), 2, lambda s: 1e-2, global_step=1, loss_scale=ls, ema=emac, tensor_norms=True)
        S = 16.0 if ls else 1.0
        for j in range(2):
            op.run([torch.from_numpy(gr[j] * F32(S)).cuda() for _, gr in data])
        assert op.last_applied
        rows.append(op.tensor_norms()[order.index(0)])
    assert np.array_equal(rows[0].view(np.uint32), rows[1].view(np.uint32)), rows


# ---- replays ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant, mode", [("adamw", "clip"), ("adamw", "noclip"), ("adam", "ls_clip"), ("lamb", "clip"),
                                           ("lamb", "ls_noclip")])
def test_repeated_launches_and_graph_replays_are_bit_identical(variant, mode):
    g = _g()
    from gaccum_b200.train_op import GaccumTrainOp
    rng = np.random.default_rng(13)
    shapes = [s for _, s in MAN]
    params = [rng.normal(0, 0.05, s).astype(F32) for s in shapes]
    windows = 3
    grads = [[torch.from_numpy(rng.normal(0, 0.1, s).astype(F32)).cuda() for s in shapes] for _ in range(windows * N)]
    counts = [torch.tensor(c, dtype=torch.float32, device="cuda") for c in (3.0, 37.0, 1000.0)]
    ls = g.LossScaleConfig(16.0, 2.0, 2) if mode.startswith("ls_") else None
    from gaccum_b200._lib import ScheduleConfig
    sched = ScheduleConfig(1e-2, 40, 4)

    def make():
        return GaccumTrainOp([torch.from_numpy(p.copy()).cuda() for p in params], [n for n, _ in MAN], _hp(variant, mode),
                             N, None, loss_scale=ls, window_weight=True, device_schedule=sched, tensor_norms=True)

    def window(op, w, static=None):
        for j in range(N):
            op.window_weight += counts[j]
            op.run_bound(op.bind(grads[w * N + j] if static is None else static[j]))

    eager = make()
    per_window = []
    for w in range(windows):
        window(eager, w)
        per_window.append(eager.tensor_norms().copy())
    # repeated launches: the same apply from the same state writes the same bits
    again = make()
    window(again, 0)
    assert np.array_equal(again.tensor_norms().view(np.uint32), per_window[0].view(np.uint32))

    gop = make()
    init = gop.state_dict()
    window(gop, 0)                                   # loads every kernel outside the capture
    gop.load_state_dict(init)
    static = [[torch.zeros_like(x) for x in grads[0]] for _ in range(N)]
    graph = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        window(gop, 0, static)
    gop._ww_state.zero_()
    for w in range(windows):
        for j in range(N):
            for dst, src in zip(static[j], grads[w * N + j]):
                dst.copy_(src)
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(gop.tensor_norms().view(np.uint32), per_window[w].view(np.uint32)), w
    _assert_same_state(gop, eager)


# ---- shapes and layouts ------------------------------------------------------------------------------------------------
def _one_window(op, grads_fn, steps=2):
    for j in range(steps):
        op.run(grads_fn(j))
    assert op.last_applied


def _check_against_oracle(man, variant, mode, views=None, nograd=(), dtype=torch.float32):
    """One window of N = 2 (global_step 1, 2): the norms of the apply against the oracle of the kernel's inputs."""
    g = _g()
    from gaccum_b200.train_op import GaccumTrainOp
    rng = np.random.default_rng(zlib.crc32(repr((len(man), variant, mode)).encode()))

    def dev(x, off):
        t = torch.from_numpy(x).to(dtype)
        if off is None:
            return t.cuda()
        buf = torch.zeros(t.numel() + off + 8, dtype=dtype, device="cuda")
        v = buf[off:off + t.numel()].view(t.shape)
        v.copy_(t)
        return v
    views = views or {}
    params = [dev(rng.normal(0, 0.05, s).astype(F32), views.get(i)) for i, (_, s) in enumerate(man)]
    op = GaccumTrainOp(params, [n for n, _ in man], _hp(variant, mode), 2, lambda s: 1e-2, global_step=1, tensor_norms=True)
    # tensors in `nograd` get a gradient on the first micro-step only: the apply reports the norm of their accumulated c
    gr = [[None if j == 1 and i in nograd else dev(rng.normal(0, 0.1, s).astype(F32), views.get(i))
           for i, (_, s) in enumerate(man)] for j in range(2)]
    op.run(gr[0])
    torch.cuda.synchronize()
    accum = [op.accum_view(i).cpu().numpy().copy() for i in range(len(man))]
    wt = (lambda i: op.master_view(i)) if op.master is not None else (lambda i: op.params[i].detach())
    before = [wt(i).float().cpu().numpy().copy() for i in range(len(man))]
    op.run(gr[1])
    after = [wt(i).float().cpu().numpy().copy() for i in range(len(man))]
    host = [None if t is None else t.float().cpu().numpy() for t in gr[1]]
    got = op.tensor_norms()
    assert_close(got, expected_norms(accum, host, 2.0, None, before, after))
    return op, got


@pytest.mark.parametrize("variant, mode", [("adamw", "clip"), ("adamw", "noclip"), ("lamb", "clip")])
def test_the_1920_entry_table(variant, mode):
    man = [(f"t{i}/{'bias' if i % 4 == 0 else 'kernel'}", (1 + (i * 37) % 300,)) for i in range(1920)]
    _check_against_oracle(man, variant, mode)


@pytest.mark.parametrize("variant, mode", [("adamw", "clip"), ("adamw", "noclip"), ("lamb", "clip")])
def test_one_30522_by_1024_tensor(variant, mode):
    _check_against_oracle([("bert/embeddings/word_embeddings", (30522, 1024)), ("b/bias", (1024,))], variant, mode)


@pytest.mark.parametrize("variant, mode", [("adamw", "clip"), ("adam", "noclip"), ("lamb", "noclip")])
def test_unaligned_views_a_tensor_without_gradient_and_a_zero_element_tensor(variant, mode):
    man = [("u/kernel", (5000,)), ("nog/kernel", (3000,)), ("empty/kernel", (0,)), ("v/kernel", (2049,))]
    op, got = _check_against_oracle(man, variant, mode, views={0: 1, 3: 3}, nograd=(1,))
    assert not got[2].any()
    assert got[1, 0] > 0 and got[1, 2] > 0


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("variant, mode", [("adamw", "clip"), ("adamw", "noclip"), ("lamb", "clip")])
def test_16_bit_model_matches_the_upcast_fp32_run(variant, mode, dtype):
    g = _g()
    from gaccum_b200.train_op import GaccumTrainOp
    man = [("a/kernel", (4 * 2048 + 333,)), ("b/bias", (77,)), ("c/kernel", (64, 65))]
    rng = np.random.default_rng(17)
    p16 = [torch.from_numpy(rng.normal(0, 0.05, s).astype(F32)).to(dtype) for _, s in man]
    g16 = [[torch.from_numpy(rng.normal(0, 0.1, s).astype(F32)).to(dtype) for _, s in man] for _ in range(2)]
    out = []
    for dt in (dtype, torch.float32):
        op = GaccumTrainOp([p.to(dt).cuda() for p in p16], [n for n, _ in man], _hp(variant, mode), 2, lambda s: 1e-2,
                           global_step=1, tensor_norms=True)
        _one_window(op, lambda j: [x.to(dt).cuda() for x in g16[j]])
        out.append(op.tensor_norms())
    assert_close(out[0], out[1])
    _check_against_oracle(man, variant, mode, dtype=dtype)


# ---- full size ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["adamw", "lamb"])
def test_bert_small_full_size_matches_the_oracle(variant):
    import oracle_np as onp
    man = onp.MANIFESTS["bert_small"]()
    _check_against_oracle(list(man), variant, "clip")


# ---- the C ABI on device plans --------------------------------------------------------------------------------------
def _L():
    from gaccum_b200 import _lib
    return _lib, _lib._load()


def _device_plan(variant=2):
    g = _g()
    hp = g.HParams(variant, 0, 0.9, 0.999, 1e-6, 0.01, 1.0)
    return g.Plan([1000, 37, 5], [True, False, True], hp, device=0)


def test_setter_is_refused_after_a_compute_call():
    lib, L = _L()
    from gaccum_b200.train_op import GaccumTrainOp
    op = GaccumTrainOp([torch.ones(8, device="cuda")], ["w"], _g().HParams.bert(), 2, lambda s: 1e-3)
    op.run([torch.ones(8, device="cuda")])
    buf = torch.zeros(4, device="cuda")
    assert L.gaccum_plan_set_tensor_norms(op.plan._h, buf.data_ptr()) == lib.EINVAL
    assert "before the plan's first compute call" in L.gaccum_last_error().decode()


OTHERS = ["ww", "lr_mult", "ema", "dtype", "loss_scale", "adapt"]


@pytest.mark.parametrize("pos", range(len(OTHERS) + 1))
@pytest.mark.parametrize("reverse", [False, True])
def test_setters_combine_in_any_order(pos, reverse):
    lib, L = _L()
    plan = _device_plan()
    buf = torch.full((3 * 3 + 4,), 7.0, device="cuda")
    calls = {
        "norms": lambda: L.gaccum_plan_set_tensor_norms(plan._h, buf.data_ptr()),
        "ww": lambda: L.gaccum_plan_set_window_weight(plan._h, 0x50000),
        "lr_mult": lambda: L.gaccum_plan_set_lr_multipliers(plan._h, C.cast((C.c_float * 3)(0.5, 0.0, 2.0), C.c_void_p)),
        "ema": lambda: L.gaccum_plan_set_ema(plan._h, C.byref(lib.EmaConfig(0.999)), 0x10000, 0x20000),
        "dtype": lambda: L.gaccum_plan_set_param_dtype(plan._h, lib.DTYPE_BF16, 0x30000),
        "loss_scale": lambda: L.gaccum_plan_set_loss_scale(plan._h, C.byref(lib.LossScaleConfig()), 0x40000),
        "adapt": lambda: L.gaccum_plan_set_layer_adaptation(plan._h, C.cast((C.c_uint8 * 3)(1, 0, 1), C.c_void_p)),
    }
    order = (OTHERS[::-1] if reverse else list(OTHERS))
    order.insert(pos, "norms")
    for what in order:
        assert calls[what]() == 0, what
    torch.cuda.synchronize()
    assert not buf[:9].any() and bool((buf[9:] == 7.0).all())          # zeroed: 3 x num_tensors floats, nothing more
    assert plan.algorithmic_bytes(True) == 56 * plan.num_elements


@pytest.mark.parametrize("variant", [0, 1, 2])
def test_algorithmic_bytes_are_unchanged(variant):
    a, b = _device_plan(variant), _device_plan(variant)
    buf = torch.zeros(16, device="cuda")
    b.set_tensor_norms(buf.data_ptr())
    for is_apply in (True, False):
        assert a.algorithmic_bytes(is_apply) == b.algorithmic_bytes(is_apply)


def test_c_entry_points_without_norms_refuse_the_plan():
    lib, L = _L()
    plan = _device_plan(variant=0)
    buf = torch.zeros(16, device="cuda")
    plan.set_tensor_norms(buf.data_ptr())
    h = C.c_void_p()
    assert L.gaccum_host_session_create(C.byref(h), plan._h) == lib.EINVAL
    assert "per-tensor norms" in L.gaccum_last_error().decode()
    comm = lib.DpComm()
    args = lib.StepArgs(0, 1, 0, 1e-3, 0.9, 0.999, 0.0)
    for fn in (L.gaccum_step_dp, L.gaccum_apply_dp):
        assert fn(plan._h, C.byref(comm), None, None, None, C.byref(args), 1, None) == lib.EINVAL
        assert "per-tensor norms" in L.gaccum_last_error().decode()


def test_data_parallel_engine_takes_the_option():
    """DataParallelTrainOp's engine is a caller-built GaccumTrainOp: it may report norms (every rank applies the same
    reduced window).  Without a process group only the construction is checked here."""
    from gaccum_b200.train_op import GaccumTrainOp
    op = GaccumTrainOp([torch.ones(8, device="cuda")], ["w"], _g().HParams.bert(), 1, lambda s: 1e-3, tensor_norms=True)
    op.apply_only([torch.ones(8, device="cuda")])
    torch.cuda.synchronize()
    assert op.tensor_norms()[0, 0] == np.sqrt(F32(8.0), dtype=F32)


# ---- the drop-in API ---------------------------------------------------------------------------------------------------
def _tiny_model():
    from gaccum_b200 import graph
    graph.reset_default_graph()
    torch.manual_seed(0)
    lin = torch.nn.Linear(16, 4).cuda()
    graph.register_module(lin, lambda n: "dense/" + ("kernel" if n == "weight" else n))
    x, y = torch.randn(8, 16, device="cuda"), torch.randn(8, 4, device="cuda")
    return lin, lambda: torch.nn.functional.mse_loss(lin(x), y)


def test_create_optimizer_with_the_module_attribute(monkeypatch):
    from gaccum_b200 import optimization as opt
    lin, loss = _tiny_model()
    monkeypatch.setattr(opt, "tensor_norms", True)
    monkeypatch.setattr(opt, "gradient_accumulation_multiplier", 2)
    op = opt.create_optimizer(loss, 1e-3, 100, 10, False)
    for _ in range(3):
        op.run()
    got = op.tensor_norms()
    assert set(got) == {v.name.split(":")[0] for v in op.tvars}
    for k, (gn, wn, un) in got.items():
        assert gn > 0 and wn > 0 and un > 0, k
    assert not op.engine.tensor_norms_tensor.isnan().any()


def test_gradient_accumulation_train_op_takes_the_option():
    from gaccum_b200 import optimization as opt
    lin, loss = _tiny_model()
    op = opt.gradient_accumulation_train_op(loss, opt.AdamOptimizer(1e-3), 2, tensor_norms=True)
    for _ in range(3):
        op.run()
    assert all(len(v) == 3 for v in op.tensor_norms().values())
    plain = opt.gradient_accumulation_train_op(loss, opt.AdamOptimizer(1e-3), 2)
    with pytest.raises(ValueError):
        plain.tensor_norms()
