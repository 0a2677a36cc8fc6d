"""The device schedule (include/gaccum.h, gaccum_plan_set_device_schedule) against the composed oracle.

a. Every dispatch key (336 cases), eagerly, with learning-rate multipliers, mixed window weights and per-tensor norms on,
   over a schedule that passes the end of warm-up and the end of decay, in ``LockStep``'s injected mode: p, m, v, the
   accumulators, the master weights and model copy, the EMA, the loss-scaling block, the device counter, the lr of every
   micro-step and the beta powers in their one home are compared bit for bit after every micro-step; the norms within
   ``tensor_norms_oracle``'s tolerance.
b. One window captured as a CUDA graph and replayed, for every (variant, mode, layout), with and without EMA: after every
   replay every buffer of the op equals, bit for bit, that of an eager twin checked against the oracle as in a.
c. Refusal and recovery in each kernel family: a launch whose kernel the device step does not select (a replayed graph
   that ends mid-window, or a launch from a front end that lost track of the step) changes no buffer; after
   ``op.global_step = g`` training continues and matches the oracle over two or more applies.
d. The int32 wrap of global_step: from 2^31 - 2N (N = 3, 5, and 4 as a control) and from 2^32 - 2N, the host-scheduled
   op, the device-scheduled op and the oracle agree bit for bit, accumulators included, with a warm-up whose int32 cast
   gives a negative lr past 2^31.  A whole-window graph replayed into the window that straddles 2^31 is refused and
   changes nothing; the documented recovery continues the run, and replays resume from the next window start.
"""
import gc
import zlib

import numpy as np
import pytest

from apply_matrix import LAYOUTS, MODES, VARIANTS, Case, LockStep, _bits_equal, matrix_cases, poison_bits
from tensor_norms_oracle import assert_close, expected_norms

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

F32 = np.float32
MAN = [("a/kernel", (2 * 2048 + 777,)), ("a/bias", (5,)), ("one/kernel", (1,)), ("empty/kernel", (0,)),
       ("LayerNorm/gamma", (33,)), ("nograd/kernel", (64,)), ("t/kernel", (3, 1367))]
NOGRAD = (5,)
TINY = [(f"tiny{i}/{'bias' if i % 3 == 0 else 'kernel'}", (1 + i % 7,)) for i in range(300)]
N = 3
SCHED = dict(init_lr=1e-2, num_train_steps=10, num_warmup_steps=4)   # applies at 0, 3, .. 12: past both ends
STEPS = 13
INF_AT = (4, 0, 1000)              # loss scaling: the window that applies at 6 overflows and is skipped
EMA = (0.9, True)
WEIGHTS = (3.0, 37.0, 1000.0, 5.0, 64.0, 11.0)
CYCLE = (0.37, 0.0, 2.5, 1.0)


def _setup(case: Case):
    layout = "packed" if case.layout == "packed" else "table"
    dtype = case.layout.split("_")[-1] if layout == "table" else "fp32"
    return layout, dtype, (MAN + TINY if case.layout.startswith("t1920") else MAN)


class Scheduled(LockStep):
    """A device-scheduled ``LockStep`` with learning-rate multipliers, window weights and per-tensor norms; every apply's
    norms are checked against ``tensor_norms_oracle`` from the accumulators, gradients, W, S and weights around it."""

    def __init__(self, case: Case, seed: int, injected: bool = True, sched=SCHED, global_step: int = 0, n: int = N,
                 device_schedule: bool = True, man=None, reset: str = "materialized"):
        layout, dtype, m = _setup(case)
        man = m if man is None else man
        super().__init__(man, case.variant, case.mode, layout, dtype, case.has_g, EMA if case.ema else None, N=n,
                         seed=seed, nograd=NOGRAD if man is not None and len(man) > 5 else (), injected=injected,
                         lr_mult=[CYCLE[i % len(CYCLE)] for i in range(len(man))], window_weight=True, tensor_norms=True,
                         sched=sched, global_step=global_step, device_schedule=device_schedule, reset=reset)
        self.step_no = 0

    def step(self, grads, launch=None) -> bool:
        applied = self.g.is_apply_step(self.g_host, self.N)
        if applied:
            host, _ = self.inputs(grads)
            S = F32(self.ref.scale) if self.ls else None
            before = ([x.copy() for x in self._slab(self.raw_accum())], [x.copy() for x in self._weights()],
                      F32(self.ref.weight))
        out = super().step(grads, launch)
        if applied:
            acc, w0, W = before
            exp = expected_norms(acc, host, W, S, w0, self._weights())
            assert_close(self.op.tensor_norms(), exp, what=f"norms at step {self.g_host - 1}")
        return out

    def micro(self, launch=None) -> bool:
        """One micro-step with the next weight of WEIGHTS and, under loss scaling, an inf at INF_AT."""
        s = self.step_no
        self.step_no += 1
        inf = INF_AT[1:] if self.ls and s == INF_AT[0] else None
        return self.wstep(self.grads(0.1, inf), WEIGHTS[s % len(WEIGHTS)], launch)


def _buffers(run):
    """Every device buffer of the op's state, and the blocks it keeps, as host tensors.  A test of the deferred reset
    reads the raw accumulators, and only mid-window: right after an apply they are unspecified."""
    from gaccum_b200 import _lib
    op = run.op
    torch.cuda.synchronize()
    accum = run.raw_accum()
    if run.reset == "deferred" and _lib.is_first_accumulate(run.g_host, run.N):
        accum = None
    out = {"accum": accum, "m": op.m, "v": op.v, "sched": op._sched_state, "ww": run.ww,
           "norms": op.tensor_norms_tensor, "stats": torch.tensor(list(op.stats().values()), dtype=torch.float32)}
    out["weights"] = op.param_slab if run.layout == "packed" else (op.master if op.master is not None else None)
    for i, p in enumerate(op.params):
        out[f"param{i}"] = p.detach()
    if op.ema is not None:
        out["ema"], out["ema_state"] = op.ema, op._ema_state
    if op._ls_state is not None:
        out["ls"] = op._ls_state
    if run.variant == "lamb":
        out["ratios"] = torch.from_numpy(op.trust_ratios())
    return {k: v.detach().cpu().clone() for k, v in out.items() if v is not None}


def _bytes(t):
    flat = torch.empty(t.numel(), dtype=t.dtype)             # stride 1 whatever t's strides
    flat.copy_(t.reshape(-1))
    return flat.view(torch.uint8)


def _assert_same(a, b, what):
    assert a.keys() == b.keys(), what
    for k in a:
        assert torch.equal(_bytes(a[k]), _bytes(b[k])), f"{what}: {k}"


def _sched_word(op, i):
    return int(op._sched_state.cpu().view(torch.int32)[i])


def _recover(run):
    """The documented recovery: read the device counter (schedule_state raises on a refused block) and write it back."""
    with pytest.raises(RuntimeError, match="refused a launch"):
        run.op.schedule_state()
    g = int(run.op._sched_state.cpu()[0])
    assert g == run.g_host
    run.op.global_step = g
    assert run.op.schedule_state()["global_step"] == g


# ---- a. every dispatch key, eagerly ------------------------------------------------------------------------------------
def test_case_count():
    assert len(matrix_cases()) == 336


# the table layouts again with the deferred reset as training runs it (the packed entry point ignores the mode)
DISPATCH_KEYS = [pytest.param(c, "materialized", id=c.id) for c in matrix_cases()] + \
    [pytest.param(c, "deferred", id=f"{c.id}-deferred") for c in matrix_cases() if c.layout != "packed"]


@pytest.mark.parametrize("case, reset", DISPATCH_KEYS)
def test_every_dispatch_key_matches_the_oracle(case: Case, reset):
    run = Scheduled(case, zlib.crc32(case.id.encode()) ^ 0x5C, reset=reset)
    applies = sum(run.micro() for _ in range(STEPS))
    assert applies == 5
    if run.ls:
        assert run.op.loss_scale_state()["skipped_windows"] == 1
    if reset == "deferred":
        assert run.first_over_poison == 4                # after the applies at steps 0, 3, 6 and 9
    run.finish()


# ---- b. one window as a CUDA graph -------------------------------------------------------------------------------------
def _capture(run, launches, weights=False, poison=None):
    """Capture ``launches`` micro-steps of ``run.op`` over static gradient buffers; returns (graph, static buffers).
    ``weights``: each micro-step's weight add is captured too, from a static device scalar (the last entry of its
    buffers), as a producer's would be; else the weights are added eagerly before each replay (``Scheduled.wstep``).
    ``poison`` (a deferred-reset run): a T-entry int32 device tensor, copied into each tensor's raw accumulators right
    after a captured apply, so every replay's first accumulate finds the values it held at that replay."""
    from gaccum_b200 import _lib
    op = run.op
    _, dev = run.inputs(run.grads(0.1))
    static = [[None if t is None else torch.zeros_like(t) for t in dev] for _ in range(launches)]
    if weights:
        for st in static:
            st.append(torch.zeros((), dtype=torch.float32, device="cuda"))
    graph = torch.cuda.CUDAGraph()
    gc.collect()               # an earlier test's plan freed (cudaFree) during the capture would invalidate it
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        for j in range(launches):
            if weights:
                run.ww[0].add_(static[j][-1])
            if run.layout == "packed":
                for p, t in zip(op.params, static[j][:len(op.params)]):
                    if t is not None:
                        p.grad.add_(t)
                op.step()
            else:
                op.run(static[j][:len(op.params)])
            if poison is not None and _lib.is_apply_step(run.g_host + j, run.N):
                for i in range(len(op.params)):
                    run.accum_view(i).view(torch.int32).copy_(poison[i])
    torch.cuda.synchronize()
    return graph, static


def _fill(static, dev, weight=None):
    for dst, src in zip(static, dev):
        if dst is not None:
            dst.copy_(src)
    if weight is not None:
        static[-1].fill_(float(weight))


GRAPH_KEYS = [(v, m, l, e) for v in VARIANTS for m in MODES for l in LAYOUTS for e in (False, True)]
GRAPH_PARAMS = [pytest.param(*k, r, id=f"{k[0]}-{k[1]}-{k[2]}-{'ema' if k[3] else 'noema'}"
                             + ("" if r == "materialized" else f"-{r}"))
                for r in ("materialized", "deferred") for k in GRAPH_KEYS if r == "materialized" or k[2] != "packed"]


@pytest.mark.parametrize("variant, mode, layout, ema, reset", GRAPH_PARAMS)
def test_one_window_replayed_matches_the_eager_run(variant, mode, layout, ema, reset):
    """``reset="deferred"``: the captured window starts with its apply, after which the graph copies a poison into the
    raw accumulators; between replays that poison is set to values other than the eager twin's, so a first accumulate
    that read it could not match the twin by reading the same garbage."""
    case = Case(variant, mode, True, layout, ema)
    seed = zlib.crc32(case.id.encode()) ^ 0x6A
    eager, graphed = Scheduled(case, seed, reset=reset), Scheduled(case, seed, reset=reset)
    for _ in range(N):                                   # an eager window: every kernel loads before the capture
        eager.micro()
        graphed.micro()
    _assert_same(_buffers(eager), _buffers(graphed), "eager window")
    deferred = reset == "deferred"
    poison = torch.zeros(len(graphed.man), dtype=torch.int32, device="cuda") if deferred else None
    graph, static = _capture(graphed, N, weights=True, poison=poison)
    assert graphed.op.global_step == N                   # nothing ran during the capture
    windows = (STEPS + 2) // N - 1
    for w in range(windows):
        if deferred:                                     # the eager twin's apply below poisons with window + 1
            poison.copy_(torch.tensor([poison_bits(i, eager.windows + 1 + 3) for i in range(len(graphed.man))]))
        for j in range(N):
            s = eager.step_no
            S = F32(eager.ref.scale) if eager.ls else F32(1.0)
            grads = eager.grads(0.1, INF_AT[1:] if eager.ls and s == INF_AT[0] else None)
            with np.errstate(over="ignore", invalid="ignore"):       # the producer scales by S, as the eager twin's
                dev = [None if x is None else graphed._device(i, torch.from_numpy(x * S).to(graphed.dtype))
                       for i, x in enumerate(grads)]
            _fill(static[j], dev, WEIGHTS[s % len(WEIGHTS)])
            eager.step_no += 1
            eager.wstep(grads, WEIGHTS[s % len(WEIGHTS)])
        graph.replay()
        _assert_same(_buffers(eager), _buffers(graphed), f"replay {w}")
    assert graphed.op.global_step == eager.g_host == N * (windows + 1)
    if deferred:
        assert eager.first_over_poison == windows + 1
        assert graphed.materializes == 0
        graphed.check_padding()
        eager.finish()


# ---- c. refusal and recovery -------------------------------------------------------------------------------------------
APPLY_FAMILIES = {
    # name: (variant, mode, layout, ema)
    "apply_kernel": ("adamw", "noclip", "t256_fp32", False),
    "apply_kernel_ema": ("adam", "noclip", "t256_bf16", True),
    "clip_apply_clip": ("adamw", "clip", "t256_fp32", False),
    "clip_apply_ls_noclip": ("adam", "ls_noclip", "t256_fp16", False),
    "clip_apply_ls_clip": ("adamw", "ls_clip", "packed", True),
    "lamb": ("lamb", "clip", "t256_fp32", False),
    "lamb_ls": ("lamb", "ls_clip", "t1920_bf16", True),
}


@pytest.mark.parametrize("name", sorted(APPLY_FAMILIES))
def test_refused_apply_changes_nothing_and_training_recovers(name):
    """A graph of one apply (it ends mid-window) replayed at the window start, then again one step later: the second
    replay's apply is refused by the kernel family under test."""
    variant, mode, layout, ema = APPLY_FAMILIES[name]
    run = Scheduled(Case(variant, mode, True, layout, ema), zlib.crc32(name.encode()))
    for _ in range(N):
        run.micro()
    graph, static = _capture(run, 1)
    assert run.micro(launch=lambda dev: (_fill(static[0], dev), graph.replay())) is True      # step 3: applies
    for t in static[0]:
        if t is not None:
            t.zero_()                             # the packed graph's producer adds +0 to the accumulators the apply zeroed
    before = _buffers(run)
    graph.replay()                                                                            # step 4: not an apply
    torch.cuda.synchronize()
    assert _sched_word(run.op, 11) == 1
    after = _buffers(run)
    before.pop("sched"); after.pop("sched")
    _assert_same(before, after, "refused apply")
    _recover(run)
    applies = sum(run.micro() for _ in range(2 * N + 1))                                     # steps 4 .. 10
    assert applies == 2


ACC_FAMILIES = {"scattered_fp32": ("t256_fp32", False), "scattered_16bit": ("t1920_fp16", False),
                "scattered_fp32_ema": ("t256_fp32", True), "packed": ("packed", False)}
# the packed op's accumulate launch only advances the schedule: it is never a first accumulate
ACC_CASES = [(name, first) for name in sorted(ACC_FAMILIES) for first in (True, False) if name != "packed" or not first]


@pytest.mark.parametrize("name, first", ACC_CASES,
                         ids=[f"{n}-{'first_accumulate' if f else 'accumulate'}" for n, f in ACC_CASES])
def test_refused_accumulate_changes_nothing_and_training_recovers(name, first):
    """A front end that lost track of the step launches an accumulate the device step does not select: the window's
    first accumulate (which does not read the accumulators) one step late, mid-window -- refused only by the check that
    a first accumulate follows an apply -- or an accumulate at an apply step."""
    from gaccum_b200 import _lib
    layout, ema = ACC_FAMILIES[name]
    run = Scheduled(Case("adam", "clip", True, layout, ema), zlib.crc32(name.encode()) ^ int(first))
    op = run.op
    for _ in range(N + 2):                            # steps 0 .. 4: the device is at 5 (mid-window)
        run.micro()
    if not first:
        run.micro()                                   # step 5: the device is at 6, an apply step
    g = run.g_host
    wrong = g - 1                                     # first accumulate at 5 (after 4), plain accumulate at 6 (after 5)
    assert _lib.is_first_accumulate(wrong, N) == first and not _lib.is_apply_step(wrong, N)
    _, dev = run.inputs(run.grads(0.1))
    before = _buffers(run)
    args = _lib.StepArgs(wrong, N, 0, 0.0, 0.0, 0.0, 0.0)
    saved = op.accum.clone()
    if layout == "packed":
        with torch.no_grad():
            for p, t in zip(op.params, dev):
                if t is not None:
                    p.grad.add_(t)                    # the producer's add: not part of the refused launch
        before = _buffers(run)
        op.plan.step_packed(0, 0, op.accum.data_ptr(), 0, 0, args, -1, op._stream())
    else:
        op.plan.step(op._grad_table(dev), op._param_ptrs, op._accum_ptr, op._m_ptr, op._v_ptr, args, op._stream())
    torch.cuda.synchronize()
    assert _sched_word(op, 11) == 1
    after = _buffers(run)
    before.pop("sched"); after.pop("sched")
    _assert_same(before, after, "refused accumulate")
    _recover(run)
    if layout == "packed":                            # the gradients the producer added stay: drop them
        op.accum.copy_(saved)
        assert all(_bits_equal(a, r) for a, r in zip(run._slab(op.accum), run.ref.accum))
    applies = sum(run.micro() for _ in range(2 * N + 1))
    assert applies >= 2


# ---- d. the int32 wrap of global_step ----------------------------------------------------------------------------------
WRAP_SCHED = dict(init_lr=1e-3, num_train_steps=2**33, num_warmup_steps=2**20)   # past 2^31: int32(g) < W, lr < 0
WRAP_KEYS = [("adamw", "noclip"), ("adamw", "clip"), ("lamb", "ls_clip")]
WRAP_MAN = MAN[:5]


WRAP_PARAMS = [pytest.param(v, m, n, base, r, id=f"{v}-{m}-{n}-{bid}" + ("" if r == "materialized" else f"-{r}"))
               for r in ("materialized", "deferred") for v, m in WRAP_KEYS for n in (3, 4, 5)
               for base, bid in ((2**31, "at_2_31"), (2**32, "at_2_32"))]


@pytest.mark.parametrize("variant, mode, n, base, reset", WRAP_PARAMS)
def test_the_int32_wrap(variant, mode, n, base, reset):
    """``reset="deferred"``: the window that straddles 2^31 is longer than N, and its first accumulate finds a poisoned
    slab all the same."""
    case = Case(variant, mode, True, "t256_fp32", False)
    g0 = base - 2 * n
    man = WRAP_MAN if reset == "materialized" else WRAP_MAN + [MAN[NOGRAD[0]]]     # + a tensor without a gradient
    runs = [Scheduled(case, 17 + n, sched=WRAP_SCHED, global_step=g0, n=n, device_schedule=d, man=man,
                      reset=reset) for d in (False, True)]
    applied = []
    for _ in range(4 * n):
        a = [r.micro() for r in runs]                 # each op against its own oracle, accumulators included
        assert a[0] == a[1]
        applied.append(a[0])
        _assert_same_ops(runs)
    assert runs[1].op.global_step == g0 + 4 * n
    if base == 2**31:
        lrs = [float(r.ref.lr(base + 1)) for r in runs]
        assert lrs[0] < 0                            # the warm-up's int32 cast, as the reference computes it
    # the straddling window (N = 3, 5): longer than N
    starts = [g0 + k for k, a in enumerate(applied) if a]
    gaps = set(np.diff(starts))
    assert gaps == ({n} if base == 2**32 or n == 4 else {n, n + 1})
    for r in runs:
        if reset == "deferred":
            assert r.first_over_poison == sum(applied[:-1])
        r.finish()


def _assert_same_ops(runs):
    a, b = (_buffers(r) for r in runs)
    a.pop("sched", None); b.pop("sched", None)
    _assert_same(a, b, "host vs device schedule")


@pytest.mark.parametrize("n", [3, 5])
def test_graph_replayed_across_the_wrap_is_refused_and_recovers(n):
    """One window captured at the apply before 2^31 and replayed: the replay that reaches the straddling window is
    refused at its apply and changes nothing; reading the step, writing it back, running the rest of that window eagerly
    and replaying again from the next window start continues the run, against the oracle."""
    from gaccum_b200 import _lib
    case = Case("adamw", "noclip", True, "t256_fp32", False)
    last = max(g for g in range(2**31 - 2 * n, 2**31) if _lib.is_apply_step(g, n))      # the last apply before 2^31
    run = Scheduled(case, 5 + n, injected=False, sched=WRAP_SCHED, global_step=last - n, n=n, man=WRAP_MAN)
    while run.g_host < last:                                     # an eager window: every kernel loads
        run.micro()
    graph, static = _capture(run, n, weights=True)

    def replay():
        """One window through the graph, the oracle stepped over the same gradients."""
        infos = []
        for j in range(n):
            s = run.step_no
            run.step_no += 1
            host, dev = run.inputs(run.grads(0.1))
            w = WEIGHTS[s % len(WEIGHTS)]
            run.ref.add_weight(w)
            _fill(static[j], dev, w)
            infos.append(run.ref.run(host))
        graph.replay()
        run.g_host += n
        run.check(infos[-1])

    replay()                                                     # last .. last + n - 1, all before or at the jump
    assert run.g_host == last + n
    for st in static:
        for t in st:
            if t is not None:
                t.zero_()                                        # the captured weight adds then add +0
    before = _buffers(run)
    graph.replay()                                               # its apply at last + n is not one by int32
    torch.cuda.synchronize()
    assert _sched_word(run.op, 11) == 1
    after = _buffers(run)
    before.pop("sched"); after.pop("sched")
    _assert_same(before, after, "refused replay")
    _recover(run)
    while not _lib.is_apply_step(run.g_host, n) or run.g_host <= 2**31:   # the rest of the straddling window, eagerly
        run.micro()
    for _ in range(2):
        replay()                                                 # whole windows again
    assert run.op.global_step == run.g_host > 2**31 + n
