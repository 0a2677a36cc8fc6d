"""The train op on a model past 2^31 elements, every element of every slab against the oracle, bit for bit.

The model is MAN: ``big`` has 2^31 + 3*2048 + 7 elements, so its tiles reach a tensor offset (TileDesc::toff) of 2^31
and end in a partial tile; ``head`` puts ``big`` at a nonzero slab offset, and ``t1`` and ``t2`` sit at slab offsets
past 2^31.  Every kernel rebuilds its addresses from toff and the slab offset soff32 * 32 in 64 bits: an int32
product or offset anywhere would wrap here and nowhere in the rest of the suite, whose largest tensor has 31 M elements.

Inputs are periodic in the tensor-local index: element i of a tensor holds ``pattern[i mod 97]`` (97 is prime, so a tile
or slab offset off by any amount shifts the residues), except five marked elements that each hold a value of their own:
``big[0]``, the first element at toff = 2^31, the first at slab index 2^31, ``big``'s last element and ``t2``'s last.
An element's result depends on its own inputs and the launch-uniform scalars only (lr, the clip scale, its tensor's
trust ratio and decay flag), so the oracle runs on a compact model of 97 + (marks) elements per tensor, in
``LockStep``'s injected mode (it takes the kernel's global norm and trust ratios), and every slab is compared with that
table on the device, in chunks, as int32 bit patterns, after every micro-step: accumulators, p, m, v, the master weights,
the bf16 model copy and the EMA, and the padding between tensors (+0).

Inputs are k * 2^-4 with k in {+-1, +-2, +-3} (+-5..7 marked) and N = 4, so every partial sum is exact: the global norm
and the per-tensor gradient norms (and the weight norms of the first window) must equal the correctly rounded norm of
the exact sum of squares (counted per residue, in ``Fraction``), bit for bit; the update norms and LAMB's trust ratios
are held to the exact sums of the oracle's values as ``tests/test_gpu_exact_norms.py`` holds them.

Each case needs 20 bytes per element (~43 GB) on one GPU; it reads the free memory first and skips, with the
figures, when there is not enough.  Test infrastructure: ``apply_matrix`` (oracles, hyper-parameters), ``ema_oracle``,
``exact_norm_oracle``.
"""
import gc
import math
import time
from fractions import Fraction
from typing import Dict, List, NamedTuple

import numpy as np
import pytest

import exact_norm_oracle as eno
import oracle_np as onp
from apply_matrix import LAMB_TIE_REL, LS_CFG, SCHED, oracle_hparams, reference_op
from composed_oracle import trust_ratio
from ema_oracle import Ema

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

F32 = np.float32
PERIOD = 97
TILE = 2048
BIG = 2 ** 31 + 3 * TILE + 7
MAN = [("head/kernel", (1000,)), ("big/kernel", (BIG,)), ("t1/bias", (5,)), ("t2/kernel", (33,))]
N = 4                          # a power of two: c = a / N is exact
G0 = 1                         # the first micro-step: windows end at global_step 4, 8 (and 12)
J = 4                          # inputs are multiples of 2^-J
CHUNK = PERIOD * (1 << 20)     # elements per device compare; a multiple of the period, so every chunk starts at residue 0
MARGIN = 2 << 30               # bytes beyond the slabs: compare buffers, the CUDA context
EMA = (0.9, True)
MARK_K = (5, -6, 7, -5, 6)     # the marked elements' k, one each, none a periodic value


class Case(NamedTuple):
    variant: str
    mode: str
    layout: str                # "packed" (PackedTrainOp, CAP 0) or "table" (GaccumTrainOp, CAP 256)
    dtype: str
    has_g: bool                # the apply step gets a gradient stream; else the gradients are added into the accumulators
    ema: bool
    norms: bool
    windows: int
    bytes_per_elem: int        # device bytes per element the case holds at once


CASES: Dict[str, Case] = {
    # accumulate_kernel (FROM_ZERO true and false) and the clip-apply with a gradient stream, packed and pointer table
    "packed_adamw_clip": Case("adamw", "clip", "packed", "fp32", True, False, False, 2, 20),      # param, accum, m, v, G
    "table_adamw_clip_norms": Case("adamw", "clip", "table", "fp32", True, False, True, 2, 20),   # param, G, accum, m, v
    # apply_kernel
    "table_adamw_noclip": Case("adamw", "noclip", "table", "fp32", True, False, False, 2, 20),
    "table_adam_noclip": Case("adam", "noclip", "table", "fp32", True, False, False, 2, 20),
    # the in-place hand-off: p.grad is the accumulator; no gradient stream, no accumulate launch (16 B/element, 20 while
    # the op copies the parameters into its slab)
    "packed_inplace_adamw_clip": Case("adamw", "clip", "packed", "fp32", False, False, False, 2, 20),
    # LAMB: big's trust ratio from more than a million tiles across many CTA ranges
    "table_lamb_noclip": Case("lamb", "noclip", "table", "fp32", True, False, False, 2, 20),
    "table_lamb_clip_norms": Case("lamb", "clip", "table", "fp32", True, False, True, 2, 20),
    # loss scaling: +inf at toff = 2^31 in the second window, which is skipped; the third applies
    "table_adamw_ls_clip_inf": Case("adamw", "ls_clip", "table", "fp32", True, False, False, 3, 20),
    # EMA: apply_only(None) on accumulators filled in place (param, accum, m, v, EMA)
    "table_adamw_clip_ema": Case("adamw", "clip", "table", "fp32", False, True, False, 2, 20),
    # a bf16 model: bf16 param and G, fp32 master, accum, m, v
    "table_adamw_clip_bf16": Case("adamw", "clip", "table", "bf16", True, False, False, 2, 20),
}
INF_STEP = 6                   # the loss-scaled case's overflowed micro-step (window 2: steps 5..8)


def _padded(n: int) -> int:
    return -(-n // 32) * 32


OFFSETS = [int(x) for x in np.cumsum([0] + [_padded(int(np.prod(s))) for _, s in MAN[:-1]])]
PADDED = OFFSETS[-1] + _padded(MAN[-1][1][0])
# tensor index -> its marked elements (tensor-local indices)
MARKS: Dict[int, List[int]] = {0: [], 1: sorted([0, 2 ** 31, 2 ** 31 - OFFSETS[1], BIG - 1]), 2: [], 3: [32]}
MARK_SLOT = {(t, pos): k for k, (t, pos) in enumerate((t, p) for t in sorted(MARKS) for p in MARKS[t])}
assert len(MARK_SLOT) == len(MARK_K)


def _counts(t: int) -> np.ndarray:
    """How many elements of tensor t each compact entry stands for: residue r, then each marked element once."""
    n = MAN[t][1][0]
    c = np.array([n // PERIOD + (1 if r < n % PERIOD else 0) for r in range(PERIOD)], np.int64)
    for pos in MARKS[t]:
        c[pos % PERIOD] -= 1
    return np.concatenate([c, np.ones(len(MARKS[t]), np.int64)])


COUNTS = [_counts(t) for t in range(len(MAN))]


def _sumsq(x: np.ndarray, counts: np.ndarray):
    """sum(x^2) over the tensor the compact x stands for, exactly (inf / NaN if a counted entry is not finite)."""
    x = np.asarray(x, F32).ravel()
    live = counts > 0
    if np.isnan(x[live]).any():
        return float("nan")
    if np.isinf(x[live]).any():
        return float("inf")
    return sum((Fraction(float(v)) ** 2 * int(c) for v, c in zip(x[live], counts[live])), Fraction(0))


def _units(rng, size: int) -> np.ndarray:
    return (rng.integers(1, 4, size=size) * rng.choice([-1, 1], size=size) * 2.0 ** -J).astype(F32)


def _compact(rng, sign: float = 1.0) -> List[np.ndarray]:
    """One input of every tensor: 97 periodic values and the marked ones."""
    return [np.concatenate([_units(rng, PERIOD),
                            np.array([sign * MARK_K[MARK_SLOT[(t, p)]] * 2.0 ** -J for p in MARKS[t]], F32)])
            for t in range(len(MAN))]


class LargeRun:
    """One train op on MAN and its oracle on the compact model, stepped together (``apply_matrix.LockStep`` in its
    injected mode, with the slabs compared on the device)."""

    def __init__(self, case: Case, seed: int):
        import gaccum_b200 as g
        from gaccum_b200.train_op import GaccumTrainOp, PackedTrainOp
        self.case, self.g, self.dev = case, g, torch.device("cuda", 0)
        self.tdtype = {"fp32": torch.float32, "bf16": torch.bfloat16}[case.dtype]
        self.rng = np.random.default_rng(seed)
        self.names = [n for n, _ in MAN]
        self.ls = case.mode.startswith("ls_")
        init = _compact(self.rng)
        params = []
        for t, (_, s) in enumerate(MAN):
            p = torch.empty(s, dtype=self.tdtype, device=self.dev)
            self._write(p, init[t], t)
            params.append(p)
        hpo = oracle_hparams(case.variant, case.mode)
        hp = g.HParams(hpo.variant, 0, hpo.beta1, hpo.beta2, hpo.epsilon, hpo.weight_decay_rate, hpo.clip_norm)
        lr_fn = lambda s: g.learning_rate(SCHED["init_lr"], SCHED["num_train_steps"], SCHED["num_warmup_steps"], s)
        kw = dict(loss_scale=g.LossScaleConfig(*LS_CFG) if self.ls else None, ema=g.EmaConfig(*EMA) if case.ema else None,
                  global_step=G0, tensor_norms=case.norms)
        if case.layout == "packed":
            self.op = PackedTrainOp(params, self.names, hp, N, lr_fn, **kw)
        else:
            self.op = GaccumTrainOp(params, self.names, hp, N, lr_fn, **kw)
        del params
        assert self.op.plan.offsets == OFFSETS and self.op.plan.padded_size == PADDED
        self.grads = None
        if case.has_g:
            if case.layout == "packed":
                self.gslab = torch.zeros_like(self.op.accum)
                self.grads = [self.op._view(self.gslab, t) for t in range(len(MAN))]
            else:
                self.grads = [torch.empty(s, dtype=self.tdtype, device=self.dev) for _, s in MAN]
        self.ref = reference_op(case.variant, case.mode, init, self.names, N,
                                adapt=self.op.adapt if case.variant == "lamb" else None, global_step=G0)
        self.tracker = Ema(self.ref.params, *EMA) if case.ema else None
        self.window = 0                # applied windows so far
        self.g_step = G0               # the step of the next micro-step

    # -- device fills: periodic chunks copied from one repeated 97-element table, the marked elements one by one --------
    def _rep(self, period: np.ndarray, dtype) -> "torch.Tensor":
        return torch.from_numpy(np.ascontiguousarray(period, F32)).to(self.dev).to(dtype).repeat(CHUNK // PERIOD)

    def _write(self, dst, compact: np.ndarray, t: int, add: bool = False) -> None:
        """dst (tensor t, any shape) = the tensor the compact values stand for; ``add``: dst += it, one fp32 add per
        element, the marked ones included."""
        flat = dst.view(-1)
        n = flat.numel()
        rep = self._rep(compact[:PERIOD], flat.dtype)
        saved = [flat[p].clone() for p in MARKS[t]] if add else None
        for k in range(0, n, CHUNK):
            L = min(CHUNK, n - k)
            (flat[k:k + L].add_ if add else flat[k:k + L].copy_)(rep[:L])
        for j, p in enumerate(MARKS[t]):
            v = torch.tensor(float(compact[PERIOD + j]), dtype=torch.float32, device=self.dev)
            flat[p] = (saved[j] + v) if add else v.to(flat.dtype)

    # -- device compares --------------------------------------------------------------------------------------------------
    def _compare(self, what: str, got, compact: np.ndarray, t: int) -> None:
        """got (tensor t's fp32 elements in some slab) == the tensor the compact oracle values stand for, bit for bit."""
        gi = got.reshape(-1).view(torch.int32)
        n = gi.numel()
        compact = np.ascontiguousarray(compact, F32)
        bits = compact.view(np.int32)
        rep = torch.from_numpy(bits[:PERIOD].copy()).to(self.dev).repeat(CHUNK // PERIOD)
        bad = []
        for k in range(0, n, CHUNK):
            ne = gi[k:k + CHUNK] != self._expected(rep, bits, t, k, min(CHUNK, n - k))
            bad.append(ne.sum())
        bad = torch.stack(bad).cpu().numpy()
        if bad.any():
            # the first and the last mismatch: an offset that wraps past 2^31 shows in both ends of the tensor
            where = []
            for c in (np.flatnonzero(bad)[0], np.flatnonzero(bad)[-1]):
                k = int(c) * CHUNK
                L = min(CHUNK, n - k)
                exp = self._expected(rep, bits, t, k, L)
                idx = torch.nonzero(gi[k:k + L] != exp).view(-1)
                for i in (k + int(idx[0]), k + int(idx[-1])):
                    where.append(f"element {i} (slab index {OFFSETS[t] + i}): got {int(gi[i]) & 0xffffffff:#010x}, "
                                 f"expected {int(exp[i - k]) & 0xffffffff:#010x}")
            pytest.fail(f"{what} of {self.names[t]} (window {self.window}): {int(bad.sum())} elements differ; the first "
                        f"at {where[0]}; the last at {where[-1]}")

    def _expected(self, rep, bits: np.ndarray, t: int, k: int, L: int):
        """Tensor t's expected int32 bits over [k, k + L): the periodic table (a view of it where no marked element
        falls in the range), with the marked elements in it."""
        marks = [(p - k, int(bits[PERIOD + j])) for j, p in enumerate(MARKS[t]) if k <= p < k + L]
        if not marks:
            return rep[:L]
        exp = rep[:L].clone()
        for i, b in marks:
            exp[i] = b
        return exp

    def _padding(self, what: str, slab) -> None:
        words = slab.view(torch.int32)
        gaps = [(OFFSETS[t] + MAN[t][1][0], OFFSETS[t + 1] if t + 1 < len(MAN) else words.numel()) for t in range(len(MAN))]
        nz = torch.stack([torch.count_nonzero(words[a:b]) for a, b in gaps]).cpu().numpy()
        assert not nz.any(), f"{what}: padding after {[self.names[t] for t in np.flatnonzero(nz)]} is not +0"

    def _model_copy(self) -> None:
        """The bf16 model copy == the master weights rounded to nearest-even."""
        for t in range(len(MAN)):
            p, m = self.op.params[t].view(-1), self.op.master_view(t).view(-1)
            for k in range(0, p.numel(), CHUNK):
                a, b = p[k:k + CHUNK].view(torch.int16), m[k:k + CHUNK].to(torch.bfloat16).view(torch.int16)
                if not torch.equal(a, b):
                    i = k + int(torch.nonzero(a != b)[0])
                    pytest.fail(f"model copy of {self.names[t]}: first mismatch at element {i}")

    def _weights(self, t: int):
        op = self.op
        if self.case.dtype != "fp32":
            return op.master_view(t)
        return op._view(op.param_slab, t) if self.case.layout == "packed" else op.params[t]

    def _slabs(self):
        op = self.op
        out = {"accumulator": op.accum, "m": op.m, "v": op.v}
        if self.case.layout == "packed":
            out["p"] = op.param_slab
        if self.case.dtype != "fp32":
            out["master"] = op.master
        if self.case.ema:
            out["average"] = op.ema
        return out

    # -- one micro-step ---------------------------------------------------------------------------------------------------
    def step(self, inf: bool = False) -> bool:
        op, ref, g = self.op, self.ref, self.g
        step = self.g_step
        applied = g.is_apply_step(step, N)
        S = F32(ref.scale) if self.ls else F32(1.0)
        host = _compact(self.rng, sign=-1.0 if step % 2 else 1.0)
        with np.errstate(over="ignore", invalid="ignore"):
            host = [(x * S).astype(F32) for x in host]
        if inf:
            host[1][PERIOD + MARKS[1].index(2 ** 31)] = np.inf
        with torch.no_grad():
            if self.grads is not None:
                for t in range(len(MAN)):
                    self._write(self.grads[t], host[t], t)
            if self.case.layout == "packed" and self.case.has_g:
                lr = op.lr_fn(step)
                op.plan.step_packed(self.gslab.data_ptr(), op.param_slab.data_ptr(), op.accum.data_ptr(), op.m.data_ptr(),
                                    op.v.data_ptr(), op._step_args(step, lr), -1, op._stream())
                if applied:
                    op._advance_beta_powers()
                op.global_step = step + 1
            elif self.case.layout == "packed":
                for t, p in enumerate(op.params):
                    self._write(p.grad, host[t], t, add=True)
                assert op.step() == applied
            elif self.case.has_g:
                assert op.run(self.grads) == applied
            else:
                for t in range(len(MAN)):
                    self._write(op.accum_view(t), host[t], t, add=True)
                if applied:
                    op.apply_only(None)
                op.global_step = step + 1
        p_before = [x.copy() for x in ref.params]
        if applied:
            st = op.stats()
            ratios = op.trust_ratios() if self.case.variant == "lamb" else None
            ref.reduced = onp.Reduced(F32(st["global_norm"]), ratios)
        info = ref.run(host)
        assert info.applied == applied
        self.g_step = step + 1
        if applied:
            self.window += 1
            if self.tracker is not None and not getattr(ref, "last_skipped", False):
                self.tracker.average(ref.params)
        self.check(info, p_before)
        return applied

    def check(self, info, p_before) -> None:
        op, ref, case = self.op, self.ref, self.case
        torch.cuda.synchronize()
        for t in range(len(MAN)):
            self._compare("accumulator", op.accum_view(t), ref.accum[t], t)
            self._compare("p", self._weights(t), ref.params[t], t)
            self._compare("m", op.m_view(t), ref.m[t], t)
            self._compare("v", op.v_view(t), ref.v[t], t)
            if self.tracker is not None:
                self._compare("average", op.ema_view(t), self.tracker.avg[t], t)
        for what, slab in self._slabs().items():
            self._padding(what, slab)
        if case.dtype != "fp32":
            self._model_copy()
        if self.ls:
            s = op.loss_scale_state()
            assert (F32(s["scale"]), s["good_windows"], s["skipped_windows"], s["last_skipped"]) == \
                (ref.scale, ref.good_windows, ref.skipped_windows, ref.last_skipped)
        if case.variant in ("adam", "lamb") and not self.ls:
            assert (F32(op.beta1_power), F32(op.beta2_power)) == (F32(ref.beta1_power), F32(ref.beta2_power))
        if not info.applied:
            return
        st = op.stats()
        assert st["applied"] and F32(st["lr"]) == F32(info.lr)
        skipped = getattr(ref, "last_skipped", False)
        if case.mode in ("clip", "ls_clip"):
            s, e = F32(st["clip_scale"]), F32(info.clip_scale)
            assert s.tobytes() == e.tobytes() or (np.isnan(s) and np.isnan(e)), (s, e)
            exact = sum((_sumsq(c, COUNTS[t]) for t, c in enumerate(ref.window_c)), Fraction(0))
            gn = F32(st["global_norm"])
            if isinstance(exact, Fraction):
                assert gn.tobytes() == eno.ref_norm(exact).tobytes(), (gn, eno.ref_norm(exact))
            else:
                assert skipped and not np.isfinite(gn), gn
        else:
            assert (st["global_norm"], st["clip_scale"]) == (0.0, 1.0)
        if case.variant == "lamb" and not skipped:
            r = op.trust_ratios()
            adapted = [t for t in range(len(MAN)) if ref.adapt[t]]
            assert len(adapted) < len(MAN) and len(ref.window_pu) == len(adapted)
            for t in range(len(MAN)):
                if not ref.adapt[t]:
                    assert r[t] == 1.0
            for t, (p, u) in zip(adapted, ref.window_pu):
                exp = [trust_ratio(wn, un) for wn in eno.norm_candidates(_sumsq(p, COUNTS[t]), LAMB_TIE_REL)
                       for un in eno.norm_candidates(_sumsq(u, COUNTS[t]), LAMB_TIE_REL)]
                assert any(r[t].tobytes() == x.tobytes() for x in exp), (self.names[t], r[t], exp)
        if case.norms:
            norms = op.tensor_norms()
            for t in range(len(MAN)):
                n = MAN[t][1][0]
                ec = _sumsq(ref.window_c[t], COUNTS[t])
                assert norms[t, 0].tobytes() == eno.ref_norm(ec).tobytes(), (self.names[t], "gradient", norms[t, 0])
                ew = _sumsq(p_before[t], COUNTS[t])
                if self.window == 1:       # p is still the k * 2^-J it started as: the sum is exact
                    assert norms[t, 1].tobytes() == eno.ref_norm(ew).tobytes(), (self.names[t], "weight", norms[t, 1])
                else:
                    assert abs(float(norms[t, 1]) - math.sqrt(ew)) <= eno.clip_norm_bound(ew, n), (self.names[t], "weight")
                d = (p_before[t] - ref.params[t]).astype(F32)
                eu = _sumsq(d, COUNTS[t])
                assert abs(float(norms[t, 2]) - math.sqrt(eu)) <= eno.clip_norm_bound(eu, n), \
                    (self.names[t], "update", float(norms[t, 2]), math.sqrt(eu))


def _free_device_memory():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def _fresh_device():
    _free_device_memory()
    yield
    _free_device_memory()


@pytest.mark.parametrize("name", list(CASES))
def test_past_2_31_elements(name):
    case = CASES[name]
    free, total = torch.cuda.mem_get_info(0)
    need = case.bytes_per_elem * PADDED + MARGIN
    if free < need:
        pytest.skip(f"{name} needs {need / 2 ** 30:.1f} GiB of device memory ({case.bytes_per_elem} B/element), "
                    f"{free / 2 ** 30:.1f} GiB of {total / 2 ** 30:.1f} GiB are free")
    torch.cuda.reset_peak_memory_stats(0)
    t0 = time.perf_counter()
    run = LargeRun(case, seed=sum(map(ord, name)))
    for s in range(N * case.windows):
        step = G0 + s
        if run.ls and step == INF_STEP:
            before = [[x.copy() for x in a] for a in (run.ref.params, run.ref.m, run.ref.v)]
            scale = F32(run.ref.scale)
        run.step(inf=run.ls and step == INF_STEP)
        if run.ls and step == 2 * N:
            # the overflowed window: skipped, p, m and v unchanged, S halved (the accumulators' +0 is checked above)
            st = run.op.loss_scale_state()
            assert st["last_skipped"] and st["skipped_windows"] == 1 and F32(st["scale"]) == scale / 2
            for a, b in zip(before, (run.ref.params, run.ref.m, run.ref.v)):
                assert all(np.array_equal(x.view(np.int32), y.view(np.int32)) for x, y in zip(a, b))
    assert run.window == case.windows
    if run.ls:
        st = run.op.loss_scale_state()
        assert not st["last_skipped"] and st["skipped_windows"] == 1
    print(f"\n{name}: {time.perf_counter() - t0:.1f} s, {free / 2 ** 30:.1f} GiB free at start, "
          f"{torch.cuda.max_memory_allocated(0) / 2 ** 30:.1f} GiB peak, {torch.cuda.get_device_name(0)}")
    del run
