"""The apply kernels' instantiation space, the schedule constants the tests aim at, and a train op stepped in lock-step
with its composed oracle.

* ``matrix_cases()`` / ``instantiation(case)``: every dispatch key of ``gaccum_abi.cu`` (optimizer x mode x gradients or
  not x layout and dtype x EMA) and the kernel template each one launches.  ``tests/test_kernel_inventory.py`` checks that
  this mapping covers exactly the apply kernels in the built library; ``tests/test_gpu_apply_matrix.py`` runs every case.
* ``Schedule``: the tile and CTA bookkeeping of the clip-apply and the LAMB kernels, for tests that place tiles on their
  boundaries (``tests/test_gpu_schedule_edges.py``).
* ``reference_op``: the expected values of one dispatch key, ``composed_oracle.ComposedReferenceTrainOp``; a 16-bit
  model is the fp32 oracle fed the upcast gradients.
* ``LockStep``: one train op on the GPU and its oracle, stepped together and compared after every micro-step.

Importable without torch (the inventory test runs without a GPU).  Test infrastructure only.
"""
from __future__ import annotations

import itertools
import math
from fractions import Fraction
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

import exact_norm_oracle as eno
import oracle_np as onp
from composed_oracle import ComposedReferenceTrainOp, trust_ratio
from ema_oracle import Ema

F32 = np.float32

# ---- the dispatch keys ------------------------------------------------------------------------------------------------
VARIANTS = ("adamw", "adam", "lamb")
MODES = ("noclip", "clip", "ls_noclip", "ls_clip")
# layout -> (pointer-table capacity CAP, 16-bit model H, parameter dtype).  CAP 0 is gaccum_step_packed (fp32 only).
LAYOUTS: Dict[str, Tuple[int, bool, str]] = {
    "packed": (0, False, "fp32"),
    "t256_fp32": (256, False, "fp32"), "t256_bf16": (256, True, "bf16"), "t256_fp16": (256, True, "fp16"),
    "t1920_fp32": (1920, False, "fp32"), "t1920_bf16": (1920, True, "bf16"), "t1920_fp16": (1920, True, "fp16"),
}

# gaccum_kernels.cuh kNoClip / kClip / kLsClip / kLsNoClip: the MODE template argument of the cooperative kernels
MODE_ARG = {"noclip": "kNoClip", "clip": "kClip", "ls_clip": "kLsClip", "ls_noclip": "kLsNoClip"}


class Case(NamedTuple):
    variant: str
    mode: str
    has_g: bool
    layout: str
    ema: bool

    @property
    def id(self) -> str:
        return f"{self.variant}-{self.mode}-{'g' if self.has_g else 'nog'}-{self.layout}-{'ema' if self.ema else 'noema'}"


def matrix_cases() -> List[Case]:
    return [Case(*k) for k in itertools.product(VARIANTS, MODES, (True, False), LAYOUTS, (False, True))]


def instantiation(case: Case, consts: Dict[str, int]) -> Tuple[str, Tuple[int, ...]]:
    """The kernel template and its arguments that ``gaccum_abi.cu`` launches for ``case``; ``consts`` maps the
    kernels' mode constants (MODE_ARG) to their values.  With or without gradients, a case runs the same kernel: a
    tensor without a gradient is one whose gradient pointer is NULL."""
    cap, h, _ = LAYOUTS[case.layout]
    h, e = int(h), int(case.ema)
    mode = consts[MODE_ARG[case.mode]]
    if case.variant == "lamb":
        return "lamb_apply_kernel", (cap, mode, h, e)
    v = 0 if case.variant == "adamw" else 1
    if case.mode == "noclip":
        return "apply_kernel", (v, cap, h, e)
    return "apply_clip_kernel", (v, cap, mode, h, e)


# ---- the schedules ----------------------------------------------------------------------------------------------------
class Schedule:
    """The tile and CTA bookkeeping of the cooperative apply kernels on a GPU with ``sms`` SMs.
    ``tests/test_kernel_inventory.py`` reads the four constants out of csrc/*.cuh and compares them with these."""
    TILE = 2048                # gaccum_kernels.cuh kTile = kThreads * 4 * kUnroll: elements per tile
    GROUPS = 3                 # gaccum_kernels.cuh kGroups: consumer groups per clip-apply CTA
    STASH_TILES = {False: 4,   # gaccum_kernels.cuh kStashTiles: a group's own tiles whose a' stays in shared memory
                   True: 3}    # ... ClipLayout<true>::kStashTiles: an EMA launch's larger pass-2 slot leaves room for 3
    LAMB_BLOCKS_PER_SM = 3     # gaccum_lamb.cuh kLambBlocksPerSm

    def __init__(self, sms: int):
        self.sms = sms

    def clip_groups(self, nt: int) -> int:
        """G: the clip-apply's grid is min(sms, ceil(nt / 3)) CTAs of 3 groups (gaccum_abi.cu launch_apply)."""
        return self.GROUPS * max(1, min(self.sms, -(-nt // self.GROUPS)))

    def pool_lo(self, nt: int, ema: bool) -> int:
        """The first tile drawn from the ticket counters; group b's own tiles are b + j*G, j < kStashTiles."""
        return min(nt, self.STASH_TILES[ema] * self.clip_groups(nt))

    def lamb_ranges(self, nt: int) -> List[Tuple[int, int]]:
        """LAMB CTA c owns tiles [nt*c/grid, nt*(c+1)/grid), grid = min(3*sms, nt) (gaccum_lamb.cuh)."""
        grid = max(1, min(self.LAMB_BLOCKS_PER_SM * self.sms, nt))
        return [(nt * c // grid, nt * (c + 1) // grid) for c in range(grid)]


def num_tiles(numels: Sequence[int]) -> int:
    return sum(-(-int(n) // Schedule.TILE) for n in numels)


# ---- the composed oracle ----------------------------------------------------------------------------------------------
CLIP = 0.5                     # clipping modes: small enough that every window's clip scale is < 1
SCHED = dict(init_lr=1e-2, num_train_steps=40, num_warmup_steps=4)
LS_CFG = (16.0, 2.0, 2)        # initial scale, multiplier, growth interval: S grows after the second applied window


def oracle_hparams(variant: str, mode: str) -> onp.HParams:
    clip = CLIP if mode in ("clip", "ls_clip") else 0.0
    if variant == "lamb":
        return onp.HParams(variant=2, clip_norm=clip)
    if variant == "adam":
        return onp.HParams(variant=onp.VARIANT_ADAM, epsilon=1e-8, weight_decay_rate=0.0, clip_norm=clip)
    return onp.HParams(clip_norm=clip)


def reference_op(variant: str, mode: str, params, names, N: int, adapt: Optional[Sequence[bool]] = None,
                 lr_mult: Optional[Sequence[float]] = None, window_weight: bool = False, ls_cfg=LS_CFG, sched=SCHED,
                 global_step: int = 0) -> ComposedReferenceTrainOp:
    """The oracle of one dispatch key, with learning-rate multipliers ``lr_mult`` and the window weight if given."""
    hp = oracle_hparams(variant, mode)
    params = [np.array(p, dtype=F32, copy=True) for p in params]
    lskw = dict(initial_scale=ls_cfg[0], multiplier=ls_cfg[1], growth_interval=ls_cfg[2]) if mode.startswith("ls_") else {}
    return ComposedReferenceTrainOp(params, names, hp, N, adapt=adapt, lr_mult=lr_mult, window_weight=window_weight,
                                    **lskw, **sched, global_step=global_step)


def rel_err(x, ref) -> float:
    x = np.asarray(x, np.float64); ref = np.asarray(ref, np.float64)
    if x.size == 0:
        return 0.0
    return float(np.max(np.abs(x - ref)) / max(float(np.max(np.abs(ref))), 1e-30))


def _bits_equal(x: np.ndarray, y: np.ndarray) -> bool:
    return x.shape == y.shape and np.array_equal(np.ascontiguousarray(x).view(np.uint32),
                                                 np.ascontiguousarray(y, dtype=F32).view(np.uint32))


# a sum of squares the LAMB kernel forms in fp64 (gaccum_lamb.cuh add_sq64) is known far better than this before its
# one rounding to fp32; only a sum this close to an fp32 rounding boundary may round to the boundary's other side
LAMB_TIE_REL = 1e-12


def check_global_norm(gn: np.float32, c: Sequence[np.ndarray]) -> None:
    """The clip-apply's gn against the exact sum of squares of the window's c (``exact_norm_oracle.clip_norm_bound``);
    a non-finite c or sum must give a non-finite gn."""
    e = sum((eno.exact_sumsq(x) for x in c), Fraction(0))
    if not isinstance(e, Fraction):
        assert not np.isfinite(gn), (gn, e)
        return
    ref = eno.ref_norm(e)
    if not np.isfinite(ref):
        assert not np.isfinite(gn) or float(gn) ** 2 >= float(e) * (1 - 1e-6), (gn, float(e))
        return
    n = sum(x.size for x in c)
    err = abs(float(gn) - math.sqrt(e))
    assert np.isfinite(gn) and err <= eno.clip_norm_bound(e, n), (float(gn), math.sqrt(e), err, eno.clip_norm_bound(e, n))


RESETS = ("materialized", "deferred", "stored")
# What a deferred-reset test writes into the raw accumulators right after an apply, as fp32 bit patterns; None is
# 1 + window.  A quiet NaN with a payload and -inf propagate into p, m, v and the norms if read; -0.0 survives only in
# a tensor without a gradient that the first accumulate left unwritten; 3e38 overflows the loss-scaling test; the
# smallest denormal and 1 + window change a sum they are added into once.
POISON = (0x7FC0BEEF, 0xFF800000, 0x80000000, int(np.array(3.0e38, F32).view(np.uint32)), 0x00000001, None)
PAD_BITS = 0x7FC0DEAD                 # the slab's padding: a NaN no kernel may read or write


def poison_bits(tensor: int, window: int) -> int:
    """The poison of tensor ``tensor`` after the apply that ends window ``window``, as a signed int32."""
    v = POISON[(tensor + window) % len(POISON)]
    if v is None:
        v = int(np.array(1 + window, F32).view(np.uint32))
    return int(np.array(v, np.uint32).view(np.int32))


def trust_ratio_candidates(p: np.ndarray, u: np.ndarray) -> List[np.float32]:
    """LAMB's r = ||p|| / ||u|| with each norm rounded to fp32 once from its exact sum of squares: one value, or, for
    a sum within LAMB_TIE_REL of a rounding boundary, the values either side of it gives."""
    return [trust_ratio(wn, un) for wn in eno.norm_candidates(eno.exact_sumsq(p), LAMB_TIE_REL)
            for un in eno.norm_candidates(eno.exact_sumsq(u), LAMB_TIE_REL)]


# ---- one train op and its oracle in lock-step -------------------------------------------------------------------------
class LockStep:
    """A train op on cuda:0 and its composed oracle, stepped together.

    ``layout`` is "packed" (PackedTrainOp; with ``has_g`` the apply gets a gradient slab through ``plan.step_packed``) or
    "table" (GaccumTrainOp; without ``has_g`` every micro-step is ``accumulate_only`` and an apply step adds
    ``apply_only(None)``).  ``views`` places tensor i (parameter and gradients) ``views[i]`` elements past an aligned
    address; ``nograd`` lists tensors that never get a gradient; ``zero`` tensors start at 0.  ``adapt_exclude`` is
    LAMB's layer-adaptation exclusion list (default: the weight-decay one).

    After every micro-step ``check`` compares: accumulators bit for bit; p (the master weights of a 16-bit model), m
    and v bit for bit while no window has clipped and the variant is not LAMB, else within 1e-5; the global norm and
    clip scale within 3e-6; trust ratios within 1e-6; the average bit for bit against ``Ema`` fed the kernel's own
    weights; the model copy bit for bit against the RNE rounding of the kernel's master weights; the loss-scaling block
    and the beta powers exactly.

    ``injected``: on an apply step the kernel runs first, and the oracle takes its global norm and trust ratios
    (``oracle_np.Reduced``).  Everything the oracle still computes is then compared bit for bit, clipped windows and
    LAMB included: p, m, v and the clip scale the oracle derives from the kernel's gn.  The reduced scalars themselves
    are held to exact sums (``exact_norm_oracle``): gn within ``clip_norm_bound`` of sqrt(sum c^2), and r equal to
    ||p|| / ||u|| with both norms rounded to fp32 once from their exact sums (either side of a tie for a sum that
    lies within 1e-12 of one).  ``init`` maps tensor indices to their initial values; ``tensor_norms`` turns the
    train op's per-tensor norms on.

    ``sched`` is the learning-rate schedule (``init_lr``, ``num_train_steps``, ``num_warmup_steps``; default ``SCHED``)
    and ``global_step`` the step both start at.  ``device_schedule``: the train op keeps global_step, the lr and the
    beta powers on the device, and every micro-step goes through the op's own entry point -- ``op.step()`` packed
    (gradients added into ``p.grad``, with or without ``has_g``), ``op.run`` with a table, where a case without
    gradients adds them into the accumulators and runs ``run([None] * T)``.  ``check`` then also compares the device
    counter, the lr in the stats of every micro-step, and the beta powers in their one home (the schedule block, or the
    loss-scaling block under loss scaling, the schedule block's then 0).

    ``reset`` (table layout, N >= 2): how the accumulators get back to zero after an apply (RESETS).
    "materialized" reads them through ``op.accum``, which stores a deferred reset's zeros after every micro-step.
    "deferred" is the path a training loop takes: nothing calls ``gaccum_accum_materialize`` (a counter on the plan
    checks it at every ``check``); the raw slab is compared only where it is defined, after a micro-step that did not
    apply; right after an apply every tensor's raw accumulators are poisoned (POISON, rotated by tensor and window), so
    a kernel that reads them, or leaves a tensor without a gradient unwritten, fails.  "stored" turns the mode off: the
    raw slab holds +0.0 right after every apply.  Both write NaN into the slab's padding at construction; ``finish``
    checks that nothing touched it and reads ``op.accum`` once.  A case without gradients runs its accumulates through
    ``op.run`` and, at an apply, adds the gradients into the raw slab (mid-window, so defined) before ``run([None] *
    T)``.  ``first_over_poison`` counts first accumulates that found a poisoned slab and a tensor without a gradient.

    ``lr_mult``: the plan gets the learning-rate table before its first compute call (``Plan.set_lr_multipliers``, what
    the train ops' ``lr_multipliers`` argument does).  ``window_weight``: the plan divides each window by W
    (``Plan.set_window_weight`` on a zeroed 16-byte block ``ww``, what the train ops' ``window_weight=True`` does);
    ``wstep(grads, w)`` adds w into the device W (an fp32 add on the stream) and into the oracle's, then steps both, and
    ``check`` also compares W and last_weight exactly.
    """

    def __init__(self, man, variant: str, mode: str, layout: str = "table", dtype: str = "fp32", has_g: bool = True,
                 ema: Optional[Tuple[float, bool]] = None, N: int = 3, seed: int = 0, views: Optional[Dict[int, int]] = None,
                 nograd: Sequence[int] = (), zero: Sequence[int] = (), adapt_exclude: Optional[Sequence[str]] = None,
                 injected: bool = False, init: Optional[Dict[int, np.ndarray]] = None, tensor_norms: bool = False,
                 ls_cfg=LS_CFG, sched: Optional[Dict[str, float]] = None, global_step: int = 0,
                 device_schedule: bool = False, reset: str = "materialized", lr_mult: Optional[Sequence[float]] = None,
                 window_weight: bool = False):
        import torch
        import gaccum_b200 as g
        from gaccum_b200.train_op import GaccumTrainOp, PackedTrainOp
        self.torch, self.g = torch, g
        self.man, self.variant, self.mode, self.layout, self.has_g, self.N = man, variant, mode, layout, has_g, N
        self.dtype = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}[dtype]
        self.views, self.nograd = dict(views or {}), set(nograd)
        self.injected = injected
        self.ls_cfg, self.sched, self.g0 = ls_cfg, dict(SCHED if sched is None else sched), int(global_step)
        self.device_schedule = device_schedule
        self.g_host = self.g0                # the step of the next micro-step, as the oracle counts it
        self.rng = np.random.default_rng(seed)
        names = [n for n, _ in man]
        params = []
        for i, (_, s) in enumerate(man):
            x = np.zeros(s, F32) if i in zero else self.rng.normal(0, 0.05, s).astype(F32)
            if init is not None and i in init:
                x = np.array(init[i], F32).reshape(s)
            params.append(torch.from_numpy(x).to(self.dtype))          # 16-bit: the model starts representable
        hpo = oracle_hparams(variant, mode)
        hp = g.HParams(hpo.variant, 0, hpo.beta1, hpo.beta2, hpo.epsilon, hpo.weight_decay_rate, hpo.clip_norm)
        self.ls = mode.startswith("ls_")
        lsc = g.LossScaleConfig(*ls_cfg) if self.ls else None
        emac = g.EmaConfig(*ema) if ema is not None else None
        sc = self.sched
        lr_fn = lambda s: g.learning_rate(sc["init_lr"], sc["num_train_steps"], sc["num_warmup_steps"], s)
        kw = dict(loss_scale=lsc, ema=emac, exclude_from_layer_adaptation=adapt_exclude, global_step=self.g0)
        if device_schedule:
            kw["device_schedule"] = g._lib.ScheduleConfig(**sc)
            lr_fn = None
        if tensor_norms:
            kw["tensor_norms"] = True
        if layout == "packed":
            assert dtype == "fp32" and not self.views
            self.op = PackedTrainOp([p.cuda() for p in params], names, hp, N, lr_fn, **kw)
            self.gslab = torch.zeros_like(self.op.accum) if has_g else None
        else:
            self.op = GaccumTrainOp([self._device(i, p) for i, p in enumerate(params)], names, hp, N, lr_fn, **kw)
        self.cap = 0 if layout == "packed" else (256 if len(man) <= 256 else 1920)
        adapt = self.op.adapt if variant == "lamb" else None
        lr_mult = None if lr_mult is None else np.asarray(lr_mult, F32)
        self.ref = reference_op(variant, mode, [p.float().numpy() for p in params], names, N, adapt=adapt,
                                lr_mult=lr_mult, window_weight=window_weight, ls_cfg=ls_cfg, sched=self.sched,
                                global_step=self.g0)
        self.tracker = Ema(self._weights(), *ema) if ema is not None else None
        self.clipped = False                 # some window so far had a clip scale other than 1
        assert reset in RESETS and (reset == "materialized" or (layout == "table" and N >= 2)), (reset, layout, N)
        self.reset = reset
        self.windows = 0                     # applies so far: the poison's rotation
        self.poisoned = False                # the raw slab holds poison (the window's first accumulate is next)
        self.first_over_poison = 0
        self.materializes = 0                # calls of gaccum_accum_materialize ...
        self.expected_materializes = 0       # ... and how many of them a test made on purpose
        if reset != "materialized":
            if reset == "stored":
                self.op._set_deferred_reset(False)
            assert self.op._deferred == (reset == "deferred")
            plan, real = self.op.plan, self.op.plan.accum_materialize

            def counted(*a):
                self.materializes += 1
                return real(*a)
            plan.accum_materialize = counted
            covered = np.zeros(self.op._accum.numel(), bool)
            for o, (_, s) in zip(self.op.plan.offsets, man):
                covered[o:o + int(np.prod(s))] = True
            self.pad_idx = torch.from_numpy(np.flatnonzero(~covered)).cuda()
            self.op._accum.view(torch.int32)[self.pad_idx] = np.array(PAD_BITS, np.uint32).view(np.int32).item()
        if lr_mult is not None:
            self.op.plan.set_lr_multipliers(lr_mult)
        self.ww = None
        if window_weight:
            self.ww = torch.zeros(4, dtype=torch.float32, device="cuda")
            self.op.plan.set_window_weight(self.ww.data_ptr())

    # -- inputs -----------------------------------------------------------------------------------------------------
    def _device(self, i: int, t):
        """Tensor i's parameter or gradient on the GPU, at its view offset."""
        torch = self.torch
        off = self.views.get(i)
        if off is None:
            return t.cuda()
        buf = torch.zeros(t.numel() + off + 8, dtype=t.dtype, device="cuda")
        v = buf[off:off + t.numel()].view(t.shape)
        v.copy_(t)
        return v

    def grads(self, sigma: float = 0.1, inf_at: Optional[Tuple[int, int]] = None):
        """This micro-step's gradients (fp32, unscaled), None for the tensors without one."""
        out = [None if i in self.nograd else self.rng.normal(0, sigma, s).astype(F32) for i, (_, s) in enumerate(self.man)]
        if inf_at is not None:
            out[inf_at[0]].reshape(-1)[inf_at[1]] = np.inf
        return out

    # -- one micro-step ---------------------------------------------------------------------------------------------
    def inputs(self, grads):
        """This micro-step's gradients as the oracle sees them (host, the upcast) and as the op gets them (dev)."""
        torch = self.torch
        S = F32(self.ref.scale) if self.ls else F32(1.0)
        host, dev = [], []
        for i, x in enumerate(grads):
            if x is None:
                host.append(None); dev.append(None)
                continue
            with np.errstate(over="ignore", invalid="ignore"):
                t = torch.from_numpy(x * S).to(self.dtype)                 # gradients of loss * S, in the model's dtype
            host.append(t.float().numpy())                                   # ... what the oracle sees: their upcast
            dev.append(self._device(i, t))
        return host, dev

    def wstep(self, grads, w, launch=None) -> bool:
        """``step`` with the micro-batch's weight w added into the device W and the oracle's first."""
        self.ref.add_weight(w)
        with self.torch.no_grad():
            self.ww[0].add_(float(w))
        return self.step(grads, launch)

    def step(self, grads, launch=None) -> bool:
        """One micro-step of the op and its oracle, then ``check``.  ``launch(dev)``, if given, runs the op's micro-step
        in place of its own entry point (e.g. by replaying a graph captured over one micro-step); a device-scheduled op
        only."""
        torch, op = self.torch, self.op
        host, dev = self.inputs(grads)
        g = self.g_host if self.device_schedule else op.global_step
        applied = self.g.is_apply_step(g, self.N)
        info = None if self.injected else self.ref.run(host)
        if launch is not None:
            assert self.device_schedule
            launch(dev)
        elif self.device_schedule:
            with torch.no_grad():
                if self.layout == "packed":
                    for p, t in zip(op.params, dev):
                        if t is not None:
                            p.grad.add_(t)
                    ran = op.step()
                elif self.has_g or (self.reset != "materialized" and not applied):
                    ran = op.run(dev)
                else:
                    for i, t in enumerate(dev):                # what the accumulate kernel adds: the widened gradient
                        if t is not None:
                            self.accum_view(i).add_(t.float())
                    ran = op.run([None] * len(dev))
            op.schedule_state()                                # raises if the device refused the launch
            assert ran == applied
        elif self.layout == "packed":
            if self.has_g:
                self.gslab.zero_()
                for i, t in enumerate(dev):
                    if t is not None:
                        op._view(self.gslab, i).copy_(t)
                lr = op.lr_fn(g)
                op.plan.step_packed(self.gslab.data_ptr(), op.param_slab.data_ptr(), op.accum.data_ptr(), op.m.data_ptr(),
                                    op.v.data_ptr(), op._step_args(g, lr), -1, op._stream())
                if applied:
                    op._advance_beta_powers()
                op.global_step = g + 1
            else:
                for p, t in zip(op.params, dev):
                    if t is not None:
                        p.grad.add_(t)
                assert op.step() == applied
        elif self.has_g or (self.reset != "materialized" and not applied):
            assert op.run(dev) == applied
        elif self.reset != "materialized":
            # the apply's gradients go in through the accumulate kernel on the raw slab, which is defined mid-window
            op.plan.accumulate(op._grad_table(dev), op._accum_ptr, op._stream())
            assert op.run([None] * len(dev))
        else:
            op.accumulate_only(dev)
            if applied:
                op.apply_only(None)
            op.global_step = g + 1
        self.g_host = g + 1
        if self.injected:
            if applied:
                st = op.stats()
                ratios = op.trust_ratios() if self.variant == "lamb" else None
                self.ref.reduced = onp.Reduced(F32(st["global_norm"]), ratios)
            info = self.ref.run(host)
        assert info.applied == applied
        if self.poisoned and any(x is None and n > 0 for x, n in zip(grads, self._sizes())):
            self.first_over_poison += 1
        self.poisoned = False
        self.check(info)
        if applied:
            self.windows += 1
            if self.reset == "deferred":
                self.poison()
        return applied

    # -- the accumulators without materializing a deferred reset ------------------------------------------------------
    def _sizes(self) -> List[int]:
        return [int(np.prod(s)) for _, s in self.man]

    def raw_accum(self):
        """The accumulator slab as the kernels left it: ``op.accum`` unless a test of the deferred reset runs."""
        return self.op.accum if self.reset == "materialized" else self.op._accum

    def accum_view(self, i: int):
        return self.op._view(self.raw_accum(), i)

    def poison(self) -> None:
        """Right after an apply of a deferred-reset op: POISON into every tensor's raw accumulators, on the op's
        stream.  The slab is logically +0 until the window's first accumulate, which must not read it."""
        torch = self.torch
        with torch.no_grad():
            for i in range(len(self.man)):
                self.accum_view(i).view(torch.int32).fill_(poison_bits(i, self.windows))
        self.poisoned = True

    def set_reset(self, reset: str) -> None:
        """Turn the op's deferred reset on ("deferred") or off ("stored") between micro-steps.  Turning it off
        materializes first."""
        assert reset in ("deferred", "stored") and self.reset != "materialized"
        if self.op._deferred and reset == "stored":
            self.expected_materializes += 1
            self.poisoned = False
        self.op._set_deferred_reset(reset == "deferred")
        self.reset = reset

    def read_accum(self) -> None:
        """The op's own read of the accumulators (``op.accum``, which materializes a deferred reset) against the
        oracle: every tensor element bit for bit, +0.0 right after an apply."""
        self.expected_materializes += self.op._deferred
        got = self._slab(self.op.accum)
        assert self.materializes == self.expected_materializes
        for i, a in enumerate(got):
            assert _bits_equal(a, self.ref.accum[i]), f"accumulator of {self.man[i][0]} read through op.accum"
        self.poisoned = False

    def finish(self) -> None:
        """The end of a case: no unplanned materialize ran, the padding is untouched, and one ``op.accum`` read
        matches the oracle."""
        if self.reset == "materialized":
            return
        assert self.materializes == self.expected_materializes
        self.check_padding()
        self.read_accum()
        self.check_padding()

    def check_padding(self) -> None:
        pad = self.op._accum.view(self.torch.int32)[self.pad_idx].cpu().numpy()
        assert (pad == np.array(PAD_BITS, np.uint32).view(np.int32)).all(), "a kernel wrote the slab's padding"

    def run(self, steps: int, inf_at: Optional[Tuple[int, int, int]] = None, sigma: float = 0.1) -> None:
        """``steps`` micro-steps; ``inf_at = (step, tensor, element)`` puts one inf into that gradient."""
        for s in range(steps):
            self.step(self.grads(sigma, inf_at[1:] if inf_at is not None and inf_at[0] == s else None))

    # -- what the kernel left ---------------------------------------------------------------------------------------
    def _slab(self, slab) -> List[np.ndarray]:
        host = slab.cpu().numpy()
        return [host[o:o + int(np.prod(s))].reshape(s) for o, (_, s) in zip(self.op.plan.offsets, self.man)]

    def _weights(self) -> List[np.ndarray]:
        op = self.op
        if getattr(op, "master", None) is not None:
            return self._slab(op.master)
        if self.layout == "packed":
            return self._slab(op.param_slab)
        flat = self.torch.cat([p.detach().reshape(-1).float() for p in op.params]).cpu().numpy()
        out, o = [], 0
        for _, s in self.man:
            n = int(np.prod(s))
            out.append(flat[o:o + n].reshape(s)); o += n
        return out

    def skipped(self) -> bool:
        return bool(self.ref.last_skipped)

    def check(self, info) -> None:
        torch, op, ref = self.torch, self.op, self.ref
        torch.cuda.synchronize()
        names = [n for n, _ in self.man]
        assert self.materializes == self.expected_materializes, "the accumulators were materialized"
        if not (self.reset == "deferred" and info.applied):    # right after a deferred reset the slab is unspecified
            for i, a in enumerate(self._slab(self.raw_accum())):
                assert _bits_equal(a, ref.accum[i]), f"accumulator of {names[i]}"
        if info.applied and not self.skipped() and (self.mode in ("clip", "ls_clip")) and info.clip_scale != F32(1.0):
            self.clipped = True
        exact = self.injected or (self.variant != "lamb" and not self.clipped)
        weights = self._weights()
        for what, got, exp in (("p", weights, ref.params), ("m", self._slab(op.m), ref.m), ("v", self._slab(op.v), ref.v)):
            # not bit-exact: within 1e-5 of the model's largest |value|.  Per tensor that would be too tight for the
            # oracle itself: its global norm adds the per-tensor sums in fp32 one by one (off by up to ~1e-6 with 300
            # tensors; the kernel's sum is exact), and a 1-element tensor whose m nearly cancels magnifies that.
            scale = max([float(np.max(np.abs(e))) for e in exp if e.size] + [1e-30])
            for i in range(len(self.man)):
                if exact:
                    assert _bits_equal(got[i], exp[i]), f"{what} of {names[i]}"
                elif got[i].size:
                    err = float(np.max(np.abs(got[i].astype(np.float64) - exp[i])))
                    assert err <= 1e-5 * scale, f"{what} of {names[i]}: {err / scale}"
        if getattr(op, "master", None) is not None:
            for i, p in enumerate(op.params):
                assert torch.equal(p.view(torch.int16), op.master_view(i).to(self.dtype).view(torch.int16)), \
                    f"model copy of {names[i]}"
        if info.applied:
            st = op.stats()
            assert st["applied"] and F32(st["lr"]) == F32(info.lr)
            if self.mode not in ("clip", "ls_clip"):
                assert (st["global_norm"], st["clip_scale"]) == (0.0, 1.0)
            elif self.injected:
                s, e = F32(st["clip_scale"]), F32(info.clip_scale)
                assert s.tobytes() == e.tobytes() or (np.isnan(s) and np.isnan(e)), (s, e)    # NaN: any payload
                check_global_norm(F32(st["global_norm"]), ref.window_c)
            else:
                for k, e in (("global_norm", info.global_norm), ("clip_scale", info.clip_scale)):
                    if np.isfinite(e):
                        assert abs(st[k] - float(e)) <= 3e-6 * abs(float(e)), (k, st[k], e)
                    else:
                        assert not np.isfinite(st[k]), (k, st[k], e)
            if self.variant == "lamb" and self.injected:
                if not self.skipped():
                    adapted = [i for i in range(len(self.man)) if ref.adapt[i]]
                    r = op.trust_ratios()
                    assert all(r[i] == 1.0 for i in range(len(self.man)) if not ref.adapt[i])
                    assert len(ref.window_pu) == len(adapted)
                    for i, (p, u) in zip(adapted, ref.window_pu):
                        exp = trust_ratio_candidates(p, u)
                        assert any(r[i].tobytes() == e.tobytes() for e in exp), (names[i], r[i], exp)
            elif self.variant == "lamb":
                r = op.trust_ratios()
                exp = np.array(ref.ratios, F32)
                # within 1e-6; once a window has clipped, 2e-4: a 1-element tensor whose u nearly cancels turns the
                # ~1e-6 difference of the two global norms (above) into up to ~1e-4 in r = |p| / |u|
                rtol = 2e-4 if self.clipped else 1e-6
                bad = np.abs(r.astype(np.float64) - exp) > rtol * np.abs(exp)
                assert not bad.any(), [(names[i], r[i], exp[i]) for i in np.flatnonzero(bad)]
        if self.ls:
            s = op.loss_scale_state()
            assert (F32(s["scale"]), s["good_windows"], s["skipped_windows"], s["last_skipped"]) == \
                (ref.scale, ref.good_windows, ref.skipped_windows, ref.last_skipped)
        if self.device_schedule:
            block = op._sched_state.cpu()
            assert int(block[0]) == int(op.global_step_tensor) == ref.global_step == self.g_host
            assert int(block.view(torch.int32)[11]) == 0, "refused"
            st = op.stats()
            assert F32(st["lr"]).tobytes() == F32(self.g.learning_rate(
                self.sched["init_lr"], self.sched["num_train_steps"], self.sched["num_warmup_steps"], ref.global_step - 1)).tobytes()
            assert st["applied"] == info.applied
            sched_b = block.view(torch.float32)[9:11].numpy()
            if self.ls:
                assert not sched_b.any(), "the schedule block holds beta powers under loss scaling"
        if self.variant in ("adam", "lamb"):
            if self.ls:
                words = op._ls_state.cpu().numpy()
                b1, b2 = words[4], words[5]
            elif self.device_schedule:
                b1, b2 = sched_b
            else:
                b1, b2 = F32(op.beta1_power), F32(op.beta2_power)
            assert (b1, b2) == (F32(ref.beta1_power), F32(ref.beta2_power))
        if self.tracker is not None:
            if info.applied and not self.skipped():
                self.tracker.average(weights)
            for i, e in enumerate(self._slab(op.ema)):
                assert _bits_equal(e, self.tracker.avg[i]), f"average of {names[i]}"
            es = op.ema_state()
            assert es["num_updates"] == self.tracker.num_updates and F32(es["decay"]) == self.tracker.decay
        if self.ww is not None:
            got = self.ww[:2].cpu().numpy()
            assert got[0].tobytes() == F32(ref.weight).tobytes(), (got[0], ref.weight)
            assert got[1].tobytes() == F32(ref.last_weight).tobytes(), (got[1], ref.last_weight)
