"""GaccumTrainOp -- the train_op object ``create_optimizer`` returns (host side, PyTorch plumbing).

Holds what the reference's graph holds as variables: ``accum_grads`` (optimization.py:78),
``adam_m`` / ``adam_v`` (optimization.py:137-148), ``global_step`` (optimization.py:27) and, for
the plain-Adam variant, TF1's ``beta{1,2}_power`` non-slot variables -- but accum/m/v are three
packed fp32 slabs in HBM instead of 3T separate variables.  ``run(grads)`` is one
``session.run(train_op)``: exactly one kernel launch through the C ABI, then ``global_step += 1``
(optimization.py:102-103).  PyTorch supplies device memory and the CUDA stream; all arithmetic is
in csrc/.
"""
from __future__ import annotations

import contextlib
from typing import Callable, Dict, Optional, Sequence, Union

import numpy as np
import torch

from . import _lib
from ._lib import ADAM, ADAM_WEIGHT_DECAY, LAMB, EmaConfig, HParams, LossScaleConfig, Plan, ScheduleConfig, StepArgs


def _f32(x) -> float:
    return float(np.float32(x))


# 16-bit models GaccumTrainOp trains with fp32 master weights (gaccum_plan_set_param_dtype)
_HALF_DTYPES = {torch.bfloat16: _lib.DTYPE_BF16, torch.float16: _lib.DTYPE_F16}


def _refuse_half(params: Sequence[torch.Tensor], what: str) -> None:
    if any(p.dtype in _HALF_DTYPES for p in params):
        raise ValueError(f"{what} does not support bf16 / fp16 parameters; use GaccumTrainOp")


def _pinned_zeros(n: int) -> torch.Tensor:
    """fp32 zeros in page-locked host memory (pageable where the CUDA runtime cannot pin)."""
    t = torch.zeros(n, dtype=torch.float32)
    try:
        return t.pin_memory()
    except Exception:
        return t


class ScheduleCursor:
    """The host's share of a device-scheduled train op: the step of its next launch, passed as StepArgs.global_step.
    gaccum_step takes from it both the branch and whether the launch is a window's first accumulate (which does not read
    the accumulators), by the int32 predicate the device checks.  The position g mod N is not enough: int32(g) jumps
    from 2^31 - 1 to -2^31 every 2^32 steps, and unless N is a power of two the window that straddles the jump is longer
    than N (for N = 3 it applies at 2^31 - 2 and next at 2^31 + 2).

    Captured launches run when the graph is replayed, any number of times, so after a capture the host does not know the
    step: the first eager launch after it reads the device counter (``read_step``, synchronous), once.  A replay made
    after that, between eager launches, leaves the tracked step behind by whole windows: the same kernels, except once
    the replays have carried the device across an int32 wrap, where the next eager launch is refused by the device
    (loudly: ``schedule_state()`` raises) and writing ``global_step`` resynchronises."""

    def __init__(self, accum_n: int, read_step: Callable[[], int]):
        self.N, self._read_step = int(accum_n), read_step
        self.step = 0                   # the next launch's step, while not stale
        self._stale = False             # a capture launched since the step was last known
        self._capturing = False

    def reset(self, g: int) -> None:
        """The device counter was written with g."""
        self.step, self._stale = int(g), False

    def launch(self, capturing: bool) -> int:
        """The step of the launch about to be enqueued.  A CUDA graph must start at a window start (an apply step):
        refused here when the capture follows eager micro-steps; a graph that starts or ends mid-window, or whose replay
        straddles the int32 wrap, is refused by the device when replayed (gaccum.h: `refused`)."""
        if capturing:
            if not self._capturing and not _lib.is_apply_step(self.step, self.N):
                raise ValueError(f"a CUDA graph of a device-scheduled train op must start at a window start: this "
                                 f"capture starts at global_step {self.step}, an accumulate step (N = {self.N})")
            self._stale = True
        elif self._stale:
            self.reset(self._read_step())
        self._capturing = capturing
        return self.step

    def advance(self) -> bool:
        """After the launch: True if it was an apply step."""
        applied = _lib.is_apply_step(self.step, self.N)
        self.step += 1
        return applied


class ScheduleLr:
    """The learning rate of a device-scheduled train op as a host function (for logging and comparisons): the same
    fp32 evaluation of create_optimizer's schedule the device performs (gaccum_learning_rate)."""

    def __init__(self, cfg: ScheduleConfig):
        self.cfg = cfg

    def __call__(self, step: int) -> float:
        return _lib.learning_rate(self.cfg.init_lr, self.cfg.num_train_steps, self.cfg.num_warmup_steps, step)


class LrTable:
    """A device schedule whose learning rates come from a table: the launch at step g uses lr = values[min(g, L - 1)]
    (gaccum_plan_set_lr_table), so a replayed CUDA graph follows any schedule the host can evaluate -- e.g. one of
    ``schedules`` (``LrTable((schedules.cosine_decay(1e-4, 10000), 10000))``).  ``values`` is a 1-D array-like of
    learning rates, or ``(lr_fn, num_steps)``: ``lr_fn.table(num_steps)`` where it has one, else ``lr_fn(g)`` for g in
    [0, num_steps).  Each value is rounded to fp32 once; ValueError unless there is at least one, and every one is finite,
    >= 0 and fits fp32.  The table is configuration, not state: checkpoints do not store it, a resumed run passes it
    again."""

    def __init__(self, values):
        if isinstance(values, tuple) and len(values) == 2 and callable(values[0]):
            fn, n = values
            n = int(n)
            if n < 1:
                raise ValueError(f"a learning-rate table needs num_steps >= 1 (got {n})")
            values = fn.table(n) if hasattr(fn, "table") else [fn(g) for g in range(n)]
        vals = np.asarray(values, dtype=np.float64)
        if vals.ndim != 1 or vals.size == 0:
            raise ValueError(f"a learning-rate table is a non-empty 1-D array (got shape {vals.shape})")
        with np.errstate(over="ignore"):
            v32 = vals.astype(np.float32)
        bad = ~(np.isfinite(vals) & (vals >= 0.0) & np.isfinite(v32))
        if bad.any():
            i = int(np.flatnonzero(bad)[0])
            raise ValueError(f"learning rate {i} of the table is {vals[i]!r}: it must be finite and >= 0, and fit fp32")
        v32.flags.writeable = False
        self.values = v32


class TableLr:
    """The learning rate of a table-scheduled train op as a host function: ``float(table[min(g, L - 1)])`` read from the
    op's device table (synchronous), so an entry rewritten on the device is what it reports."""

    def __init__(self, table: torch.Tensor):
        self.table = table

    def __call__(self, step: int) -> float:
        return float(self.table[min(int(step), self.table.numel() - 1)])


# the state_dict key of a weighted train op's running window weight W (an fp32 scalar)
WINDOW_WEIGHT_KEY = "gradient_accumulation/window_weight"


def _stats_dict(buf: torch.Tensor) -> Dict[str, float]:
    """The 16-byte gaccum_stats block as ``stats()`` reports it."""
    a, lr, gn, s = buf.tolist()
    return {"applied": bool(a), "lr": lr, "global_norm": gn, "clip_scale": s}


class _TrainOpCore:
    """What every train op keeps besides its slabs: the plan, the hyper-parameters, ``global_step``
    (optimization.py:27) and TF1's ``beta{1,2}_power`` non-slot variables, with the per-step scalars built from them."""

    def __init__(self, params: Sequence[torch.Tensor], names: Sequence[str], hp: HParams, accum_n: int,
                 lr_fn: Callable[[int], float], exclude_from_weight_decay: Optional[Sequence[str]],
                 global_step: int, device: int, exclude_from_layer_adaptation: Optional[Sequence[str]] = None):
        if len(params) != len(names):
            raise ValueError("params and names differ in length")
        self.params = list(params)
        # optimization.py:135-143 names slots after _get_variable_name(param.name): the ":0" tensor suffix is stripped
        self.names = [_lib._variable_name(n) for n in names]
        self.hp, self.N, self.lr_fn, self.global_step = hp, int(accum_n), lr_fn, int(global_step)
        self.decay = _lib.decay_mask(names, hp.weight_decay_rate, exclude_from_weight_decay) \
            if hp.variant in (ADAM_WEIGHT_DECAY, LAMB) else [False] * len(params)
        self.plan = Plan([p.numel() for p in params], self.decay, hp, device=device)
        # LAMB: the layer-adaptation mask; as in TF-Addons, its exclusions default to the weight-decay ones, and it is
        # evaluated by name whatever the weight-decay rate
        self.adapt: Optional[list] = None
        if hp.variant == LAMB:
            excl = exclude_from_layer_adaptation if exclude_from_layer_adaptation is not None else exclude_from_weight_decay
            self.adapt = _lib.adaptation_mask(names, excl)
            self.plan.set_layer_adaptation(self.adapt)
        # TF1 AdamOptimizer._create_slots: beta powers start at beta
        self.beta1_power, self.beta2_power = _f32(hp.beta1), _f32(hp.beta2)
        self._stats_host = _pinned_zeros(4)
        self._ls_state: Optional[torch.Tensor] = None    # the loss-scaling block, when loss scaling is on
        self.loss_scale: Optional[torch.Tensor] = None

    def _step_args(self, g: int, lr: float) -> StepArgs:
        return StepArgs(g, self.N, 0, lr, self.beta1_power, self.beta2_power, 0.0)

    def _advance_beta_powers(self) -> None:
        """TF1 AdamOptimizer._finish: beta_power <- beta_power * beta (fp32) after the updates of an apply step.
        Under loss scaling the beta powers live in the device block and the apply kernel advances them, on applied
        windows only."""
        if self.hp.variant in (ADAM, LAMB) and self._ls_state is None:
            self.beta1_power = _f32(np.float32(self.beta1_power) * np.float32(self.hp.beta1))
            self.beta2_power = _f32(np.float32(self.beta2_power) * np.float32(self.hp.beta2))


class _DeviceTrainOp(_TrainOpCore):
    """A train op whose parameters live on one CUDA device and whose Adam moments are packed HBM slabs."""

    def __init__(self, params, names, hp, accum_n, lr_fn, exclude_from_weight_decay, global_step,
                 loss_scale: Optional[LossScaleConfig] = None, exclude_from_layer_adaptation=None,
                 lr_multipliers: Optional[Sequence[float]] = None, window_weight: bool = False,
                 device_schedule: Union[ScheduleConfig, LrTable, None] = None, tensor_norms: bool = False):
        self.ema: Optional[torch.Tensor] = None          # the moving average of the weights, when one is kept
        self._ema_state: Optional[torch.Tensor] = None
        self._sched_state: Optional[torch.Tensor] = None  # the device schedule's block, when one is kept
        self.lr_table: Optional[torch.Tensor] = None       # the device copy of an LrTable schedule (writable)
        if not params:
            raise ValueError("no trainable variables")
        # checked before the plan exists, so a bad table fails without touching the device
        mult = _lib.lr_multiplier_array(lr_multipliers, len(params)) if lr_multipliers is not None else None
        self.device = params[0].device
        if self.device.type != "cuda":
            raise _lib.GaccumError(_lib.ENODEVICE, "parameters must live on a CUDA device: the train_op has no CPU fallback")
        super().__init__(params, names, hp, accum_n, lr_fn, exclude_from_weight_decay, global_step,
                         self.device.index or 0, exclude_from_layer_adaptation)
        self.m = self._zeros_slab()
        self.v = self._zeros_slab()
        # per-tensor learning rates lr_t = fp32(lr * mult[t]) (gaccum_plan_set_lr_multipliers); configuration, not state:
        # checkpoints do not store them
        self._lr_multipliers = np.ones(len(params), np.float32) if mult is None else mult
        self._lr_multipliers.flags.writeable = False
        if mult is not None:
            self.plan.set_lr_multipliers(mult)
        if loss_scale is not None:
            # gaccum_loss_scale_state: 8 x 4 bytes; `loss_scale` views its first word, S, so a producer can write
            # (loss * op.loss_scale).backward() without reading S back to the host
            self._ls_state = torch.zeros(8, dtype=torch.float32, device=self.device)
            self.plan.set_loss_scale(loss_scale, self._ls_state.data_ptr())
            self.plan.loss_scale_init(self._ls_state.data_ptr(), self._stream())
            self.loss_scale = self._ls_state[0]
        self._ww_state: Optional[torch.Tensor] = None
        self.window_weight: Optional[torch.Tensor] = None
        if window_weight:
            # gaccum_window_weight_state: 4 x 4 bytes, zeroed; `window_weight` views its first word, W, so a producer adds
            # each micro-batch's weight on the device (op.window_weight += count) without a host round trip
            self._ww_state = torch.zeros(4, dtype=torch.float32, device=self.device)
            self.plan.set_window_weight(self._ww_state.data_ptr())
            self.window_weight = self._ww_state[0]
        if device_schedule is not None:
            # gaccum_schedule_state: 6 x 8 bytes.  From here on global_step, the lr and (without loss scaling) the beta
            # powers live on the device; the host tracks the step only to pick each launch's kernel (ScheduleCursor)
            table = isinstance(device_schedule, LrTable)
            if lr_fn is not None and (table or not isinstance(lr_fn, ScheduleLr)):
                raise ValueError("a device-scheduled train op computes its learning rate on the device: pass "
                                 "lr_fn=None" + ("" if table else " (or device_schedule_lr(cfg))"))
            # a table schedule still sets a valid config, whose init_lr and step counts the table then ignores
            cfg = ScheduleConfig(0.0, 0, 0) if table else device_schedule
            self._sched_state = torch.zeros(6, dtype=torch.int64, device=self.device)
            self.plan.set_device_schedule(cfg, self._sched_state.data_ptr())
            if table:
                self.lr_table = torch.from_numpy(device_schedule.values.copy()).to(self.device)
                self.plan.set_lr_table(self.lr_table.data_ptr(), self.lr_table.numel())
                self.lr_fn = TableLr(self.lr_table)
            else:
                self.lr_fn = ScheduleLr(cfg)
            self._cursor = ScheduleCursor(self.N, lambda: self._read_schedule()["global_step"])
            self._write_schedule(self._step, self.beta1_power, self.beta2_power)
        self._norms: Optional[torch.Tensor] = None
        if tensor_norms:
            # T x 3 fp32 on the device, rewritten by every apply: statistics, not state (checkpoints do not store them)
            self._norms = torch.zeros((len(params), 3), dtype=torch.float32, device=self.device)
            self.plan.set_tensor_norms(self._norms.data_ptr())

    @property
    def tensor_norms_tensor(self) -> torch.Tensor:
        """The per-tensor norms of the last apply as a (T, 3) fp32 CUDA tensor -- columns gradient, weight, update --
        without a copy or a sync (e.g. for a captured loop).  Every apply overwrites it."""
        if self._norms is None:
            raise ValueError("this train op does not report per-tensor norms (tensor_norms=False)")
        return self._norms

    def tensor_norms(self) -> np.ndarray:
        """Synchronously read the per-tensor norms of the last apply: a (T, 3) np.float32 array in tensor order with
        columns gradient (||c||, c before the clip scale), weight (||p|| before the update) and update
        (||p_before - p_after||); zeros before the first apply (gaccum.h, gaccum_plan_set_tensor_norms)."""
        return self.tensor_norms_tensor.cpu().numpy().copy()

    # -- global_step: a host int, or the device schedule's counter ---------------------------------------------------
    @property
    def global_step(self) -> int:
        """The pre-increment step of the next micro-step.  With a device schedule this is a SYNCHRONOUS read of the
        device counter: a training loop that wants the step without waiting reads ``global_step_tensor`` instead."""
        if self._sched_state is None:
            return self._step
        return self.schedule_state()["global_step"]

    @global_step.setter
    def global_step(self, g: int) -> None:
        g = int(g)
        sched = getattr(self, "_sched_state", None) is not None
        # deferred reset: the accumulators may be logically zero only while the next launch is a window's first
        # accumulate, which does not read them; a launch at any other new step would
        if getattr(self, "_deferred", False) and (sched or g != self._step) and not _lib.is_first_accumulate(g, self.N):
            self._materialize()
        self._step = g
        if sched:
            st = self._read_schedule()      # keeps the beta powers; a refused schedule starts afresh
            self._write_schedule(self._step, st["beta1_power"], st["beta2_power"])

    @property
    def device_schedule(self) -> bool:
        return self._sched_state is not None

    @property
    def global_step_tensor(self) -> torch.Tensor:
        """The device counter as a 0-d int64 CUDA tensor (a view: no copy, no sync).  Device-scheduled ops only."""
        if self._sched_state is None:
            raise ValueError("this train op keeps global_step on the host (device_schedule=None)")
        return self._sched_state[0]

    def _write_schedule(self, g: int, beta1_power: float, beta2_power: float) -> None:
        """gaccum_schedule_init: the step, the beta powers (ignored under loss scaling, whose block holds them) and
        refused = 0, stream-ordered on the current stream."""
        self.plan.schedule_init(self._sched_state.data_ptr(), g, beta1_power, beta2_power, self._stream())
        self._cursor.reset(g)

    def schedule_state(self) -> Dict[str, float]:
        """Synchronously read the device schedule: global_step, beta1_power and beta2_power (under loss scaling the
        loss-scaling block's) and refused.  Raises RuntimeError if a launch was refused (see gaccum.h)."""
        if self._sched_state is None:
            raise ValueError("this train op keeps global_step on the host (device_schedule=None)")
        out = self._read_schedule()
        if out["refused"]:
            raise RuntimeError(f"the device schedule refused a launch at global_step {out['global_step']}: it found the "
                               "step selecting the other branch (a CUDA graph captured or replayed across a window "
                               "boundary?).  Every launch since was a no-op; nothing after that step was computed")
        return out

    def _read_schedule(self) -> Dict[str, float]:
        words = self._sched_state.cpu()
        f, i = words.view(torch.float32), words.view(torch.int32)
        out = {"global_step": int(words[0]), "beta1_power": float(f[9]), "beta2_power": float(f[10]),
               "refused": bool(i[11])}
        if self._ls_state is not None:
            ls = self._ls_state.cpu()
            out["beta1_power"], out["beta2_power"] = float(ls[4]), float(ls[5])
        return out

    def _scheduled_step_args(self) -> StepArgs:
        """The host's share of a device-scheduled micro-step: its step, from which gaccum_step picks the branch and
        the first-accumulate kernel (ScheduleCursor.launch)."""
        g = self._cursor.launch(torch.cuda.is_current_stream_capturing())
        return StepArgs(g, self.N, 0, 0.0, 0.0, 0.0, 0.0)

    def _scheduled_after(self) -> bool:
        self.last_applied = self._cursor.advance()
        return self.last_applied

    def _init_ema(self, cfg: EmaConfig, weights: Callable[[int], torch.Tensor]) -> None:
        """Keep an exponential moving average of ``weights(i)`` (the fp32 weights the apply updates).  TF initialises
        a shadow variable to its variable's value: the average starts at the weights, and n at 0."""
        self.ema = self._zeros_slab()
        with torch.no_grad():
            for i in range(len(self.params)):
                self.ema_view(i).copy_(weights(i))
        self._ema_state = torch.zeros(2, dtype=torch.int64, device=self.device)    # gaccum_ema_state: 16 bytes
        self.plan.set_ema(cfg, self.ema.data_ptr(), self._ema_state.data_ptr())
        self.plan.ema_init(self._ema_state.data_ptr(), 0, self._stream())

    @property
    def lr_multipliers(self) -> np.ndarray:
        """Tensor t's learning-rate multiplier: the apply trains it with lr_t = fp32(lr * mult[t]) (np.float32,
        read-only; ones unless ``lr_multipliers`` was given)."""
        return self._lr_multipliers

    def window_weight_state(self) -> Dict[str, float]:
        """Synchronously read the window-weight block: weight (W, the running window's total so far) and last_weight
        (the W the last apply step divided by)."""
        if self._ww_state is None:
            raise ValueError("this train op does not weight its windows (window_weight=False)")
        words = self._ww_state.cpu()
        return {"weight": float(words[0]), "last_weight": float(words[1])}

    def _add_weight(self, weight, stream: Optional[int] = None) -> None:
        """Add a micro-batch's weight into W (an fp32 add on the op's stream), after checking it against the op: a
        weighted op needs one on every micro-step, an unweighted op takes none."""
        if self._ww_state is None:
            if weight is not None:
                raise ValueError("a weight was given to a train op that divides each window by N (window_weight=False)")
            return
        if weight is None:
            raise ValueError("this train op divides each window by its total weight (window_weight=True): "
                             "every micro-step needs its weight")
        ctx = torch.cuda.stream(torch.cuda.ExternalStream(stream, device=self.device)) if stream is not None \
            else contextlib.nullcontext()
        if isinstance(weight, torch.Tensor):
            weight = weight.to(device=self.device, dtype=torch.float32)   # fp32(w) first: the add is an fp32 add
        else:
            weight = float(np.float32(weight))
        with ctx, torch.no_grad():
            self.window_weight.add_(weight)

    def _window_weight_state_dict(self, out: Dict[str, torch.Tensor]) -> None:
        """The running W: a checkpoint taken mid-window needs it, as it needs the accumulators."""
        out[WINDOW_WEIGHT_KEY] = self._ww_state[0].detach().cpu().clone()

    def _load_window_weight(self, sd: Dict[str, torch.Tensor], strict: bool) -> None:
        """W from a checkpoint; non-strict, a checkpoint without it starts the window at W = 0."""
        if WINDOW_WEIGHT_KEY in sd:
            w = torch.as_tensor(sd[WINDOW_WEIGHT_KEY], dtype=torch.float32).reshape(())
        elif strict:
            raise KeyError(WINDOW_WEIGHT_KEY)
        else:
            w = torch.zeros((), dtype=torch.float32)
        with torch.no_grad():
            self._ww_state[0].copy_(w)

    def _zeros_slab(self) -> torch.Tensor:
        return torch.zeros(max(self.plan.padded_size, 32), dtype=torch.float32, device=self.device)

    def _materialize(self) -> None:
        """A deferred-reset op (GaccumTrainOp): store the zeros its last apply left logical, if it did, on the current
        stream (gaccum_accum_materialize; no sync)."""
        if getattr(self, "_deferred", False):
            self.plan.accum_materialize(self._accum_ptr, self._stream())

    def _stream(self, stream: Optional[int] = None) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream

    # -- views under the reference's variable names (read self.accum / m / v when called) -------------
    def _view(self, slab: torch.Tensor, i: int) -> torch.Tensor:
        o = self.plan.offsets[i]
        return slab[o:o + self.params[i].numel()].view(self.params[i].shape)

    def accum_view(self, i: int) -> torch.Tensor:
        return self._view(self.accum, i)

    def m_view(self, i: int) -> torch.Tensor:
        return self._view(self.m, i)

    def v_view(self, i: int) -> torch.Tensor:
        return self._view(self.v, i)

    def ema_view(self, i: int) -> torch.Tensor:
        """The moving average of parameter i (fp32; of the master weights on a 16-bit model)."""
        if self.ema is None:
            raise ValueError("this train op keeps no moving average (ema=None)")
        return self._view(self.ema, i)

    def ema_state(self) -> Dict[str, float]:
        """Synchronously read the moving average's state: num_updates (windows averaged so far) and decay (the d of
        the last averaged window, 0 before the first)."""
        if self._ema_state is None:
            raise ValueError("this train op keeps no moving average (ema=None)")
        words = self._ema_state.cpu()
        return {"num_updates": int(words[0]), "decay": float(words.view(torch.float32)[2])}

    @contextlib.contextmanager
    def averaged_weights(self):
        """Evaluate with the averaged weights: inside the block the parameters hold the moving averages (a 16-bit
        model: rounded to nearest-even); on leaving it they are restored bit for bit (a 16-bit model: from the master
        weights, as the apply leaves them).  Do not train inside the block."""
        if self.ema is None:
            raise ValueError("this train op keeps no moving average (ema=None)")
        master = getattr(self, "master", None)
        with torch.no_grad():
            saved = [p.detach().clone() for p in self.params] if master is None else None
            for i, p in enumerate(self.params):
                p.copy_(self.ema_view(i))
        try:
            yield self
        finally:
            with torch.no_grad():
                for i, p in enumerate(self.params):
                    p.copy_(saved[i] if master is None else self._view(master, i))

    def stats(self) -> Dict[str, float]:
        """Synchronously read what the last step computed (applied, lr, global_norm, clip_scale)."""
        stream = torch.cuda.current_stream(self.device)
        self.plan.read_stats(self._stats_host.data_ptr(), stream.cuda_stream)
        stream.synchronize()
        return _stats_dict(self._stats_host)

    def trust_ratios(self) -> np.ndarray:
        """LAMB: synchronously read the per-tensor trust ratios r of the last applied window (1 for tensors without
        layer adaptation, and before the first apply) -- what LAMB users log per layer."""
        if self.hp.variant != LAMB:
            raise ValueError("trust ratios exist for LAMB train ops only")
        out = _pinned_zeros(len(self.params))
        stream = torch.cuda.current_stream(self.device)
        self.plan.read_trust_ratios(out.data_ptr(), stream.cuda_stream)
        stream.synchronize()
        return out.numpy().copy()

    def loss_scale_state(self) -> Dict[str, float]:
        """Synchronously read the loss-scaling block (for logging): scale, good_windows, skipped_windows and
        last_skipped (True if the last apply step skipped its window)."""
        if self._ls_state is None:
            raise ValueError("loss scaling is off for this train op")
        words = self._ls_state.cpu()
        ints = words.view(torch.int32)
        return {"scale": float(words[0]), "good_windows": int(ints[1]),
                "skipped_windows": int(ints[2]) & 0xFFFFFFFF, "last_skipped": bool(ints[3])}

    def _loss_scale_state_dict(self, out: Dict[str, torch.Tensor]) -> None:
        """TF 2 LossScaleOptimizer's variable names; the beta powers come from the device block."""
        words = self._ls_state.cpu()
        out["loss_scale/current_loss_scale"] = words[0].clone()
        out["loss_scale/good_steps"] = torch.tensor(int(words.view(torch.int32)[1]), dtype=torch.int64)
        if self.hp.variant in (ADAM, LAMB):
            out["beta1_power"] = words[4].clone()
            out["beta2_power"] = words[5].clone()

    def _load_loss_scale_state(self, sd: Dict[str, torch.Tensor]) -> None:
        words = self._ls_state.cpu()
        if "loss_scale/current_loss_scale" in sd:
            s = float(sd["loss_scale/current_loss_scale"])
            m, e = np.frexp(s)
            if not (m == 0.5 and 1 <= e <= 128):
                raise ValueError(f"loss_scale/current_loss_scale must be a power of two in [1, 2^127], got {s!r}")
            words[0] = s
            words.view(torch.int32)[1] = int(sd["loss_scale/good_steps"])
        if self.hp.variant in (ADAM, LAMB) and "beta1_power" in sd:
            words[4] = float(sd["beta1_power"])
            words[5] = float(sd["beta2_power"])
        self._ls_state.copy_(words)


class GaccumTrainOp(_DeviceTrainOp):
    """The train op over scattered parameter and gradient tensors.

    A bf16 or fp16 model (every parameter of one of these dtypes) is trained with fp32 master weights: gradients of
    the parameters' dtype are accumulated in fp32, the apply updates the master weights (``master_view``) exactly as
    an fp32 model's parameters, then rewrites the model's tensors with them rounded to nearest-even.  The master
    weights are the truth: an edit of the model's tensors between applies is overwritten by the next apply (write
    checkpoints through ``load_state_dict``, which refreshes both)."""

    def __init__(self, params: Sequence[torch.Tensor], names: Sequence[str], hp: HParams, accum_n: int,
                 lr_fn: Callable[[int], float],
                 exclude_from_weight_decay: Optional[Sequence[str]] = ("LayerNorm", "layer_norm", "bias"),
                 global_step: int = 0, accum: Optional[torch.Tensor] = None,
                 loss_scale: Optional[LossScaleConfig] = None,
                 exclude_from_layer_adaptation: Optional[Sequence[str]] = None, ema: Optional[EmaConfig] = None,
                 lr_multipliers: Optional[Sequence[float]] = None, window_weight: bool = False,
                 device_schedule: Union[ScheduleConfig, LrTable, None] = None, tensor_norms: bool = False):
        dtypes = {p.dtype for p in params}
        if len(dtypes) > 1 and dtypes & set(_HALF_DTYPES):
            raise ValueError(f"parameters of mixed dtypes ({', '.join(sorted(str(d) for d in dtypes))}): "
                             "a 16-bit model must be all bf16 or all fp16")
        self.param_dtype = params[0].dtype if len(dtypes) == 1 and params[0].dtype in _HALF_DTYPES else torch.float32
        super().__init__(params, names, hp, accum_n, lr_fn, exclude_from_weight_decay, global_step, loss_scale,
                         exclude_from_layer_adaptation, lr_multipliers, window_weight, device_schedule, tensor_norms)
        for p in self.params:
            if p.dtype != self.param_dtype or not p.is_contiguous() or p.device != self.device:
                if self.param_dtype != torch.float32:
                    raise ValueError("parameters must be contiguous tensors of one dtype on one device")
                raise ValueError("parameters must be contiguous fp32 tensors on one device")
        self.master: Optional[torch.Tensor] = None
        if self.param_dtype != torch.float32:
            # the fp32 master weights: a slab in the plan's layout, starting at the exact upcast of the model
            self.master = self._zeros_slab()
            with torch.no_grad():
                for i, p in enumerate(self.params):
                    self.master_view(i).copy_(p)
            self.plan.set_param_dtype(_HALF_DTYPES[self.param_dtype], self.master.data_ptr())
        if ema is not None:
            self._init_ema(ema, self._weights)
        if accum is not None:          # caller-provided slab (e.g. NVLink peer-mapped symmetric memory)
            if accum.numel() < self.m.numel() or accum.dtype != torch.float32 or accum.device != self.device:
                raise ValueError("accum must be an fp32 tensor of at least plan.padded_size elements on the params' device")
            self.accum = accum
        else:
            self.accum = self._zeros_slab()
        self._accum_ptr, self._m_ptr, self._v_ptr = self.accum.data_ptr(), self.m.data_ptr(), self.v.data_ptr()
        self._param_ptrs = Plan.ptr_array([p.data_ptr() for p in self.params])
        self._param_key = tuple(p.data_ptr() for p in self.params)
        self._grad_key = None
        self._grad_ptrs = None
        self.last_lr = 0.0
        self.last_applied = False
        # N >= 2: the apply leaves the accumulators logically zero instead of storing zeros (4 B/param less HBM traffic
        # per window); the window's first accumulate, which does not read them, stores +0 + G.  With N = 1 every step
        # applies and reads them.
        self._deferred = False
        if self.N >= 2:
            self._set_deferred_reset(True)

    @property
    def accum(self) -> torch.Tensor:
        """The accumulator slab (optimization.py:78), in the plan's layout.  After an apply of a deferred-reset op it is
        first zeroed on the current stream (no sync), so every reader and writer sees the zeros the reference's apply
        stores."""
        self._materialize()
        return self._accum

    @accum.setter
    def accum(self, t: torch.Tensor) -> None:
        self._accum = t

    def _set_deferred_reset(self, on: bool) -> None:
        """Front ends whose collectives read or write the slab between launches keep the apply's zero store."""
        if not on:
            self._materialize()
        self.plan.set_deferred_reset(on)
        self._deferred = bool(on)

    def _grad_table(self, grads: Sequence[Optional[torch.Tensor]]):
        key = tuple(0 if g is None else g.data_ptr() for g in grads)
        if key != self._grad_key:
            for g, p in zip(grads, self.params):
                if g is None:
                    continue
                if self.param_dtype != torch.float32 and g.dtype != self.param_dtype:
                    raise ValueError(f"gradients of a {self.param_dtype} model must be {self.param_dtype} (got {g.dtype})")
                if g.dtype != self.param_dtype or not g.is_contiguous() or g.numel() != p.numel() or g.device != self.device:
                    raise ValueError("gradients must be contiguous fp32 tensors shaped like their parameter")
            self._grad_ptrs = Plan.ptr_array(list(key))
            self._grad_key = key
        return self._grad_ptrs

    def _refresh_param_table(self):
        key = tuple(p.data_ptr() for p in self.params)
        if key != self._param_key:
            self._param_ptrs = Plan.ptr_array(list(key))
            self._param_key = key

    # -- one micro-step -------------------------------------------------------------------
    def run(self, grads: Sequence[Optional[torch.Tensor]], weight=None) -> bool:
        """One ``session.run(train_op)`` (optimization.py:91-104).  Returns True if it applied.  A weighted op
        (window_weight=True) takes the micro-batch's weight -- a number or a device scalar, typically its count of loss
        tokens -- and adds it into W before the step; ``grads`` are then the gradients of the summed loss."""
        self._add_weight(weight)
        self._refresh_param_table()
        return self.run_bound(self._grad_table(grads))

    def bind(self, grads: Sequence[Optional[torch.Tensor]]):
        """Validate a gradient list once and return its device-pointer table.  A graph-mode caller
        (TF hands the op raw pointers) pays nothing per step; Python callers whose gradient buffers
        are persistent can do the same with ``run_bound(bind(grads))``."""
        self._grad_key = None
        table = self._grad_table(grads)
        self._grad_key = None
        return table

    def run_bound(self, grad_table, stream: Optional[int] = None) -> bool:
        """``run`` with a pointer table from ``bind`` (no per-step Python work over T tensors).
        Parameters must not have been re-allocated since construction / the last ``run``."""
        if self._sched_state is not None:
            # device schedule: the launch reads the step, lr and beta powers from the block and advances them
            args = self._scheduled_step_args()
            self.plan.step(grad_table, self._param_ptrs, self._accum_ptr, self._m_ptr, self._v_ptr, args,
                           self._stream(stream))
            return self._scheduled_after()
        g = self.global_step
        lr = self.lr_fn(g)
        if stream is None:
            stream = torch.cuda.current_stream(self.device).cuda_stream
        self.plan.step(grad_table, self._param_ptrs, self._accum_ptr, self._m_ptr, self._v_ptr,
                       self._step_args(g, lr), stream)
        return self._after(g, _lib.is_apply_step(g, self.N), lr)

    def accumulate_only(self, grads: Sequence[Optional[torch.Tensor]]) -> None:
        """The false branch alone (used by the data-parallel driver); does not touch global_step.  Reads the
        accumulators: ``self.accum`` materializes a deferred reset first."""
        self._refuse_schedule("accumulate_only")
        self.plan.accumulate(self._grad_table(grads), self.accum.data_ptr(), self._stream())

    def apply_only(self, grads: Optional[Sequence[Optional[torch.Tensor]]] = None) -> None:
        """The true branch alone; ``grads=None`` applies the accumulators as they are (``self.accum`` materializes a
        deferred reset first)."""
        self._refuse_schedule("apply_only")
        lr = _f32(self.lr_fn(self.global_step))
        self._refresh_param_table()
        self.plan.apply(self._grad_table(grads) if grads is not None else None, self._param_ptrs,
                        self.accum.data_ptr(), self.m.data_ptr(), self.v.data_ptr(),
                        self._step_args(self.global_step, lr), self._stream())
        self.last_lr, self.last_applied = lr, True
        self._advance_beta_powers()
        if not _lib.is_first_accumulate(self._step, self.N):
            self._materialize()      # global_step is unchanged: its launch may read the accumulators

    def _after(self, g: int, applied: bool, lr: float) -> bool:
        """Bookkeeping once micro-step ``g`` is launched."""
        self.last_lr, self.last_applied = lr, applied
        if applied:
            self._advance_beta_powers()
        # optimization.py:102-103.  Not through the setter: after an apply, step g + 1 is a window's first accumulate
        # (N >= 2), which does not read the accumulators, so a deferred reset stays deferred
        self._step = g + 1
        return applied

    __call__ = run

    # -- host-buffer entry point (what a CPU-resident caller such as the TF CPU graph sees) ----
    def _host_init(self):
        n = self.accum.numel()
        self._stage = [torch.empty(n, dtype=torch.float32, device=self.device) for _ in range(2)]
        self._stage_views = [[self._view(s, i) for i in range(len(self.params))] for s in self._stage]
        self._copy_stream = torch.cuda.Stream(self.device)
        self._d2h_stream = torch.cuda.Stream(self.device)
        self._buf_free = [torch.cuda.Event() for _ in range(2)]
        self._h2d_done = [torch.cuda.Event() for _ in range(2)]
        self._k_done, self._d2h_done = torch.cuda.Event(), torch.cuda.Event()
        self._host_calls = 0
        self._stats_ring = _pinned_zeros(4)

    def _refuse_schedule(self, what: str) -> None:
        if self._sched_state is not None:
            raise ValueError(f"{what} does not support a device schedule: a device-scheduled train op steps with run()")

    def run_host(self, host_grads: Sequence[Optional[torch.Tensor]],
                 host_params_out: Optional[Sequence[torch.Tensor]] = None) -> bool:
        """One micro-step whose gradients live in (pinned) HOST memory.

        H2D of this step's gradients (copy stream, double-buffered so it overlaps the previous
        kernel), one kernel launch, D2H of the 16-byte stats block, and -- on apply steps -- D2H of
        the updated parameters into ``host_params_out``.  Everything is stream-ordered; the caller's
        current stream observes completion.  Returns True if the step applied.
        """
        if self.master is not None:
            raise ValueError("run_host stages fp32 gradients: it does not support bf16 / fp16 parameters")
        if not hasattr(self, "_stage"):
            self._host_init()
        main = torch.cuda.current_stream(self.device)
        b = self._host_calls & 1
        self._host_calls += 1
        self._copy_stream.wait_event(self._buf_free[b])
        with torch.cuda.stream(self._copy_stream):
            for view, hg in zip(self._stage_views[b], host_grads):
                if hg is not None:
                    view.copy_(hg.view(view.shape), non_blocking=True)
            self._h2d_done[b].record(self._copy_stream)
        main.wait_event(self._h2d_done[b])
        grads = [v if hg is not None else None for v, hg in zip(self._stage_views[b], host_grads)]
        applied = self.run(grads)
        self._buf_free[b].record(main)
        self.plan.read_stats(self._stats_ring.data_ptr(), main.cuda_stream)
        if applied and host_params_out is not None:
            self._k_done.record(main)
            self._d2h_stream.wait_event(self._k_done)
            with torch.cuda.stream(self._d2h_stream):
                for hp_, p in zip(host_params_out, self.params):
                    hp_.copy_(p, non_blocking=True)
                self._d2h_done.record(self._d2h_stream)
            main.wait_event(self._d2h_done)
        return applied

    def master_view(self, i: int) -> torch.Tensor:
        """The fp32 master weights of parameter i (16-bit models only)."""
        if self.master is None:
            raise ValueError("fp32 parameters have no master copy")
        return self._view(self.master, i)

    def _weights(self, i: int) -> torch.Tensor:
        """The fp32 weights the apply updates: parameter i, or its master weights on a 16-bit model."""
        return self.params[i] if self.master is None else self.master_view(i)

    def _refresh_model(self) -> None:
        """The model's 16-bit tensors = the master weights rounded to nearest-even, as the apply leaves them."""
        with torch.no_grad():
            for i, p in enumerate(self.params):
                p.copy_(self.master_view(i))

    # -- checkpoint compatibility: the reference's Saver sees per-variable tensors --------
    def state_dict(self) -> Dict[str, torch.Tensor]:
        """Per-tensor copies under the reference's names (optimization.py:78, 137-148).  A 16-bit model stores its
        fp32 master weights under the variables' names, as TF mixed precision saves its fp32 variables, so fp32 and
        16-bit checkpoints load into each other."""
        sched = self.schedule_state() if self._sched_state is not None else None
        g = self.global_step if sched is None else sched["global_step"]
        out: Dict[str, torch.Tensor] = {"global_step": torch.tensor(g, dtype=torch.int64)}
        for i, n in enumerate(self.names):
            out[n] = self.params[i].detach().clone() if self.master is None else self.master_view(i).clone()
            out[n + "/adam_m"] = self.m_view(i).clone()
            out[n + "/adam_v"] = self.v_view(i).clone()
            out[n + "/accum_grad"] = self.accum_view(i).clone()
        if self.hp.variant in (ADAM, LAMB):
            b1, b2 = (self.beta1_power, self.beta2_power) if sched is None else (sched["beta1_power"], sched["beta2_power"])
            out["beta1_power"] = torch.tensor(b1, dtype=torch.float32)
            out["beta2_power"] = torch.tensor(b2, dtype=torch.float32)
        if self._ls_state is not None:
            self._loss_scale_state_dict(out)
        if self.ema is not None:
            # tf.train.ExponentialMovingAverage's shadow-variable names
            for i, n in enumerate(self.names):
                out[n + "/ExponentialMovingAverage"] = self.ema_view(i).clone()
            out["ExponentialMovingAverage/num_updates"] = torch.tensor(self.ema_state()["num_updates"], dtype=torch.int64)
        if self._ww_state is not None:
            self._window_weight_state_dict(out)
        return out

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True) -> None:
        self.global_step = int(sd["global_step"])
        for i, n in enumerate(self.names):
            with torch.no_grad():
                if n in sd:
                    (self.params[i] if self.master is None else self.master_view(i)).copy_(sd[n])
                for suffix, view in (("/adam_m", self.m_view), ("/adam_v", self.v_view), ("/accum_grad", self.accum_view)):
                    if n + suffix in sd:
                        view(i).copy_(sd[n + suffix])
                    elif strict:
                        raise KeyError(n + suffix)
        if self._ls_state is not None:
            self._load_loss_scale_state(sd)
        elif self.hp.variant in (ADAM, LAMB) and "beta1_power" in sd:
            self.beta1_power = float(sd["beta1_power"])
            self.beta2_power = float(sd["beta2_power"])
            if self._sched_state is not None:        # the beta powers' home is the schedule block
                self._write_schedule(int(sd["global_step"]), self.beta1_power, self.beta2_power)
        if self.ema is not None:
            self._load_ema_state(sd, strict)
        if self._ww_state is not None:
            self._load_window_weight(sd, strict)
        if self.master is not None:
            self._refresh_model()

    def _load_ema_state(self, sd: Dict[str, torch.Tensor], strict: bool) -> None:
        """The averages and n from a checkpoint.  Non-strict, a checkpoint without them (a pre-trained model, or a run
        without an EMA) starts the average afresh, as TF creates a shadow variable from its variable's restored value:
        each tensor whose weights were loaded but whose average was not averages from the loaded fp32 weights (the
        master weights of a 16-bit model), and without a stored n the count restarts at 0."""
        for i, n in enumerate(self.names):
            key = n + "/ExponentialMovingAverage"
            if key in sd:
                with torch.no_grad():
                    self.ema_view(i).copy_(sd[key])
            elif strict:
                raise KeyError(key)
            elif n in sd:
                with torch.no_grad():
                    self.ema_view(i).copy_(self._weights(i))
        key = "ExponentialMovingAverage/num_updates"
        if key in sd:
            n = int(sd[key])
            if n < 0:
                raise ValueError(f"{key} must be >= 0, got {n}")
        elif strict:
            raise KeyError(key)
        else:
            n = 0
        self.plan.ema_init(self._ema_state.data_ptr(), n, self._stream())


class PackedTrainOp(_DeviceTrainOp):
    """SURVEY.md 8(f) #2 -- gradient hand-off without the scatter.

    The reference keeps T parameters, T gradients and T ``accum_grads`` as separate tensors
    (optimization.py:70-71, 78) and adds gradient to accumulator with T ``assign_add`` ops per micro-step (:81, 93).
    Here the parameters are re-pointed at views of ONE flat slab in the plan's layout and every ``p.grad`` is a view
    of the packed accumulator slab, so the producer (autograd's ``AccumulateGrad``: ``grad += new_grad``, one fp32
    rounding per micro-step -- the same arithmetic as ``assign_add``) accumulates IN PLACE, straight into ``accum``:
      * accumulate micro-steps launch nothing from this library (12 -> 0 B/param of train_op traffic),
      * the apply micro-step runs the slab-to-slab kernel with no gradient stream and no pointer table
        (``gaccum_step_packed(grad_slab=NULL)``: 32 B/param instead of 36) and leaves ``accum`` == ``p.grad`` zeroed
        for the next window.
    Call ``step()`` once per micro-step, after ``loss.backward()``.  Never set the gradients to ``None``
    (``zero_grad(set_to_none=True)``) -- the views are the accumulator.
    """

    def __init__(self, params: Sequence[torch.Tensor], names: Sequence[str], hp: HParams, accum_n: int,
                 lr_fn: Callable[[int], float],
                 exclude_from_weight_decay: Optional[Sequence[str]] = ("LayerNorm", "layer_norm", "bias"),
                 global_step: int = 0, loss_scale: Optional[LossScaleConfig] = None,
                 exclude_from_layer_adaptation: Optional[Sequence[str]] = None, ema: Optional[EmaConfig] = None,
                 lr_multipliers: Optional[Sequence[float]] = None, window_weight: bool = False,
                 device_schedule: Union[ScheduleConfig, LrTable, None] = None, tensor_norms: bool = False):
        # autograd accumulates a 16-bit parameter's gradient in its own dtype: it cannot add into an fp32 slab
        _refuse_half(params, "PackedTrainOp")
        super().__init__(params, names, hp, accum_n, lr_fn, exclude_from_weight_decay, global_step, loss_scale,
                         exclude_from_layer_adaptation, lr_multipliers, window_weight, device_schedule, tensor_norms)
        self.param_slab = self._zeros_slab()
        self.accum = self._zeros_slab()
        with torch.no_grad():
            for i, p in enumerate(self.params):
                if p.dtype != torch.float32:
                    raise ValueError("parameters must be fp32")
                view = self._view(self.param_slab, i)
                view.copy_(p)
                p.data = view                          # the caller's tensors now alias the slab
                p.grad = self.accum_view(i)            # autograd accumulates straight into accum_grads
        if ema is not None:
            self._init_ema(ema, lambda i: self._view(self.param_slab, i))
        self.launches = 0

    def step(self, stream: Optional[int] = None, weight=None) -> bool:
        """One ``session.run(train_op)`` AFTER the backward pass has added this micro-batch's gradient into
        ``p.grad`` (== accum).  Returns True if it applied (optimization.py:91, pre-increment predicate).  A weighted op
        (window_weight=True) takes the micro-batch's weight, as ``GaccumTrainOp.run`` does."""
        self._add_weight(weight, stream)
        sched = self._sched_state is not None
        args = self._scheduled_step_args() if sched else None
        g = args.global_step if sched else self.global_step
        applied = _lib.is_apply_step(g, self.N)
        if sched and not applied:
            # the gradients are already in accum: the launch only advances the device schedule (one CTA)
            self.plan.step_packed(0, 0, self.accum.data_ptr(), 0, 0, args, -1, self._stream(stream))
            self.launches += 1
            return self._scheduled_after()
        if applied:
            for p, o in zip(self.params, self.plan.offsets):     # a caller that dropped the views broke the contract
                # (a zero-element view reports data_ptr() 0 wherever it points: there is nothing it could alias)
                if p.grad is None or (p.numel() > 0 and p.grad.data_ptr() != self.accum.data_ptr() + 4 * o):
                    raise RuntimeError("p.grad no longer aliases the packed accumulator (zero_grad(set_to_none=True)?)")
            if sched:
                self.plan.step_packed(0, self.param_slab.data_ptr(), self.accum.data_ptr(), self.m.data_ptr(),
                                      self.v.data_ptr(), args, -1, self._stream(stream))
                self.launches += 1
                return self._scheduled_after()
            lr = self.lr_fn(g)
            self.plan.step_packed(0, self.param_slab.data_ptr(), self.accum.data_ptr(), self.m.data_ptr(), self.v.data_ptr(),
                                  self._step_args(g, lr), 1, self._stream(stream))
            self.launches += 1
            self._advance_beta_powers()
        self.global_step = g + 1
        return applied


class HostTrainOp(_TrainOpCore):
    """The train_op for a caller whose parameters and gradients live in HOST memory (the reference's
    CPU placement, distributedExample/02 "1 worker CPU").  A thin state holder over the C ABI's
    ``gaccum_host_session``: gradients go H2D every micro-step (double-buffered), the kernel runs,
    updated parameters come back D2H on apply steps, the 16-byte stats block every step.
    ``host_params`` are updated in place; pin them (and the gradients) for asynchronous copies."""

    @staticmethod
    def pinned_arena(shapes: Sequence[Sequence[int]], hp: HParams):
        """One pinned host buffer laid out like the device slabs (plan offsets, 128-byte aligned tensors) and the
        per-tensor views into it.  Gradients / parameters kept in such an arena cross PCIe with ONE copy per
        direction (gaccum_step_host coalesces tensors whose host spacing equals their slab spacing)."""
        numels = [int(np.prod(s)) for s in shapes]
        layout = Plan(numels, None, hp, device=-1)
        flat = _pinned_zeros(max(layout.padded_size, 32))
        views = [flat[o:o + n].view(tuple(s)) for o, n, s in zip(layout.offsets, numels, shapes)]
        return flat, views

    def connect_data_parallel(self, process_group=None) -> None:
        """04's MultiWorkerMirroredStrategy for host-resident tensors: exchange the sessions' CUDA-IPC records over
        torch.distributed (any transport would do: they are plain bytes) and switch the apply step to the fused
        exchange + apply kernel.  Every rank must hold identical parameters and step in lock-step."""
        import torch.distributed as dist
        world, rank = dist.get_world_size(process_group), dist.get_rank(process_group)
        if world < 2:
            return
        mine = self.session.dp_export(world)
        records = [None] * world
        dist.all_gather_object(records, mine, group=process_group)
        self.session.dp_connect(rank, world, records)
        dist.barrier(group=process_group)
        self.world = world

    def __init__(self, host_params: Sequence[torch.Tensor], names: Sequence[str], hp: HParams, accum_n: int,
                 lr_fn: Callable[[int], float],
                 exclude_from_weight_decay: Optional[Sequence[str]] = ("LayerNorm", "layer_norm", "bias"),
                 global_step: int = 0, device: int = 0, loss_scale: Optional[LossScaleConfig] = None,
                 ema: Optional[EmaConfig] = None, lr_multipliers: Optional[Sequence[float]] = None,
                 window_weight: bool = False, device_schedule: Optional[ScheduleConfig] = None,
                 tensor_norms: bool = False):
        if tensor_norms:
            raise ValueError("HostTrainOp does not report per-tensor norms; use GaccumTrainOp")
        if device_schedule is not None:
            raise ValueError("HostTrainOp does not support a device schedule; use GaccumTrainOp")
        if ema is not None:
            raise ValueError("HostTrainOp does not keep a moving average of the weights; use GaccumTrainOp")
        if window_weight:
            raise ValueError("HostTrainOp does not support a window weight; use GaccumTrainOp")
        if lr_multipliers is not None:
            raise ValueError("HostTrainOp does not support per-tensor learning-rate multipliers; use GaccumTrainOp")
        if loss_scale is not None:   # host-resident models have no fp16 autocast: nothing to loss-scale
            raise ValueError("HostTrainOp does not support loss scaling")
        if hp.variant == LAMB:
            raise ValueError("HostTrainOp does not support LAMB; use GaccumTrainOp")
        _refuse_half(host_params, "HostTrainOp")
        self.world = 1
        for p in host_params:
            if p.device.type != "cpu" or p.dtype != torch.float32 or not p.is_contiguous():
                raise ValueError("host_params must be contiguous fp32 CPU tensors")
        super().__init__(host_params, names, hp, accum_n, lr_fn, exclude_from_weight_decay, global_step, device)
        self.session = _lib.HostSession(self.plan)
        self._param_ptrs = Plan.ptr_array([p.data_ptr() for p in self.params])
        self.session.set_params(self._param_ptrs)

    def bind(self, host_grads: Sequence[Optional[torch.Tensor]]):
        for g, p in zip(host_grads, self.params):
            if g is not None and (g.device.type != "cpu" or g.dtype != torch.float32 or not g.is_contiguous() or g.numel() != p.numel()):
                raise ValueError("host gradients must be contiguous fp32 CPU tensors shaped like their parameter")
        return Plan.ptr_array([0 if g is None else g.data_ptr() for g in host_grads])

    def run(self, host_grads: Sequence[Optional[torch.Tensor]]) -> bool:
        return self.run_bound(self.bind(host_grads))

    def run_bound(self, grad_ptrs) -> bool:
        g = self.global_step
        lr = self.lr_fn(g)
        self.session.step(grad_ptrs, self._param_ptrs, self._step_args(g, lr), self._stats_host.data_ptr())
        applied = _lib.is_apply_step(g, self.N)
        if applied:
            self._advance_beta_powers()
        self.global_step = g + 1
        return applied

    def sync(self) -> None:
        self.session.sync()

    def stats(self) -> Dict[str, float]:
        self.sync()
        return _stats_dict(self._stats_host)
