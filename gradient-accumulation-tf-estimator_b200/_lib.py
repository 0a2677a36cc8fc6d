"""ctypes binding of include/gaccum.h -- the only way Python reaches the kernels."""
from __future__ import annotations

import ctypes as C
import math
import os
import re
from typing import List, Optional, Sequence

from . import build as _build

ADAM_WEIGHT_DECAY = 0   # reference optimization.py:107-194
ADAM = 1                # tf.train.AdamOptimizer (02:41, 04:42, another-example.py:135)
LAMB = 2                # LAMB (You et al. 2019), TF-Addons' form with AdamWeightDecay's op order (gaccum.h)

OK, EINVAL, ENODEVICE, ECUDA, ENCCL, ENOMEM = 0, -1, -2, -3, -4, -5

DTYPE_F32, DTYPE_BF16, DTYPE_F16 = 0, 1, 2   # element type of the model's weights and gradients


class GaccumError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libgaccum error {code}: {msg}")
        self.code = code


class HParams(C.Structure):
    """gaccum_hparams; defaults = what create_optimizer hard-codes (optimization.py:59-65, 84)."""
    _fields_ = [("variant", C.c_int32), ("reserved", C.c_int32), ("beta1", C.c_double),
                ("beta2", C.c_double), ("epsilon", C.c_double), ("weight_decay_rate", C.c_double),
                ("clip_norm", C.c_double)]

    @classmethod
    def bert(cls) -> "HParams":
        return cls(ADAM_WEIGHT_DECAY, 0, 0.9, 0.999, 1e-6, 0.01, 1.0)

    @classmethod
    def lamb(cls, beta1=0.9, beta2=0.999, epsilon=1e-6, weight_decay_rate=0.01, clip_norm=1.0) -> "HParams":
        return cls(LAMB, 0, beta1, beta2, epsilon, weight_decay_rate, clip_norm)

    @classmethod
    def tf_adam(cls, beta1=0.9, beta2=0.999, epsilon=1e-8) -> "HParams":
        return cls(ADAM, 0, beta1, beta2, epsilon, 0.0, 0.0)


class StepArgs(C.Structure):
    _fields_ = [("global_step", C.c_int64), ("accum_n", C.c_int32), ("reserved", C.c_int32),
                ("lr", C.c_float), ("beta1_power", C.c_float), ("beta2_power", C.c_float),
                ("reserved2", C.c_float)]


MAX_RANKS = 8
DP_CTRL_BYTES = 256


class DpComm(C.Structure):
    """gaccum_dp_comm: the local accumulator slab + peer base pointers for the fused data-parallel apply."""
    _fields_ = [("rank", C.c_int32), ("world", C.c_int32), ("accum", C.c_void_p),
                ("param_peers", C.c_void_p * MAX_RANKS), ("stage_peers", C.c_void_p * MAX_RANKS),
                ("ctrl_peers", C.c_void_p * MAX_RANKS), ("stage_elements", C.c_int64)]


class DpIpc(C.Structure):
    """gaccum_dp_ipc: what one rank's host session exports for the others (plain bytes)."""
    _fields_ = [("param", C.c_ubyte * 64), ("stage", C.c_ubyte * 64), ("ctrl", C.c_ubyte * 64),
                ("stage_elements", C.c_int64), ("padded_size", C.c_int64)]


class Stats(C.Structure):
    _fields_ = [("applied", C.c_float), ("lr", C.c_float), ("global_norm", C.c_float),
                ("clip_scale", C.c_float)]


class LossScaleConfig(C.Structure):
    """gaccum_loss_scale_config: dynamic loss scaling as TF 2's ``DynamicLossScale`` does it, counted in windows
    (defaults are TF 2's).  ``initial_scale`` and ``multiplier`` must be powers of two."""
    _fields_ = [("initial_scale", C.c_double), ("multiplier", C.c_double), ("growth_interval", C.c_int32),
                ("reserved", C.c_int32)]

    def __init__(self, initial_scale: float = 2.0 ** 15, multiplier: float = 2.0, growth_interval: int = 2000,
                 reserved: int = 0):
        super().__init__(float(initial_scale), float(multiplier), int(growth_interval), int(reserved))


class LossScaleState(C.Structure):
    """gaccum_loss_scale_state: the 32-byte device block the apply launches update."""
    _fields_ = [("scale", C.c_float), ("good_windows", C.c_int32), ("skipped_windows", C.c_uint32),
                ("last_skipped", C.c_int32), ("beta1_power", C.c_float), ("beta2_power", C.c_float),
                ("reserved", C.c_float * 2)]


class EmaConfig(C.Structure):
    """gaccum_ema_config: an exponential moving average of the weights, updated by the apply step once per applied
    window (TF1 ``ExponentialMovingAverage(decay, num_updates=...)``, ``zero_debias=False``).  ``num_updates=True``
    turns on TF's warm-up ``d = min(decay, (1 + n) / (10 + n))``, n counting the windows averaged so far."""
    _fields_ = [("decay", C.c_double), ("num_updates", C.c_int32), ("reserved", C.c_int32)]

    def __init__(self, decay: float = 0.9999, num_updates: bool = False, reserved: int = 0):
        super().__init__(float(decay), int(num_updates), int(reserved))


class ScheduleConfig(C.Structure):
    """gaccum_schedule_config: create_optimizer's learning-rate schedule (optimization.py:29-52), evaluated on the device
    by every launch of a device-scheduled plan (``end_lr`` 0 and ``power`` 1 are the only values it takes)."""
    _fields_ = [("init_lr", C.c_double), ("num_train_steps", C.c_int64), ("num_warmup_steps", C.c_int64),
                ("end_lr", C.c_double), ("power", C.c_double)]

    def __init__(self, init_lr: float, num_train_steps: int, num_warmup_steps: Optional[int] = 0,
                 end_lr: float = 0.0, power: float = 1.0):
        super().__init__(float(init_lr), int(num_train_steps), int(num_warmup_steps or 0), float(end_lr), float(power))


class ScheduleState(C.Structure):
    """gaccum_schedule_state: the 48-byte device block of a device-scheduled plan."""
    _fields_ = [("global_step", C.c_int64), ("num_train_steps", C.c_int64), ("num_warmup_steps", C.c_int64),
                ("init_lr", C.c_float), ("end_lr", C.c_float), ("power", C.c_float), ("beta1_power", C.c_float),
                ("beta2_power", C.c_float), ("refused", C.c_int32)]


_lib = None


def lib_path() -> str:
    _load()                 # make sure it exists (built on demand) before anyone dlopens the path
    return _build.LIB


def _load():
    global _lib
    if _lib is not None:
        return _lib
    override = os.environ.get("GACCUM_LIB")    # measurement builds (build.build_variant), never a fallback
    if override:
        if not os.path.exists(override):
            raise ImportError(f"GACCUM_LIB={override} does not exist")
        _build.LIB = override
    try:
        path = override or _build.build_libgaccum()
    except Exception as e:  # no nvcc and no prebuilt library: fail loudly, never fall back
        if not os.path.exists(_build.LIB):
            raise ImportError(f"libgaccum.so is missing and cannot be built ({e}); "
                              "there is no CPU/PyTorch fallback for the train_op") from e
        path = _build.LIB
    L = C.CDLL(path)
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    sig = {
        "gaccum_version": (C.c_int, []),
        "gaccum_last_error": (C.c_char_p, []),
        "gaccum_device_count": (C.c_int, []),
        "gaccum_learning_rate": (C.c_float, [C.c_double, i64, i64, i64]),
        "gaccum_is_apply_step": (C.c_int, [i64, i32]),
        "gaccum_decay_mask": (C.c_int, [i32, vp, C.c_double, vp, i32, vp]),
        "gaccum_plan_create": (C.c_int, [C.POINTER(vp), i32, vp, vp, C.POINTER(HParams), i32]),
        "gaccum_plan_destroy": (C.c_int, [vp]),
        "gaccum_padded_size": (i64, [vp]),
        "gaccum_offsets": (C.c_int, [vp, vp]),
        "gaccum_num_tensors": (i32, [vp]),
        "gaccum_num_elements": (i64, [vp]),
        "gaccum_num_tiles": (i32, [vp]),
        "gaccum_algorithmic_bytes": (i64, [vp, i32]),
        "gaccum_step": (C.c_int, [vp, vp, vp, vp, vp, vp, C.POINTER(StepArgs), vp]),
        "gaccum_accumulate": (C.c_int, [vp, vp, vp, vp]),
        "gaccum_apply": (C.c_int, [vp, vp, vp, vp, vp, vp, C.POINTER(StepArgs), vp]),
        "gaccum_step_packed": (C.c_int, [vp, vp, vp, vp, vp, vp, C.POINTER(StepArgs), i32, vp]),
        "gaccum_read_stats": (C.c_int, [vp, vp, vp]),
        "gaccum_host_session_create": (C.c_int, [C.POINTER(vp), vp]),
        "gaccum_host_session_destroy": (C.c_int, [vp]),
        "gaccum_host_session_set_params": (C.c_int, [vp, vp]),
        "gaccum_step_host": (C.c_int, [vp, vp, vp, C.POINTER(StepArgs), vp]),
        "gaccum_host_session_sync": (C.c_int, [vp]),
        "gaccum_host_session_slabs": (C.c_int, [vp, vp]),
        "gaccum_host_session_dp_export": (C.c_int, [vp, i32, C.POINTER(DpIpc)]),
        "gaccum_host_session_dp_connect": (C.c_int, [vp, i32, i32, C.POINTER(DpIpc)]),
        "gaccum_dp_shard_range": (C.c_int, [vp, i32, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i64)]),
        "gaccum_dp_stage_elements": (i64, [vp, i32]),
        "gaccum_apply_dp": (C.c_int, [vp, C.POINTER(DpComm), vp, vp, vp, C.POINTER(StepArgs), C.c_uint32, vp]),
        "gaccum_step_dp": (C.c_int, [vp, C.POINTER(DpComm), vp, vp, vp, C.POINTER(StepArgs), C.c_uint32, vp]),
        "gaccum_plan_set_loss_scale": (C.c_int, [vp, C.POINTER(LossScaleConfig), vp]),
        "gaccum_loss_scale_init": (C.c_int, [vp, vp, vp]),
        "gaccum_plan_set_param_dtype": (C.c_int, [vp, i32, vp]),
        "gaccum_plan_set_layer_adaptation": (C.c_int, [vp, vp]),
        "gaccum_read_trust_ratios": (C.c_int, [vp, vp, vp]),
        "gaccum_plan_set_ema": (C.c_int, [vp, C.POINTER(EmaConfig), vp, vp]),
        "gaccum_ema_init": (C.c_int, [vp, vp, i64, vp]),
        "gaccum_plan_set_lr_multipliers": (C.c_int, [vp, vp]),
        "gaccum_plan_set_window_weight": (C.c_int, [vp, vp]),
        "gaccum_plan_set_device_schedule": (C.c_int, [vp, C.POINTER(ScheduleConfig), vp]),
        "gaccum_schedule_init": (C.c_int, [vp, vp, i64, C.c_float, C.c_float, vp]),
        "gaccum_plan_set_tensor_norms": (C.c_int, [vp, vp]),
        "gaccum_plan_set_lr_table": (C.c_int, [vp, vp, i64]),
        "gaccum_plan_set_deferred_reset": (C.c_int, [vp, i32]),
        "gaccum_accum_materialize": (C.c_int, [vp, vp, vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    _lib = L
    return L


def _check(rc: int) -> None:
    if rc != 0:
        raise GaccumError(rc, (_load().gaccum_last_error() or b"").decode())


def version() -> int:
    return _load().gaccum_version()


def device_count() -> int:
    return _load().gaccum_device_count()


def learning_rate(init_lr: float, num_train_steps: int, num_warmup_steps: Optional[int], global_step: int) -> float:
    """optimization.py:29-54 in fp32 (host)."""
    return float(_load().gaccum_learning_rate(float(init_lr), int(num_train_steps),
                                              int(num_warmup_steps or 0), int(global_step)))


def is_apply_step(global_step: int, accum_n: int) -> bool:
    """optimization.py:77,91: the step is cast to int32 (two's-complement wraparound) before the modulo.  The same
    decision as ``gaccum_is_apply_step`` without a foreign call, so every Python front end can take it per
    micro-step.  Divisibility does not depend on whether ``%`` truncates (C) or floors (Python)."""
    step32 = (int(global_step) + 0x80000000) % 0x100000000 - 0x80000000
    return accum_n > 0 and step32 % accum_n == 0


def is_first_accumulate(global_step: int, accum_n: int) -> bool:
    """The first accumulate of a window, which gaccum_step runs without reading the accumulators (gaccum_abi.cu
    first_of_window): the step does not apply and the one before it did, both by the int32 predicate."""
    return not is_apply_step(global_step, accum_n) and is_apply_step(int(global_step) - 1, accum_n)


def _c_strs(strs: Sequence[str]):
    arr = (C.c_char_p * len(strs))()
    arr[:] = [s.encode() for s in strs]
    return arr


def _variable_name(name: str) -> str:
    """optimization.py:189-194 (``_get_variable_name``): a trailing ``:<digits>`` is stripped."""
    m = re.match("^(.*):\\d+$", name)
    return name if m is None else m.group(1)


def _use_weight_decay(name: str, weight_decay_rate: float, exclude: Optional[Sequence[str]]) -> bool:
    """optimization.py:179-187 (``_do_use_weight_decay``)."""
    if not weight_decay_rate:
        return False
    return not any(re.search(r, name) is not None for r in exclude or ())


def decay_mask(names: Sequence[str], weight_decay_rate: float,
               exclude: Optional[Sequence[str]] = ("LayerNorm", "layer_norm", "bias")) -> List[bool]:
    """optimization.py:179-194, with the reference's own regular-expression engine: Python ``re.search`` on the
    name with a trailing ``:<digits>`` stripped.  (The C helper ``gaccum_decay_mask`` is for non-Python callers and
    speaks POSIX ERE: identical for the reference's plain substrings, different for Python-only syntax such as
    ``\\d`` or look-arounds -- both Python bindings therefore evaluate the patterns here.)"""
    return [_use_weight_decay(_variable_name(n), weight_decay_rate, exclude) for n in names]


def adaptation_mask(names: Sequence[str], exclude: Optional[Sequence[str]]) -> List[bool]:
    """LAMB's layer-adaptation mask (TF-Addons ``_do_layer_adaptation``): tensor i adapts unless a pattern of ``exclude``
    is found (Python ``re.search``) in its name with a trailing ``:<digits>`` stripped.  Unlike the decay mask it does not
    depend on the weight-decay rate."""
    return [not any(re.search(r, _variable_name(n)) is not None for r in exclude or ()) for n in names]


def lr_multiplier_array(mult: Sequence[float], num_tensors: int):
    """The T per-tensor learning-rate multipliers as the kernels see them: an np.float32 array, each value rounded to
    fp32 once.  ValueError for the wrong length, or a value that is negative, not finite, or overflows fp32."""
    import numpy as np
    vals = [float(x) for x in mult]
    if len(vals) != num_tensors:
        raise ValueError(f"{len(vals)} learning-rate multipliers for {num_tensors} tensors")
    with np.errstate(over="ignore"):
        out = np.array(vals, dtype=np.float64).astype(np.float32)
    for i, (x, x32) in enumerate(zip(vals, out)):
        if not (math.isfinite(x) and x >= 0.0 and np.isfinite(x32)):
            raise ValueError(f"learning-rate multiplier {i} is {x!r}: it must be finite and >= 0, and fit fp32")
    return out


def decay_mask_c(names: Sequence[str], weight_decay_rate: float,
                 exclude: Optional[Sequence[str]] = ("LayerNorm", "layer_norm", "bias")) -> List[bool]:
    """The C ABI's ``gaccum_decay_mask`` (POSIX extended regular expressions)."""
    exclude = list(exclude or [])
    out = (C.c_uint8 * len(names))()
    n, e = _c_strs(names), _c_strs(exclude)
    _check(_load().gaccum_decay_mask(len(names), C.cast(n, C.c_void_p), float(weight_decay_rate),
                                     C.cast(e, C.c_void_p), len(exclude), C.cast(out, C.c_void_p)))
    return [bool(x) for x in out]


class Plan:
    """gaccum_plan: slab layout + tile table for T tensors.  device=-1 -> layout-only."""

    def __init__(self, numels: Sequence[int], decay: Optional[Sequence[bool]], hp: HParams, device: int = -1):
        L = _load()
        self.T = len(numels)
        self.hp = hp
        self.device = device
        ne = (C.c_int64 * self.T)(*[int(n) for n in numels])
        dm = (C.c_uint8 * self.T)(*[1 if d else 0 for d in (decay or [0] * self.T)])
        h = C.c_void_p()
        _check(L.gaccum_plan_create(C.byref(h), self.T, C.cast(ne, C.c_void_p), C.cast(dm, C.c_void_p),
                                    C.byref(hp), int(device)))
        self._h = h
        self.numels = [int(n) for n in numels]
        self.padded_size = int(L.gaccum_padded_size(h))
        self.num_elements = int(L.gaccum_num_elements(h))
        self.num_tiles = int(L.gaccum_num_tiles(h))
        off = (C.c_int64 * self.T)()
        _check(L.gaccum_offsets(h, C.cast(off, C.c_void_p)))
        self.offsets = [int(x) for x in off]

    def algorithmic_bytes(self, is_apply: bool) -> int:
        return int(_load().gaccum_algorithmic_bytes(self._h, 1 if is_apply else 0))

    @staticmethod
    def ptr_array(ptrs: Sequence[int]):
        return (C.c_void_p * len(ptrs))(*[p if p else None for p in ptrs])

    def step(self, grads, params, accum: int, m: int, v: int, args: StepArgs, stream: int = 0) -> None:
        _check(_load().gaccum_step(self._h, grads, params, accum, m, v, C.byref(args), stream))

    def accumulate(self, grads, accum: int, stream: int = 0) -> None:
        _check(_load().gaccum_accumulate(self._h, grads, accum, stream))

    def apply(self, grads, params, accum: int, m: int, v: int, args: StepArgs, stream: int = 0) -> None:
        _check(_load().gaccum_apply(self._h, grads, params, accum, m, v, C.byref(args), stream))

    def step_packed(self, grad_slab: int, param_slab: int, accum: int, m: int, v: int, args: StepArgs,
                    force_branch: int = -1, stream: int = 0) -> None:
        _check(_load().gaccum_step_packed(self._h, grad_slab or None, param_slab or None, accum, m, v,
                                          C.byref(args), force_branch, stream))

    def dp_shard_range(self, world: int, rank: int):
        lo, hi, n = C.c_int32(), C.c_int32(), C.c_int64()
        _check(_load().gaccum_dp_shard_range(self._h, world, rank, C.byref(lo), C.byref(hi), C.byref(n)))
        return lo.value, hi.value, n.value

    def dp_stage_elements(self, world: int) -> int:
        n = int(_load().gaccum_dp_stage_elements(self._h, world))
        if n < 0:
            _check(n)
        return n

    def apply_dp(self, comm: "DpComm", grads, m: int, v: int, args: StepArgs, epoch: int, stream: int = 0) -> None:
        _check(_load().gaccum_apply_dp(self._h, C.byref(comm), grads, m, v, C.byref(args), epoch, stream))

    def step_dp(self, comm: "DpComm", grads, m: int, v: int, args: StepArgs, epoch: int, stream: int = 0) -> None:
        _check(_load().gaccum_step_dp(self._h, C.byref(comm), grads, m, v, C.byref(args), epoch, stream))

    def read_stats(self, host_ptr: int, stream: int = 0) -> None:
        _check(_load().gaccum_read_stats(self._h, host_ptr, stream))

    def set_deferred_reset(self, on: bool) -> None:
        """Applies leave the accumulators logically zero instead of storing zeros (gaccum_plan_set_deferred_reset);
        whatever reads or writes the slab outside a window's first accumulate calls ``accum_materialize`` first."""
        _check(_load().gaccum_plan_set_deferred_reset(self._h, 1 if on else 0))

    def accum_materialize(self, accum: int, stream: int = 0) -> None:
        """Store the zeros a deferred-reset apply left logical, if it did (asynchronous on ``stream``)."""
        _check(_load().gaccum_accum_materialize(self._h, accum, stream))

    def set_loss_scale(self, cfg: LossScaleConfig, device_state: int) -> None:
        """Turn dynamic loss scaling on (before the first compute call); ``device_state`` points to 32 bytes of
        device memory that ``loss_scale_init`` fills."""
        _check(_load().gaccum_plan_set_loss_scale(self._h, C.byref(cfg), device_state or None))

    def loss_scale_init(self, device_state: int, stream: int = 0) -> None:
        _check(_load().gaccum_loss_scale_init(self._h, device_state or None, stream))

    def set_param_dtype(self, dtype: int, master_slab: int) -> None:
        """Train a bf16 / fp16 model (DTYPE_BF16 / DTYPE_F16) with fp32 master weights (before the first compute
        call); ``master_slab`` points to ``padded_size`` floats of device memory in the plan's layout, 16-byte
        aligned.  The step calls then take 16-bit gradient and parameter pointers."""
        _check(_load().gaccum_plan_set_param_dtype(self._h, int(dtype), master_slab or None))

    def set_layer_adaptation(self, adapt: Sequence[bool]) -> None:
        """LAMB: which tensors are scaled by their trust ratio (before the first compute call; default all)."""
        if len(adapt) != self.T:
            raise ValueError(f"the adaptation mask has {len(adapt)} entries, the plan {self.T} tensors")
        arr = (C.c_uint8 * max(self.T, 1))(*[1 if a else 0 for a in adapt])
        _check(_load().gaccum_plan_set_layer_adaptation(self._h, C.cast(arr, C.c_void_p)))

    def read_trust_ratios(self, host_ptr: int, stream: int = 0) -> None:
        """LAMB: copy the last applied window's T trust ratios (fp32) to ``host_ptr``, asynchronously on ``stream``."""
        _check(_load().gaccum_read_trust_ratios(self._h, host_ptr or None, stream))

    def set_ema(self, cfg: EmaConfig, ema_slab: int, device_state: int) -> None:
        """Keep an exponential moving average of the weights (before the first compute call): ``ema_slab`` points to
        ``padded_size`` floats of device memory in the plan's layout holding the initial averages, ``device_state`` to
        16 bytes of device memory that ``ema_init`` fills."""
        _check(_load().gaccum_plan_set_ema(self._h, C.byref(cfg), ema_slab or None, device_state or None))

    def ema_init(self, device_state: int, num_updates: int = 0, stream: int = 0) -> None:
        _check(_load().gaccum_ema_init(self._h, device_state or None, int(num_updates), stream))

    def set_lr_multipliers(self, mult: Sequence[float]) -> None:
        """Tensor t trains with lr_t = fp32(lr * mult[t]) (before the first compute call; default 1.0 everywhere)."""
        m32 = lr_multiplier_array(mult, self.T)
        arr = (C.c_float * max(self.T, 1))(*m32.tolist())
        _check(_load().gaccum_plan_set_lr_multipliers(self._h, C.cast(arr, C.c_void_p)))

    def set_window_weight(self, device_state: int) -> None:
        """Divide each window by the producer's total weight W instead of N (before the first compute call):
        ``device_state`` points to the 16-byte gaccum_window_weight_state in device memory, zeroed to start."""
        _check(_load().gaccum_plan_set_window_weight(self._h, device_state or None))

    def set_device_schedule(self, cfg: ScheduleConfig, block: int) -> None:
        """Keep global_step, the learning rate and the beta powers on the device (before the first compute call):
        ``block`` points to the 48-byte gaccum_schedule_state in device memory that ``schedule_init`` fills."""
        _check(_load().gaccum_plan_set_device_schedule(self._h, C.byref(cfg), block or None))

    def schedule_init(self, block: int, global_step: int, beta1_power: float, beta2_power: float,
                      stream: int = 0) -> None:
        _check(_load().gaccum_schedule_init(self._h, block or None, int(global_step), float(beta1_power),
                                            float(beta2_power), stream))

    def set_lr_table(self, ptr: int, length: int) -> None:
        """Take every launch's learning rate from ``length`` fp32 values of device memory at ``ptr`` (4-byte aligned):
        lr = table[min(global_step, length - 1)] in place of the device schedule's formula (before the first compute
        call; the plan must be device-scheduled by then).  The table is read at launch time."""
        _check(_load().gaccum_plan_set_lr_table(self._h, ptr or None, int(length)))

    def set_tensor_norms(self, device_out: int) -> None:
        """Write per-tensor gradient, weight and update norms on every apply (before the first compute call):
        ``device_out`` points to 3 x T floats of 16-byte aligned device memory, row t = (gradient, weight, update)."""
        _check(_load().gaccum_plan_set_tensor_norms(self._h, device_out or None))

    def close(self) -> None:
        if getattr(self, "_h", None):
            _load().gaccum_plan_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class HostSession:
    """gaccum_host_session: the train_op for a caller whose tensors live in host memory."""

    def __init__(self, plan: Plan):
        self.plan = plan
        h = C.c_void_p()
        _check(_load().gaccum_host_session_create(C.byref(h), plan._h))
        self._h = h

    def set_params(self, host_ptrs) -> None:
        _check(_load().gaccum_host_session_set_params(self._h, host_ptrs))

    def step(self, host_grad_ptrs, host_param_out_ptrs, args: StepArgs, stats_ptr: int = 0) -> None:
        _check(_load().gaccum_step_host(self._h, host_grad_ptrs, host_param_out_ptrs, C.byref(args), stats_ptr or None))

    def sync(self) -> None:
        _check(_load().gaccum_host_session_sync(self._h))

    def dp_export(self, world: int) -> bytes:
        rec = DpIpc()
        _check(_load().gaccum_host_session_dp_export(self._h, world, C.byref(rec)))
        return bytes(rec)

    def dp_connect(self, rank: int, world: int, records: Sequence[bytes]) -> None:
        arr = (DpIpc * world)()
        for w, r in enumerate(records):
            C.memmove(C.byref(arr[w]), r, C.sizeof(DpIpc))
        _check(_load().gaccum_host_session_dp_connect(self._h, rank, world, arr))

    def slabs(self):
        out = (C.c_void_p * 4)()
        _check(_load().gaccum_host_session_slabs(self._h, out))
        return [int(x) for x in out]

    def close(self) -> None:
        if getattr(self, "_h", None):
            _load().gaccum_host_session_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
