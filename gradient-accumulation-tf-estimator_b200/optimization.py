"""Drop-in host mirror of the reference's ``optimization.py`` (same names, same arguments).

    train_op = create_optimizer(loss, init_lr, num_train_steps, num_warmup_steps, use_tpu)

keeps the reference signature (optimization.py:25).  Where the reference builds a ``tf.cond`` over
``assign_add`` / ``clip_by_global_norm`` / ``AdamWeightDecayOptimizer.apply_gradients`` and returns
a ``tf.Operation``, this returns a :class:`TrainOp` whose ``run()`` is one ``session.run(train_op)``:
forward + backward of ``loss`` (PyTorch autograd -- not our path) followed by exactly ONE launch of
the sm_90a kernel behind ``include/gaccum.h``.  State (accumulators, adam_m, adam_v, global_step)
lives where the reference keeps it: in variables owned by the graph, here packed HBM slabs.

``loss`` is the symbolic loss of graph mode: a zero-argument callable that evaluates the loss on
the next micro-batch (or an already-evaluated scalar tensor for a single run).
Trainable variables and the global step come from :mod:`graph` collections, as
``tf.trainable_variables()`` / ``tf.train.get_or_create_global_step()`` do (optimization.py:27,70).

There is no CPU fallback: variables must be CUDA tensors.
"""
from __future__ import annotations

import os
import re
from typing import Callable, Dict, Iterable, List, Optional, Sequence, Tuple, Union

import torch

from . import _lib, graph, schedules
from ._lib import ADAM, ADAM_WEIGHT_DECAY, LAMB, EmaConfig, HParams, LossScaleConfig
from .train_op import GaccumTrainOp

# optimization.py:76 hard-codes 8 (README.md:17,34 says 4).  The signature has no argument for
# it, so it is a module attribute (and GACCUM_MULTIPLIER in the environment) -- default as shipped.
gradient_accumulation_multiplier = int(os.environ.get("GACCUM_MULTIPLIER", "8"))
clip_norm = 1.0   # optimization.py:84
# Dynamic loss scaling for fp16 mixed precision (a LossScaleConfig), off by default; create_optimizer reads it.
loss_scale: Optional[LossScaleConfig] = None
# The optimizer create_optimizer builds: "adam" (the reference's AdamWeightDecayOptimizer) or "lamb" (LAMBOptimizer with
# the same hyper-parameters and exclusions, for large effective batches).
optimizer_type = "adam"
# The decay of an exponential moving average of the weights (ExponentialMovingAverage), off by default; create_optimizer
# reads it.
moving_average_decay: Optional[float] = None
# ELECTRA's layer-wise learning-rate decay (layerwise_lr_multipliers), off by default; create_optimizer reads it and takes
# the number of encoder layers from the trainable variables' names.
layerwise_lr_decay: Optional[float] = None
# Divide each window by its total weight (typically its number of loss tokens) instead of N: the loss callable returns
# (summed loss, weight).  Off by default; create_optimizer reads it.
window_weight = False
# Report per-tensor gradient, weight and update norms from every apply step (``train_op.tensor_norms()``).  Off by
# default; create_optimizer reads it.
tensor_norms = False
# NVIDIA BERT's polynomial decay of the learning rate after warm-up (``polynomial_decay(power=poly_power,
# end_learning_rate=end_learning_rate)``; its LAMB recipe uses poly_power = 0.5).  The defaults are the reference's
# linear decay to 0; create_optimizer reads them.
poly_power = 1.0
end_learning_rate = 0.0

LossLike = Union[torch.Tensor, Callable[[], torch.Tensor]]
LrLike = Union[float, Callable[[int], float]]


def _lr_callable(lr: LrLike) -> Callable[[int], float]:
    return lr if callable(lr) else (lambda step, _v=float(lr): _v)


def layerwise_lr_multipliers(layer_decay: float, num_layers: int) -> Dict[str, float]:
    """ELECTRA's layer-wise learning-rate decay (``_get_layer_lrs``) as multipliers of the scheduled lr, keyed by
    variable-name substring: the embeddings get ``layer_decay ** (L + 2)``, encoder layer i ``layer_decay ** (L + 1 - i)``
    and the task head (``task_specific/``) 1.  The powers are Python doubles; each is rounded to fp32 once, as TF
    converts the constant it multiplies the learning rate by."""
    L = int(num_layers)
    depths = {"/embeddings/": 0, "/embeddings_project/": 0, "task_specific/": L + 2}
    for i in range(L):
        depths[f"encoder/layer_{i}/"] = i + 1
    return {key: float(layer_decay) ** (L + 2 - depth) for key, depth in depths.items()}


def lr_multipliers_for(names: Sequence[str], multipliers: Optional[Dict[str, float]]) -> Optional[List[float]]:
    """The per-tensor list of ``multipliers`` (ELECTRA's key -> rate dict, as multipliers of the scheduled lr): each
    variable takes the multiplier of the key that is a substring of its name.  Two deliberate departures from ELECTRA:
    a variable that matches no key trains at the scheduled lr (1.0) -- ELECTRA raises, so BERT's pooler and
    ``output_weights`` would each need a key -- and a variable that matches two keys raises ValueError -- ELECTRA would
    silently update it once per key.  None stays None: the train op then keeps a single learning rate."""
    if multipliers is None:
        return None
    out = []
    for name in names:
        keys = [k for k in multipliers if k in name]
        if len(keys) > 1:
            raise ValueError(f"variable {name!r} matches more than one learning-rate key: {keys}")
        out.append(float(multipliers[keys[0]]) if keys else 1.0)
    return out


def _num_encoder_layers(names: Sequence[str]) -> int:
    """1 + the largest i of an ``encoder/layer_<i>/`` in the names."""
    layers = [int(m.group(1)) for n in names for m in [re.search(r"encoder/layer_(\d+)/", n)] if m is not None]
    if not layers:
        raise ValueError("layerwise_lr_decay is set, but no trainable variable is named like encoder/layer_<i>/")
    return max(layers) + 1


def bert_learning_rate(init_lr: float, num_train_steps: int, num_warmup_steps: Optional[int]) -> Callable[[int], float]:
    """optimization.py:29-54 as a function of the pre-increment global step (fp32 op order)."""
    return lambda step: _lib.learning_rate(init_lr, num_train_steps, num_warmup_steps, step)


class _OptimizerBase:
    """What every optimizer shares: turning (grad, var) pairs into one kernel launch.  ``lr_multipliers`` is ELECTRA's
    per-variable learning-rate dict as multipliers of the scheduled lr (``lr_multipliers_for``): a constructor argument
    of LAMBOptimizer and AdamOptimizer, an attribute to set on AdamWeightDecayOptimizer (whose constructor keeps the
    reference's signature).  It is read when the train op is built."""
    variant = ADAM_WEIGHT_DECAY

    def _hparams(self, clip: float) -> HParams:
        raise NotImplementedError

    def __init__(self, lr_multipliers: Optional[Dict[str, float]] = None):
        self.lr_multipliers = dict(lr_multipliers) if lr_multipliers is not None else None
        self._direct_op: Optional[GaccumTrainOp] = None
        self._direct_key = None

    def apply_gradients(self, grads_and_vars: Iterable[Tuple[Optional[torch.Tensor], graph.Variable]],
                        global_step=None, name=None):
        """Apply one update NOW (the reference's method builds the op; eager here).

        Pairs whose grad or var is None are skipped (optimization.py:132-133).  ``global_step`` is
        accepted and ignored exactly as the reference does (optimization.py:128, comment :99-101).
        Implemented as the apply branch of the train_op with N=1, no clipping and zero accumulators,
        i.e. the same fused kernel."""
        pairs = [(g, v) for g, v in grads_and_vars if g is not None and v is not None]
        if not pairs:
            return None
        vars_ = [v for _, v in pairs]
        key = tuple(id(v) for v in vars_)
        if self._direct_op is None or self._direct_key != key:
            self._direct_op = GaccumTrainOp([v.tensor for v in vars_], [v.name for v in vars_],
                                            self._hparams(0.0), 1, _lr_callable(self.learning_rate),
                                            exclude_from_weight_decay=getattr(self, "exclude_from_weight_decay", None),
                                            exclude_from_layer_adaptation=getattr(self, "exclude_from_layer_adaptation", None),
                                            lr_multipliers=lr_multipliers_for([v.name for v in vars_], self.lr_multipliers))
            self._direct_key = key
        op = self._direct_op
        gs = graph.get_global_step()
        step_for_lr = int(gs) if gs is not None else 0
        saved = op.global_step
        op.global_step = 0                      # N=1: every step applies; lr comes from the graph's step
        op.lr_fn = lambda _s, _f=_lr_callable(self.learning_rate), _g=step_for_lr: _f(_g)
        op.run([g.contiguous() for g, _ in pairs])
        op.global_step = saved
        return op


class AdamWeightDecayOptimizer(_OptimizerBase):
    """optimization.py:107-194: Adam without bias correction + decoupled weight decay."""
    variant = ADAM_WEIGHT_DECAY

    def __init__(self, learning_rate: LrLike, weight_decay_rate=0.0, beta_1=0.9, beta_2=0.999, epsilon=1e-6,
                 exclude_from_weight_decay: Optional[Sequence[str]] = None, name="AdamWeightDecayOptimizer"):
        # the reference's signature: per-variable learning rates are set as the ``lr_multipliers`` attribute
        super().__init__()
        self.learning_rate = learning_rate
        self.weight_decay_rate = weight_decay_rate
        self.beta_1 = beta_1
        self.beta_2 = beta_2
        self.epsilon = epsilon
        self.exclude_from_weight_decay = exclude_from_weight_decay
        self.name = name

    def _hparams(self, clip: float) -> HParams:
        return HParams(ADAM_WEIGHT_DECAY, 0, self.beta_1, self.beta_2, self.epsilon, self.weight_decay_rate, clip)

    def _do_use_weight_decay(self, param_name: str) -> bool:
        """optimization.py:179-187."""
        return _lib._use_weight_decay(param_name, self.weight_decay_rate, self.exclude_from_weight_decay)

    def _get_variable_name(self, param_name: str) -> str:
        """optimization.py:189-194."""
        return _lib._variable_name(param_name)


class LAMBOptimizer(_OptimizerBase):
    """LAMB (You et al. 2019, "Large Batch Optimization for Deep Learning") in TF-Addons' form: bias-corrected Adam
    moments, decoupled weight decay, and each tensor's update scaled by its trust ratio ||p|| / ||u||.
    ``exclude_from_layer_adaptation`` defaults to ``exclude_from_weight_decay``, as in TF-Addons."""
    variant = LAMB

    def __init__(self, learning_rate: LrLike, weight_decay_rate=0.01, beta_1=0.9, beta_2=0.999, epsilon=1e-6,
                 exclude_from_weight_decay: Optional[Sequence[str]] = None,
                 exclude_from_layer_adaptation: Optional[Sequence[str]] = None, name="LAMBOptimizer",
                 lr_multipliers: Optional[Dict[str, float]] = None):
        super().__init__(lr_multipliers)
        self.learning_rate = learning_rate
        self.weight_decay_rate = weight_decay_rate
        self.beta_1 = beta_1
        self.beta_2 = beta_2
        self.epsilon = epsilon
        self.exclude_from_weight_decay = exclude_from_weight_decay
        self.exclude_from_layer_adaptation = exclude_from_layer_adaptation if exclude_from_layer_adaptation is not None \
            else exclude_from_weight_decay
        self.name = name

    def _hparams(self, clip: float) -> HParams:
        return HParams(LAMB, 0, self.beta_1, self.beta_2, self.epsilon, self.weight_decay_rate, clip)

    def _do_use_weight_decay(self, param_name: str) -> bool:
        return _lib._use_weight_decay(param_name, self.weight_decay_rate, self.exclude_from_weight_decay)

    def _do_layer_adaptation(self, param_name: str) -> bool:
        """TF-Addons LAMB._do_layer_adaptation: by name only, whatever the weight-decay rate."""
        return _lib.adaptation_mask([param_name], self.exclude_from_layer_adaptation)[0]

    def _get_variable_name(self, param_name: str) -> str:
        return _lib._variable_name(param_name)


class AdamOptimizer(_OptimizerBase):
    """``tf.train.AdamOptimizer`` as the example scripts use it (02:41, 04:42, another-example.py:135)."""
    variant = ADAM

    def __init__(self, learning_rate: LrLike = 0.001, beta1=0.9, beta2=0.999, epsilon=1e-8, name="Adam",
                 lr_multipliers: Optional[Dict[str, float]] = None):
        super().__init__(lr_multipliers)
        self.learning_rate = learning_rate
        self.beta1, self.beta2, self.epsilon, self.name = beta1, beta2, epsilon, name

    def _hparams(self, clip: float) -> HParams:
        return HParams(ADAM, 0, self.beta1, self.beta2, self.epsilon, 0.0, clip)


class ExponentialMovingAverage:
    """``tf.train.ExponentialMovingAverage(decay, num_updates=...)`` (``zero_debias=False``) for the train op: pass it as
    ``gradient_accumulation_train_op(..., ema=)``.  The TF idiom ``with tf.control_dependencies([train_op]):
    ema.apply(tvars)`` would average on every micro-step; here the apply step averages every trainable variable once per
    applied window, on the device, after the update (the fp32 master weights of a bf16 / fp16 model).  With
    ``num_updates=True`` the decay is TF's ``min(decay, (1 + n) / (10 + n))``, n counting the windows averaged so far."""

    def __init__(self, decay: float, num_updates: bool = False, name: str = "ExponentialMovingAverage"):
        self.decay, self.num_updates, self.name = float(decay), bool(num_updates), name
        self._train_op: Optional["TrainOp"] = None

    def config(self) -> EmaConfig:
        return EmaConfig(self.decay, self.num_updates)

    def average_name(self, var: graph.Variable) -> str:
        return _lib._variable_name(var.name) + "/" + self.name

    def average(self, var: graph.Variable) -> torch.Tensor:
        """The moving average of ``var`` (a view of the train op's device slab)."""
        if self._train_op is None:
            raise ValueError("this ExponentialMovingAverage is not attached to a train op")
        ids = [id(v) for v in self._train_op.tvars]
        if id(var) not in ids:
            raise KeyError(f"{var.name} is not averaged")
        return self._train_op.engine.ema_view(ids.index(id(var)))

    def variables_to_restore(self):
        """{shadow-variable name: variable}: what a Saver restoring the averages into the variables maps (TF's
        evaluation idiom); ``TrainOp.engine.averaged_weights()`` does the same swap in place."""
        tv = self._train_op.tvars if self._train_op is not None else graph.trainable_variables()
        return {self.average_name(v): v for v in tv}


class TrainOp:
    """The object ``create_optimizer`` returns; ``run()`` == ``session.run(train_op)``."""

    def __init__(self, loss: LossLike, tvars: Sequence[graph.Variable], optimizer: _OptimizerBase,
                 accum_n: int, clip: Optional[float], global_step: graph.GlobalStep, process_group=None,
                 dp_mode: str = "fused", loss_scale: Optional[LossScaleConfig] = None,
                 ema: Optional[ExponentialMovingAverage] = None, window_weight: bool = False,
                 tensor_norms: bool = False):
        self.loss = loss
        self.window_weight = bool(window_weight)
        self.tvars = list(tvars)
        self.optimizer = optimizer
        self.global_step = global_step
        tensors, names = [v.tensor for v in self.tvars], [v.name for v in self.tvars]
        hp = optimizer._hparams(clip or 0.0)
        lr_fn = _lr_callable(optimizer.learning_rate)
        exclude = getattr(optimizer, "exclude_from_weight_decay", None)
        adapt_kw = {"exclude_from_layer_adaptation": getattr(optimizer, "exclude_from_layer_adaptation", None)} \
            if hp.variant == LAMB else {}
        self.ema = ema
        ema_cfg = ema.config() if ema is not None else None
        mult = lr_multipliers_for(names, getattr(optimizer, "lr_multipliers", None))
        self.dp = None
        if process_group is not None:
            # reference 04: MultiWorkerMirroredStrategy.  "fused": the exchange happens inside the apply
            # kernel over NVLink peer memory; "allreduce": NCCL all-reduce of the slab + replicated apply.
            from .distributed import DataParallelTrainOp, FusedDataParallelTrainOp
            pg = None if process_group is True else process_group
            if dp_mode == "fused":
                self.dp = FusedDataParallelTrainOp(tensors, names, hp, accum_n, lr_fn, pg, exclude, int(global_step),
                                                   loss_scale=loss_scale, ema=ema_cfg, lr_multipliers=mult,
                                                   window_weight=window_weight, tensor_norms=tensor_norms)
                self.engine = self.dp.engine
            else:
                self.engine = GaccumTrainOp(tensors, names, hp, accum_n, lr_fn, exclude, int(global_step),
                                            loss_scale=loss_scale, ema=ema_cfg, lr_multipliers=mult,
                                            window_weight=window_weight, tensor_norms=tensor_norms, **adapt_kw)
                self.dp = DataParallelTrainOp(self.engine, pg)
        else:
            self.engine = GaccumTrainOp(tensors, names, hp, accum_n, lr_fn, exclude, int(global_step),
                                        loss_scale=loss_scale, ema=ema_cfg, lr_multipliers=mult,
                                        window_weight=window_weight, tensor_norms=tensor_norms, **adapt_kw)
        if ema is not None:
            ema._train_op = self
        self.last_loss: Optional[torch.Tensor] = None
        self._weight = None          # window_weight: the weight the loss callable returned with last_loss

    def tensor_norms(self) -> Dict[str, Tuple[float, float, float]]:
        """Synchronously read the per-tensor norms of the last apply step, keyed by variable name (``:0`` stripped):
        (gradient, weight, update) -- ||c|| before the clip scale, ||p|| before the update, ||p_before - p_after||.
        ValueError unless the train op was built with ``tensor_norms=True``."""
        vals = self.engine.tensor_norms()
        return {_lib._variable_name(v.name): (float(r[0]), float(r[1]), float(r[2])) for v, r in zip(self.tvars, vals)}

    @property
    def accum_n(self) -> int:
        return self.engine.N

    def state_dict(self):
        """Checkpoint under the reference's variable names; correct under data parallelism (collective there)."""
        self.engine.global_step = int(self.global_step)
        return self.dp.state_dict() if self.dp is not None else self.engine.state_dict()

    def load_state_dict(self, sd, strict: bool = True) -> None:
        (self.dp if self.dp is not None else self.engine).load_state_dict(sd, strict)
        self.global_step.assign(int(sd["global_step"]))

    def gradients(self) -> List[Optional[torch.Tensor]]:
        """``tf.gradients(loss, tvars)`` (optimization.py:71): evaluated every micro-step.  Under loss scaling these
        are the gradients of ``loss * S``, S read on the device; ``last_loss`` stays unscaled.  With ``window_weight``
        the loss is a pair (summed loss, weight): the gradients are those of the summed loss, ``last_loss`` is the
        summed loss as returned, and the weight goes to the next ``run_with_grads``."""
        loss = self.loss() if callable(self.loss) else self.loss
        if self.window_weight:
            if not (isinstance(loss, (tuple, list)) and len(loss) == 2):
                raise ValueError("with window_weight=True the loss must be a pair (summed loss, weight)")
            loss, self._weight = loss
        self.last_loss = loss.detach()
        if self.engine.loss_scale is not None:
            loss = loss * self.engine.loss_scale
        grads = torch.autograd.grad(loss, [v.tensor for v in self.tvars], allow_unused=True)
        return [None if g is None else g.contiguous() for g in grads]

    def run_with_grads(self, grads: Sequence[Optional[torch.Tensor]], weight=None) -> bool:
        """One micro-step with ``grads``; with ``window_weight`` it takes the micro-batch's weight -- by default the one
        the loss callable returned to the last ``gradients()``."""
        if weight is None and self.window_weight:
            weight, self._weight = self._weight, None
        self.engine.global_step = int(self.global_step)
        kw = {} if weight is None else {"weight": weight}
        applied = self.dp.run(grads, **kw) if self.dp is not None else self.engine.run(grads, **kw)
        self.global_step.assign(self.engine.global_step)          # optimization.py:102-103
        return applied

    def run(self) -> Optional[torch.Tensor]:
        self.run_with_grads(self.gradients())
        return self.last_loss

    __call__ = run


def gradient_accumulation_train_op(loss: LossLike, optimizer: _OptimizerBase, gradient_accumulation_multiplier: int,
                                   clip_norm: Optional[float] = None, global_step: Optional[graph.GlobalStep] = None,
                                   tvars: Optional[Sequence[graph.Variable]] = None, process_group=None,
                                   dp_mode: str = "fused", loss_scale: Optional[LossScaleConfig] = None,
                                   ema: Optional[ExponentialMovingAverage] = None, window_weight: bool = False,
                                   tensor_norms: bool = False) -> TrainOp:
    """The recipe the example scripts inline (02:47-73, 04:48-74, another-example.py:126-155):
    N from ``params``, optimizer given, no clipping unless asked.  ``loss_scale`` turns on dynamic loss scaling for
    fp16 mixed precision: gradients are taken of ``loss * S`` and a window that overflows is skipped on the device.
    ``ema`` keeps an exponential moving average of the trainable variables, updated by the apply step.
    ``window_weight`` divides each window by its total weight instead of N: ``loss`` returns (summed loss, weight), the
    weight typically the micro-batch's number of loss tokens, so a window trains on the per-token mean of its tokens.
    ``tensor_norms`` makes every apply step report per-tensor gradient, weight and update norms (``tensor_norms()``)."""
    gs = global_step or graph.get_or_create_global_step()
    tv = list(tvars) if tvars is not None else graph.trainable_variables()
    if not tv:
        raise ValueError("no trainable variables registered (graph.add_variable / graph.register_module)")
    return TrainOp(loss, tv, optimizer, int(gradient_accumulation_multiplier), clip_norm, gs, process_group, dp_mode,
                   loss_scale, ema, window_weight, tensor_norms)


def create_optimizer(loss, init_lr, num_train_steps, num_warmup_steps, use_tpu):
    """Creates an optimizer training op -- reference optimization.py:25-104, same arguments.

    Schedule :29-54; AdamWeightDecayOptimizer(0.01, 0.9, 0.999, 1e-6, exclude LayerNorm/layer_norm/
    bias) :59-65; window ``gradient_accumulation_multiplier`` :76; apply branch (/N, clip 1.0,
    apply_gradients, zero) :80-88; ``tf.cond`` on the pre-increment step :91-94; step++ :102-103.
    With the module attribute ``optimizer_type = "lamb"`` the optimizer is a LAMBOptimizer with the same
    hyper-parameters and exclusions (layer adaptation excludes what weight decay excludes).  With the module attribute
    ``moving_average_decay`` set, the train op keeps an ExponentialMovingAverage of the variables (``train_op.ema``).
    With the module attribute ``layerwise_lr_decay`` set, each variable trains at ELECTRA's layer-wise decayed rate
    (``layerwise_lr_multipliers``), the number of encoder layers taken from the trainable variables' names.
    With the module attribute ``window_weight`` set, ``loss`` returns (summed loss, weight) and each window is divided by
    its total weight instead of N.  With the module attribute ``tensor_norms`` set, every apply step reports per-tensor
    gradient, weight and update norms (``train_op.tensor_norms()``).  The module attributes ``poly_power`` and
    ``end_learning_rate`` set the polynomial decay after warm-up (``schedules.polynomial_decay``); at their defaults (1.0,
    0.0) the schedule is the reference's, bit for bit.
    """
    if use_tpu:
        # optimization.py:67-68 wraps the optimizer in tf.contrib.tpu.CrossShardOptimizer: TPU-only.
        raise ValueError("use_tpu=True is not supported: this train_op targets H100 GPUs")
    global_step = graph.get_or_create_global_step()
    if optimizer_type not in ("adam", "lamb"):
        raise ValueError(f"optimizer_type must be 'adam' or 'lamb' (got {optimizer_type!r})")
    mult = None
    if layerwise_lr_decay is not None:
        mult = layerwise_lr_multipliers(layerwise_lr_decay,
                                        _num_encoder_layers([v.name for v in graph.trainable_variables()]))
    cls = LAMBOptimizer if optimizer_type == "lamb" else AdamWeightDecayOptimizer
    optimizer = cls(
        learning_rate=schedules.with_bert_warmup(
            schedules.polynomial_decay(init_lr, num_train_steps, end_learning_rate, poly_power), init_lr,
            num_warmup_steps),
        weight_decay_rate=0.01, beta_1=0.9, beta_2=0.999, epsilon=1e-6,
        exclude_from_weight_decay=["LayerNorm", "layer_norm", "bias"])
    optimizer.lr_multipliers = mult
    ema = ExponentialMovingAverage(moving_average_decay) if moving_average_decay is not None else None
    return gradient_accumulation_train_op(loss, optimizer, gradient_accumulation_multiplier,
                                          clip_norm=clip_norm, global_step=global_step, loss_scale=loss_scale, ema=ema,
                                          window_weight=window_weight, tensor_norms=tensor_norms)
