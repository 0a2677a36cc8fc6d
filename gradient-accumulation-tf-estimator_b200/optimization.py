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
from typing import Callable, Iterable, List, Optional, Sequence, Tuple, Union

import torch

from . import _lib, graph
from ._lib import ADAM, ADAM_WEIGHT_DECAY, HParams
from .train_op import GaccumTrainOp

# optimization.py:76 hard-codes 8 (README.md:17,34 says 4).  The signature has no argument for
# it, so it is a module attribute (and GACCUM_MULTIPLIER in the environment) -- default as shipped.
gradient_accumulation_multiplier = int(os.environ.get("GACCUM_MULTIPLIER", "8"))
clip_norm = 1.0   # optimization.py:84

LossLike = Union[torch.Tensor, Callable[[], torch.Tensor]]
LrLike = Union[float, Callable[[int], float]]


def _lr_callable(lr: LrLike) -> Callable[[int], float]:
    return lr if callable(lr) else (lambda step, _v=float(lr): _v)


def bert_learning_rate(init_lr: float, num_train_steps: int, num_warmup_steps: Optional[int]) -> Callable[[int], float]:
    """optimization.py:29-54 as a function of the pre-increment global step (fp32 op order)."""
    return lambda step: _lib.learning_rate(init_lr, num_train_steps, num_warmup_steps, step)


class _OptimizerBase:
    """What both optimizers share: turning (grad, var) pairs into one kernel launch."""
    variant = ADAM_WEIGHT_DECAY

    def _hparams(self, clip: float) -> HParams:
        raise NotImplementedError

    def __init__(self):
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
                                            exclude_from_weight_decay=getattr(self, "exclude_from_weight_decay", None))
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
        if not self.weight_decay_rate:
            return False
        if self.exclude_from_weight_decay:
            for r in self.exclude_from_weight_decay:
                if re.search(r, param_name) is not None:
                    return False
        return True

    def _get_variable_name(self, param_name: str) -> str:
        """optimization.py:189-194."""
        m = re.match("^(.*):\\d+$", param_name)
        if m is not None:
            param_name = m.group(1)
        return param_name


class AdamOptimizer(_OptimizerBase):
    """``tf.train.AdamOptimizer`` as the example scripts use it (02:41, 04:42, another-example.py:135)."""
    variant = ADAM

    def __init__(self, learning_rate: LrLike = 0.001, beta1=0.9, beta2=0.999, epsilon=1e-8, name="Adam"):
        super().__init__()
        self.learning_rate = learning_rate
        self.beta1, self.beta2, self.epsilon, self.name = beta1, beta2, epsilon, name

    def _hparams(self, clip: float) -> HParams:
        return HParams(ADAM, 0, self.beta1, self.beta2, self.epsilon, 0.0, clip)


class TrainOp:
    """The object ``create_optimizer`` returns; ``run()`` == ``session.run(train_op)``."""

    def __init__(self, loss: LossLike, tvars: Sequence[graph.Variable], optimizer: _OptimizerBase,
                 accum_n: int, clip: Optional[float], global_step: graph.GlobalStep, process_group=None,
                 dp_mode: str = "fused"):
        self.loss = loss
        self.tvars = list(tvars)
        self.optimizer = optimizer
        self.global_step = global_step
        tensors, names = [v.tensor for v in self.tvars], [v.name for v in self.tvars]
        hp = optimizer._hparams(clip or 0.0)
        lr_fn = _lr_callable(optimizer.learning_rate)
        exclude = getattr(optimizer, "exclude_from_weight_decay", None)
        self.dp = None
        if process_group is not None:
            # reference 04: MultiWorkerMirroredStrategy.  "fused": the exchange happens inside the apply
            # kernel over NVLink peer memory; "allreduce": NCCL all-reduce of the slab + replicated apply.
            from .distributed import DataParallelTrainOp, FusedDataParallelTrainOp
            pg = None if process_group is True else process_group
            if dp_mode == "fused":
                self.dp = FusedDataParallelTrainOp(tensors, names, hp, accum_n, lr_fn, pg, exclude, int(global_step))
                self.engine = self.dp.engine
            else:
                self.engine = GaccumTrainOp(tensors, names, hp, accum_n, lr_fn, exclude, int(global_step))
                self.dp = DataParallelTrainOp(self.engine, pg)
        else:
            self.engine = GaccumTrainOp(tensors, names, hp, accum_n, lr_fn, exclude, int(global_step))
        self.last_loss: Optional[torch.Tensor] = None

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
        """``tf.gradients(loss, tvars)`` (optimization.py:71): evaluated every micro-step."""
        loss = self.loss() if callable(self.loss) else self.loss
        self.last_loss = loss.detach()
        grads = torch.autograd.grad(loss, [v.tensor for v in self.tvars], allow_unused=True)
        return [None if g is None else g.contiguous() for g in grads]

    def run_with_grads(self, grads: Sequence[Optional[torch.Tensor]]) -> bool:
        self.engine.global_step = int(self.global_step)
        applied = self.dp.run(grads) if self.dp is not None else self.engine.run(grads)
        self.global_step.assign(self.engine.global_step)          # optimization.py:102-103
        return applied

    def run(self) -> Optional[torch.Tensor]:
        self.run_with_grads(self.gradients())
        return self.last_loss

    __call__ = run


def gradient_accumulation_train_op(loss: LossLike, optimizer: _OptimizerBase, gradient_accumulation_multiplier: int,
                                   clip_norm: Optional[float] = None, global_step: Optional[graph.GlobalStep] = None,
                                   tvars: Optional[Sequence[graph.Variable]] = None, process_group=None,
                                   dp_mode: str = "fused") -> TrainOp:
    """The recipe the example scripts inline (02:47-73, 04:48-74, another-example.py:126-155):
    N from ``params``, optimizer given, no clipping unless asked."""
    gs = global_step or graph.get_or_create_global_step()
    tv = list(tvars) if tvars is not None else graph.trainable_variables()
    if not tv:
        raise ValueError("no trainable variables registered (graph.add_variable / graph.register_module)")
    return TrainOp(loss, tv, optimizer, int(gradient_accumulation_multiplier), clip_norm, gs, process_group, dp_mode)


def create_optimizer(loss, init_lr, num_train_steps, num_warmup_steps, use_tpu):
    """Creates an optimizer training op -- reference optimization.py:25-104, same arguments.

    Schedule :29-54; AdamWeightDecayOptimizer(0.01, 0.9, 0.999, 1e-6, exclude LayerNorm/layer_norm/
    bias) :59-65; window ``gradient_accumulation_multiplier`` :76; apply branch (/N, clip 1.0,
    apply_gradients, zero) :80-88; ``tf.cond`` on the pre-increment step :91-94; step++ :102-103.
    """
    if use_tpu:
        # optimization.py:67-68 wraps the optimizer in tf.contrib.tpu.CrossShardOptimizer: TPU-only.
        raise ValueError("use_tpu=True is not supported: this train_op targets H100 GPUs")
    global_step = graph.get_or_create_global_step()
    optimizer = AdamWeightDecayOptimizer(
        learning_rate=bert_learning_rate(init_lr, num_train_steps, num_warmup_steps),
        weight_decay_rate=0.01, beta_1=0.9, beta_2=0.999, epsilon=1e-6,
        exclude_from_weight_decay=["LayerNorm", "layer_norm", "bias"])
    return gradient_accumulation_train_op(loss, optimizer, gradient_accumulation_multiplier,
                                          clip_norm=clip_norm, global_step=global_step)
