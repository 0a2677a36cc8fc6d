"""CPU oracle (numpy, fp32) for the gradient-accumulation train_op.

TEST INFRASTRUCTURE ONLY.  Nothing in the shipped package imports this module:
only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may use it, and only as the checker / CPU stopwatch.

PARITY STATUS: the reference (hpandana/gradient-accumulation-tf-estimator, commit 74ae92b8) ships no tests, no
golden vectors and no fixtures, and its arithmetic executes inside TensorFlow 1.14/1.15,
which is neither vendored nor installable here.  This restatement is therefore pinned in
two ways only:
  (1) against fixtures produced by executing the reference's *own* ``optimization.py``
      (imported unmodified from a reference checkout) on top of ``oracle/tf_stub`` -- a
      numpy-backed emulation of the ~40 TF1 graph primitives that file touches -- see
      ``tests/golden/make_golden.py``.  This pins op order, window logic, constants and
      the Python-side double->fp32 conversions of the reference's code; the semantics of
      the TF primitives themselves (``polynomial_decay``, ``clip_by_global_norm``,
      ``tf.train.AdamOptimizer``/``ApplyAdam``) are restated from TF 1.15 and remain
      **unpinned by a real TensorFlow run**  ("parity unpinned" at the TF-primitive level);
  (2) against hand-derived known-answer vectors (tests/test_oracle_kat.py).

Every function cites the reference line(s) it follows, relative to the reference repository's root.
One numpy ufunc per TF op, temporaries materialised -- this mirrors the reference's
un-fused graph and is what ``cpu_baseline`` times (kind="port").
"""
from __future__ import annotations

import re
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

F32 = np.float32

VARIANT_ADAM_WEIGHT_DECAY = 0   # optimization.py:107-194  (BERT path, "variant A")
VARIANT_ADAM = 1                # tf.train.AdamOptimizer   (02:41, 04:42, another-example.py:135; "variant B")


# --------------------------------------------------------------------------------------
# a2 -- learning-rate schedule                                   optimization.py:29-54
# --------------------------------------------------------------------------------------
def learning_rate(init_lr: float, num_train_steps: int, num_warmup_steps: Optional[int],
                  global_step: int) -> np.float32:
    """lr used by the micro-step whose pre-increment step counter is ``global_step``.

    optimization.py:29   tf.constant(init_lr, float32)
    optimization.py:32-38 tf.train.polynomial_decay(power=1, end=0, cycle=False):
        gs = cast(step, f32); ds = cast(decay_steps, f32); gs = min(gs, ds); p = gs / ds
        lr = (lr0 - 0) * pow(1 - p, 1) + 0            [TF 1.15 PolynomialDecay.__call__]
    optimization.py:42-54 warm-up blend, all fp32; the int32 compare picks one side exactly.
    """
    lr0 = F32(init_lr)
    gs = F32(np.int64(global_step))
    ds = F32(num_train_steps)
    gs = np.minimum(gs, ds)
    p = F32(gs / ds)
    one_minus_p = F32(F32(1.0) - p)
    # pow(x, 1.0f) == x exactly; (lr0 - 0) == lr0; (+ 0) is exact.
    lr = F32(F32(lr0 - F32(0.0)) * one_minus_p) + F32(0.0)
    lr = F32(lr)
    if num_warmup_steps:                                   # optimization.py:42 (Python truthiness)
        g_i = np.int32(np.int64(global_step))              # :43  cast(global_step, int32)
        w_i = np.int32(num_warmup_steps)                   # :44
        g_f = F32(g_i)                                     # :46
        w_f = F32(w_i)                                     # :47
        pct = F32(g_f / w_f)                               # :49
        wlr = F32(F32(init_lr) * pct)                      # :50  python float -> fp32 const, fp32 Mul
        is_w = F32(1.0) if g_i < w_i else F32(0.0)         # :52
        lr = F32(F32(F32(F32(1.0) - is_w) * lr) + F32(is_w * wlr))   # :53-54
    return F32(lr)


# --------------------------------------------------------------------------------------
# a10 -- weight-decay mask from variable names                 optimization.py:179-194
# --------------------------------------------------------------------------------------
DEFAULT_EXCLUDE = ("LayerNorm", "layer_norm", "bias")      # optimization.py:65


def get_variable_name(param_name: str) -> str:
    """optimization.py:189-194 -- strip the ``:0`` tensor suffix."""
    m = re.match("^(.*):\\d+$", param_name)
    if m is not None:
        param_name = m.group(1)
    return param_name


def do_use_weight_decay(param_name: str, weight_decay_rate: float,
                        exclude: Optional[Sequence[str]] = DEFAULT_EXCLUDE) -> bool:
    """optimization.py:179-187."""
    if not weight_decay_rate:
        return False
    if exclude:
        for r in exclude:
            if re.search(r, param_name) is not None:
                return False
    return True


# --------------------------------------------------------------------------------------
# a8 -- tf.clip_by_global_norm                                  optimization.py:84
# --------------------------------------------------------------------------------------
def global_norm(tensors: Sequence[np.ndarray]) -> np.float32:
    """TF 1.15 ``tf.linalg.global_norm``: sqrt(2 * sum_i l2_loss(t_i)), l2_loss = sum(t^2)/2.

    The order of an fp32 reduction inside TF (Eigen) is unspecified; the oracle defines the
    per-tensor sum as the correctly-rounded one (float64 accumulation, one rounding to fp32),
    then adds the T per-tensor halves sequentially in fp32 (``Pack`` + ``Sum``).
    """
    half = F32(0.0)
    for t in tensors:
        x = np.asarray(t, dtype=F32).ravel()
        s = float(np.dot(x.astype(np.float64), x.astype(np.float64))) if x.size else 0.0
        half = F32(half + F32(s / 2.0))
    return F32(np.sqrt(F32(half * F32(2.0))))


def clip_scale(gn: np.float32, clip_norm: float) -> np.float32:
    """scale = clip * min(1/gn, 1/clip) + (gn - gn)     [TF 1.15 clip_ops.py]

    No epsilon.  gn == 0 -> 1/0 = inf -> min picks 1/clip -> scale 1.  gn = inf/NaN -> NaN.
    """
    c = F32(clip_norm)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = F32(F32(1.0) / gn)
        s = F32(c * np.minimum(inv, F32(F32(1.0) / c)))
        s = F32(s + F32(gn - gn))
    return s


# --------------------------------------------------------------------------------------
# a9 -- AdamWeightDecayOptimizer.apply_gradients               optimization.py:128-177
# --------------------------------------------------------------------------------------
def adam_weight_decay_update(p, m, v, c, lr, beta1, beta2, eps, wd, use_decay):
    """One tensor, un-fused, fp32.  Returns (p', m', v').

    :151-152 next_m = b1*m + (1-b1)*c     ((1-b1) evaluated in Python double, then fp32)
    :153-155 next_v = b2*v + (1-b2)*c^2
    :157     update = next_m / (sqrt(next_v) + eps)
    :166-167 update += wd * p            (old p; only when the name is not excluded)
    :169     update_with_lr = lr * update
    :171     next_param = p - update_with_lr
    """
    b1 = F32(beta1); b2 = F32(beta2)
    omb1 = F32(1.0 - float(beta1)); omb2 = F32(1.0 - float(beta2))
    t1 = np.multiply(b1, m, dtype=F32)
    t2 = np.multiply(omb1, c, dtype=F32)
    next_m = np.add(t1, t2, dtype=F32)
    sq = np.square(c, dtype=F32)
    t3 = np.multiply(b2, v, dtype=F32)
    t4 = np.multiply(omb2, sq, dtype=F32)
    next_v = np.add(t3, t4, dtype=F32)
    rt = np.sqrt(next_v, dtype=F32)
    den = np.add(rt, F32(eps), dtype=F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        update = np.divide(next_m, den, dtype=F32)
    if use_decay:
        wdp = np.multiply(F32(wd), p, dtype=F32)
        update = np.add(update, wdp, dtype=F32)
    uwl = np.multiply(F32(lr), update, dtype=F32)
    next_p = np.subtract(p, uwl, dtype=F32)
    return next_p, next_m, next_v


# --------------------------------------------------------------------------------------
# a14 -- tf.train.AdamOptimizer (TF1 ApplyAdam, use_nesterov=False)   02:41,61  04:42,62
# --------------------------------------------------------------------------------------
def adam_update(p, m, v, c, lr, beta1, beta2, eps, beta1_power, beta2_power):
    """TF 1.15 core/kernels/training_ops.cc ApplyAdam functor, fp32, un-fused:

        alpha = lr * sqrt(1 - beta2_power) / (1 - beta1_power)
        m += (g - m) * (1 - beta1)          (1 - beta1 evaluated in fp32)
        v += (g*g - v) * (1 - beta2)
        var -= (m * alpha) / (sqrt(v) + eps)
    """
    b1 = F32(beta1); b2 = F32(beta2)
    alpha = F32(F32(F32(lr) * np.sqrt(F32(F32(1.0) - F32(beta2_power)))) / F32(F32(1.0) - F32(beta1_power)))
    omb1 = F32(F32(1.0) - b1); omb2 = F32(F32(1.0) - b2)
    d1 = np.subtract(c, m, dtype=F32)
    next_m = np.add(m, np.multiply(d1, omb1, dtype=F32), dtype=F32)
    sq = np.multiply(c, c, dtype=F32)
    d2 = np.subtract(sq, v, dtype=F32)
    next_v = np.add(v, np.multiply(d2, omb2, dtype=F32), dtype=F32)
    num = np.multiply(next_m, alpha, dtype=F32)
    den = np.add(np.sqrt(next_v, dtype=F32), F32(eps), dtype=F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        next_p = np.subtract(p, np.divide(num, den, dtype=F32), dtype=F32)
    return next_p, next_m, next_v


# --------------------------------------------------------------------------------------
# a4-a7, a11-a13 -- the train_op itself                          optimization.py:76-104
# --------------------------------------------------------------------------------------
@dataclass
class HParams:
    variant: int = VARIANT_ADAM_WEIGHT_DECAY
    beta1: float = 0.9                   # optimization.py:62
    beta2: float = 0.999                 # :63
    epsilon: float = 1e-6                # :64   (1e-8 for tf.train.AdamOptimizer)
    weight_decay_rate: float = 0.01      # :61
    clip_norm: float = 1.0               # :84   (<= 0: no clip -- 02:59-61, 04:60-62)

    @staticmethod
    def bert() -> "HParams":
        return HParams()

    @staticmethod
    def tf_adam() -> "HParams":
        """tf.train.AdamOptimizer defaults as used by 02:41, 04:42, another-example.py:135."""
        return HParams(variant=VARIANT_ADAM, beta1=0.9, beta2=0.999, epsilon=1e-8,
                       weight_decay_rate=0.0, clip_norm=0.0)


@dataclass
class StepInfo:
    global_step: int
    applied: bool
    lr: np.float32
    global_norm: np.float32 = F32(0.0)
    clip_scale: np.float32 = F32(1.0)


@dataclass
class Reduced:
    """The scalars a device reduced for one applied window: the global norm gn and, LAMB, the per-tensor trust ratios
    (r of the tensors without layer adaptation is ignored: it is 1)."""
    global_norm: np.float32
    ratios: Optional[Sequence[np.float32]] = None


class ReferenceTrainOp:
    """State + one ``run(grads)`` per micro-step, op-for-op as optimization.py:76-104.

    ``params`` are updated in place (list of fp32 arrays).  ``names`` feed the decay mask.
    ``lr_fn(g)`` overrides the BERT schedule (variant B scripts use a constant lr).

    Opt-in: set ``reduced`` before the ``run`` of an apply step and that window takes its gn (and LAMB's r) from it
    instead of reducing them itself; the clip scale and everything after it are still computed here.  Such a window
    keeps its c before the clip scale in ``window_c`` (LAMB: each adapted tensor's p before the update and u in
    ``window_pu``).  ``run`` clears ``reduced`` once the window is applied.
    """
    reduced: Optional[Reduced] = None
    window_c: Optional[List[np.ndarray]] = None

    def _global_norm(self, c: Sequence[np.ndarray]) -> np.float32:
        """gn of the window's c: ``reduced.global_norm`` if it was given, else ``global_norm(c)``."""
        if self.reduced is None:
            return global_norm(c)
        self.window_c = list(c)
        return F32(self.reduced.global_norm)

    def __init__(self, params: List[np.ndarray], names: Sequence[str], hp: HParams,
                 accum_n: int, init_lr: float = 0.0, num_train_steps: int = 1,
                 num_warmup_steps: Optional[int] = 0, constant_lr: Optional[float] = None,
                 exclude: Optional[Sequence[str]] = DEFAULT_EXCLUDE, global_step: int = 0):
        self.params = [np.ascontiguousarray(p, dtype=F32) for p in params]
        self.names = [get_variable_name(n) for n in names]
        self.hp = hp
        self.N = int(accum_n)                                     # optimization.py:76
        self.init_lr, self.num_train_steps, self.num_warmup_steps = init_lr, num_train_steps, num_warmup_steps
        self.constant_lr = constant_lr
        self.global_step = int(global_step)                       # :27
        self.accum = [np.zeros_like(p) for p in self.params]      # :78
        self.m = [np.zeros_like(p) for p in self.params]          # :137-142
        self.v = [np.zeros_like(p) for p in self.params]          # :143-148
        self.decay = [do_use_weight_decay(n, hp.weight_decay_rate, exclude) for n in self.names]
        # tf.train.AdamOptimizer non-slot variables, initialised to beta (TF1 _create_slots)
        self.beta1_power = F32(hp.beta1)
        self.beta2_power = F32(hp.beta2)

    def lr(self, g: int) -> np.float32:
        if self.constant_lr is not None:
            return F32(self.constant_lr)
        return learning_rate(self.init_lr, self.num_train_steps, self.num_warmup_steps, g)

    def run(self, grads: Sequence[Optional[np.ndarray]]) -> StepInfo:
        g = self.global_step
        hp = self.hp
        lr = self.lr(g)
        is_apply = (int(np.int32(np.int64(g))) % self.N) == 0     # :77, :91 (pre-increment)
        # :81 / :93 -- assign_add in both branches (grad None == tf.gradients returned None:
        # TF would raise in assign_add; we treat it as "no contribution", the only sane reading)
        for a, gr in zip(self.accum, grads):
            if gr is not None:
                np.add(a, np.asarray(gr, dtype=F32).reshape(a.shape), out=a, dtype=F32)
        info = StepInfo(global_step=g, applied=is_apply, lr=lr)
        if is_apply:
            nf = F32(self.N)
            # :83  1.0*accum_grad / N   (Mul by 1.0 exact, then RealDiv by fp32(N))
            normalized = [np.divide(np.multiply(F32(1.0), a, dtype=F32), nf, dtype=F32) for a in self.accum]
            if hp.clip_norm and hp.clip_norm > 0:                 # :84
                gn = self._global_norm(normalized)
                s = clip_scale(gn, hp.clip_norm)
                clipped = [np.multiply(n, s, dtype=F32) for n in normalized]
                info.global_norm, info.clip_scale = gn, s
            else:
                clipped = normalized
            # :85 optimizer.apply_gradients
            for i, c in enumerate(clipped):
                if hp.variant == VARIANT_ADAM_WEIGHT_DECAY:
                    p2, m2, v2 = adam_weight_decay_update(
                        self.params[i], self.m[i], self.v[i], c, lr, hp.beta1, hp.beta2,
                        hp.epsilon, hp.weight_decay_rate, self.decay[i])
                else:
                    p2, m2, v2 = adam_update(
                        self.params[i], self.m[i], self.v[i], c, lr, hp.beta1, hp.beta2,
                        hp.epsilon, self.beta1_power, self.beta2_power)
                self.params[i][...] = p2; self.m[i][...] = m2; self.v[i][...] = v2   # :173-176
            if hp.variant == VARIANT_ADAM:
                # TF1 AdamOptimizer._finish: beta_power *= beta after the var updates
                self.beta1_power = F32(self.beta1_power * F32(hp.beta1))
                self.beta2_power = F32(self.beta2_power * F32(hp.beta2))
            for a in self.accum:                                  # :86-87
                a[...] = F32(0.0)
            self.reduced = None
        self.global_step = g + 1                                  # :102-103
        return info


# --------------------------------------------------------------------------------------
# Shape manifests (names matter: the decay mask comes from them).  Upstream BERT variable
# names (google-research/bert modeling.py, referenced by README.md:14) in
# tf.trainable_variables() creation order; MNIST CNN from distributedExample/02:22-28.
# --------------------------------------------------------------------------------------
def bert_manifest(num_layers: int, hidden: int, intermediate: Optional[int] = None,
                  vocab: int = 30522, max_pos: int = 512, type_vocab: int = 2, num_labels: int = 2):
    inter = intermediate or 4 * hidden
    out = []
    e = "bert/embeddings/"
    out += [(e + "word_embeddings", (vocab, hidden)),
            (e + "token_type_embeddings", (type_vocab, hidden)),
            (e + "position_embeddings", (max_pos, hidden)),
            (e + "LayerNorm/beta", (hidden,)), (e + "LayerNorm/gamma", (hidden,))]
    for l in range(num_layers):
        b = f"bert/encoder/layer_{l}/"
        for nm in ("query", "key", "value"):
            out += [(b + f"attention/self/{nm}/kernel", (hidden, hidden)),
                    (b + f"attention/self/{nm}/bias", (hidden,))]
        out += [(b + "attention/output/dense/kernel", (hidden, hidden)),
                (b + "attention/output/dense/bias", (hidden,)),
                (b + "attention/output/LayerNorm/beta", (hidden,)),
                (b + "attention/output/LayerNorm/gamma", (hidden,)),
                (b + "intermediate/dense/kernel", (hidden, inter)),
                (b + "intermediate/dense/bias", (inter,)),
                (b + "output/dense/kernel", (inter, hidden)),
                (b + "output/dense/bias", (hidden,)),
                (b + "output/LayerNorm/beta", (hidden,)),
                (b + "output/LayerNorm/gamma", (hidden,))]
    out += [("bert/pooler/dense/kernel", (hidden, hidden)), ("bert/pooler/dense/bias", (hidden,)),
            ("output_weights", (num_labels, hidden)), ("output_bias", (num_labels,))]
    return out


def mnist_cnn_manifest():
    """distributedExample/02:22-28 -- Conv2D(32,3) -> MaxPool -> Flatten -> Dense(64) -> Dense(10)."""
    return [("conv2d/kernel", (3, 3, 1, 32)), ("conv2d/bias", (32,)),
            ("dense/kernel", (5408, 64)), ("dense/bias", (64,)),
            ("dense_1/kernel", (64, 10)), ("dense_1/bias", (10,))]


MANIFESTS = {
    "mnist_cnn": mnist_cnn_manifest,
    "bert_small": lambda: bert_manifest(4, 512),
    "bert_base": lambda: bert_manifest(12, 768),
    "bert_large": lambda: bert_manifest(24, 1024),
}
