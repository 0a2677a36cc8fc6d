# coding=utf-8
"""Drop-in replacement for the reference's ``optimization.py`` on a machine that HAS TensorFlow.

Put this file where ``run_classifier.py`` imports ``optimization`` from (or the inline recipes of
distributedExample/02,04 call ``gaccum_train_op``) -- nothing else in the caller changes:

    train_op = optimization.create_optimizer(total_loss, learning_rate, num_train_steps,
                                             num_warmup_steps, use_tpu)

Same five arguments, same return type (a ``tf.Operation``), same checkpointed state (variables),
but instead of the ``tf.cond`` over 3T ``assign_add`` / ~17T un-fused Adam ops
(reference optimization.py:76-94, 128-177) the graph contains ONE stateful custom-op node,
``GaccumStep`` (gaccum_tf_op.cc), that calls ``gaccum_step`` in libgaccum.so.

CANNOT BE EXECUTED IN THIS REPOSITORY'S IMAGE (TensorFlow is not installable; tests/
test_tf_shim.py activates wherever ``import tensorflow`` works).  Written against
``tf.compat.v1`` so it runs on TF 1.15 and TF 2.x alike.
"""
from __future__ import absolute_import, division, print_function

import os
import re

import tensorflow as _tf

tf = _tf.compat.v1 if hasattr(_tf, "compat") and hasattr(_tf.compat, "v1") else _tf

_HERE = os.path.dirname(os.path.abspath(__file__))
_ops = None

# optimization.py:76 hard-codes 8 (README.md:17,34 says 4); no argument exists for it.
gradient_accumulation_multiplier = int(os.environ.get("GACCUM_MULTIPLIER", "8"))


def _load():
    global _ops
    if _ops is None:
        _ops = tf.load_op_library(os.path.join(_HERE, "libgaccum_tf.so"))
    return _ops


def _decay_mask(names, weight_decay_rate, exclude):
    """optimization.py:179-194."""
    out = []
    for n in names:
        m = re.match("^(.*):\\d+$", n)
        n = m.group(1) if m is not None else n
        use = bool(weight_decay_rate)
        for r in (exclude or []):
            if re.search(r, n) is not None:
                use = False
        out.append(use)
    return out


def _slab_size(tvars):
    return sum((int(v.shape.num_elements()) + 31) // 32 * 32 for v in tvars)


def _is_resource(v):
    """TF2-style variables (what Keras layers create in distributedExample/02, 04 under TF >= 2) are resource handles."""
    return "Resource" in type(v).__name__ or getattr(getattr(v, "dtype", None), "name", "") == "resource"


def gaccum_train_op(loss, learning_rate, accum_n, variant=0, beta1=0.9, beta2=0.999, epsilon=1e-6,
                    weight_decay_rate=0.01, clip_norm=1.0, exclude_from_weight_decay=None,
                    global_step=None, increment_global_step=True, grads_and_vars=None):
    """The accumulate-then-apply train_op as one node (the recipe of 02:47-73 / 04:48-74 /
    optimization.py:70-104)."""
    if grads_and_vars is None:
        tvars = tf.trainable_variables()                               # optimization.py:70
        grads = tf.gradients(loss, tvars)                              # optimization.py:71
        grads_and_vars = zip(grads, tvars)
    pairs = [(g, v) for g, v in grads_and_vars if g is not None and v is not None]    # optimization.py:132-133
    grads, tvars = [g for g, _ in pairs], [v for _, v in pairs]
    if global_step is None and (increment_global_step or variant == 0 or accum_n > 1):
        global_step = tf.train.get_or_create_global_step()
    n = _slab_size(tvars)
    resource = any(_is_resource(v_) for v_ in tvars)
    with tf.variable_scope("gaccum", reuse=tf.AUTO_REUSE):
        mk = lambda name: tf.get_variable(name, shape=[n], dtype=tf.float32, trainable=False,
                                          initializer=tf.zeros_initializer(), use_resource=resource)
        accum, m, v = mk("accum_grads"), mk("adam_m"), mk("adam_v")   # :78, :137-148 packed
        beta_powers = tf.get_variable("beta_powers", dtype=tf.float32, trainable=False, use_resource=False,
                                      initializer=tf.constant([beta1, beta2], dtype=tf.float32))
    mask = _decay_mask([v_.name for v_ in tvars], weight_decay_rate if variant == 0 else 0.0,
                       exclude_from_weight_decay)
    # ONE read of the step counter feeds the op, the beta-power update and the increment: whatever order the executor
    # picks for the unordered ops below, they all see the PRE-increment value (optimization.py:77, 91)
    step_before = tf.identity(global_step) if global_step is not None else tf.constant(0, dtype=tf.int64)
    op_fn = _load().gaccum_step_v2 if resource and hasattr(_load(), "gaccum_step_v2") else _load().gaccum_step
    # hyper-parameters travel as strings: a float attr is fp32 in the GraphDef and would lose the reference's
    # double -> fp32 conversion points (`1.0 - beta_1` is evaluated in double, optimization.py:152)
    step_op = op_fn(
        params=tvars, grads=grads, accum=accum, m=m, v=v, global_step=step_before,
        lr=tf.cast(learning_rate, tf.float32), beta_powers=beta_powers, accum_n=accum_n, variant=variant,
        beta1=repr(float(beta1)), beta2=repr(float(beta2)), epsilon=repr(float(epsilon)),
        weight_decay_rate=repr(float(weight_decay_rate)), clip_norm=repr(float(clip_norm or 0.0)), decay_mask=mask)
    tail = [step_op]
    if variant == 1:
        # TF1 AdamOptimizer._finish: beta powers advance after every APPLY; the predicate uses step_before, the update
        # waits for the kernel (which reads the current powers)
        with tf.control_dependencies([step_op]):
            is_apply = tf.equal(tf.cast(step_before, tf.int32) % accum_n, 0)
            tail = [tf.cond(is_apply,
                            lambda: beta_powers.assign(beta_powers * tf.constant([beta1, beta2], tf.float32)),
                            lambda: tf.identity(beta_powers))]
    if increment_global_step:
        with tf.control_dependencies(tail + [step_before]):           # after everything that consumes the old value
            tail = tail + [global_step.assign(step_before + 1)]       # optimization.py:102-103
    return tf.group(*tail)


def create_optimizer(loss, init_lr, num_train_steps, num_warmup_steps, use_tpu):
    """Creates an optimizer training op (same signature as the reference, optimization.py:25)."""
    if use_tpu:
        raise ValueError("use_tpu=True is not supported by the H100 train_op")
    global_step = tf.train.get_or_create_global_step()
    # optimization.py:29-54 verbatim semantics (this IS TensorFlow, so the schedule stays in-graph)
    learning_rate = tf.constant(value=init_lr, shape=[], dtype=tf.float32)
    learning_rate = tf.train.polynomial_decay(learning_rate, global_step, num_train_steps,
                                              end_learning_rate=0.0, power=1.0, cycle=False)
    if num_warmup_steps:
        global_steps_int = tf.cast(global_step, tf.int32)
        warmup_steps_int = tf.constant(num_warmup_steps, dtype=tf.int32)
        warmup_percent_done = tf.cast(global_steps_int, tf.float32) / tf.cast(warmup_steps_int, tf.float32)
        warmup_learning_rate = init_lr * warmup_percent_done
        is_warmup = tf.cast(global_steps_int < warmup_steps_int, tf.float32)
        learning_rate = (1.0 - is_warmup) * learning_rate + is_warmup * warmup_learning_rate
    return gaccum_train_op(loss, learning_rate, gradient_accumulation_multiplier, variant=0,
                           beta1=0.9, beta2=0.999, epsilon=1e-6, weight_decay_rate=0.01, clip_norm=1.0,
                           exclude_from_weight_decay=["LayerNorm", "layer_norm", "bias"],
                           global_step=global_step)


class AdamWeightDecayOptimizer(object):
    """Reference optimization.py:107-194 with the same constructor and the same ``apply_gradients`` contract:
    one un-clipped AdamWeightDecay update of the given (grad, var) pairs, pairs with a None member skipped (:132-133),
    ``global_step`` accepted and NOT incremented (:128, comment :99-101).  The update is the same GaccumStep node with a
    window of 1 (every run applies), so ``optimization.AdamWeightDecayOptimizer(...).apply_gradients(...)`` -- legal
    against the reference -- works against this file too."""

    def __init__(self, learning_rate, weight_decay_rate=0.0, beta_1=0.9, beta_2=0.999, epsilon=1e-6,
                 exclude_from_weight_decay=None, name="AdamWeightDecayOptimizer"):
        self.learning_rate, self.weight_decay_rate = learning_rate, weight_decay_rate
        self.beta_1, self.beta_2, self.epsilon = beta_1, beta_2, epsilon
        self.exclude_from_weight_decay, self.name = exclude_from_weight_decay, name

    def apply_gradients(self, grads_and_vars, global_step=None, name=None):
        return gaccum_train_op(None, self.learning_rate, accum_n=1, variant=0, beta1=self.beta_1, beta2=self.beta_2,
                               epsilon=self.epsilon, weight_decay_rate=self.weight_decay_rate, clip_norm=0.0,
                               exclude_from_weight_decay=self.exclude_from_weight_decay, global_step=None,
                               increment_global_step=False, grads_and_vars=list(grads_and_vars))

    def _do_use_weight_decay(self, param_name):
        """optimization.py:179-187."""
        return _decay_mask([param_name], self.weight_decay_rate, self.exclude_from_weight_decay)[0]

    def _get_variable_name(self, param_name):
        """optimization.py:189-194."""
        m = re.match("^(.*):\\d+$", param_name)
        return m.group(1) if m is not None else param_name
