"""A numpy-backed stand-in for the ~40 TensorFlow-1.x graph primitives that the reference's
``optimization.py`` touches.  TEST INFRASTRUCTURE ONLY (see oracle/README.md).

Purpose: TensorFlow cannot be installed in this image, so the reference cannot be executed as is.
With this package first on ``sys.path`` the reference's OWN file (optimization.py of a reference checkout,
imported unmodified) builds its graph against these primitives, and ``Session.run`` evaluates it in
IEEE fp32 with one rounding per op.  That pins everything the reference's Python decides -- op
order, window logic (pre-increment ``global_step % N``), constants, Python double -> fp32
conversions, control dependencies, the name-based decay mask -- into golden vectors
(tests/golden/make_golden.py).  What it cannot pin is TensorFlow's own semantics for the
composite functions restated below from TF 1.15 (``polynomial_decay``, ``clip_by_global_norm``):
those stay "[TF-memory]" (SURVEY.md 8(c)).

Model: a lazy dataflow graph.  ``Tensor.eval(run)`` memoises per ``Session.run``; control
dependencies are evaluated before the op; variable reads are never memoised (a ref-variable read
yields whatever the buffer holds when the consumer runs, which is what control_dependencies rely
on); ``cond`` evaluates only the taken branch's ops.  Binary operators convert Python scalars to
the tensor operand's dtype exactly like ``ops.convert_to_tensor`` does.
"""
from __future__ import annotations

import contextlib
import types

import numpy as np

__version__ = "1.15.0-stub"


# ------------------------------------------------------------------------------------------ dtypes
class DType:
    def __init__(self, np_dtype, name):
        self.np = np.dtype(np_dtype)
        self.name = name

    @property
    def base_dtype(self):
        return self

    def __repr__(self):
        return f"tf.{self.name}"

    def __eq__(self, o):
        return isinstance(o, DType) and o.np == self.np

    def __hash__(self):
        return hash(self.np)


float32 = DType(np.float32, "float32")
float64 = DType(np.float64, "float64")
int32 = DType(np.int32, "int32")
int64 = DType(np.int64, "int64")
bool_ = DType(np.bool_, "bool")
_BY_NP = {d.np: d for d in (float32, float64, int32, int64, bool_)}


def _dt(np_dtype):
    return _BY_NP[np.dtype(np_dtype)]


class TensorShape(tuple):
    def as_list(self):
        return list(self)

    def num_elements(self):
        return int(np.prod(self, dtype=np.int64)) if len(self) else 1


# ------------------------------------------------------------------------------------------- graph
_control_stack = []          # stack of lists of ops (tf.control_dependencies)
REVERSE_UNORDERED = False    # tests flip this to evaluate unordered op sets (tf.group inputs) in reverse: exposes missing control dependencies


class _Run:
    def __init__(self, feeds):
        self.memo = {}
        self.feeds = feeds


class Tensor:
    def __init__(self, fn, inputs=(), dtype=None, shape=(), name=None):
        self._fn = fn
        self._inputs = tuple(inputs)
        self.dtype = dtype
        self.shape = TensorShape(shape)
        self.name = name or "op"
        self._control = tuple(op for frame in _control_stack for op in frame)

    def eval(self, run: _Run):
        k = id(self)
        if k in run.memo:
            return run.memo[k]
        for c in self._control:
            c.eval(run)
        vals = [i.eval(run) for i in self._inputs]
        out = self._fn(run, *vals)
        run.memo[k] = out
        return out

    # python operators -> the TF ops they dispatch to
    def __add__(self, o): return _binary(np.add, self, o, "add")
    def __radd__(self, o): return _binary(np.add, o, self, "add")
    def __sub__(self, o): return _binary(np.subtract, self, o, "sub")
    def __rsub__(self, o): return _binary(np.subtract, o, self, "sub")
    def __mul__(self, o): return _binary(np.multiply, self, o, "mul")
    def __rmul__(self, o): return _binary(np.multiply, o, self, "mul")
    def __truediv__(self, o): return _binary(_realdiv, self, o, "truediv")
    def __rtruediv__(self, o): return _binary(_realdiv, o, self, "truediv")
    def __mod__(self, o): return _binary(np.mod, self, o, "floormod")      # FloorMod
    def __lt__(self, o): return _binary(np.less, self, o, "less", out_dtype=bool_)
    def __neg__(self): return Tensor(lambda r, x: np.negative(x), [self], self.dtype, self.shape)
    __hash__ = object.__hash__


def _realdiv(x, y):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.divide(x, y)


def convert_to_tensor(v, dtype=None, name=None):
    if isinstance(v, Tensor):
        return v
    if v is None:
        raise ValueError("None values not supported.")          # what TF's make_tensor_proto raises
    if dtype is None:
        if isinstance(v, bool):
            dtype = bool_
        elif isinstance(v, (int, np.integer)):
            dtype = int32
        elif isinstance(v, (float, np.floating)):
            dtype = float32
        else:
            dtype = _dt(np.asarray(v).dtype)
    arr = np.asarray(v, dtype=dtype.np)       # Python double -> fp32 happens HERE, once
    return Tensor(lambda r, _a=arr: _a, (), dtype, arr.shape, name or "Const")


def _binary(ufunc, a, b, name, out_dtype=None):
    # ops.convert_to_tensor with the tensor operand's dtype as the preferred dtype
    if isinstance(a, Tensor) and not isinstance(b, Tensor):
        b = convert_to_tensor(b, a.dtype)
    elif isinstance(b, Tensor) and not isinstance(a, Tensor):
        a = convert_to_tensor(a, b.dtype)
    if a.dtype != b.dtype:
        raise TypeError(f"{name}: dtype mismatch {a.dtype} vs {b.dtype} (TF would raise too)")
    dt = out_dtype or a.dtype
    shape = a.shape if len(a.shape) >= len(b.shape) else b.shape

    def fn(r, x, y):
        out = ufunc(x, y)
        return np.asarray(out, dtype=dt.np)
    return Tensor(fn, [a, b], dt, shape, name)


# --------------------------------------------------------------------------------------- variables
class _Collections:
    def __init__(self):
        self.all, self.by_name, self.placeholders = [], {}, []
        self.global_step = None


_g = _Collections()


def reset_default_graph():
    global _g
    _g = _Collections()
    del _control_stack[:]


class VariableAggregation:
    NONE, SUM, MEAN, ONLY_FIRST_REPLICA = range(4)


class Variable(Tensor):
    _auto = 0

    def __init__(self, initial_value=None, trainable=True, name=None, dtype=None, aggregation=None):
        if isinstance(initial_value, Tensor):
            init = initial_value.eval(_Run({}))           # initializers need no feeds
        else:
            init = np.asarray(initial_value, dtype=(dtype.np if dtype else None))
        if name is None:
            Variable._auto += 1
            name = f"Variable_{Variable._auto}"
        self.value = np.array(init, copy=True)
        self._initial = np.array(init, copy=True)
        self.trainable = trainable
        Tensor.__init__(self, None, (), _dt(self.value.dtype), self.value.shape, name + ":0")
        self._control = ()
        _g.all.append(self)
        _g.by_name[name] = self

    def eval(self, run):                                  # never memoised
        return self.value

    def initialized_value(self):
        return Tensor(lambda r, _a=self._initial: _a, (), self.dtype, self.shape, "initialized_value")

    def assign(self, v, **kw):
        v = convert_to_tensor(v, self.dtype)

        def fn(r, x):
            self.value = np.array(np.broadcast_to(x, self.value.shape), dtype=self.value.dtype, copy=True)
            return self.value
        return Tensor(fn, [v], self.dtype, self.shape, "Assign")

    def assign_add(self, v, **kw):
        v = convert_to_tensor(v, self.dtype)

        def fn(r, x):
            self.value = np.add(self.value, x, dtype=self.value.dtype)     # AssignAdd: one rounding
            return self.value
        return Tensor(fn, [v], self.dtype, self.shape, "AssignAdd")


def zeros_initializer():
    return lambda shape, dtype: np.zeros(shape, dtype=dtype.np)


AUTO_REUSE = "AUTO_REUSE"
_scope_stack = []


@contextlib.contextmanager
def variable_scope(name, reuse=None, **kw):
    _scope_stack.append((name, reuse))
    try:
        yield
    finally:
        _scope_stack.pop()


def get_variable(name, shape=None, dtype=float32, trainable=True, initializer=None, **kw):
    if _scope_stack:
        name = "/".join(n for n, _ in _scope_stack) + "/" + name
    if name in _g.by_name:
        if any(r is AUTO_REUSE or r is True for _, r in _scope_stack):
            return _g.by_name[name]
        raise ValueError(f"Variable {name} already exists (no reuse scope)")
    if isinstance(initializer, Tensor):
        init = np.asarray(initializer.eval(_Run({})), dtype=dtype.np)
    elif callable(initializer):
        init = initializer(tuple(shape), dtype)
    else:
        init = np.asarray(initializer, dtype=dtype.np).reshape(tuple(shape))
    return Variable(init, trainable=trainable, name=name, dtype=dtype)


def trainable_variables():
    return [v for v in _g.all if v.trainable]


def global_variables():
    return list(_g.all)


# --------------------------------------------------------------------------------------------- ops
def constant(value, dtype=None, shape=None, name=None):
    t = convert_to_tensor(value, dtype)
    if shape is not None and tuple(shape) != tuple(t.shape):
        arr = np.broadcast_to(t.eval(_Run({})), tuple(shape)).copy()
        t = convert_to_tensor(arr, dtype)
    return t


def cast(x, dtype, name=None):
    x = convert_to_tensor(x)
    return Tensor(lambda r, v: np.asarray(v).astype(dtype.np), [x], dtype, x.shape, "Cast")


def multiply(x, y, name=None):
    return _binary(np.multiply, x, y, "Mul")


def square(x, name=None):
    x = convert_to_tensor(x)
    return Tensor(lambda r, v: np.multiply(v, v), [x], x.dtype, x.shape, "Square")


def sqrt(x, name=None):
    x = convert_to_tensor(x)

    def fn(r, v):
        with np.errstate(invalid="ignore"):
            return np.sqrt(v)
    return Tensor(fn, [x], x.dtype, x.shape, "Sqrt")


def zeros_like(x, name=None):
    x = convert_to_tensor(x)
    return Tensor(lambda r, v: np.zeros_like(v), [x], x.dtype, x.shape, "ZerosLike")


def minimum(x, y, name=None):
    return _binary(np.minimum, x, y, "Minimum")


def identity(x, name=None):
    x = convert_to_tensor(x)
    return Tensor(lambda r, v: v, [x], x.dtype, x.shape, "Identity")


def group(*inputs, **kw):
    flat = []
    for i in inputs:
        flat.extend(i) if isinstance(i, (list, tuple)) else flat.append(i)
    flat = [f for f in flat if f is not None]
    if REVERSE_UNORDERED:          # tf.group imposes no order on its inputs: an adversarial executor may run them backwards
        flat = flat[::-1]

    def fn(r, *vals):
        return None
    return Tensor(fn, flat, None, (), kw.get("name") or "group")


@contextlib.contextmanager
def control_dependencies(ops):
    _control_stack.append(list(ops))
    try:
        yield
    finally:
        _control_stack.pop()


def cond(pred, true_fn=None, false_fn=None, name=None):
    t_out, f_out = true_fn(), false_fn()       # both branches are BUILT; only one is RUN

    def fn(r, p):
        return (t_out if bool(p) else f_out).eval(r)
    out = Tensor(fn, [convert_to_tensor(pred)], None, (), "cond")
    return out


def gradients(ys, xs, **kw):
    """The model's backward pass is not on this path: gradients are placeholders fed per run."""
    outs = []
    for x in xs:
        ph = placeholder(x.dtype, x.shape, name="grad/" + x.name)
        outs.append(ph)
    return outs


def placeholder(dtype, shape=(), name=None):
    t = Tensor(None, (), dtype, shape, name or "Placeholder")

    def ev(run, _t=t):
        if _t not in run.feeds:
            raise KeyError(f"placeholder {_t.name} was not fed")
        return np.asarray(run.feeds[_t], dtype=dtype.np)
    t.eval = ev
    _g.placeholders.append(t)
    return t


def l2_loss(t):
    """sum(t**2)/2.  TF's reduction order is unspecified; defined here as the correctly rounded
    sum (fp64 accumulation, one rounding) -- the same definition the oracle uses."""
    t = convert_to_tensor(t)

    def fn(r, v):
        x = np.asarray(v, dtype=np.float64).ravel()
        return np.float32(float(np.dot(x, x)) / 2.0)
    return Tensor(fn, [t], t.dtype, (), "L2Loss")


def global_norm(t_list, name=None):
    """TF 1.15 clip_ops.global_norm: sqrt(2 * reduce_sum(stack([l2_loss(t) ...])))."""
    halves = [l2_loss(t) for t in t_list if t is not None]

    def fn(r, *vals):
        acc = np.float32(0.0)
        for v in vals:                          # Pack + Sum: sequential fp32
            acc = np.float32(acc + v)
        return np.sqrt(np.float32(acc * np.float32(2.0)))
    return Tensor(fn, halves, float32, (), "global_norm")


def clip_by_global_norm(t_list, clip_norm, use_norm=None, name=None):
    """TF 1.15 clip_ops.clip_by_global_norm:
        scale_for_finite = clip_norm * minimum(1.0 / use_norm, 1.0 / clip_norm)
        scale = scale_for_finite + (use_norm - use_norm)
        values_clipped = [identity(v * scale) ...]"""
    t_list = list(t_list)
    if use_norm is None:
        use_norm = global_norm(t_list)
    one = constant(1.0, dtype=use_norm.dtype)
    scale_for_finite = clip_norm * minimum(1.0 / use_norm, one / clip_norm)
    scale = scale_for_finite + (use_norm - use_norm)
    clipped = [None if v is None else identity(v * scale) for v in t_list]
    return clipped, use_norm


# ------------------------------------------------------------------------------------ tf.train etc.
def _polynomial_decay(learning_rate, global_step, decay_steps, end_learning_rate=0.0001, power=1.0,
                      cycle=False, name=None):
    """TF 1.15 learning_rate_schedule.PolynomialDecay.__call__ (cycle=False branch)."""
    if cycle:
        raise NotImplementedError("cycle=True is not used by the reference")
    lr = convert_to_tensor(learning_rate)
    dtype = lr.dtype
    end_lr = cast(end_learning_rate, dtype)
    pw = cast(power, dtype)
    gs = cast(global_step, dtype)
    ds = cast(decay_steps, dtype)
    gs = minimum(gs, convert_to_tensor(decay_steps, dtype))
    p = gs / ds
    one_minus_p = 1 - p
    powed = Tensor(lambda r, b, e: np.asarray(np.power(b, e), dtype=dtype.np), [one_minus_p, pw], dtype, (), "Pow")
    return multiply(lr - end_lr, powed) + end_lr


class Optimizer:
    """tf.train.Optimizer: only what AdamWeightDecayOptimizer.__init__ calls."""

    def __init__(self, use_locking, name):
        self._use_locking = use_locking
        self._name = name


class AdamOptimizer(Optimizer):
    """``tf.train.AdamOptimizer`` / ``tf.compat.v1.train.AdamOptimizer`` as TF 1.15 runs it on dense fp32
    variables (python/training/adam.py + core/kernels/training_ops.cc, ApplyAdam, use_nesterov=False).
    RESTATEMENT of TensorFlow (not of the reference): listed in tests/golden/MANIFEST.json.

    adam.py:  _create_slots: non-slot variables beta1_power = beta1, beta2_power = beta2; slots m, v = 0
              _prepare:      lr, beta1, beta2, epsilon -> tensors (cast to the variable dtype at use)
              _apply_dense:  training_ops.apply_adam(var, m, v, beta1_power, beta2_power, lr, beta1, beta2, eps, grad)
              _finish:       after all updates: beta1_power *= beta1; beta2_power *= beta2
    training_ops.cc (ApplyAdam functor, T = float):
              alpha = lr * sqrt(T(1) - beta2_power) / (T(1) - beta1_power)
              m += (grad - m) * (T(1) - beta1)
              v += (grad.square() - v) * (T(1) - beta2)
              var -= (m * alpha) / (v.sqrt() + epsilon)
    apply_gradients(..., global_step=None) leaves the step counter alone (02:61 relies on it)."""

    def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8, use_locking=False, name="Adam"):
        Optimizer.__init__(self, use_locking, name)
        self._lr, self._beta1, self._beta2, self._epsilon = learning_rate, beta1, beta2, epsilon
        self._slots = {}
        self._beta1_power = self._beta2_power = None

    def get_slot(self, var, name):
        return self._slots[(id(var), name)]

    def _get_beta_accumulators(self):
        return self._beta1_power, self._beta2_power

    def apply_gradients(self, grads_and_vars, global_step=None, name=None):
        pairs = [(g, v) for g, v in grads_and_vars if g is not None]      # optimizer.py: vars with no grad are skipped
        if not pairs:
            raise ValueError("No gradients provided for any variable")
        if self._beta1_power is None:
            self._beta1_power = Variable(np.float32(self._beta1), trainable=False, name=f"{self._name}/beta1_power", dtype=float32)
            self._beta2_power = Variable(np.float32(self._beta2), trainable=False, name=f"{self._name}/beta2_power", dtype=float32)
        f32 = np.float32
        lr_t = convert_to_tensor(self._lr, float32) if not isinstance(self._lr, Tensor) else self._lr
        b1, b2, eps = f32(self._beta1), f32(self._beta2), f32(self._epsilon)
        b1p, b2p = self._beta1_power, self._beta2_power
        updates = []
        for g, var in pairs:
            base = var.name.split(":")[0]
            for sl in ("m", "v"):
                if (id(var), sl) not in self._slots:
                    self._slots[(id(var), sl)] = Variable(np.zeros(var.value.shape, np.float32), trainable=False,
                                                          name=f"{base}/{self._name}" + ("" if sl == "m" else "_1"), dtype=float32)
            m, v = self._slots[(id(var), "m")], self._slots[(id(var), "v")]

            def fn(r, grad, lr, _var=var, _m=m, _v=v):
                grad = np.asarray(grad, dtype=f32)
                one = f32(1.0)
                with np.errstate(divide="ignore", invalid="ignore"):
                    alpha = f32(f32(f32(lr) * np.sqrt(f32(one - f32(b2p.value)))) / f32(one - f32(b1p.value)))
                    _m.value = np.add(_m.value, np.multiply(np.subtract(grad, _m.value, dtype=f32), f32(one - b1), dtype=f32), dtype=f32)
                    _v.value = np.add(_v.value, np.multiply(np.subtract(np.multiply(grad, grad, dtype=f32), _v.value, dtype=f32),
                                                            f32(one - b2), dtype=f32), dtype=f32)
                    _var.value = np.subtract(_var.value, np.divide(np.multiply(_m.value, alpha, dtype=f32),
                                                                   np.add(np.sqrt(_v.value, dtype=f32), eps, dtype=f32), dtype=f32), dtype=f32)
                return None
            updates.append(Tensor(fn, [convert_to_tensor(g, float32), lr_t], None, (), "ApplyAdam"))
        with control_dependencies(updates):                        # _finish
            up1 = b1p.assign(b1p * b1)
            up2 = b2p.assign(b2p * b2)
        ops = updates + [up1, up2]
        if global_step is not None:
            with control_dependencies(ops):
                ops = ops + [global_step.assign_add(1)]
        return group(*ops, name=name or self._name)


def assign_add(ref, value, use_locking=None, name=None):
    return ref.assign_add(value)


def _get_or_create_global_step():
    if _g.global_step is None:
        _g.global_step = Variable(np.int64(0), trainable=False, name="global_step", dtype=int64)
    return _g.global_step


train = types.SimpleNamespace(
    Optimizer=Optimizer,
    AdamOptimizer=AdamOptimizer,
    polynomial_decay=_polynomial_decay,
    get_or_create_global_step=_get_or_create_global_step,
    get_global_step=lambda: _g.global_step,
)
import sys as _sys_mod
compat = types.SimpleNamespace(v1=_sys_mod.modules[__name__])       # `tf.compat.v1.<anything>` is this module
math = types.SimpleNamespace(
    equal=lambda x, y, name=None: _binary(np.equal, x, y, "Equal", out_dtype=bool_),
)


def equal(x, y, name=None):
    return _binary(np.equal, x, y, "Equal", out_dtype=bool_)


# ---------------------------------------------------------------------------------- tf.load_op_library
class _GaccumOps:
    """What ``tf.load_op_library("libgaccum_tf.so")`` returns, emulated: the ``GaccumStep`` node of
    tf_shim/gaccum_tf_op.cc with the semantics of the C ABI's ``gaccum_step`` (include/gaccum.h), evaluated with the
    CPU oracle's per-op functions on the packed slabs.  TEST INFRASTRUCTURE: it lets tests execute the Python half
    of the TensorFlow shim (graph wiring, variable creation, ordering of the scalar updates) without TensorFlow."""

    @staticmethod
    def gaccum_step(params, grads, accum, m, v, global_step, lr, beta_powers, accum_n, variant, beta1, beta2, epsilon,
                    weight_decay_rate, clip_norm, decay_mask, name=None, **unused):
        import os as _os
        import sys as _sys
        _oracle = _os.path.dirname(_os.path.dirname(_os.path.dirname(_os.path.abspath(__file__))))
        if _oracle not in _sys.path:
            _sys.path.insert(0, _oracle)
        import oracle_np as onp
        n = len(params)
        b1, b2, eps, wd, clip = (float(x) for x in (beta1, beta2, epsilon, weight_decay_rate, clip_norm))   # str or float attrs
        sizes = [int(np.prod(p.value.shape)) for p in params]
        offs, o = [], 0
        for sz in sizes:
            offs.append(o)
            o += (sz + 31) // 32 * 32
        f32 = np.float32

        def fn(r, *vals):
            gs, step, lr_v, bp = vals[:n], int(vals[n]), f32(vals[n + 1]), np.asarray(vals[n + 2], dtype=f32)
            A, M, V = accum.value.copy(), m.value.copy(), v.value.copy()
            view = lambda S, i: S[offs[i]:offs[i] + sizes[i]].reshape(params[i].value.shape)
            for i in range(n):
                if gs[i] is not None:
                    view(A, i)[...] = np.add(view(A, i), np.asarray(gs[i], dtype=f32), dtype=f32)      # optimization.py:81,93
            if int(np.int32(np.int64(step))) % int(accum_n) == 0:                                      # :77,91 pre-increment
                normalized = [np.divide(np.multiply(f32(1.0), view(A, i), dtype=f32), f32(accum_n), dtype=f32) for i in range(n)]
                if clip > 0:
                    s_ = onp.clip_scale(onp.global_norm(normalized), clip)
                    normalized = [np.multiply(x, s_, dtype=f32) for x in normalized]
                for i in range(n):
                    if int(variant) == 0:
                        p2, m2, v2 = onp.adam_weight_decay_update(params[i].value, view(M, i), view(V, i), normalized[i], lr_v,
                                                                  b1, b2, eps, wd, bool(decay_mask[i]))
                    else:
                        p2, m2, v2 = onp.adam_update(params[i].value, view(M, i), view(V, i), normalized[i], lr_v, b1, b2, eps,
                                                     f32(bp[0]), f32(bp[1]))
                    params[i].value = np.asarray(p2, dtype=f32)
                    view(M, i)[...] = m2; view(V, i)[...] = v2
                    view(A, i)[...] = f32(0.0)
            accum.value, m.value, v.value = A, M, V
            return None
        ins = [convert_to_tensor(g) for g in grads] + [convert_to_tensor(global_step), convert_to_tensor(lr), convert_to_tensor(beta_powers)]
        return Tensor(fn, ins, None, (), name or "GaccumStep")


def load_op_library(path):
    return _GaccumOps()


def _no_tpu(*a, **k):
    raise NotImplementedError("tf.contrib.tpu.CrossShardOptimizer: TPU path is out of scope")


contrib = types.SimpleNamespace(tpu=types.SimpleNamespace(CrossShardOptimizer=_no_tpu))


class Session:
    def run(self, fetches, feed_dict=None):
        run = _Run(dict(feed_dict or {}))
        if isinstance(fetches, (list, tuple)):
            return [f.eval(run) for f in fetches]
        return fetches.eval(run)

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False
