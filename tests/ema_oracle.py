"""numpy oracle of the exponential moving average the apply step keeps (include/gaccum.h, gaccum_ema_config).

TF1 ``tf.train.ExponentialMovingAverage(decay, num_updates=...)`` with ``zero_debias=False``, one correctly rounded fp32
op per TF op -- one numpy ufunc with ``dtype=float32`` each:

    d = fp32(decay);  num_updates mode: nf = fp32(n), d = min(d, (1 + nf) / (10 + nf));  c = 1 - d
    e = e - (e - p) * c

once per APPLIED window, after the update, on every tensor.  ``EmaReferenceTrainOp`` layers it on any reference train op
of this repository (``oracle_np.ReferenceTrainOp``, ``composed_oracle.ComposedReferenceTrainOp``, the C oracle): it
averages the reference's parameters whenever a step applied and loss scaling did not skip its window.
"""
from typing import List, Sequence, Tuple

import numpy as np

F32 = np.float32


def ema_coefficients(decay: float, num_updates: bool, n: int) -> Tuple[np.float32, np.float32]:
    """(d, c = 1 - d) of the window averaged after n others."""
    d = F32(decay)                                                     # convert_to_tensor of the Python float
    if num_updates:
        nf = F32(n)                                                    # TF's cast of the counter: round to nearest
        w = np.divide(np.add(F32(1.0), nf, dtype=F32), np.add(F32(10.0), nf, dtype=F32), dtype=F32)
        d = np.minimum(d, w, dtype=F32)
    return F32(d), np.subtract(F32(1.0), d, dtype=F32)


def ema_update(e: np.ndarray, p: np.ndarray, c: np.float32) -> np.ndarray:
    """assign_moving_average: e - (e - p) * c, three fp32 ops."""
    return np.subtract(e, np.multiply(np.subtract(e, p, dtype=F32), c, dtype=F32), dtype=F32)


class Ema:
    """The averages and the state block (num_updates, decay) of gaccum_ema_state."""

    def __init__(self, weights: Sequence[np.ndarray], decay: float, num_updates: bool = False, n: int = 0):
        self.avg: List[np.ndarray] = [np.array(w, dtype=F32, copy=True) for w in weights]
        self.decay_cfg, self.num_updates_mode = decay, bool(num_updates)
        self.num_updates, self.decay = int(n), F32(0.0)

    def average(self, weights: Sequence[np.ndarray]) -> None:
        d, c = ema_coefficients(self.decay_cfg, self.num_updates_mode, self.num_updates)
        for i, w in enumerate(weights):
            self.avg[i] = ema_update(self.avg[i], np.asarray(w, dtype=F32).reshape(self.avg[i].shape), c)
        self.num_updates += 1
        self.decay = d


class EmaReferenceTrainOp:
    """A reference train op plus the moving average of its parameters."""

    def __init__(self, ref, decay: float, num_updates: bool = False):
        self.ref = ref
        self.ema = Ema(ref.params, decay, num_updates)

    def __getattr__(self, name):
        return getattr(self.ref, name)

    def run(self, grads):
        info = self.ref.run(grads)
        if info.applied and not getattr(self.ref, "last_skipped", False):
            self.ema.average(self.ref.params)
        return info
