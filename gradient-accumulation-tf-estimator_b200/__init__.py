"""gradient-accumulation-tf-estimator_b200 -- the H100-native accumulate-then-apply train_op.

One hot path of hpandana/gradient-accumulation-tf-estimator, rebuilt for sm_90a:
``create_optimizer``'s tf.cond train_op (reference optimization.py:25-104) with
``AdamWeightDecayOptimizer.apply_gradients`` (optimization.py:128-177) and the plain-Adam variant
of the distributedExample scripts, as hand-written CUDA kernels behind a C ABI
(``include/gaccum.h`` / ``csrc/libgaccum.so``).  Import it as ``gaccum_b200``.

There is no CPU fallback anywhere in this package: importing works without a GPU (layout and
scalar host logic are usable), every compute call raises ``GaccumError`` without one.
"""
from ._lib import (ADAM, ADAM_WEIGHT_DECAY, GaccumError, HParams, Plan, StepArgs, decay_mask,
                   device_count, is_apply_step, learning_rate, lib_path, version)

__all__ = ["ADAM", "ADAM_WEIGHT_DECAY", "GaccumError", "HParams", "Plan", "StepArgs", "decay_mask",
           "device_count", "is_apply_step", "learning_rate", "lib_path", "version"]
