#!/usr/bin/env python
"""The reference's another-example.py recipe (a custom-Estimator regressor whose ``_train_op_fn`` accumulates gradients,
another-example.py:126-155) on the H100 train_op -- a thin launch script, not a re-implementation of tf.estimator.

  python examples/another_example.py --steps 600 --model-dir /tmp/housing           # fresh run (RESUME_TRAINING = False, :323-325)
  python examples/another_example.py --steps 600 --model-dir /tmp/housing --resume  # continue from model_dir (:326-327)

What is kept from the reference: the model (Dense 16 -> 8 -> 4 -> 1 with ReLU, hidden_units :276, :110-116), the
regression head's loss (mean squared error over the batch), BATCH_SIZE 59 (:272), gradient_accumulation_multiplier 3
(:275), ``tf.train.AdamOptimizer()`` with its DEFAULT learning rate 1e-3 (:135), no clipping, ``global_step=None`` inside
apply_gradients and one increment per micro-step (:142, :153), tf_random_seed 19830610 (:285), and a ``model_dir`` that
holds TensorFlow-format checkpoints under the variable names a Saver over the reference's graph would use
(``dense/kernel``, ``dense/kernel/Adam``, ``Variable`` ..., ``beta1_power``, ``global_step``), so ``--resume`` works
mid-window.  What is not: the housing CSV and its feature columns (no data ships with the reference, no network here);
inputs are synthetic 13-feature rows with a fixed nonlinear target, so the loss still has to fall.
"""
import argparse
import os
import shutil
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaccum_b200 import graph, optimization, tf_checkpoint  # noqa: E402

HIDDEN_UNITS = [16, 8, 4]          # another-example.py:276
BATCH_SIZE = 59                    # :272
FEATURES = 13


def tf_name(torch_name: str) -> str:
    """net.0.kernel -> dense/kernel, net.2.bias -> dense_1/bias, ... (Keras' default layer names)"""
    idx, kind = torch_name.split(".")[1:]
    layer = int(idx) // 2
    return ("dense" if layer == 0 else f"dense_{layer}") + "/" + kind


class Dense(nn.Module):
    """tf.keras.layers.Dense: kernel [in, out] (TensorFlow's layout, so checkpoints hold what a TF run would), Glorot
    uniform kernel, zero bias."""

    def __init__(self, n_in, n_out):
        super().__init__()
        limit = (6.0 / (n_in + n_out)) ** 0.5
        self.kernel = nn.Parameter((torch.rand(n_in, n_out) * 2 - 1) * limit)
        self.bias = nn.Parameter(torch.zeros(n_out))

    def forward(self, x):
        return x @ self.kernel + self.bias


class Regressor(nn.Module):
    def __init__(self):
        super().__init__()
        layers, prev = [], FEATURES
        for h in HIDDEN_UNITS:                                                      # :110-113
            layers += [Dense(prev, h), nn.ReLU()]
            prev = h
        layers.append(Dense(prev, 1))                                              # :116
        self.net = nn.Sequential(*layers)

    def forward(self, x):
        return self.net(x)


def synthetic_batch(gen, dev, global_step):
    gen.manual_seed(19830610 + global_step)           # the batch is a function of the micro-step: a resumed run sees the same data
    x = torch.randn(BATCH_SIZE, FEATURES, device=dev, generator=gen)
    y = 1.0 + 0.5 * x[:, :1] - 0.25 * x[:, 1:2] * x[:, 2:3] + 0.3 * torch.relu(x[:, 3:4])
    return x, y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=600, help="micro-steps to run in this invocation")
    ap.add_argument("--accum", type=int, default=3)                                # :275
    ap.add_argument("--model-dir", default=None)
    ap.add_argument("--resume", action="store_true")                               # RESUME_TRAINING, :209
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(19830610)                                                    # :285
    model = Regressor().to(dev)
    graph.reset_default_graph()
    graph.register_module(model, tf_name)
    state = {}
    gen = torch.Generator(device=dev)

    def loss_fn():
        x, y = synthetic_batch(gen, dev, int(graph.get_global_step()))
        loss = torch.mean((model(x) - y) ** 2)                                      # regression_head: MSE, SUM_OVER_BATCH_SIZE
        state["loss"] = loss.detach()
        return loss

    train_op = optimization.gradient_accumulation_train_op(loss_fn, optimization.AdamOptimizer(), args.accum)   # :135: default lr 1e-3
    if args.model_dir and not args.resume:
        shutil.rmtree(args.model_dir, ignore_errors=True)                          # "Removing previous artifacts..." :324-325
    if args.model_dir and args.resume:
        prefix = tf_checkpoint.restore(args.model_dir, train_op)
        print(f"Resuming training... restored {os.path.basename(prefix)}")
    for step in range(args.steps):
        train_op.run()
        g = int(graph.get_global_step())
        if step % 100 == 0 or step == args.steps - 1:
            print(f"global_step {g}  loss {float(state['loss']):.4f}")
    if args.model_dir:
        os.makedirs(args.model_dir, exist_ok=True)
        print(f"saved {os.path.basename(tf_checkpoint.save(args.model_dir, train_op))}")


if __name__ == "__main__":
    main()
