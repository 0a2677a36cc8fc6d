#!/usr/bin/env python
"""The reference's distributedExample/02 (single worker) and /04 (multi worker) recipes on the
H100 train_op -- a thin launch script, not a re-implementation of tf.estimator.

  python examples/mnist_gaccum.py --steps 200                       # 02: 1 worker, batch 100, N=2
  torchrun --nproc-per-node 2 examples/mnist_gaccum.py --steps 200  # 04: 2 workers, batch 50 each

Model: Conv2D(32,3) -> MaxPool -> Flatten -> Dense(64) -> Dense(10)  (02:22-28), loss
sum(xent) / BATCH_SIZE [/ num_workers] (02:43-45, 04:46), tf.train.AdamOptimizer(1e-4) without
clipping (02:41,59-61), gradient_accumulation_multiplier from params (02:48,110).  MNIST files are
not shipped with the reference (README.md:128) and there is no network here: inputs are synthetic
MNIST-shaped tensors with a learnable rule, so the loss still has to fall.
"""
import argparse
import os
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaccum_b200 import graph, optimization  # noqa: E402

TF_NAMES = {"conv.weight": "conv2d/kernel", "conv.bias": "conv2d/bias", "fc1.weight": "dense/kernel",
            "fc1.bias": "dense/bias", "fc2.weight": "dense_1/kernel", "fc2.bias": "dense_1/bias"}


class MnistCnn(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(1, 32, 3)
        self.fc1 = nn.Linear(32 * 13 * 13, 64)
        self.fc2 = nn.Linear(64, 10)

    def forward(self, x):
        x = F.max_pool2d(F.relu(self.conv(x)), 2)
        return self.fc2(F.relu(self.fc1(x.flatten(1))))


def synthetic_batch(batch, gen, dev):
    y = torch.randint(0, 10, (batch,), device=dev, generator=gen)
    x = torch.randn(batch, 1, 28, 28, device=dev, generator=gen) * 0.3
    for k in range(10):                       # class k lights up a 2x28 stripe: learnable
        x[y == k, :, 2 * k + 4:2 * k + 6, :] += 1.0
    return x, y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--batch-size", type=int, default=100)          # 02:101
    ap.add_argument("--accum", type=int, default=2)                 # 02:110
    ap.add_argument("--lr", type=float, default=1e-4)               # 02:110
    args = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    group = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
        group = True
    torch.manual_seed(19830610)                                     # 02:106 tf_random_seed
    model = MnistCnn().to(dev)
    graph.reset_default_graph()
    graph.register_module(model, lambda n: TF_NAMES[n])
    per_worker = args.batch_size // world                           # 04:124 BATCH_SIZE per worker
    gen = torch.Generator(device=dev); gen.manual_seed(1000 * rank + 7)
    state = {}

    def loss_fn():
        x, y = synthetic_batch(per_worker, gen, dev)
        loss = F.cross_entropy(model(x), y, reduction="sum") * (1.0 / per_worker / world)   # 02:45 / 04:46
        state["loss"] = loss.detach() * world
        return loss

    train_op = optimization.gradient_accumulation_train_op(
        loss_fn, optimization.AdamOptimizer(learning_rate=args.lr), args.accum, process_group=group)
    for step in range(args.steps):
        train_op.run()
        if rank == 0 and (step % 50 == 0 or step == args.steps - 1):
            print(f"global_step {int(graph.get_global_step())}  loss {float(state['loss']):.4f}")
    if world > 1:
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
