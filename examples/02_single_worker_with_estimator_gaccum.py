#!/usr/bin/env python
"""distributedExample/02_single_worker_with_estimator_gaccum.py on the H100 train_op, keeping the
reference's structure: input_fn / model_fn(features, labels, mode, params) -> EstimatorSpec /
RunConfig / Estimator / train_and_evaluate.  Synthetic MNIST-shaped data (the MNIST files are not
shipped with the reference and there is no network here).

    python examples/02_single_worker_with_estimator_gaccum.py
"""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaccum_b200 import estimator as est, graph, optimization  # noqa: E402
from mnist_gaccum import TF_NAMES, MnistCnn, synthetic_batch  # noqa: E402  (same directory)


def input_fn(mode, num_steps, batch_size, seed=0, start=0):
    def gen():
        g = torch.Generator(device="cuda"); g.manual_seed(19830610 + seed)
        for i in range(start + num_steps):
            batch = synthetic_batch(batch_size, g, torch.device("cuda"))
            if i >= start:
                yield batch
    return gen


def model_fn(features, labels, mode, params):
    model = MnistCnn().cuda()                                         # 02:22-28
    graph.register_module(model, lambda n: TF_NAMES[n])
    logits = lambda: model(features.get())                            # 02:29
    BATCH_SIZE = params['batch_size']
    optimizer = optimization.AdamOptimizer(learning_rate=params['learning_rate'])              # 02:41
    loss = lambda: F.cross_entropy(logits(), labels.get(), reduction="sum") * (1. / BATCH_SIZE)   # 02:43-45
    train_op = optimization.gradient_accumulation_train_op(                                   # 02:47-73
        loss, optimizer, params['gradient_accumulation_multiplier'])
    accuracy = lambda: (logits().argmax(1) == labels.get()).float().mean()                    # 02:75-76
    return est.EstimatorSpec(mode=mode, loss=loss, train_op=train_op, eval_metric_ops={'accuracy': accuracy})


if __name__ == "__main__":
    OUTDIR = 'tmp/singleworkergaccum'
    import shutil
    shutil.rmtree(OUTDIR, ignore_errors=True)                         # 02:99
    BATCH_SIZE = 100                                                  # 02:101
    config = est.RunConfig(log_step_count_steps=100, tf_random_seed=19830610, model_dir=OUTDIR)    # 02:104-108
    hparams = dict({'learning_rate': 1e-3, 'batch_size': BATCH_SIZE, 'gradient_accumulation_multiplier': 2})
    classifier = est.Estimator(model_fn=model_fn, config=config, params=hparams)
    result = est.train_and_evaluate(classifier,
                                    input_fn(est.ModeKeys.TRAIN, 600, BATCH_SIZE),
                                    input_fn(est.ModeKeys.EVAL, 10, 1000, seed=1))
    for step, loss, rate in classifier.log:
        print(f"global_step {step}  loss {loss:.4f}  {rate:.0f} global_step/sec")
    print("eval:", result)
