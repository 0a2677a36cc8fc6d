"""Micro-steps per second of BERT-Small training at N = 4 with the schedule on the host, on the device, and as one captured
CUDA graph of a window replayed (gaccum_plan_set_device_schedule), with and without the model's forward + backward.

Arms (create_optimizer's AdamWeightDecay, clipping at 1.0, BERT's schedule):
  host    eager, host-scheduled: lr and the step on the host, one launch per micro-step
  device  eager, device-scheduled: the same launches, lr / step / beta powers read and advanced on the device
  graph   the device-scheduled op's window -- N micro-steps -- captured once and replayed

Modes:
  optimizer   the train op alone on fixed gradient buffers (what the schedule's host work and launch overhead cost)
  producer    tools/bert_producer.py's forward + backward (micro-batch 8 x 128) feeding the train op; the graph arm
              captures forward, backward and train op of the whole window

Each round times --windows windows of every arm with CUDA events, one arm after the other, so clock and power drift hit
them alike; the medians over --rounds rounds are reported with p10 / p90 and the GPU's name and power limit.

    python tools/graph_window_bench.py [--rounds 15] [--windows 8] [--modes optimizer,producer] [--json OUT]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np
import torch

import gaccum_b200 as g
from gaccum_b200 import _lib
from gaccum_b200.optimization import bert_learning_rate
from gaccum_b200.train_op import GaccumTrainOp
from bert_producer import Bert, synthetic_batch, tf_names
from loss_scale_bench import gpu_info

N = 4
SCHED = dict(init_lr=2e-5, num_train_steps=100000, num_warmup_steps=10000)
ARMS = ("host", "device", "graph")


class Arm:
    """One train op (and, in producer mode, one model) and a function that runs one window of N micro-steps."""

    def __init__(self, kind, mode, gen):
        self.kind = kind
        model = Bert("bert_small").cuda()
        named = tf_names(model)
        params = [p for _, p in named]
        for p in params:
            p.requires_grad_(mode == "producer")
        kw = {"device_schedule": _lib.ScheduleConfig(**SCHED)} if kind != "host" else {}
        self.op = GaccumTrainOp([p.data for p in params], [n for n, _ in named], g.HParams.bert(), N,
                                None if kind != "host" else bert_learning_rate(**SCHED), **kw)
        if mode == "producer":
            batches = [synthetic_batch(8, 128, "cuda", gen) for _ in range(N)]

            def micro(i):
                loss = model(*batches[i])
                grads = torch.autograd.grad(loss, params)
                self.op.run(grads)
        else:
            grads = [torch.randn(p.shape, device="cuda", generator=gen) * 1e-3 for p in params]
            table = self.op.bind(grads)

            def micro(i):
                self.op.run_bound(table)
        self.window = lambda: [micro(i) for i in range(N)]
        # warm-up window on a side stream (autograd's buffers, lazy kernel loading, the apply kernel's grid fit)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            self.window()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = None
        if kind == "graph":
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self.window()
            torch.cuda.synchronize()

    def run(self, windows):
        for _ in range(windows):
            if self.graph is not None:
                self.graph.replay()
            else:
                self.window()


def run_mode(mode, rounds, windows, gen, info):
    arms = {k: Arm(k, mode, gen) for k in ARMS}
    times = {k: [] for k in ARMS}
    for r in range(rounds + 2):
        for k in ARMS:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            arms[k].run(windows)
            e1.record()
            e1.synchronize()
            if r >= 2:
                times[k].append(e0.elapsed_time(e1) / 1e3)
    steps = windows * N
    out = {"mode": mode, "N": N, "gpu": info, "micro_steps_per_round": steps}
    for k in ARMS:
        rate = steps / np.array(times[k])
        out[k] = {"median_micro_steps_per_s": float(np.median(rate)), "p10": float(np.percentile(rate, 10)),
                  "p90": float(np.percentile(rate, 90)), "n": int(rate.size)}
    for k in ("device", "graph"):
        out[f"{k}_over_host"] = out[k]["median_micro_steps_per_s"] / out["host"]["median_micro_steps_per_s"]
    # every arm ran the same number of micro-steps: the device counters agree with the host's
    gs = {k: arms[k].op.global_step for k in ARMS}
    assert len(set(gs.values())) == 1, gs
    del arms
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--windows", type=int, default=8)
    ap.add_argument("--modes", default="optimizer,producer")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    gen = torch.Generator(device="cuda").manual_seed(0)
    info = gpu_info()
    print(f"GPU: {info}; BERT-Small, N = {N}; {a.rounds} rounds x {a.windows} windows per arm")
    results = []
    for mode in a.modes.split(","):
        row = run_mode(mode, a.rounds, a.windows, gen, info)
        results.append(row)
        print(f"{mode:9s} " + " | ".join(
            f"{k} {row[k]['median_micro_steps_per_s']:8.1f}/s (p10 {row[k]['p10']:.1f}, p90 {row[k]['p90']:.1f})"
            for k in ARMS) + f" | device/host {row['device_over_host']:.3f} | graph/host {row['graph_over_host']:.3f}")
    print(json.dumps(results))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
