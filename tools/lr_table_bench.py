"""What a learning-rate table (gaccum_plan_set_lr_table) costs a device-scheduled train op against the formula it
replaces, on BERT-Small and BERT-Large shapes, for the AdamWeightDecay clip-apply and for LAMB, N = 4.  Two arms, the
same kernels each time:

  formula  device_schedule=ScheduleConfig: every CTA's prologue evaluates create_optimizer's schedule (schedule_lr)
  table    device_schedule=LrTable of the same values: every CTA's prologue loads table[min(g, L - 1)] instead

Both arms hold the same learning rates, so they do the same work; the table adds one dependent 4-byte load per CTA.
Two measurements, each with CUDA events:
  eager  every launch of a window on its own (the apply, the window's first accumulate, the other accumulates);
  graph  one captured window (3 accumulates + the apply) replayed, the way a device-scheduled run is driven.
Every arm keeps --sets independent state sets and the timed launches rotate through them, so no launch finds its inputs
in L2; arms alternate window by window, so clock and power drift hit them alike.  The GPU's name and power limit are
printed with the numbers.

    python tools/lr_table_bench.py [--reps 100] [--sets 3] [--models bert_small,bert_large] [--json OUT]
"""
import argparse
import gc
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np
import torch

import gaccum_b200 as g
from gaccum_b200._lib import ScheduleConfig
from gaccum_b200.manifests import MANIFESTS
from gaccum_b200.train_op import GaccumTrainOp, LrTable
from loss_scale_bench import gpu_info

N = 4
HP = {"adamw": g.HParams.bert, "lamb": g.HParams.lamb}
SCHED = dict(init_lr=1e-4, num_train_steps=100000, num_warmup_steps=10000)
ARMS = ("formula", "table")
WARM = 5


def make_arm(man, sets, gen, variant, arm, table):
    names = [n for n, _ in man]
    out = []
    for _ in range(sets):
        params = [torch.randn(s, device="cuda", generator=gen) * 0.02 for _, s in man]
        grads = [torch.randn(s, device="cuda", generator=gen) * 1e-3 for _, s in man]
        ds = ScheduleConfig(**SCHED) if arm == "formula" else table
        op = GaccumTrainOp(params, names, HP[variant](), N, None, device_schedule=ds)
        # bind() keeps only the pointers: the gradients must outlive every launch and graph that reads them
        out.append((op, op.bind(grads), grads))
    return out


def summary(t):
    t = np.array(t)
    return {"median_us": float(np.median(t)), "p10_us": float(np.percentile(t, 10)),
            "p90_us": float(np.percentile(t, 90)), "n": int(t.size)}


def run_model(name, variant, reps, sets, gen, info, table):
    man = MANIFESTS[name]()
    P = sum(int(np.prod(s)) for _, s in man)
    arms = {k: make_arm(man, sets, gen, variant, k, table) for k in ARMS}
    kinds = ("apply", "first_accumulate", "accumulate")
    ev = []
    for rep in range(reps + WARM):                       # eager windows, launch by launch
        for s in range(sets):
            for k in ARMS:
                op, ptrs, _ = arms[k][s]
                for j in range(N):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    op.run_bound(ptrs)
                    e1.record()
                    if rep >= WARM:
                        ev.append((k, kinds[min(j, 2)], e0, e1))
    torch.cuda.synchronize()
    t = {(k, kind): [] for k in ARMS for kind in kinds}
    for k, kind, e0, e1 in ev:
        t[(k, kind)].append(e0.elapsed_time(e1) * 1e3)
    graphs = {}
    gc.collect()
    torch.cuda.synchronize()
    for k in ARMS:                                       # one window per state set, captured at a window start
        for s in range(sets):
            op, ptrs, _ = arms[k][s]
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(N):
                    op.run_bound(ptrs)
            graphs[(k, s)] = graph
    torch.cuda.synchronize()
    gev = []
    for rep in range(reps + WARM):
        for s in range(sets):
            for k in ARMS:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                graphs[(k, s)].replay()
                e1.record()
                if rep >= WARM:
                    gev.append((k, e0, e1))
    torch.cuda.synchronize()
    gt = {k: [] for k in ARMS}
    for k, e0, e1 in gev:
        gt[k].append(e0.elapsed_time(e1) * 1e3)
    # both arms ran the same steps with the same rates, and no launch was refused (schedule_state raises)
    steps = {k: arms[k][0][0].schedule_state()["global_step"] for k in ARMS}
    lrs = {k: arms[k][0][0].stats()["lr"] for k in ARMS}
    assert steps["formula"] == steps["table"] == N * (2 * (reps + WARM)) and lrs["formula"] == lrs["table"], (steps, lrs)
    row = {"model": name, "optimizer": variant, "P": P, "gpu": info, "N": N,
           "eager": {k: {kind: summary(t[(k, kind)]) for kind in kinds} for k in ARMS},
           "graph_window": {k: summary(gt[k]) for k in ARMS}}
    row["table_over_formula"] = {kind: row["eager"]["table"][kind]["median_us"] / row["eager"]["formula"][kind]["median_us"]
                                 for kind in kinds}
    row["table_over_formula"]["graph_window"] = (row["graph_window"]["table"]["median_us"]
                                                 / row["graph_window"]["formula"]["median_us"])
    del arms, graphs
    gc.collect()
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--sets", type=int, default=3)
    ap.add_argument("--models", default="bert_small,bert_large")
    ap.add_argument("--optimizers", default="adamw,lamb")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    if a.sets < 1 or a.reps < 1:
        sys.exit("--sets and --reps must be >= 1")
    gen = torch.Generator(device="cuda").manual_seed(0)
    info = gpu_info()
    vals = [g.learning_rate(SCHED["init_lr"], SCHED["num_train_steps"], SCHED["num_warmup_steps"], s)
            for s in range(SCHED["num_train_steps"])]
    table = LrTable(vals)
    print(f"GPU: {info}; {a.sets} state sets per arm; {a.reps} windows per set and arm; N = {N}")
    results = []
    for name in a.models.split(","):
        for variant in a.optimizers.split(","):
            row = run_model(name, variant, a.reps, a.sets, gen, info, table)
            results.append(row)
            r = row["table_over_formula"]
            print(f"{name:10s} {variant:5s} " + " | ".join(
                f"{kind} {row['eager']['formula'][kind]['median_us']:8.1f} -> {row['eager']['table'][kind]['median_us']:8.1f} us"
                for kind in ("apply", "first_accumulate", "accumulate"))
                + f" | graph window {row['graph_window']['formula']['median_us']:8.1f} -> "
                  f"{row['graph_window']['table']['median_us']:8.1f} us | table/formula "
                + " ".join(f"{k} {v:.3f}" for k, v in r.items()))
    print(json.dumps(results))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
