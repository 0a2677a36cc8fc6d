"""What dividing each window by its total weight W (gaccum_plan_set_window_weight) costs on the apply step, on BERT-Small
and BERT-Large shapes, for the AdamWeightDecay clip-apply and for LAMB (clipping at 1.0, as create_optimizer does), N = 4.
Three arms, the same kernel each time:

  unweighted  a train op without the block: c = a'/N, N = 4 (an exact multiply by 1/4)
  w4          window_weight=True with W = 4: the power-of-two path (an exact multiply by 1/W)
  w148        window_weight=True with W = 4*37: the division path (__fdiv_rn per element)

Timed with CUDA events around the apply launch alone; the weighted arms set W (a one-element fill) before the first
event.  Every arm keeps --sets independent state sets and the timed launches rotate through them, so no launch finds its
inputs in L2; arms alternate launch by launch, so clock and power drift hit them alike.  The GPU's name and power limit
are printed with the numbers.

    python tools/window_weight_bench.py [--reps 200] [--sets 3] [--models bert_small,bert_large] [--arms ...] [--json OUT]
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
from gaccum_b200.manifests import MANIFESTS
from gaccum_b200.train_op import GaccumTrainOp
from loss_scale_bench import gpu_info

N = 4
HP = {"adamw": g.HParams.bert, "lamb": g.HParams.lamb}
ARMS = {"unweighted": None, "w4": 4.0, "w148": 4.0 * 37.0}


def make_arm(man, sets, gen, variant, weight):
    names = [n for n, _ in man]
    arm = []
    for _ in range(sets):
        params = [torch.randn(s, device="cuda", generator=gen) * 0.02 for _, s in man]
        grads = [torch.randn(s, device="cuda", generator=gen) * 1e-3 for _, s in man]
        op = GaccumTrainOp(params, names, HP[variant](), N, lambda s: 1e-4, window_weight=weight is not None)
        arm.append((op, op.bind(grads)))
    return arm


def summary(t, bytes_per_param, P):
    t = np.array(t)
    med = float(np.median(t))
    return {"median_us": med, "p10_us": float(np.percentile(t, 10)), "p90_us": float(np.percentile(t, 90)),
            "GB_per_s": bytes_per_param * P / med / 1e3, "n": int(t.size)}


def run_model(name, variant, reps, sets, gen, info, kinds):
    man = MANIFESTS[name]()
    P = sum(int(np.prod(s)) for _, s in man)
    arms = {k: make_arm(man, sets, gen, variant, ARMS[k]) for k in kinds}
    bpp = float(arms[kinds[0]][0][0].plan.algorithmic_bytes(True)) / P
    ev = []
    for rep in range(reps + 5):
        for s in range(sets):
            for k in kinds:
                w = ARMS[k]
                op, table = arms[k][s]
                if w is not None:
                    op.window_weight.fill_(w)              # the window's total, outside the timed region
                op.global_step = 0                         # g = 0: the apply branch
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                op.run_bound(table)
                e1.record()
                if rep >= 5:
                    ev.append((k, e0, e1))
    torch.cuda.synchronize()
    for k in kinds:                                       # every weighted launch read W and reset it
        if ARMS[k] is not None:
            st = arms[k][0][0].window_weight_state()
            assert st == {"weight": 0.0, "last_weight": ARMS[k]}, st
    t = {k: [] for k in kinds}
    for k, e0, e1 in ev:
        t[k].append(e0.elapsed_time(e1) * 1e3)
    row = {"model": name, "optimizer": variant, "P": P, "gpu": info,
           "apply": {k: summary(t[k], bpp, P) for k in kinds}}
    for k in ("w4", "w148"):
        if k in kinds and "unweighted" in kinds:
            row[f"{k}_over_unweighted"] = row["apply"][k]["median_us"] / row["apply"]["unweighted"]["median_us"]
    del arms
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--sets", type=int, default=3)
    ap.add_argument("--models", default="bert_small,bert_large")
    ap.add_argument("--optimizers", default="adamw,lamb")
    ap.add_argument("--arms", default=",".join(ARMS))
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    gen = torch.Generator(device="cuda").manual_seed(0)
    info = gpu_info()
    kinds = a.arms.split(",")
    print(f"GPU: {info}; {a.sets} state sets per arm; {a.reps} applies per set and arm; N = {N}")
    results = []
    for name in a.models.split(","):
        for variant in a.optimizers.split(","):
            row = run_model(name, variant, a.reps, a.sets, gen, info, kinds)
            results.append(row)
            r = row["apply"]
            print(f"{name:10s} {variant:5s} " + " | ".join(
                f"{k} {r[k]['median_us']:9.1f} us (p10 {r[k]['p10_us']:.1f}, p90 {r[k]['p90_us']:.1f})" for k in r)
                + "".join(f" | {k}/unweighted {row[k + '_over_unweighted']:.3f}" for k in ("w4", "w148")
                          if k + "_over_unweighted" in row))
    print(json.dumps(results))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
