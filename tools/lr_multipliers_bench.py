"""What per-tensor learning rates cost on the apply step, on BERT-Small and BERT-Large shapes, for the AdamWeightDecay
clip-apply and for LAMB (clipping at 1.0, as create_optimizer does).  Three arms:

  ones     one train op with a table of ones (lr_multipliers=[1] * T)
  electra  one train op with ELECTRA's layer-wise table at decay 0.8 (optimization.layerwise_lr_multipliers)
  split    the workaround without the table: one train op per learning-rate group (the embeddings, each encoder layer,
           the rest), each with its own constant lr, launched one after the other.  NOT EQUIVALENT: every group clips by
           its own global norm instead of the model's, so it computes something else; it is timed for its launch count.

Timed with CUDA events.  Every arm keeps --sets independent state sets and the timed launches rotate through them, so no
launch finds its inputs in L2; arms alternate launch by launch, so clock and power drift hit them alike.  The GPU's name
and power limit are printed with the numbers.

    python tools/lr_multipliers_bench.py [--reps 200] [--sets 3] [--models bert_small,bert_large] [--json OUT]
"""
import argparse
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np
import torch

import gaccum_b200 as g
from gaccum_b200 import optimization as opt
from gaccum_b200.manifests import MANIFESTS
from gaccum_b200.train_op import GaccumTrainOp
from loss_scale_bench import gpu_info

N = 4
DECAY = 0.8
HP = {"adamw": g.HParams.bert, "lamb": g.HParams.lamb}


def groups(names):
    """Tensor indices per learning-rate group: the embeddings, each encoder layer, everything else."""
    out = {}
    for i, n in enumerate(names):
        m = re.search(r"encoder/layer_(\d+)/", n)
        key = "embeddings" if "/embeddings/" in n else (f"layer_{m.group(1)}" if m else "rest")
        out.setdefault(key, []).append(i)
    return list(out.values())


def make_arm(man, sets, gen, variant, kind):
    names = [n for n, _ in man]
    L = 1 + max(int(m.group(1)) for n in names for m in [re.search(r"encoder/layer_(\d+)/", n)] if m)
    table = opt.lr_multipliers_for(names, opt.layerwise_lr_multipliers(DECAY, L))
    arm = []
    for _ in range(sets):
        params = [torch.randn(s, device="cuda", generator=gen) * 0.02 for _, s in man]
        grads = [torch.randn(s, device="cuda", generator=gen) * 1e-3 for _, s in man]
        if kind == "split":
            ops = []
            for idx in groups(names):
                lr = 1e-4 * table[idx[0]]
                op = GaccumTrainOp([params[i] for i in idx], [names[i] for i in idx], HP[variant](), N, lambda s, _l=lr: _l)
                ops.append((op, op.bind([grads[i] for i in idx])))
        else:
            mult = [1.0] * len(man) if kind == "ones" else table
            op = GaccumTrainOp(params, names, HP[variant](), N, lambda s: 1e-4, lr_multipliers=mult)
            ops = [(op, op.bind(grads))]
        arm.append(ops)
    return arm


def summary(t, bytes_per_param, P):
    t = np.array(t)
    med = float(np.median(t))
    return {"median_us": med, "p10_us": float(np.percentile(t, 10)), "p90_us": float(np.percentile(t, 90)),
            "GB_per_s": bytes_per_param * P / med / 1e3, "n": int(t.size)}


def run_model(name, variant, reps, sets, gen, info):
    man = MANIFESTS[name]()
    P = sum(int(np.prod(s)) for _, s in man)
    kinds = ("ones", "electra", "split")
    arms = {k: make_arm(man, sets, gen, variant, k) for k in kinds}
    bpp = float(arms["ones"][0][0][0].plan.algorithmic_bytes(True)) / P
    ev = []
    for rep in range(reps + 5):
        for s in range(sets):
            for k in kinds:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for op, table in arms[k][s]:
                    op.global_step = 0                      # g = 0: the apply branch
                    op.run_bound(table)
                e1.record()
                if rep >= 5:
                    ev.append((k, e0, e1))
    torch.cuda.synchronize()
    t = {k: [] for k in kinds}
    for k, e0, e1 in ev:
        t[k].append(e0.elapsed_time(e1) * 1e3)
    row = {"model": name, "optimizer": variant, "P": P, "gpu": info, "launches": {k: len(arms[k][0]) for k in kinds},
           "apply": {k: summary(t[k], bpp, P) for k in kinds}}
    row["electra_over_ones"] = row["apply"]["electra"]["median_us"] / row["apply"]["ones"]["median_us"]
    row["split_over_ones"] = row["apply"]["split"]["median_us"] / row["apply"]["ones"]["median_us"]
    del arms
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--sets", type=int, default=3)
    ap.add_argument("--models", default="bert_small,bert_large")
    ap.add_argument("--optimizers", default="adamw,lamb")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    gen = torch.Generator(device="cuda").manual_seed(0)
    info = gpu_info()
    print(f"GPU: {info}; {a.sets} state sets per arm; {a.reps} applies per set and arm; "
          "'split' clips per group: NOT equivalent to the other two arms")
    results = []
    for name in a.models.split(","):
        for variant in a.optimizers.split(","):
            row = run_model(name, variant, a.reps, a.sets, gen, info)
            results.append(row)
            r = row["apply"]
            print(f"{name:10s} {variant:5s} " + " | ".join(
                f"{k} {r[k]['median_us']:9.1f} us (p10 {r[k]['p10_us']:.1f}, p90 {r[k]['p90_us']:.1f}, "
                f"{row['launches'][k]} launch{'es' if row['launches'][k] > 1 else ''})" for k in r)
                + f" | electra/ones {row['electra_over_ones']:.3f}, split/ones {row['split_over_ones']:.3f}")
    print(json.dumps(results))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
