"""What the exponential moving average costs on the apply step, three arms on BERT-Small and BERT-Large shapes (the
AdamWeightDecay clip-apply, clipping at 1.0 as create_optimizer does):

  plain    the apply launch without an EMA                                          (36 B/param)
  fused    the apply launch of an EMA train op: e = e - (e - p) * c in the kernel   (44 B/param)
  foreach  the plain apply followed by the same EMA in torch._foreach_* ops, what a user without the fused EMA runs
           (e - p, * c, e - that: three passes over the tensors, plus the host-side c of a TF-style num_updates rule)

Timed with CUDA events.  Every arm keeps --sets independent state sets (params, m, v, accumulators, gradients, EMA) and
the timed launches rotate through them, so no launch finds its inputs in L2; arms alternate launch by launch, so clock
and power drift hit them alike.  GB/s are on the fused arm's algorithmic bytes for both EMA arms.  The GPU's name and
power limit are printed with the numbers.

    python tools/ema_bench.py [--reps 300] [--sets 3] [--models bert_small,bert_large] [--json OUT]
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
DECAY = 0.9999


def make_arm(man, sets, gen, ema):
    arm = []
    for _ in range(sets):
        params = [torch.randn(s, device="cuda", generator=gen) * 0.02 for _, s in man]
        op = GaccumTrainOp(params, [n for n, _ in man], g.HParams.bert(), N, lambda s: 1e-4,
                           ema=g.EmaConfig(DECAY) if ema else None)
        grads = [torch.randn(s, device="cuda", generator=gen) * 1e-3 for _, s in man]
        avg = [p.detach().clone() for p in params] if not ema else None
        arm.append((op, op.bind(grads), avg))
    return arm


def foreach_ema(op, avg):
    """The EMA a user runs after the apply today: c from the decay on the host, then three foreach passes."""
    c = float(np.float32(1.0) - np.float32(DECAY))
    delta = torch._foreach_sub(avg, op.params)
    torch._foreach_mul_(delta, c)
    torch._foreach_sub_(avg, delta)


def summary(t, bytes_per_param, P):
    t = np.array(t)
    med = float(np.median(t))
    return {"median_us": med, "p10_us": float(np.percentile(t, 10)), "p90_us": float(np.percentile(t, 90)),
            "GB_per_s": bytes_per_param * P / med / 1e3, "n": int(t.size)}


def run_model(name, reps, sets, gen, info):
    man = MANIFESTS[name]()
    P = sum(int(np.prod(s)) for _, s in man)
    arms = {"plain": make_arm(man, sets, gen, False), "fused": make_arm(man, sets, gen, True),
            "foreach": make_arm(man, sets, gen, False)}
    bpp = {"plain": 36.0, "fused": 44.0, "foreach": 44.0}
    assert arms["fused"][0][0].plan.algorithmic_bytes(True) == 44 * P
    ev = []
    for rep in range(reps + 5):
        for s in range(sets):
            for k in arms:
                op, table, avg = arms[k][s]
                op.global_step = 0                          # g = 0: the apply branch
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                op.run_bound(table)
                if k == "foreach":
                    foreach_ema(op, avg)
                e1.record()
                if rep >= 5:
                    ev.append((k, e0, e1))
    torch.cuda.synchronize()
    assert arms["fused"][0][0].ema_state()["num_updates"] == reps + 5
    t = {k: [] for k in arms}
    for k, e0, e1 in ev:
        t[k].append(e0.elapsed_time(e1) * 1e3)
    row = {"model": name, "P": P, "gpu": info, "apply": {k: summary(t[k], bpp[k], P) for k in arms}}
    row["fused_ratio"] = row["apply"]["fused"]["median_us"] / row["apply"]["plain"]["median_us"]
    row["foreach_ratio"] = row["apply"]["foreach"]["median_us"] / row["apply"]["plain"]["median_us"]
    del arms
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=300)
    ap.add_argument("--sets", type=int, default=3)
    ap.add_argument("--models", default="bert_small,bert_large")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    gen = torch.Generator(device="cuda").manual_seed(0)
    info = gpu_info()
    print(f"GPU: {info}; {a.sets} state sets per arm; {a.reps} apply launches per set and arm")
    results = []
    for name in a.models.split(","):
        row = run_model(name, a.reps, a.sets, gen, info)
        results.append(row)
        r = row["apply"]
        print(f"{name:10s} " + " | ".join(f"{k} {r[k]['median_us']:9.1f} us (p10 {r[k]['p10_us']:.1f}, p90 {r[k]['p90_us']:.1f}, "
                                          f"{r[k]['GB_per_s']:.0f} GB/s)" for k in r)
              + f" | fused/plain {row['fused_ratio']:.3f}, foreach/plain {row['foreach_ratio']:.3f}")
    print(json.dumps(results))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
