"""What LAMB costs on the apply step: the AdamWeightDecay clip-apply launch against the LAMB apply launch (clipping on in
both), timed with CUDA events on BERT-Small and BERT-Large shapes, and one whole window (N = 4 micro-steps) of each.

Every arm keeps --sets independent state sets (params, m, v, accumulators and gradients) and the timed launches rotate
through them, so no launch finds its inputs in L2.  Arms alternate launch by launch, so clock and power drift hit them
alike.  GB/s are on the algorithmic bytes of each arm (36 B/param AdamWeightDecay, 48 B/param LAMB).  The GPU's name
and power limit are printed with the numbers.

    python tools/lamb_bench.py [--reps 300] [--sets 3] [--models bert_small,bert_large] [--json OUT]
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


def make_arm(man, hp, sets, gen):
    arm = []
    for _ in range(sets):
        params = [torch.randn(s, device="cuda", generator=gen) * 0.02 for _, s in man]
        op = GaccumTrainOp(params, [n for n, _ in man], hp, N, lambda s: 1e-4)
        grads = [torch.randn(s, device="cuda", generator=gen) * 1e-3 for _, s in man]
        arm.append((op, op.bind(grads)))
    return arm


def summary(t, bytes_per_param, P):
    t = np.array(t)
    med = float(np.median(t))
    return {"median_us": med, "p10_us": float(np.percentile(t, 10)), "p90_us": float(np.percentile(t, 90)),
            "GB_per_s": bytes_per_param * P / med / 1e3, "n": int(t.size)}


def run_model(name, reps, sets, gen, info):
    man = MANIFESTS[name]()
    P = sum(int(np.prod(s)) for _, s in man)
    arms = {"adamw": make_arm(man, g.HParams.bert(), sets, gen), "lamb": make_arm(man, g.HParams.lamb(), sets, gen)}
    bpp = {"adamw": 36.0, "lamb": 48.0}
    assert arms["lamb"][0][0].plan.algorithmic_bytes(True) == 48 * P
    apply_ev, window_ev = [], []
    for rep in range(reps + 5):
        for s in range(sets):
            for k in arms:
                op, table = arms[k][s]
                op.global_step = 0                          # g = 0: the apply branch
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                op.run_bound(table)
                e1.record()
                if rep >= 5:
                    apply_ev.append((k, e0, e1))
    for rep in range(max(reps // 10, 20) + 2):              # whole windows: 3 accumulates and the apply
        for s in range(sets):
            for k in arms:
                op, table = arms[k][s]
                op.global_step = 1
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(N):
                    op.run_bound(table)
                e1.record()
                if rep >= 2:
                    window_ev.append((k, e0, e1))
    torch.cuda.synchronize()
    for k in arms:
        assert arms[k][0][0].stats()["applied"]
    ta = {k: [] for k in arms}
    tw = {k: [] for k in arms}
    for k, e0, e1 in apply_ev:
        ta[k].append(e0.elapsed_time(e1) * 1e3)
    for k, e0, e1 in window_ev:
        tw[k].append(e0.elapsed_time(e1) * 1e3)
    row = {"model": name, "P": P, "gpu": info,
           "apply": {k: summary(ta[k], bpp[k], P) for k in arms},
           "window_n4": {k: summary(tw[k], 8 + 12 * (N - 2) + bpp[k], P) for k in arms}}
    row["apply_ratio"] = row["apply"]["lamb"]["median_us"] / row["apply"]["adamw"]["median_us"]
    row["window_ratio"] = row["window_n4"]["lamb"]["median_us"] / row["window_n4"]["adamw"]["median_us"]
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
        for what in ("apply", "window_n4"):
            r = row[what]
            print(f"{name:10s} {what:9s} AdamWeightDecay {r['adamw']['median_us']:9.1f} us (p10 {r['adamw']['p10_us']:.1f}, "
                  f"p90 {r['adamw']['p90_us']:.1f}, {r['adamw']['GB_per_s']:.0f} GB/s) | LAMB {r['lamb']['median_us']:9.1f} us "
                  f"(p10 {r['lamb']['p10_us']:.1f}, p90 {r['lamb']['p90_us']:.1f}, {r['lamb']['GB_per_s']:.0f} GB/s) | "
                  f"ratio {row['apply_ratio' if what == 'apply' else 'window_ratio']:.3f}")
    print(json.dumps(results))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
