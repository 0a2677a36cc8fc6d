"""Cost of the per-tensor norms (gaccum_plan_set_tensor_norms) in the apply step, against the unfused torch equivalent.

Shapes: BERT-Small and BERT-Large.  Kernels: AdamWeightDecay with clipping (the clip-apply), AdamWeightDecay without
clipping (apply_kernel), LAMB with clipping.  Arms:
  off       apply_only(G): the apply launch of a plan without norms
  on        apply_only(G): the same launch on a plan with norms
  unfused   a plan without norms, the window split so torch can see the gradient: accumulate_only(G); the _foreach_norm
            of the accumulator views times 1/N; a clone of p; apply_only(None); _foreach_sub and _foreach_norm

Each arm keeps 3 state sets (train op, parameters, gradients) used in rotation, so no launch finds its inputs in L2;
arms alternate launch by launch, so clock and power drift hit them alike.  Every launch is timed with CUDA events;
medians with p10 / p90 over --iters launches per arm.  The GPU's name and power limit are printed with the numbers.

    python tools/tensor_norms_bench.py [--iters 30] [--shapes bert_small,bert_large] [--json OUT]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.dirname(os.path.abspath(__file__))):
    sys.path.insert(0, p)

import numpy as np
import torch

import gaccum_b200 as g
import oracle_np as onp
from gaccum_b200.train_op import GaccumTrainOp
from loss_scale_bench import gpu_info

N = 4
SETS = 3
KERNELS = {
    "adamw_clip": lambda: g.HParams.bert(),
    "adamw_noclip": lambda: g.HParams(g.ADAM_WEIGHT_DECAY, 0, 0.9, 0.999, 1e-6, 0.01, 0.0),
    "lamb_clip": lambda: g.HParams.lamb(),
}
ARMS = ("off", "on", "unfused")


def make_sets(man, hp, norms, gen):
    out = []
    for _ in range(SETS):
        params = [torch.randn(s, device="cuda", generator=gen) * 0.02 for _, s in man]
        op = GaccumTrainOp(params, [n for n, _ in man], hp, N, lambda s: 1e-4, tensor_norms=norms)
        grads = [torch.randn(s, device="cuda", generator=gen) * 1e-3 for _, s in man]
        out.append((op, grads))
    return out


def launch(arm, op, grads):
    if arm != "unfused":
        op.apply_only(grads)
        return
    op.accumulate_only(grads)
    views = [op.accum_view(i) for i in range(len(op.params))]
    gn = torch._foreach_norm(views)
    torch._foreach_mul_(gn, 1.0 / N)
    before = [p.detach().clone() for p in op.params]
    op.apply_only(None)
    torch._foreach_norm(before)
    torch._foreach_norm(torch._foreach_sub(before, [p.detach() for p in op.params]))


def bench(man, hp, iters, gen):
    sets = {arm: make_sets(man, hp, arm == "on", gen) for arm in ARMS}
    for arm in ARMS:                                   # warm-up: load every kernel, allocate torch's workspaces
        for op, grads in sets[arm]:
            launch(arm, op, grads)
    torch.cuda.synchronize()
    times = {arm: [] for arm in ARMS}
    for it in range(iters):
        for arm in ARMS:
            op, grads = sets[arm][it % SETS]
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            launch(arm, op, grads)
            b.record()
            b.synchronize()
            times[arm].append(a.elapsed_time(b))
    return {arm: {"median_ms": float(np.median(t)), "p10_ms": float(np.percentile(t, 10)),
                  "p90_ms": float(np.percentile(t, 90))} for arm, t in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--shapes", default="bert_small,bert_large")
    ap.add_argument("--kernels", default=",".join(KERNELS))
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    gen = torch.Generator(device="cuda").manual_seed(0)
    out = {"gpu": gpu_info(), "N": N, "results": {}}
    print(out["gpu"])
    for shape in args.shapes.split(","):
        man = onp.MANIFESTS[shape]()
        P = sum(int(np.prod(s)) for _, s in man)
        for kern in args.kernels.split(","):
            r = bench(man, KERNELS[kern](), args.iters, gen)
            out["results"][f"{shape}/{kern}"] = r
            off = r["off"]["median_ms"]
            print(f"{shape:10s} {kern:13s} P={P:>10d}  " + "  ".join(
                f"{arm} {r[arm]['median_ms']:.3f} ms [{r[arm]['p10_ms']:.3f}-{r[arm]['p90_ms']:.3f}]" for arm in ARMS) +
                f"  on-off {r['on']['median_ms'] - off:+.3f} ms, unfused-off {r['unfused']['median_ms'] - off:+.3f} ms",
                flush=True)
            torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
