"""What dynamic loss scaling costs on the apply step of BERT-Small: the apply launch timed with CUDA events, with and
without loss scaling, for AdamWeightDecay with clipping (the clip kernel either way) and for tf_adam without clipping
(the single-pass apply kernel against the two-pass kernel that loss scaling needs).

Every arm keeps --sets independent state sets (params, m, v, accumulators and gradients; ~580 MB each, far above the
50 MB L2) and the timed launches rotate through them, so no launch finds its inputs in L2.  Arms alternate launch by
launch, so clock and power drift hit them alike.  The GPU's name and power limit are printed with the numbers.

    python tools/loss_scale_bench.py [--reps 200] [--sets 3] [--json OUT]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np
import torch

import gaccum_b200 as g
from gaccum_b200.manifests import MANIFESTS
from gaccum_b200.train_op import GaccumTrainOp


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + " (power limit not readable)"


def make_arm(man, hp, loss_scale, sets, gen):
    arm = []
    for _ in range(sets):
        params = [torch.randn(s, device="cuda", generator=gen) * 0.02 for _, s in man]
        op = GaccumTrainOp(params, [n for n, _ in man], hp, 4, lambda s: 1e-4, loss_scale=loss_scale)
        grads = [torch.randn(s, device="cuda", generator=gen) * 1e-3 for _, s in man]
        arm.append((op, grads))
    return arm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--sets", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    man = MANIFESTS["bert_small"]()
    P = sum(int(np.prod(s)) for _, s in man)
    gen = torch.Generator(device="cuda").manual_seed(0)
    # growth_interval so large that S never changes: every timed window is applied, none skipped
    ls = g.LossScaleConfig(2.0 ** 15, 2.0, 1 << 30)
    info = gpu_info()
    print(f"GPU: {info}; BERT-Small P = {P}; {a.sets} state sets per arm; {a.reps} launches per set")
    results = []
    for label, hp in (("AdamWeightDecay, clip 1.0", g.HParams.bert()), ("tf_adam, no clip", g.HParams.tf_adam())):
        arms = {"off": make_arm(man, hp, None, a.sets, gen), "loss_scale": make_arm(man, hp, ls, a.sets, gen)}
        tables = {k: [op.bind(gr) for op, gr in v] for k, v in arms.items()}
        times = {k: [] for k in arms}
        ev = []
        for rep in range(a.reps + 5):
            for s in range(a.sets):
                for k in arms:
                    op = arms[k][s][0]
                    op.global_step = 0                  # g = 0: the apply branch
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    op.run_bound(tables[k][s])
                    e1.record()
                    if rep >= 5:                        # the first launches warm up every kernel and state set
                        ev.append((k, e0, e1))
        torch.cuda.synchronize()
        for k, e0, e1 in ev:
            times[k].append(e0.elapsed_time(e1) * 1e3)
        for k in arms:
            st = arms[k][0][0].stats()
            assert st["applied"]
            if k == "loss_scale":
                assert arms[k][0][0].loss_scale_state()["skipped_windows"] == 0
        row = {"config": label, "gpu": info}
        for k, t in times.items():
            t = np.array(t)
            row[k] = {"median_us": float(np.median(t)), "mean_us": float(t.mean()), "p10_us": float(np.percentile(t, 10)),
                      "p90_us": float(np.percentile(t, 90)), "GB_per_s": 36.0 * P / float(np.median(t)) / 1e3}
        row["overhead_pct"] = 100.0 * (row["loss_scale"]["median_us"] / row["off"]["median_us"] - 1.0)
        results.append(row)
        print(f"{label:28s} off {row['off']['median_us']:8.1f} us (p10 {row['off']['p10_us']:.1f}, p90 {row['off']['p90_us']:.1f})"
              f" | loss scaling {row['loss_scale']['median_us']:8.1f} us (p10 {row['loss_scale']['p10_us']:.1f},"
              f" p90 {row['loss_scale']['p90_us']:.1f}) | {row['overhead_pct']:+.2f} %")
        del arms, tables
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
