"""What a bf16 model costs the train op against an fp32 one on BERT-Small (P = 28 764 674): each launch timed with CUDA
events -- the first accumulate of a window, a later accumulate, and the apply -- with clipping on (AdamWeightDecay,
clip 1.0: the two-pass clip kernel) and off (the single-pass apply kernel).

Every arm keeps --sets independent state sets (params, master weights, m, v, accumulators and gradients; > 400 MB each,
far above the 50 MB L2) and the timed launches rotate through them, so no launch finds its inputs in L2.  Arms
alternate launch by launch, so clock and power drift hit them alike.  The GPU's name and power limit are printed with
the numbers.

    python tools/half_params_bench.py [--reps 100] [--sets 3] [--json OUT]
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

N = 4
# global_step -> which launch: g = 0 applies, g = 1 is the first accumulate of a window, g = 2 a later one
LAUNCHES = {"accumulate_first": 1, "accumulate": 2, "apply": 0}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + " (power limit not readable)"


def make_arm(man, hp, dtype, sets, gen):
    arm = []
    for _ in range(sets):
        params = [(torch.randn(s, device="cuda", generator=gen) * 0.02).to(dtype) for _, s in man]
        op = GaccumTrainOp(params, [n for n, _ in man], hp, N, lambda s: 1e-4)
        grads = [(torch.randn(s, device="cuda", generator=gen) * 1e-3).to(dtype) for _, s in man]
        arm.append((op, op.bind(grads)))
    return arm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--sets", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    man = MANIFESTS["bert_small"]()
    P = sum(int(np.prod(s)) for _, s in man)
    gen = torch.Generator(device="cuda").manual_seed(0)
    info = gpu_info()
    print(f"GPU: {info}; BERT-Small P = {P}; N = {N}; {a.sets} state sets per arm; {a.reps} launches per set and kind")
    results = []
    for label, hp in (("AdamWeightDecay, clip 1.0", g.HParams.bert()), ("AdamWeightDecay, no clip", g.HParams.bert())):
        if label.endswith("no clip"):
            hp.clip_norm = 0.0
        arms = {"fp32": make_arm(man, hp, torch.float32, a.sets, gen), "bf16": make_arm(man, hp, torch.bfloat16, a.sets, gen)}
        bytes_per = {k: {kind: arms[k][0][0].plan.algorithmic_bytes(kind == "apply") for kind in LAUNCHES} for k in arms}
        for k in arms:                                   # the first accumulate moves 4 B/param less than the others
            bytes_per[k]["accumulate_first"] -= 4 * P
        times = {(k, kind): [] for k in arms for kind in LAUNCHES}
        ev = []
        for rep in range(a.reps + 3):
            for kind, gs in LAUNCHES.items():
                for s in range(a.sets):
                    for k in arms:
                        op, table = arms[k][s]
                        op.global_step = gs
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        op.run_bound(table)
                        e1.record()
                        if rep >= 3:                     # the first launches warm up every kernel and state set
                            ev.append((k, kind, e0, e1))
        torch.cuda.synchronize()
        for k, kind, e0, e1 in ev:
            times[(k, kind)].append(e0.elapsed_time(e1) * 1e3)
        for kind in LAUNCHES:
            row = {"config": label, "launch": kind, "gpu": info}
            for k in arms:
                t = np.array(times[(k, kind)])
                med = float(np.median(t))
                row[k] = {"median_us": med, "p10_us": float(np.percentile(t, 10)), "p90_us": float(np.percentile(t, 90)),
                          "algorithmic_bytes_per_param": bytes_per[k][kind] / P, "GB_per_s": bytes_per[k][kind] / med / 1e3}
            row["bf16_vs_fp32_pct"] = 100.0 * (row["bf16"]["median_us"] / row["fp32"]["median_us"] - 1.0)
            results.append(row)
            print(f"{label:26s} {kind:17s} fp32 {row['fp32']['median_us']:8.1f} us (p10 {row['fp32']['p10_us']:.1f},"
                  f" p90 {row['fp32']['p90_us']:.1f}, {row['fp32']['GB_per_s']:.0f} GB/s)"
                  f" | bf16 {row['bf16']['median_us']:8.1f} us (p10 {row['bf16']['p10_us']:.1f},"
                  f" p90 {row['bf16']['p90_us']:.1f}, {row['bf16']['GB_per_s']:.0f} GB/s) | {row['bf16_vs_fp32_pct']:+.2f} %")
        del arms
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
