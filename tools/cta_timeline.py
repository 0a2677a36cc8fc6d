#!/usr/bin/env python
"""Per-CTA timeline of the clip-apply kernel: where does each CTA wait?  Needs the experiments build
(python gradient-accumulation-tf-estimator_b200/build.py --variant exp GACCUM_EXPERIMENTS), which this
script selects through GACCUM_LIB; the shipped libgaccum.so carries no timestamp code."""
import ctypes as C, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ.setdefault("GACCUM_LIB", os.path.join(ROOT, "gradient-accumulation-tf-estimator_b200", "csrc", "libgaccum_exp.so"))
sys.path.insert(0, ROOT)
import numpy as np, torch
import gaccum_b200 as g
from gaccum_b200.manifests import MANIFESTS
from gaccum_b200.train_op import GaccumTrainOp
from gaccum_b200 import _lib
man = MANIFESTS["bert_small"]()
dev = torch.device("cuda:0")
sets = []
for r in range(3):
    params = [torch.randn(s, device=dev) * 0.02 for _, s in man]
    op = GaccumTrainOp(params, [n for n, _ in man], g.HParams.bert(), 4, lambda s: 1e-5, global_step=100001)
    grads = [torch.randn(s, device=dev) * 1e-3 for _, s in man]
    sets.append((op, op.bind(grads)))
L = _lib._load()
L.gaccum_debug_read.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
for it in range(12):
    for op, b in sets:
        op.run_bound(b)
torch.cuda.synchronize()
op = sets[0][0]
props = torch.cuda.get_device_properties(dev)
nsm = props.multi_processor_count      # one clip-apply CTA per SM
sm_mhz = props.clock_rate / 1000.0     # peak SM clock of the device the kernel ran on
buf = (C.c_ulonglong * (16 * nsm))()
assert L.gaccum_debug_read(op.plan._h, buf, 16 * nsm) == 0
raw = np.array(buf, dtype=np.float64).reshape(nsm, 16)
t = raw[:, :4].copy()
cyc = raw[:, 4:16] / sm_mhz        # cycles -> us at the maximum SM clock
t0 = t[:, 0].min()
t = (t - t0) / 1e3
for name, col in (("start", 0), ("pass1 done", 1), ("barrier out", 2), ("pass2 done", 3)):
    c = t[:, col]
    print(f"{name:12s} min {c.min():7.1f}  median {np.median(c):7.1f}  max {c.max():7.1f} us   spread {c.max()-c.min():6.1f}")
p1 = t[:, 1] - t[:, 0]; p2 = t[:, 3] - t[:, 2]
print(f"pass1 duration per CTA: min {p1.min():.1f} median {np.median(p1):.1f} max {p1.max():.1f}; waiting at barrier: mean {np.mean(t[:,2]-t[:,1]):.1f} us")
print(f"pass2 duration per CTA: min {p2.min():.1f} median {np.median(p2):.1f} max {p2.max():.1f}; idle before kernel end: mean {np.mean(t[:,3].max()-t[:,3]):.1f} us")
for name, lo in (("consumers waiting for G (per group)", 0), ("producer waiting for a free slot", 3), ("group pass-1 duration", 6), ("producer: all copies issued after", 9)):
    c = cyc[:, lo:lo + 3]
    print(f"{name:36s} min {c.min():6.1f}  median {np.median(c):6.1f}  max {c.max():6.1f} us")
