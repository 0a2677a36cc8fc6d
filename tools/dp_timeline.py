#!/usr/bin/env python
"""Per-block timeline of dp_apply_kernel (experiments build): torchrun --nproc-per-node W tools/dp_timeline.py"""
import ctypes as C, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ.setdefault("GACCUM_LIB", os.path.join(ROOT, "gradient-accumulation-tf-estimator_b200", "csrc", "libgaccum_exp.so"))
sys.path.insert(0, ROOT)
import numpy as np, torch, torch.distributed as dist
import gaccum_b200 as g
from gaccum_b200.manifests import MANIFESTS
from gaccum_b200.distributed import FusedDataParallelTrainOp
from gaccum_b200 import _lib
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
wl = sys.argv[1] if len(sys.argv) > 1 else "bert_small"
man = MANIFESTS[wl]()
N = 4
sets = []
for r in range(3):
    params = [torch.randn(s, device=dev) * 0.02 for _, s in man]
    dp = FusedDataParallelTrainOp(params, [n for n, _ in man], g.HParams.bert(), N, lambda s: 1e-5, global_step=1)
    grads = [torch.randn(s, device=dev) * 1e-3 for _, s in man]
    sets.append((dp, dp.bind(grads)))
L = _lib._load()
L.gaccum_debug_read.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
for it in range(3 * N):
    for dp, b in sets:
        dp.run_bound(b)
torch.cuda.synchronize(); dist.barrier()
dp = sets[0][0]
nb = 16 * torch.cuda.get_device_properties(dev).multi_processor_count      # the plan's largest grid
buf = (C.c_ulonglong * (16 * nb))()
assert L.gaccum_debug_read(dp.plan._h, buf, 16 * nb) == 0
raw = np.array(buf, dtype=np.float64).reshape(nb, 16)
raw = raw[raw[:, 0] > 0]
t0 = raw[:, 0].min()
t = (raw[:, :8] - t0) / 1e3
names = ["start", "A: local a+=G, pushes issued", "A: fence + counter", "flag 0 seen (all ranks pushed)", "B: shard reduced", "flag 1 seen (norms)", "C: update + pushes issued", "end"]
for rr in range(world):
    if rank == rr:
        print(f"rank {rank} of {world} {wl}: {len(raw)} blocks")
        for i, nme in enumerate(names):
            c = t[:, i]
            print(f"{nme:34s} min {c.min():7.1f}  median {np.median(c):7.1f}  max {c.max():7.1f} us")
        for col, nme in ((9, "B: block fenced + counted"), (8, "B: last block starts publishing"), (10, "B: last block raised the flags")):
            c = raw[:, col][raw[:, col] > 0]
            if len(c):
                c = (c - t0) / 1e3
                print(f"{nme:34s} min {c.min():7.1f}  median {np.median(c):7.1f}  max {c.max():7.1f} us")
        sys.stdout.flush()
    dist.barrier()
# event-timed duration of ONE apply launch on an idle stream, ranks aligned by a barrier: launch overhead + kernel
stream = torch.cuda.current_stream(dev)
iso = []
for rep in range(6):
    dp, b = sets[rep % 3]
    while dp.global_step % N != 0:
        dp.run_bound(b)
    torch.cuda.synchronize(); dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream); dp.run_bound(b); e1.record(stream)
    torch.cuda.synchronize()
    iso.append(e0.elapsed_time(e1) * 1e3)
# (an idle stream makes the GPU wait for the host between the two events: this is launch latency, not kernel time)
dist.barrier()
dist.destroy_process_group()
