"""Minimal workload for ncu: N forward steps of the bench configuration (L12 x2, 256 48x48 tiles), nothing else."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "dcscn-super-resolution_b200"))
import bench  # noqa: E402
from helper import engine as E  # noqa: E402

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
batch = int(sys.argv[2]) if len(sys.argv) > 2 else bench.BATCH
prec = E.PRECISION_F16X1 if (len(sys.argv) > 3 and sys.argv[3] == "f16x1") else E.PRECISION_F16X3
eng = E.Engine(E.make_config(precision=prec))
eng.set_params(bench.load_weights())
eng.set_option("graph", 0)                      # one kernel launch per layer for ncu's -k / -s / -c filters
for kv in filter(None, os.environ.get("DCSCN_OPTS", "").split(",")):   # e.g. DCSCN_OPTS=seg_chunks=1,fuse_last=0
    k, v = kv.split("=")
    eng.set_option(k, int(v))
g = torch.Generator().manual_seed(0)
x = (torch.rand(batch, 48, 48, 1, generator=g) * 255).cuda()
x2 = (torch.rand(batch, 96, 96, 1, generator=g) * 255).cuda()
y = torch.empty_like(x2)
for _ in range(steps):
    eng.forward(x, x2, y)
torch.cuda.synchronize()
print("done", eng.launch_count)
