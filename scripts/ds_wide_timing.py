"""Forward time of the depthwise-separable L12 x2 graph (the reference's default flags with --depthwise_separable, He-init
weights) next to the dense L12 x2 graph, at the benchmark shape (256 tiles of 48x48), alternating the two; then the
per-launch times of one wide depthwise-separable forward; then the L12 x4 train step on 64 tiles of 48x48, the
depthwise-separable graph (composed dense step) next to the dense one.  Needs a GPU.  Usage: python scripts/ds_wide_timing.py [rounds]"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "dcscn-super-resolution_b200"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import dcscn_oracle as O  # noqa: E402
from helper import engine as E  # noqa: E402


def build(ds, **kw):
    kw = dict(kw, depthwise_separable=ds)
    eng = E.Engine(E.make_config(**kw))
    eng.set_params(O.he_init_weights(O.OracleConfig(**kw), seed=0))
    return eng


def time_forward(eng, x, x2, y, iters=20):
    for _ in range(3):
        eng.forward(x, x2, y)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        eng.forward(x, x2, y)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    g = torch.Generator().manual_seed(2)
    x = (torch.rand(256, 48, 48, 1, generator=g) * 255).cuda()
    x2 = (torch.rand(256, 96, 96, 1, generator=g) * 255).cuda()
    y = torch.empty_like(x2)
    engines = {"dense": build(False), "ds": build(True)}
    px = 256 * 48 * 48
    for r in range(rounds):
        for name, eng in engines.items():
            ms = time_forward(eng, x, x2, y)
            print("round %d %-5s L12 x2 forward %.3f ms  %.1f Mpixel/s (LR)" % (r, name, ms, px / ms / 1e3))
    eng = engines["ds"]
    eng.set_option("timing", 1)
    for _ in range(3):
        eng.forward(x, x2, y)
    torch.cuda.synchronize()
    tm = eng.timings()
    print("ds per launch: total %.3f ms  " % sum(t for _, t in tm) + " ".join("%s=%.3f" % kv for kv in tm))
    for eng in engines.values():
        eng.close()

    x = (torch.rand(64, 48, 48, 1, generator=g) * 255).cuda()
    x2 = (torch.rand(64, 192, 192, 1, generator=g) * 255).cuda()
    y = (x2 + 2.0).contiguous()
    engines = {"dense": build(False, scale=4), "ds": build(True, scale=4)}
    for r in range(rounds):
        for name, eng in engines.items():
            for i in range(3):
                eng.train_step(x, x2, y, 1e-4, i)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for i in range(10):
                eng.train_step(x, x2, y, 1e-4, 10 + i)
            b.record()
            torch.cuda.synchronize()
            print("round %d %-5s L12 x4 train step (64 x 48^2) %.3f ms" % (r, name, a.elapsed_time(b) / 10))
    for eng in engines.values():
        eng.close()


if __name__ == "__main__":
    main()
