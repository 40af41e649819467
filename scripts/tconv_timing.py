"""The two upsamplers side by side: the L12 graph (the reference's default flags) with the pixel shuffler (Up-PS, and
Up-PS2 at x4) and with --pixel_shuffler=false (Up-TCNN, one transposed convolution run as a 3x3 LR layer into s*s*C
columns).  Times x2 and x4 inference on 256 tiles of 48x48 and the x4 train step on 64 tiles of 48x48, alternating the
two graphs, with CUDA events; then the per-launch times of one forward of each x4 graph.  Prints the card's name and
power limit first.  Needs a GPU.  Usage: python scripts/tconv_timing.py [rounds]"""
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dcscn-super-resolution_b200"))
import DCSCN  # noqa: E402
from helper import engine as E  # noqa: E402


def build(tconv, **kw):
    eng = E.Engine(E.make_config(transposed_upsampler=tconv, **kw))
    g = np.random.RandomState(0)
    for name, shape in eng.param_shapes().items():
        if name.endswith("/Tconv_W"):
            w = DCSCN.upscale_weight(shape)
        elif name.endswith("/conv_W"):
            w = np.clip(g.randn(*shape), -2, 2) * math.sqrt(2.0 / (shape[0] * shape[1] * shape[2]))
        elif name.endswith("/conv_B"):
            w = np.zeros(shape)
        else:
            w = np.full(shape, 0.1)
        eng.set_param(name, w.astype(np.float32))
    return eng


def events(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(iters):
        fn(i)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    g = torch.Generator().manual_seed(2)
    for s in (2, 4):
        x = (torch.rand(256, 48, 48, 1, generator=g) * 255).cuda()
        x2 = (torch.rand(256, 48 * s, 48 * s, 1, generator=g) * 255).cuda()
        y = torch.empty_like(x2)
        engines = {"Up-PS": build(False, scale=s), "Up-TCNN": build(True, scale=s)}
        for eng in engines.values():
            for _ in range(3):
                eng.forward(x, x2, y)
        for r in range(rounds):
            for name, eng in engines.items():
                ms = events(lambda i: eng.forward(x, x2, y), 20)
                print("round %d %-8s L12 x%d forward (256 x 48^2) %.3f ms" % (r, name, s, ms))
        if s == 4:
            for name, eng in engines.items():
                eng.set_option("timing", 1)
                eng.forward(x, x2, y)
                torch.cuda.synchronize()
                tm = eng.timings()
                print("%s per launch: total %.3f ms  " % (name, sum(t for _, t in tm)) + " ".join("%s=%.3f" % kv for kv in tm))
                eng.set_option("timing", 0)
        for eng in engines.values():
            eng.close()

    x = (torch.rand(64, 48, 48, 1, generator=g) * 255).cuda()
    x2 = (torch.rand(64, 192, 192, 1, generator=g) * 255).cuda()
    y = (x2 + 2.0).contiguous()
    engines = {"Up-PS": build(False, scale=4), "Up-TCNN": build(True, scale=4)}
    for eng in engines.values():
        for i in range(3):
            eng.train_step(x, x2, y, 1e-4, i)
    for r in range(rounds):
        for name, eng in engines.items():
            ms = events(lambda i: eng.train_step(x, x2, y, 1e-4, 10 + i), 10)
            print("round %d %-8s L12 x4 train step (64 x 48^2) %.3f ms" % (r, name, ms))
    for eng in engines.values():
        eng.close()


if __name__ == "__main__":
    main()
