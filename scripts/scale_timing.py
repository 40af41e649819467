"""x4 against x8: the L12 graph (the reference's default flags, He-initialised) at --scale=4 (two x2 pixel-shuffler stages)
and --scale=8 (one Up-PS of 64 * 96 = 6144 columns), alternating the two, with CUDA events.  Times inference on 256 tiles
of 48x48 and the train step on the default 20 patches of 48x48, and prints ms, output (HR) Mpixels/s and
dcscn_device_bytes (activation workspace) for each.  Prints the card's name and power limit first.  Needs a GPU.
Usage: python scripts/scale_timing.py [rounds]"""
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dcscn-super-resolution_b200"))
from helper import engine as E  # noqa: E402


def build(**kw):
    eng = E.Engine(E.make_config(**kw))
    g = np.random.RandomState(0)
    for name, shape in eng.param_shapes().items():
        if name.endswith("/conv_W"):
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
    for what, n, iters in (("forward", 256, 10), ("train step", 20, 10)):
        cases = {}
        for s in (4, 8):
            x = (torch.rand(n, 48, 48, 1, generator=g) * 255).cuda()
            x2 = (torch.rand(n, 48 * s, 48 * s, 1, generator=g) * 255).cuda()
            y = torch.empty_like(x2) if what == "forward" else (x2 + 2.0).contiguous()
            eng = build(scale=s, dropout_keep=0.8)
            if what == "forward":
                run = (lambda e, a, b, c: lambda i: e.forward(a, b, c))(eng, x, x2, y)
            else:
                run = (lambda e, a, b, c: lambda i: e.train_step(a, b, c, 1e-4, 10 + i))(eng, x, x2, y)
            for i in range(3):
                run(i)
            torch.cuda.synchronize()
            cases[s] = (eng, run, n * (48 * s) ** 2)
            print("L12 x%d %s (%d x 48^2): dcscn_device_bytes %.1f MB" % (s, what, n, eng.device_bytes / 2 ** 20))
        for r in range(rounds):
            for s, (eng, run, hr_px) in cases.items():
                ms = events(run, iters)
                print("round %d L12 x%d %s (%d x 48^2) %.3f ms  %.1f output Mpixels/s" % (r, s, what, n, ms, hr_px / ms / 1e3))
        for eng, _, _ in cases.values():
            eng.close()
        del cases
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
