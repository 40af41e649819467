"""Cost of each --activator on the flagship shapes: L12 x2 inference on 256 tiles of 48 x 48 and the L12 x4 train step on
64 patches of 48 x 48, one engine per activator, the activators alternating round by round, CUDA events around each
call.  Prints the card's name and power limit from the same run, then one line per (workload, activator): the median
and the spread of the per-round times.

    python scripts/activator_timing.py [--rounds 7] [--reps 10] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dcscn-super-resolution_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from helper import engine as E  # noqa: E402
import activator_oracle as A  # noqa: E402
import dcscn_oracle as O  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("activator_timing: needs a CUDA device")
    g = torch.Generator(device="cuda").manual_seed(0)
    work = {}
    for act in A.ACTIVATORS:
        inf = E.Engine(E.make_config(scale=2, activator=act))
        inf.set_params(A.he_init_weights(O.OracleConfig(scale=2), act, seed=0))
        x = torch.rand(256, 48, 48, 1, device="cuda", generator=g) * 255
        x2 = torch.rand(256, 96, 96, 1, device="cuda", generator=g) * 255
        y = torch.empty_like(x2)
        tr = E.Engine(E.make_config(scale=4, dropout_keep=0.8, activator=act))
        tr.set_params(A.he_init_weights(O.OracleConfig(scale=4), act, seed=0))
        tx = torch.rand(64, 48, 48, 1, device="cuda", generator=g) * 255
        tx2 = torch.rand(64, 192, 192, 1, device="cuda", generator=g) * 255
        ty = tx2 + torch.randn(64, 192, 192, 1, device="cuda", generator=g)
        work[act] = {
            "inference L12 x2, 256 x 48^2": (inf, lambda e=inf, x=x, x2=x2, y=y: e.forward(x, x2, y)),
            "train step L12 x4, 64 x 48^2": (tr, lambda e=tr, a=tx, b=tx2, c=ty: e.train_step(a, b, c, lr=1e-4, seed=1,
                                                                                             apply_update=False)),
        }
    for act in A.ACTIVATORS:                      # warm-up: plans, graphs, workspaces
        for _, fn in work[act].values():
            for _ in range(3):
                fn()
    torch.cuda.synchronize()
    times = {(w, a): [] for a in A.ACTIVATORS for w in work[a]}
    for r in range(args.rounds):
        order = A.ACTIVATORS if r % 2 == 0 else A.ACTIVATORS[::-1]
        for act in order:
            for w, (_, fn) in work[act].items():
                times[(w, act)].append(timed(fn, args.reps))
    dev = card()
    print("device:", dev)
    rows = []
    for (w, act), t in times.items():
        t = np.array(t)
        rows.append({"workload": w, "activator": act, "median_ms": float(np.median(t)), "min_ms": float(t.min()),
                     "max_ms": float(t.max())})
        print("%-30s %-11s median %8.3f ms  (min %.3f, max %.3f)" % (w, act, np.median(t), t.min(), t.max()))
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"device": dev, "rounds": args.rounds, "reps": args.reps, "rows": rows}, f, indent=1)
    for act in A.ACTIVATORS:
        for e, _ in work[act].values():
            e.close()


if __name__ == "__main__":
    main()
