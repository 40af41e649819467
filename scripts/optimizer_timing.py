"""Cost of each --optimizer on the flagship train step: L12 x4 on 64 patches of 48 x 48, dropout keep 0.8, one engine per
optimizer, the optimizers alternating round by round, CUDA events around each call.  Two workloads: the whole train step
(forward, backward, clip and update), and `apply_gradients` alone (global norm, update and the device refresh of the
packed weights).  Prints the card's name and power limit from the same run, then one line per (workload, optimizer): the
median and the spread of the per-round times.

    python scripts/optimizer_timing.py [--rounds 7] [--reps 10] [--out result.json]
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
sys.path.insert(0, os.path.join(ROOT, "oracle"))

from helper import engine as E  # noqa: E402
import dcscn_oracle as O  # noqa: E402

OPTIMIZERS = ["adam", "gd", "momentum", "adadelta", "adagrad", "rmsprop"]


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
        sys.exit("optimizer_timing: needs a CUDA device")
    g = torch.Generator(device="cuda").manual_seed(0)
    tx = torch.rand(64, 48, 48, 1, device="cuda", generator=g) * 255
    tx2 = torch.rand(64, 192, 192, 1, device="cuda", generator=g) * 255
    ty = tx2 + torch.randn(64, 192, 192, 1, device="cuda", generator=g)
    wts = O.he_init_weights(O.OracleConfig(scale=4), seed=0)
    work = {}
    for opt in OPTIMIZERS:
        tr = E.Engine(E.make_config(scale=4, dropout_keep=0.8, optimizer=opt))
        tr.set_params(wts)
        # a learning rate small enough that no optimizer moves a layer out of its packed scale during the run
        work[opt] = (tr, {
            "train step L12 x4, 64 x 48^2": lambda e=tr: e.train_step(tx, tx2, ty, lr=1e-6, seed=1),
            "apply_gradients L12 x4": lambda e=tr: e.apply_gradients(1e-6),
        })
    for opt in OPTIMIZERS:                        # warm-up: plans, workspaces, the first host pack
        for fn in work[opt][1].values():
            for _ in range(3):
                fn()
    torch.cuda.synchronize()
    times = {(w, o): [] for o in OPTIMIZERS for w in work[o][1]}
    for r in range(args.rounds):
        order = OPTIMIZERS if r % 2 == 0 else OPTIMIZERS[::-1]
        for opt in order:
            for w, fn in work[opt][1].items():
                times[(w, opt)].append(timed(fn, args.reps))
    dev = card()
    print("device:", dev)
    rows = []
    for (w, opt), t in times.items():
        t = np.array(t)
        rows.append({"workload": w, "optimizer": opt, "median_ms": float(np.median(t)), "min_ms": float(t.min()),
                     "max_ms": float(t.max())})
        print("%-30s %-9s median %8.3f ms  (min %.3f, max %.3f)" % (w, opt, np.median(t), t.min(), t.max()))
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"device": dev, "rounds": args.rounds, "reps": args.reps, "rows": rows}, f, indent=1)
    for e, _ in work.values():
        e.close()


if __name__ == "__main__":
    main()
