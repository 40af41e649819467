"""Set5 PSNR of c-DCSCN x2 over 200 steps on Set14 patches per --optimizer, with the protocol of
tests/test_gpu_convergence.py (train_200 in tests/test_gpu_optimizers.py), at the reference's default learning rate
and any others given.  Prints the card's name and power limit, then one line per (optimizer, lr): the PSNR at steps
0/50/100/150/200 and the running mean loss.

    python scripts/optimizer_convergence.py [--lr 0.002 0.02] [--optimizers gd momentum ...] [--out result.json]
"""
import argparse
import json
import os
import pathlib
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in ("dcscn-super-resolution_b200", "oracle", "tests"):
    sys.path.insert(0, os.path.join(ROOT, p))

from test_gpu_optimizers import train_200  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lr", type=float, nargs="+", default=[0.002])
    ap.add_argument("--optimizers", nargs="+", default=["adam", "gd", "momentum", "adadelta", "adagrad", "rmsprop"])
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("optimizer_convergence: needs a CUDA device")
    dev = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    print("device:", dev)
    rows = []
    for lr in args.lr:
        for opt in args.optimizers:
            with tempfile.TemporaryDirectory() as d:
                curve, losses = train_200(pathlib.Path(d), opt, lr)
            rows.append({"optimizer": opt, "lr": lr, "psnr": curve, "loss": losses})
            print("%-9s lr %-7g PSNR %s  loss %s" % (opt, lr, " ".join("%.2f" % p for p in curve),
                                                     " ".join("%.1f" % v for v in losses)), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"device": dev, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
