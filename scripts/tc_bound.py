"""Where the K loop of each conv_tc_kernel launch of the bench headline is bound: per-launch median times of the product
build against two diagnostic builds of the same sources, fill only (-DDCSCN_TC_BOUND=1: the consumers release every
slot without issuing wgmma) and math only (-DDCSCN_TC_BOUND=2: after the first fill of each ring the producer arrives
without copying).  A launch whose normal time sits near its fill-only time is bound by what the SM takes in; near its
math-only time, by the wgmma.  The three engines alternate in one process, as in scripts/ab_libs.py.  The outputs of the
diagnostic builds are meaningless and are never compared.

usage: python scripts/tc_bound.py [--src DIR | --libs NORMAL FILL MATH] [--precision f16x3|f16x1] [--rounds R]
--src compiles the three libraries from DIR/dcscn-super-resolution_b200/csrc (default: this tree) into a temporary
directory (a few minutes); --libs takes prebuilt ones."""
import argparse
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANTS = ("normal", "fill-only", "math-only")


def build(src_root, out_dir):
    csrc = os.path.join(src_root, "dcscn-super-resolution_b200", "csrc")

    def one(i):
        lib = os.path.join(out_dir, "libdcscn_b200_bound%d.so" % i)
        cmd = [os.environ.get("NVCC", "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
               "-Xcompiler", "-fPIC", "-shared", "-o", lib, os.path.join(csrc, "engine.cu")]
        if i:
            cmd.insert(1, "-DDCSCN_TC_BOUND=%d" % i)
        subprocess.check_call(cmd, cwd=csrc)
        return lib
    with ThreadPoolExecutor(3) as ex:
        return list(ex.map(one, range(3)))


def run(libs, precision, rounds):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "dcscn-super-resolution_b200"))
    import torch
    import bench
    from helper import engine as E
    prec = E.PRECISION_F16X1 if precision == "f16x1" else E.PRECISION_F16X3
    w = bench.load_weights()
    engs = []
    for p in libs:
        E._lib = None
        E.load_library(os.path.abspath(p))
        eng = E.Engine(E.make_config(precision=prec))
        eng.set_params(w)
        eng.set_option("timing", 1)
        engs.append(eng)
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(256, 48, 48, 1, generator=g) * 255).cuda()
    x2 = (torch.rand(256, 96, 96, 1, generator=g) * 255).cuda()
    y = torch.empty_like(x2)
    acc = [{} for _ in engs]
    for eng in engs:
        for _ in range(3):
            eng.forward(x, x2, y)
    for _ in range(rounds):
        for i, eng in enumerate(engs):
            for _ in range(3):
                eng.forward(x, x2, y)
                for n, t in eng.timings():
                    acc[i].setdefault(n, []).append(t)
    for eng in engs:
        eng.close()
    return [{n: sorted(v)[len(v) // 2] for n, v in a.items()} for a in acc]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default=ROOT)
    ap.add_argument("--libs", nargs=3, default=None, metavar=("NORMAL", "FILL", "MATH"))
    ap.add_argument("--precision", default="f16x3", choices=["f16x3", "f16x1"])
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        libs = a.libs or build(os.path.abspath(a.src), tmp)
        med = run(libs, a.precision, a.rounds)
    print("%-10s %9s %9s %9s %7s %7s" % ("launch", "normal", "fill", "math", "fill/n", "math/n"))
    for n in med[0]:
        t = [m[n] for m in med]
        print("%-10s %9.4f %9.4f %9.4f %7.2f %7.2f" % (n, t[0], t[1], t[2], t[1] / t[0], t[2] / t[0]))


if __name__ == "__main__":
    main()
