"""Where the cycles of each conv_tc_kernel launch of the bench headline go: a diagnostic build of the library
(-DDCSCN_TC_PHASES) sums clock64() per phase over the consumer warpgroups of every CTA, and this script prints, per
launch, the K loop and the consumers' epilogue cycles per item, the epilogue's share of the item, and the busy cycles
per item of an epilogue warp (builds that run the epilogue on warps 1-3 of the producer warpgroup).

usage: python scripts/tc_phases.py [--lib LIB] [--precision f16x3|f16x1] [--reps R] [--workload infer|train]
Without --lib the diagnostic library is compiled from the tree into a temporary directory (about a minute or more).
The diagnostic build waits for every launch, so its timings are not the product's; only the shares are meaningful."""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dcscn-super-resolution_b200", "csrc")


def build_diag(out_dir):
    lib = os.path.join(out_dir, "libdcscn_b200_phases.so")
    cmd = [os.environ.get("NVCC", "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
           "-DDCSCN_TC_PHASES", "-Xcompiler", "-fPIC", "-shared", "-o", lib, os.path.join(CSRC, "engine.cu")]
    subprocess.check_call(cmd, cwd=CSRC)
    return lib


def run(lib, precision, reps, workload):
    """One headline forward (or bench.py's L12 x4 train step) per rep with the diagnostic library; returns the stderr
    lines it wrote."""
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "dcscn-super-resolution_b200"))
    import torch
    import bench
    from helper import engine as E
    E.load_library(lib)
    prec = E.PRECISION_F16X1 if precision == "f16x1" else E.PRECISION_F16X3
    g = torch.Generator().manual_seed(0)
    if workload == "train":
        eng = E.Engine(E.make_config(scale=4, precision=prec))
        eng.set_params(bench.load_weights(bench.MODEL_X4))
        x = (torch.rand(64, 48, 48, 1, generator=g) * 255).cuda()
        x2 = (torch.rand(64, 192, 192, 1, generator=g) * 255).cuda()
        y = (torch.rand(64, 192, 192, 1, generator=g) * 255).cuda()
        step = lambda i: eng.train_step_data_parallel(x, x2, y, lr=1e-6, seed=i)
    else:
        eng = E.Engine(E.make_config(precision=prec))
        eng.set_params(bench.load_weights())
        x = (torch.rand(256, 48, 48, 1, generator=g) * 255).cuda()
        x2 = (torch.rand(256, 96, 96, 1, generator=g) * 255).cuda()
        y = torch.empty_like(x2)
        step = lambda i: eng.forward(x, x2, y)
    eng.set_option("graph", 0)   # the report synchronises after each launch, which a captured graph cannot
    with tempfile.TemporaryFile(mode="w+") as f:
        saved = os.dup(2)
        sys.stderr.flush()
        os.dup2(f.fileno(), 2)
        try:
            for i in range(1 + reps):      # the first call plans and loads modules; its counters count too
                step(i)
            torch.cuda.synchronize()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        lines = [ln for ln in f.read().splitlines() if ln.startswith("tc_phase ")]
    eng.close()
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="a library built with -DDCSCN_TC_PHASES")
    ap.add_argument("--precision", default="f16x3", choices=["f16x3", "f16x1"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workload", default="infer", choices=["infer", "train"],
                    help="the bench headline forward, or bench.py's L12 x4 train step (64 patches of 48x48)")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        lib = a.lib or build_diag(tmp)
        lines = run(os.path.abspath(lib), a.precision, a.reps, a.workload)
    if not lines:
        sys.exit("no tc_phase lines: %s is not a -DDCSCN_TC_PHASES build" % lib)
    acc, plan, order = {}, {}, []
    for ln in lines:
        kv = dict(re.findall(r"(\w+)=(\S+)", ln))
        name = ln.split()[1]
        if name not in acc:
            order.append(name)
            acc[name] = [0, 0, 0, 0]
        for i, key in enumerate(("k", "epi", "items", "epw")):
            acc[name][i] += int(kv[key])
        plan[name] = "N=%s x%s %s a=%s w=%s smem=%s" % (kv["n_pad"], kv["n_tiles"], kv["patch"], kv["a_slots"],
                                                         kv["w_slots"], kv["smem"])
    print("%-12s %-44s %10s %10s %10s %7s" % ("launch", "plan", "K cyc/item", "epi/item", "epw/item", "epi %"))
    for name in order:
        k, e, n, w = acc[name]
        n = max(n, 1)
        # k, e and n count per consumer warpgroup (2 per item), w per epilogue warp (3 per item)
        print("%-12s %-44s %10.0f %10.0f %10.0f %6.1f%%" % (name, plan[name], k / n, e / n, w / (1.5 * n),
                                                           100.0 * e / (k + e)))


if __name__ == "__main__":
    main()
