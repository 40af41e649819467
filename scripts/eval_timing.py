"""Per-image wall time of SuperResolution.do_for_evaluate (evaluate.py --save_results=false) on Set5 and Set14, host path
(_do_for_evaluate_host: numpy / scipy / Pillow around the device self-ensemble) against the device path (decode on the
host, everything after it on the GPU).  The two paths alternate over several rounds; median and range of the per-round
mean ms per image are printed, then a torch.profiler split of the device path's kernels over one Set14 pass.

    python scripts/eval_timing.py [--rounds 5] [--out timing.json]
"""
import argparse
import glob
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dcscn-super-resolution_b200"))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CD = ["--layers=7", "--filters=32", "--min_filters=8", "--filters_decay_gamma=1.2", "--nin_filters=24",
      "--nin_filters2=8", "--reconstruct_layers=0", "--pixel_shuffler_filters=1"]
CASES = [("L12 x2, ensemble 8", ["--scale=2", "--self_ensemble=8"]), ("L12 x2, ensemble 1", ["--scale=2", "--self_ensemble=1"]),
         ("c-DCSCN x2, ensemble 8", ["--scale=2", "--self_ensemble=8"] + CD)]


def build_model(tmp, flag_args):
    from helper import args as A
    import DCSCN
    f = A._Flags()
    for name, (kind, default, help_text) in A.FLAGS._defs.items():
        f._define(name, default, help_text, kind)
    f.parse(["prog", "--checkpoint_dir=" + os.path.join(GOLDEN, "models"), "--log_filename=" + os.path.join(tmp, "log.txt"),
             "--tf_log_dir=" + os.path.join(tmp, "tf"), "--graph_dir=" + os.path.join(tmp, "g"),
             "--output_dir=" + os.path.join(tmp, "out")] + flag_args)
    m = DCSCN.SuperResolution(f, model_name=f.model_name)
    m.build_graph()
    m.build_summary_saver()
    m.init_all_variables()
    m.load_model(f.load_model_name)
    return m


def per_image_ms(fn, files):
    t0 = time.perf_counter()
    for f in files:
        fn(f)
    return (time.perf_counter() - t0) * 1e3 / len(files)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    sets = {s: sorted(glob.glob(os.path.join(GOLDEN, "data", s, "*.png"))) for s in ("set5", "set14")}
    rows = []
    tmp = tempfile.mkdtemp()
    for label, flags in CASES:
        m = build_model(tmp, flags)
        for name, files in sets.items():
            for f in files:                   # warm-up: launch plans of every image shape, both paths
                assert m.do_for_evaluate(f) == m._do_for_evaluate_host(f)
            host, dev = [], []
            for _ in range(a.rounds):
                host.append(per_image_ms(m._do_for_evaluate_host, files))
                dev.append(per_image_ms(m.do_for_evaluate, files))
            row = {"case": label, "set": name, "host_ms": [float(np.median(host)), min(host), max(host)],
                   "device_ms": [float(np.median(dev)), min(dev), max(dev)]}
            rows.append(row)
            print("%-24s %-5s host %7.2f ms (%.2f-%.2f)  device %7.2f ms (%.2f-%.2f)" % (
                label, name, *row["host_ms"], *row["device_ms"]), flush=True)
        if label.startswith("L12 x2, ensemble 8"):
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for f in sets["set14"]:
                    m.do_for_evaluate(f)
                torch.cuda.synchronize()
            split = {}
            for e in prof.key_averages():
                if e.device_type == torch.autograd.DeviceType.CUDA and ("kernel" in e.key or "Memcpy" in e.key):
                    split[e.key.split("(")[0].split("<")[0]] = split.get(e.key.split("(")[0].split("<")[0], 0.0) + \
                        e.device_time_total / 1e3 / len(sets["set14"])
            print("device time per Set14 image (ms), %s:" % label)
            for k, v in sorted(split.items(), key=lambda kv: -kv[1]):
                print("  %-40s %8.3f" % (k, v))
            rows.append({"case": label, "set": "set14", "kernel_ms_per_image": split})
        m.engine.close()
    if a.out:
        json.dump({"gpu": torch.cuda.get_device_name(0), "rows": rows}, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
