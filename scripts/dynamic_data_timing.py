"""Training step time on random-crop data (loader.DynamicDataSets, train.py without --build_batch): the host loader
(decode, crop, RGB -> Y, mirror and two Pillow resizes per patch in Python, then train_step_host) against the device image
store (draw_crop on the host, train_step_crops).  Each step is timed to a device synchronise; the two paths alternate over
rounds.  Then, in a run of its own, torch.profiler's kernel time of the crop pipeline, and the image-store upload.

Data: the in-tree Set14, and 32 synthetic 2040 x 1356 PNGs (DIV2K-sized files, so decoding costs what it does on real
training data) generated from a seed into --out.

    python scripts/dynamic_data_timing.py --out /tmp/dynamic_data
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dcscn-super-resolution_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))

SHAPES = {"train.py default (L12 x2, 20 x 48^2)": (2, 20, 48), "bench (L12 x4, 64 x 48^2)": (4, 64, 48)}
CROP_KERNELS = ("crop_gather_kernel", "crop_place_kernel", "pil_resample_h_kernel", "pil_resample_v_kernel",
                "pil_resample8_h_kernel", "pil_resample8_v_kernel")


def synthetic_pngs(out_dir, count=32, seed=0):
    from PIL import Image
    os.makedirs(out_dir, exist_ok=True)
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:1356, 0:2040].astype(np.float32)
    for i in range(count):
        path = os.path.join(out_dir, "img_%03d.png" % i)
        if os.path.isfile(path):
            continue
        f = rs.rand(3, 3) * 0.02
        base = np.stack([127 + 100 * np.sin(f[c, 0] * xx + f[c, 1] * yy + f[c, 2] * xx * yy / 500) for c in range(3)], -1)
        noise = rs.normal(0, 12, base.shape)
        Image.fromarray(np.clip(base + noise, 0, 255).astype(np.uint8), "RGB").save(path)
    return out_dir


def make_engine(scale):
    import dcscn_oracle as O
    from helper import engine as E
    eng = E.Engine(E.make_config(scale=scale))
    eng.set_params(O.he_init_weights(O.OracleConfig(scale=scale), seed=1))
    return eng


def host_step(eng, ds, batch, step):
    b = [ds.load_batch_image(255.0) for _ in range(batch)]
    x, x2, y = (np.ascontiguousarray(np.stack([v[j] for v in b]), dtype=np.float32) for j in range(3))
    return eng.train_step_host(x, x2, y, lr=1e-4, seed=step)


def device_step(eng, ds, batch, step):
    crops = np.array([ds.draw_crop() for _ in range(batch)], np.int32)
    return eng.train_step_crops(crops, ds.batch_image_size, lr=1e-4, seed=step)


def timed(fn, steps):
    import torch
    out = []
    for s in range(steps):
        t0 = time.perf_counter()
        fn(s)
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--host-steps", type=int, default=4, dest="host_steps")
    ap.add_argument("--device-steps", type=int, default=20, dest="device_steps")
    args = ap.parse_args()
    import torch
    from helper import loader
    assert torch.cuda.is_available(), "needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    print("card:", card)
    data = {"set14": os.path.join(ROOT, "tests", "golden", "data", "set14"),
            "synthetic 2040x1356 x32": synthetic_pngs(os.path.join(args.out, "synthetic"))}
    results = []
    for data_name, data_dir in data.items():
        for shape_name, (scale, batch, size) in SHAPES.items():
            eng = make_engine(scale)
            ds = loader.DynamicDataSets(scale, size)
            ds.set_data_dir(data_dir)
            images = ds.decoded_images()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.set_image_store(images)
            torch.cuda.synchronize()
            upload_ms = (time.perf_counter() - t0) * 1e3
            store_bytes = int(sum(im.size for im in images))
            random.seed(0)
            for s in range(2):                                    # warm both shapes of both paths
                host_step(eng, ds, batch, s)
                device_step(eng, ds, batch, s)
            host, dev = [], []
            for _ in range(args.rounds):
                host += timed(lambda s: host_step(eng, ds, batch, s), args.host_steps)
                dev += timed(lambda s: device_step(eng, ds, batch, s), args.device_steps)
            rec = dict(data=data_name, shape=shape_name, card=card, host_ms_median=float(np.median(host)),
                       host_ms_range=[float(min(host)), float(max(host))], device_ms_median=float(np.median(dev)),
                       device_ms_range=[float(min(dev)), float(max(dev))], upload_ms=upload_ms, store_bytes=store_bytes)
            print(json.dumps(rec), flush=True)
            results.append(rec)
            eng.close()
    # crop pipeline kernel time, in a run of its own (bench shape, synthetic data)
    from torch.profiler import ProfilerActivity, profile
    scale, batch, size = SHAPES["bench (L12 x4, 64 x 48^2)"]
    eng = make_engine(scale)
    ds = loader.DynamicDataSets(scale, size)
    ds.set_data_dir(data["synthetic 2040x1356 x32"])
    eng.set_image_store(ds.decoded_images())
    for s in range(3):
        device_step(eng, ds, batch, s)
    torch.cuda.synchronize()
    steps = 10
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for s in range(steps):
            device_step(eng, ds, batch, s)
        torch.cuda.synchronize()
    kernels, total = {}, 0.0
    for ev in prof.key_averages():
        if any(k in ev.key for k in CROP_KERNELS):
            us = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            kernels[ev.key.split("(")[0].split("::")[-1]] = dict(us_per_step=us / steps, calls=ev.count)
            total += us / steps
    rec = dict(profile="crop pipeline, bench shape, synthetic data", card=card, kernels=kernels, us_per_step=total)
    print(json.dumps(rec), flush=True)
    results.append(rec)
    eng.close()
    with open(os.path.join(args.out, "timing.json"), "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
