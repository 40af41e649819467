"""Tiled inference (option "workspace_mb") on one GPU: ms per forward of 1080p LR images through the L12 x2 / x4
checkpoints, whole-image (where its workspace is at most 16 GiB) and tiled at 1, 2, 4 and 8 GiB; a 2160p x2 forward and
the 8-flip ensemble of the 1080p image tiled at 4 GiB.  Prints one JSON line.

Per tiled run: windows per image and halo overhead (window pixels / image pixels) of the window plan, restated from
plan_tiles in csrc/engine.cu and checked against the number of batches the engine reports with option "timing";
device_bytes; whether the output equals the whole-image forward bit for bit (where the whole image ran), and whether a
256 x 256 core at the image centre equals the untiled forward of that crop with its halo (every run)."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dcscn-super-resolution_b200"))
from helper import engine as E, tf_bundle  # noqa: E402

MiB, GiB = 1 << 20, 1 << 30
MODELS = {2: "dcscn_L12_F196to48_NIN_A64_PS_R1F32", 4: "dcscn_L12_F196to48_Sc4_NIN_A64_PS_R1F32"}
REPS, WARMUP = 10, 2


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, clock = [v.strip() for v in q.split(",")]
    return {"gpu": name, "power_limit_w": float(power), "max_sm_clock_mhz": int(float(clock))}


def engine(scale):
    r = tf_bundle.BundleReader(os.path.join(ROOT, "tests", "golden", "models", MODELS[scale] + ".ckpt"))
    eng = E.Engine(E.make_config(scale=scale))
    eng.set_params({k: r.get_tensor(k) for k in r.keys()})
    return eng


def ws_bytes_per_px(scale):
    eng = engine(scale)
    eng.forward(torch.zeros(1, 8, 8, 1, device="cuda"), torch.zeros(1, 8 * scale, 8 * scale, 1, device="cuda"))
    torch.cuda.synchronize()
    b = eng.device_bytes // 64
    eng.close()
    return b


def tile_count(D, T, r):
    return 1 if T >= D else 2 + max(0, -(-(D - 2 * T + 2 * r) // (T - 2 * r)))


def plan(n, H, W, s, ws_px, budget, r, vec4=True):
    """plan_tiles of csrc/engine.cu: (th, tw, windows per image, windows per batch)."""
    max_px = budget // (ws_px + 4 * (1 + 2 * s * s))
    min_th = min(H, 16 + 2 * r)
    min_tw = min(W, ((16 + 2 * r + 3) & ~3) if vec4 else 16 + 2 * r)
    best = None
    th = min_th
    while th <= H and th * min_tw <= max_px:
        tw = min(W, max_px // th)
        if tw < W and vec4:
            tw &= ~3
        if tw >= min_tw:
            my, mx = tile_count(H, th, r), tile_count(W, tw, r)
            key = (my * mx * th * tw, -th * tw)
            if best is None or key < best[0]:
                best = (key, th, tw, my * mx)
        th += 1
    _, th, tw, per = best
    return th, tw, per, max(1, min(n * per, max_px // (th * tw)))


def image(h, w, s, seed):
    """Noise over a diagonal gradient (LR), and its HR companion x2."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    yy = torch.linspace(0, 1, h, device="cuda").view(h, 1)
    xx = torch.linspace(0, 1, w, device="cuda").view(1, w)
    x = (160 * (yy + xx) / 2 + 60 * torch.rand(h, w, device="cuda", generator=g)).view(1, h, w, 1).contiguous()
    x2 = (255 * torch.rand(1, s * h, s * w, 1, device="cuda", generator=g)).contiguous()
    return x, x2


def time_ms(fn):
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(REPS):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / REPS


def batches_reported(eng, fn):
    eng.set_option("timing", 1)
    fn()
    torch.cuda.synchronize()
    n = sum(name == "tile_gather" for name, _ in eng.timings())
    eng.set_option("timing", 0)
    return n


def centre_core_matches(eng, mb, x, x2, y, s, r, c=256):
    h, w = x.shape[1], x.shape[2]
    a0, b0 = (h - c) // 2, (w - c) // 2
    xc = x[:, a0 - r:a0 + c + r, b0 - r:b0 + c + r].contiguous()
    x2c = x2[:, s * (a0 - r):s * (a0 + c + r), s * (b0 - r):s * (b0 + c + r)].contiguous()
    eng.set_option("workspace_mb", 0)
    yc = eng.forward(xc, x2c)
    torch.cuda.synchronize()
    eng.set_option("workspace_mb", mb)
    return bool(torch.equal(yc[:, s * r:s * (r + c), s * r:s * (r + c)], y[:, s * a0:s * (a0 + c), s * b0:s * (b0 + c)]))


def tiled_run(scale, x, x2, gib, ws_px, y_whole=None, ensemble=False):
    eng = engine(scale)                             # fresh handle: device_bytes is this run's
    r = eng.tile_halo()
    n, H, W = x.shape[0], x.shape[1], x.shape[2]
    eng.set_option("workspace_mb", gib * 1024)
    if ensemble:
        out = torch.empty((scale * H, scale * W), dtype=torch.float64, device="cuda")
        xe, x2e = x[0, :, :, 0].contiguous(), x2[0, :, :, 0].contiguous()
        fn = lambda: eng.forward_ensemble(xe, x2e, 8, out=out)  # noqa: E731
    else:
        y = torch.empty_like(x2)
        fn = lambda: eng.forward(x, x2, y)  # noqa: E731
    ms = time_ms(fn)
    th, tw, per, batch = plan(n, H, W, scale, ws_px, gib * GiB, r)
    rec = {"workspace_gib": gib, "ms": round(ms, 3), "window": [th, tw], "windows_per_image": per,
           "windows_per_batch": batch, "halo_overhead": round(per * th * tw / (H * W), 4),
           "device_bytes": eng.device_bytes}
    if not ensemble:
        rec["batches"] = batches_reported(eng, fn)
        rec["batches_planned"] = -(-n * per // batch)
        rec["centre_core_bit_identical"] = centre_core_matches(eng, gib * 1024, x, x2, y, scale, r)
        if y_whole is not None:
            rec["bit_identical_to_whole"] = bool(torch.equal(y, y_whole))
    eng.close()
    return rec


def main():
    assert torch.cuda.is_available(), "tile_timing.py needs a GPU"
    out = gpu_info()
    out["reps"] = REPS
    H, W = 1080, 1920
    for s in (2, 4):
        ws_px = ws_bytes_per_px(s)
        x, x2 = image(H, W, s, seed=s)
        res = {"lr": [H, W], "workspace_bytes_per_lr_px": ws_px, "whole_workspace_bytes": ws_px * H * W}
        y_whole = None
        if ws_px * H * W <= 16 * GiB:
            eng = engine(s)
            y_whole = torch.empty_like(x2)
            res["whole_ms"] = round(time_ms(lambda: eng.forward(x, x2, y_whole)), 3)
            torch.cuda.synchronize()
            eng.close()
        else:                                      # the left half fits: its rate stands in for the whole image
            eng = engine(s)
            xl, x2l = x[:, :, :W // 2].contiguous(), x2[:, :, :s * W // 2].contiguous()
            res["whole_ms_from_left_half"] = round(2 * time_ms(lambda: eng.forward(xl, x2l)), 3)
            eng.close()
        base = res.get("whole_ms", res.get("whole_ms_from_left_half"))
        res["tiled"] = []
        for gib in (1, 2, 4, 8):
            rec = tiled_run(s, x, x2, gib, ws_px, y_whole)
            rec["predicted_ms"] = round(base * rec["halo_overhead"], 3)
            rec["ms_over_predicted"] = round(rec["ms"] / rec["predicted_ms"], 4)
            res["tiled"].append(rec)
        out["x%d_1080p" % s] = res
        del y_whole
        torch.cuda.empty_cache()
    ws2 = ws_bytes_per_px(2)
    x, x2 = image(2160, 3840, 2, seed=7)
    out["x2_2160p_4gib"] = tiled_run(2, x, x2, 4, ws2)
    del x, x2
    torch.cuda.empty_cache()
    x, x2 = image(H, W, 2, seed=2)
    out["x2_1080p_ensemble8_4gib"] = tiled_run(2, x, x2, 4, ws2, ensemble=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
