"""
Parity where an activation buffer holds more than 2^31 (and 2^32) elements per plane (run with `-m gpu` on an H100).

The feature concat buffer of an L12 graph is feat_pitch = sum pad16(filters) = 1408 channels per LR pixel, so it
crosses 2^31 elements above 1,525,201 LR pixels and 2^32 above 3,050,402: one 1920 x 1080 LR frame at x2 (sr.py to
4K), the self-ensemble of a 960 x 540 frame (transforms 0-3 run as one n = 4 forward) and a x2 train step of 704
48 x 48 patches all get there.  Every kernel forms its plane offsets in 64 bits, except last_dgrad_s2d_kernel and
s2d_planes_kernel, whose 32-bit index math the train step's guard (case 5) keeps in range.  An offset that lost its top
bit would write the bottom of the frame over its top, or read gradients from the wrong pixels, and nothing at the
smaller shapes of the rest of the suite would notice.  Each case here asserts that it crosses its boundary, computed
from the config, and prints that figure with the engine's device_bytes:

  1. one 1920 x 1080 LR frame of real content at x2, f16x3 and f16x1: the whole-image forward equals the tiled forward
     (windows far below 2^28 elements) bit for bit, two more forwards into the same output replay the CUDA graph and
     equal it, the device bicubic equals Pillow's; f16x3: the fp64 oracle on a corner crop at each of the four corners
     (tile_halo pixels of context, so the crop's core is the frame's) within 1e-3 - the bottom-right core holds the
     highest offsets;
  2. four 1280 x 720 frames at x2 (5.19e9 elements): every image bit-identical to its own batch-1 forward, and the
     bottom corners of the last image, whose feature offsets lie past 2^32, at the fp64 oracle;
  3. the self-ensemble of a 960 x 540 LR frame: equal to the tiled ensemble and to the serial loop of eight batch-1
     forwards (none of which crosses 2^31) bit for bit, and evaluate_image equal to the host's do_for_evaluate;
  4. a x2 train step of 704 real 48 x 48 patches (keep 1): split into 8 sub-batches of 88, the loss count and the
     power-of-two loss scale G = 2^round(log2(count / 2)) both move by exactly 8, so dY = (y_ - y) 2 G / count is the
     same per image, and so is every per-pixel plane after it: the big step's fp64 reference is the mean of the
     sub-batches' (test_gpu_backward_paths.check_step on each, which also checks each sub-batch's own planes).  Every
     filter, bias and slope gradient of the big step lies within its own bar, assembled from the sub-batches' sums of
     |terms| (S is additive over pixels) with the big launch's chunk count and ksplit, and the loss is within fp32
     rounding of the mean of the sub-batch losses;
  5. the train step's guard: a x2 batch with more than 4e9 gradient elements in its widest tensor (1536 M, 1,131
     patches) is refused before it launches or allocates anything, and the same handle then runs case 4.

Each case first checks that the device has the memory it needs (it skips, with the numbers, when it has not) and closes
its engines before the next.
"""
import gc
import glob
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image

import dcscn_oracle as O
from conftest import GOLDEN, MODEL_FLAGS, load_golden_weights
from test_gpu_backward_paths import (L12, U24, Checker, capture_step, check_step, finalized,  # noqa: F401
                                     real_patches, release_reference_memory, report)  # (an autouse fixture)
from test_gpu_eval import MODELS, build_model, same
from test_gpu_tiled import budget_mb, run_entry, tiled_then_whole
from test_gpu_work_items import batch_one_mismatches

pytestmark = pytest.mark.gpu

GiB = 1 << 30
MiB = 1 << 20
I31, I32 = 2 ** 31, 2 ** 32
X2 = L12[2]
CELL = 224            # mosaic cells: every Set5 / Set14 fixture is at least this large on both sides
CORE = 64             # LR pixels per side of each corner crop's core
WINDOW_PX = 1 << 17   # LR pixels per batch of windows in the tiled runs: 2^17 * 1408 = 1.8e8 < 2^28 elements
# device bytes per LR pixel of an L12 x2 train step, with room: the handle of the 704-patch step below held 34.1 GB
# (21 KB per LR pixel) on an H100 80GB HBM3
TRAIN_PX_BYTES = 26 << 10


def pad16(v):
    return (v + 15) // 16 * 16


def feat_pitch(kw):
    return sum(pad16(f) for f in O.feature_filters(O.OracleConfig(**kw)))


def need_memory(what, need):
    """Skips the case, with the numbers, when the device has less than `need` bytes free."""
    free, total = torch.cuda.mem_get_info()
    print("%s: needs about %.1f GB, %.1f GB of %.1f GB free" % (what, need / 1e9, free / 1e9, total / 1e9))
    if free < need:
        pytest.skip("%s needs about %.1f GB of device memory; %.1f GB of %.1f GB are free" % (what, need / 1e9, free / 1e9,
                                                                                              total / 1e9))


@pytest.fixture
def engines():
    """Engines a case opens; closed, and torch's cache emptied, before the next case."""
    opened = []
    yield opened
    for eng in opened:
        eng.close()
    opened.clear()
    gc.collect()
    torch.cuda.empty_cache()


def new_engine(engines, precision=0):
    """The L12 x2 checkpoint, and its workspace bytes per LR pixel measured on an 8 x 8 forward (test_gpu_tiled)."""
    from helper import engine as E
    eng = E.Engine(E.make_config(precision=precision, **MODEL_FLAGS[X2]))
    engines.append(eng)
    eng.set_params(load_golden_weights(X2))
    eng.forward(torch.zeros(1, 8, 8, 1, device="cuda"), torch.zeros(1, 16, 16, 1, device="cuda"))
    torch.cuda.synchronize()
    return eng, eng.device_bytes // 64


def inference_need(m, ws_px):
    """Workspace of an m-pixel x2 forward, the fp32 images around it (input, bicubic, outputs, staging), 2 GB over."""
    return m * (ws_px + 4 * (1 + 4 * 4)) + 2 * GiB


def mosaic(tmp_path, name, height, width):
    """A height x width RGB frame of real content: CELL x CELL crops of the Set5 and Set14 fixtures in turn, as a PNG."""
    files = sorted(glob.glob(os.path.join(GOLDEN, "data", "set5", "*.png"))) + \
        sorted(glob.glob(os.path.join(GOLDEN, "data", "set14", "*.png")))
    frame = np.zeros((height, width, 3), np.uint8)
    k = 0
    for y0 in range(0, height, CELL):
        for x0 in range(0, width, CELL):
            img = np.asarray(Image.open(files[k % len(files)]).convert("RGB"))
            k += 1
            hh, ww = min(CELL, height - y0), min(CELL, width - x0)
            frame[y0:y0 + hh, x0:x0 + ww] = img[:hh, :ww]
    path = str(tmp_path / name)
    Image.fromarray(frame).save(path)
    return path


def frame_inputs(path):
    """LR and bicubic inputs of a frame as the evaluate pipeline forms them (Pillow resize), [1, h, w, 1] fp32."""
    inp, bic, _ = O.build_inputs_for_evaluate(path, 2)
    return np.array(inp[None], dtype=np.float32), np.array(bic[None], dtype=np.float32)


@pytest.fixture(scope="module")
def frame_4k(tmp_path_factory):
    """A 3840 x 2160 frame: its LR input is one 1920 x 1080 frame."""
    return frame_inputs(mosaic(tmp_path_factory.mktemp("frames"), "uhd.png", 2160, 3840))


def corner_errors(kw, w, r, x, x2, y, corners=((0, 0), (0, 1), (1, 0), (1, 1))):
    """max |y - fp64 oracle| over the CORE x CORE LR core at each (bottom, right) corner of one image (x [h, w], x2 and y
    [2h, 2w] numpy): the oracle runs on the crop with r pixels of context on its inner sides, on the GPU."""
    cfg = O.OracleConfig(**kw)
    params = {k: torch.from_numpy(np.asarray(v, dtype=np.float64)).cuda() for k, v in w.items()}
    orc = O.Oracle(cfg, params, torch.float64)
    h, wd = x.shape
    out = {}
    for bottom, right in corners:
        y0, x0 = (h - CORE if bottom else 0), (wd - CORE if right else 0)
        a, b = max(0, y0 - r), max(0, x0 - r)
        e, f = min(h, y0 + CORE + r), min(wd, x0 + CORE + r)
        xc = torch.from_numpy(x[a:e, b:f].copy()).cuda().double()[None, None]
        x2c = torch.from_numpy(x2[2 * a:2 * e, 2 * b:2 * f].copy()).cuda().double()[None, None]
        with torch.no_grad():
            ref = orc.forward_nchw(xc, x2c, params=params)[0, 0].cpu().numpy()
        core = ref[2 * (y0 - a):2 * (y0 - a + CORE), 2 * (x0 - b):2 * (x0 - b + CORE)]
        got = y[2 * y0:2 * (y0 + CORE), 2 * x0:2 * (x0 + CORE)].astype(np.float64)
        out[(bottom, right)] = float(np.abs(got - core).max())
    return out


# ------------------------------------------------------------------------------ 1. one 1920 x 1080 LR frame ----
@pytest.mark.parametrize("precision", [0, 1], ids=["f16x3", "f16x1"])
def test_1080p_frame_at_x2(frame_4k, engines, precision):
    x, x2 = frame_4k
    n, h, w = x.shape[:3]
    assert (h, w) == (1080, 1920)
    m, fp = n * h * w, feat_pitch(MODEL_FLAGS[X2])
    assert m * fp > I31
    eng, ws_px = new_engine(engines, precision)
    need_memory("1920x1080 at x2", inference_need(m, ws_px))
    kw = {"scale": 2, **MODEL_FLAGS[X2]}
    mb = budget_mb(kw, ws_px, WINDOW_PX)
    assert mb * MiB // ws_px * fp < 2 ** 28, "a batch of windows would reach 2^28 elements"
    y_tiled, y_whole, _, _, _ = tiled_then_whole(eng, mb, "forward", x, x2)
    print("1920x1080 %s: M = %d, feat %d elements (%.2f x 2^31), device_bytes %.2f GB" % (
        ("f16x3", "f16x1")[precision], m, m * fp, m * fp / I31, eng.device_bytes / 1e9))
    assert np.isfinite(y_whole).all()
    assert np.array_equal(y_tiled, y_whole), float(np.abs(y_tiled.astype(np.float64) - y_whole).max())
    print("  tiled (%d MiB) == whole: bit for bit" % mb)

    xd, x2d = torch.from_numpy(x).cuda(), torch.from_numpy(x2).cuda()
    y = eng.forward(xd, x2d)
    torch.cuda.synchronize()
    y0 = y.cpu().numpy()
    assert np.array_equal(y0, y_whole)
    r0 = eng.graph_replays
    for _ in range(2):                     # the second forward of one input captures the front, the third replays it
        eng.forward(xd, x2d, y)
        torch.cuda.synchronize()
        assert torch.equal(y.cpu(), torch.from_numpy(y0))
    assert eng.graph_replays - r0 == 2
    print("  two forwards into the same output through the CUDA graph: bit for bit")
    del xd, x2d, y

    y_bic = run_entry(eng, "host_bicubic", x, x2)
    assert np.array_equal(y_bic, y_whole), float(np.abs(y_bic.astype(np.float64) - y_whole).max())
    print("  forward(x, None) (device bicubic) == forward with Pillow's x2: bit for bit")

    if precision == 0:
        r = eng.tile_halo()
        br = ((h - CORE) * w + (w - CORE)) * fp      # the bottom-right core's first feature offset
        assert br > I31
        err = corner_errors(kw, load_golden_weights(X2), r, x[0, :, :, 0], x2[0, :, :, 0], y_whole[0, :, :, 0])
        print("  fp64 oracle on the corner cores (bottom-right from feat offset %.2f x 2^31): max |y - fp64| %s, "
              "error / bar %.3f" % (br / I31, {k: "%.2e" % v for k, v in err.items()}, max(err.values()) / 1e-3))
        assert max(err.values()) <= 1e-3, err


# --------------------------------------------------------------------------- 2. four 1280 x 720 frames, 2^32 ----
def test_four_720p_frames_past_2_32(frame_4k, engines):
    xf, x2f = frame_4k
    h, w = 720, 1280
    corners = [(0, 0), (0, 1920 - w), (1080 - h, 0), (1080 - h, 1920 - w)]     # four different frames of the mosaic
    x = np.ascontiguousarray(np.stack([xf[0, a:a + h, b:b + w] for a, b in corners]))
    x2 = np.ascontiguousarray(np.stack([x2f[0, 2 * a:2 * (a + h), 2 * b:2 * (b + w)] for a, b in corners]))
    n = x.shape[0]
    m, fp = n * h * w, feat_pitch(MODEL_FLAGS[X2])
    assert m == 3686400 and m * fp > I32
    bottom = ((n - 1) * h * w + (h - CORE) * w) * fp     # the last image's bottom cores start past 2^32
    assert bottom > I32
    eng, ws_px = new_engine(engines, 0)
    need_memory("4 x 1280x720 at x2", inference_need(m, ws_px) + m * 4 * 4)
    xd, x2d = torch.from_numpy(x).cuda(), torch.from_numpy(x2).cuda()
    y = eng.forward(xd, x2d)
    torch.cuda.synchronize()
    print("4 x 1280x720 f16x3: M = %d, feat %d elements (%.2f x 2^32), device_bytes %.2f GB" % (
        m, m * fp, m * fp / I32, eng.device_bytes / 1e9))
    assert torch.isfinite(y).all()
    bad = batch_one_mismatches(eng, xd, x2d, y)
    print("  images differing from their batch-1 forward: %s" % bad)
    assert bad == []
    kw = {"scale": 2, **MODEL_FLAGS[X2]}
    err = corner_errors(kw, load_golden_weights(X2), eng.tile_halo(), x[-1, :, :, 0], x2[-1, :, :, 0],
                        y[-1, :, :, 0].cpu().numpy())
    print("  last image, fp64 oracle on the corner cores (bottom ones from feat offset %.3f x 2^32): max |y - fp64| %s, "
          "error / bar %.3f" % (bottom / I32, {k: "%.2e" % v for k, v in err.items()}, max(err.values()) / 1e-3))
    assert max(err.values()) <= 1e-3, err


# ------------------------------------------------------------------- 3. self-ensemble of a 960 x 540 LR frame ----
def test_self_ensemble_of_a_540p_frame(tmp_path, engines):
    from helper import utilty as util
    path = mosaic(tmp_path, "fhd.png", 1080, 1920)
    x, x2 = frame_inputs(path)
    h, w = x.shape[1:3]
    assert (h, w) == (540, 960)
    fp = feat_pitch(MODEL_FLAGS[X2])
    m = 4 * h * w                                     # transforms 0-3 (and 4-7) run as one n = 4 forward
    assert m * fp > I31 and h * w * fp < I31
    eng, ws_px = new_engine(engines, 0)
    need_memory("self-ensemble of 960x540 at x2", inference_need(m, ws_px) + 8 * m * 4 * 4)
    kw = {"scale": 2, **MODEL_FLAGS[X2]}
    mb = budget_mb(kw, ws_px, WINDOW_PX)
    assert mb * MiB // ws_px * fp < 2 ** 28
    y_tiled, y_whole, _, _, _ = tiled_then_whole(eng, mb, "ensemble8", x, x2)
    print("ensemble 960x540: M = %d per batch, feat %d elements (%.2f x 2^31), device_bytes %.2f GB" % (
        m, m * fp, m * fp / I31, eng.device_bytes / 1e9))
    assert np.isfinite(y_whole).all()
    assert np.array_equal(y_tiled, y_whole), float(np.abs(y_tiled - y_whole).max())
    print("  tiled ensemble (%d MiB) == whole: bit for bit" % mb)

    y_ens = eng.forward_ensemble_host(x[0], x2[0], 8)         # Pillow's x2, as the serial loop below takes it
    assert np.array_equal(y_ens, y_whole)
    ref = np.zeros_like(y_ens)
    for i in range(8):
        c = lambda a: np.ascontiguousarray(a[None], dtype=np.float32)
        yi = eng.forward_host(c(util.flip(x[0], i)), c(util.flip(x2[0], i)))
        ref += util.flip(yi[0], i, invert=True)
    ref /= 8
    print("  serial loop of 8 batch-1 forwards: max |ensemble - loop| %.3g" % float(np.abs(y_ens - ref).max()))
    assert np.array_equal(y_ens, ref)
    for e in engines:
        e.close()
    engines.clear()
    torch.cuda.empty_cache()

    mdl = build_model(tmp_path, MODELS["L12x2"])
    engines.append(mdl.engine)
    mdl.self_ensemble = 8
    got, want = mdl.do_for_evaluate(path), mdl._do_for_evaluate_host(path)
    print("  evaluate_image (PSNR, SSIM) %s, host do_for_evaluate %s" % (got, want))
    assert same(got, want)


# -------------------------------------------------------------------- 4 and 5. the x2 train step past 2^31 ----
N_BIG, N_SUB, N_REFUSED = 704, 88, 1131
PATCH = 48


def widest_gradient(kw, m):
    """Elements of the widest gradient tensor of an m-pixel train step, as the engine's guard counts them."""
    cfg = O.OracleConfig(**kw)
    cps = cfg.nin_filters + cfg.nin_filters2
    return m * cfg.scale ** 2 * max(cfg.pixel_shuffler_filters or cps, 4 * cps)


@pytest.fixture(scope="module")
def big_step():
    """One handle: a small step, the refused batch of N_REFUSED patches, then the step of N_BIG patches (keep 1, no
    update).  Returns what the refusal left and the big step's loss and gradients; the handle is closed."""
    from helper import engine as E
    kw = MODEL_FLAGS[X2]
    m = N_BIG * PATCH * PATCH
    need_memory("x2 train step of %d patches" % N_BIG, m * TRAIN_PX_BYTES + 2 * GiB)
    x, x2, y = real_patches(2, N_REFUSED, PATCH, PATCH, 24)
    wts = load_golden_weights(X2)
    free0 = torch.cuda.mem_get_info()[0]
    eng = E.Engine(E.make_config(dropout_keep=1.0, **kw))
    eng.set_params(wts)
    out = {}
    try:
        eng.train_step_host(x[:1], x2[:1], y[:1], lr=0.002, seed=3, apply_update=False)
        l0, d0 = eng.launch_count, eng.device_bytes
        with pytest.raises(E.EngineError) as ei:
            eng.train_step_host(x, x2, y, lr=0.002, seed=3, apply_update=False)
        out["refusal"] = (str(ei.value), eng.launch_count - l0, eng.device_bytes - d0)
        x, x2, y = x[:N_BIG], x2[:N_BIG], y[:N_BIG]
        out["loss"] = eng.train_step_host(x, x2, y, lr=0.002, seed=3, apply_update=False)[0]
        out["device_bytes"] = eng.device_bytes        # the activation workspace
        out["engine_bytes"] = free0 - torch.cuda.mem_get_info()[0]   # everything the handle holds, gradient planes too
        out["grads"] = {name: eng.get_grad(name) for name in eng.param_shapes()}
    finally:
        eng.close()
    gc.collect()
    torch.cuda.empty_cache()
    out.update(x=x, x2=x2, y=y, weights=wts)
    return out


def test_train_step_guard_refuses_past_4e9(big_step):
    kw = MODEL_FLAGS[X2]
    assert widest_gradient(kw, N_REFUSED * PATCH * PATCH) >= 4e9 > widest_gradient(kw, (N_REFUSED - 1) * PATCH * PATCH)
    msg, launches, dbytes = big_step["refusal"]
    print("refused %d patches (%d gradient elements): %s; launches %+d, device_bytes %+d" % (
        N_REFUSED, widest_gradient(kw, N_REFUSED * PATCH * PATCH), msg, launches, dbytes))
    assert "too large" in msg and "%d 48x48" % N_REFUSED in msg
    assert launches == 0 and dbytes == 0


def test_x2_train_step_past_2_31(big_step):
    kw = MODEL_FLAGS[X2]
    x, x2, y, wts = big_step["x"], big_step["x2"], big_step["y"], big_step["weights"]
    m, fp = N_BIG * PATCH * PATCH, feat_pitch(kw)
    assert m * fp > I31 and widest_gradient(kw, m) < 4e9
    print("x2 train step of %d patches: M = %d, feat / dconcat / zneg %d elements (%.2f x 2^31), device_bytes %.2f GB, "
          "%.2f GB held by the handle" % (N_BIG, m, m * fp, m * fp / I31, big_step["device_bytes"] / 1e9,
                                          big_step["engine_bytes"] / 1e9))
    subs = N_BIG // N_SUB
    count_big, count_sub = N_BIG * 4 * PATCH * PATCH, N_SUB * 4 * PATCH * PATCH
    g_big, g_sub = (2.0 ** round(math.log2(c / 2.0)) for c in (count_big, count_sub))
    assert g_big == subs * g_sub        # dY = (y_ - y) 2 G / count: the same per image in the big step and its parts

    from helper import engine as E
    eng = E.Engine(E.make_config(dropout_keep=1.0, **kw))
    sums, losses = {}, []
    try:
        eng.set_params(wts)
        for i in range(subs):
            sl = slice(i * N_SUB, (i + 1) * N_SUB)
            losses.append(capture_step(eng, x[sl], x2[sl], y[sl], 1.0, 3)[0])
            chk = check_step(eng, kw, wts, x[sl], x2[sl], y[sl], 1.0, 3, Checker(), bar_n=N_BIG)
            assert not chk.bad(), (i, chk.bad())
            for name, (s, b, dec) in chk.sums.items():
                acc = sums.setdefault(name, [0.0, 0.0, dec])
                acc[0], acc[1] = acc[0] + s, acc[1] + b
            del chk
    finally:
        eng.close()

    worst, bad = {}, []
    for name, (s, b, dec) in sums.items():     # sum / G_big = (sum over the parts of sum_i / G_sub) / subs
        ref, bar = finalized(s / subs, b / subs, dec)
        got = torch.from_numpy(big_step["grads"][name]).cuda().double()
        ratio = float(((got - ref).abs() / bar).max())
        kind = name.rsplit("/", 1)[-1].split("_")[-1]
        worst[kind] = max(worst.get(kind, 0.0), ratio)
        if not ratio <= 1.0:
            bad.append((name, ratio))
    assert sorted(sums) == sorted(big_step["grads"])
    print("  gradients against the mean of %d sub-batch references, error / bar: %s" % (
        subs, " ".join("%s %.3f" % kv for kv in sorted(worst.items()))))
    mean = float(np.mean(np.asarray(losses, np.float64)))
    loss = big_step["loss"]
    lbar = U24 * (abs(loss) + abs(mean)) + 1e-12 * abs(mean)
    print("  loss %.9g, mean of the sub-batch losses %.9g: error / bar %.3f" % (loss, mean, abs(loss - mean) / lbar))
    assert not bad, bad
    assert abs(loss - mean) <= lbar
