"""
Isolated per-layer forward parity where every tensor-core CTA runs many work items.

conv_tc_kernel is persistent: add_tc_launch (engine.cu) launches min(items, SMs) CTAs for
items = n * tiles_x * tiles_y * n_tiles, and each CTA walks items blockIdx.x, blockIdx.x + gridDim.x, ...  The TMA
ring slots and phases, the deferred slot releases and the epilogue exchange buffer carry over from one item to the
next; the image, the pixel tile (partial right and bottom tiles included) and the column tile n_tile, which selects
the weights, bias and slopes, change.  The other isolated checks run shapes small enough that every CTA computes one
item, so none of them reaches a CTA's second item.  Here every case has n H W >= 3 * 128 * SMs: a patch covers 128
pixels, so every tensor-core launch has at least n H W / 128 items and every CTA of every layer runs at least three,
whichever patch choose_patch picks and however many SMs the part has.

  * every TC_CASES configuration of test_gpu_forward_paths.py at such a batch of its images, each side odd, so that
    every side a patch tiles more than one pixel wide ends in a partial tile (a 1 x 201 or 129 x 1 image has one
    such side only), f16x3 and f16x1, seg_chunks 0 and 1, fused and unfused, and the
    folded-launch reference where the fold ran: every layer at its isolated bar, the kernels reached, and every image
    bit-identical to its own batch-1 forward;
  * bench.py's headline exactly as bench builds it (L12 x2 checkpoint, 256 uniform-noise 48 x 48 tiles, CUDA-graph
    replays): every replay bit-identical to the eager forward, every tile to its batch-1 forward, every layer at its
    isolated bar and y against the fp64 oracle (max 1.5e-3 at the default promotion periods, STRICT_HEADLINE at
    seg_chunks = 1, RMS HEADLINE_RMS; test_headline_batch says why 1e-3 does not hold at seg_chunks = 1);
  * the train step's forward at bench's train shape (L12 x4, 64 real 48 x 48 patches, keep 0.8): every layer, the
    zneg planes and the PReLU slope gradients (its backward is test_gpu_backward_paths.py's);
  * bench's depthwise-separable record (c-DCSCN DS L7 x4, 256 tiles): every layer, and repeated forwards into one
    output buffer bit-identical, issued eagerly (no CUDA-graph replay on that path).

The fp64 references run on the GPU a slice of images at a time, which keeps them to a few GB of device memory.
"""
import numpy as np
import pytest
import torch

import dcscn_oracle as O
from conftest import MODEL_FLAGS, load_golden_weights
from test_gpu_backward_paths import (L12, after_dropout, output_gradient, real_patches,  # noqa: F401
                                     release_reference_memory)  # (an autouse fixture)
from test_gpu_fold import folded_filter, folded_launch_ratios, gather9
from test_gpu_forward import TOL_DEFAULT_STRESS, check_depthwise_separable_layers, make_engine
from test_gpu_forward_paths import TC_CASES, col, conv, isolated_layers, nchw, prelu, quantise
from test_gpu_train import FAST, assert_kernels_ran, launched_kernels
from test_gpu_train_forward_paths import SlopeSums, captured_step, zneg_ratio

pytestmark = pytest.mark.gpu

GATHERS = ("conv_last_gather_kernel", "conv_last_gather4_kernel")
# Layers whose column-tile count does not divide 132 or 114, so a CTA's consecutive items change n_tile (the tile
# counts TC_CASES documents): x3-rdot1's Up-PS is 288 columns as 5 tiles of 64 (f16x1 and unfused; the f16x3 fold
# replaces it by one 96-column tile), ps128's Up-PS 512 columns as 5 tiles of 112.
COLUMN_TILES = {"x3-rdot1": 5, "x3-rdot1-1x200": 5, "ps128": 5}
# |y - fp64| over bench's 256 headline tiles (test_headline_batch): the strict setting's max, and the RMS of both f16x3
# settings, with about 25 % headroom over what an H100 measured (2.0e-3; RMS 1.2e-4 strict, 9.6e-5 default).
STRICT_HEADLINE = 2.5e-3
HEADLINE_RMS = 1.5e-4
CHUNK = 32          # images per slice of the fp64 references at the 48 x 48 tile shapes


def dev():
    return torch.device("cuda")


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def assert_many_items(n, h, w):
    """Every tensor-core launch of an n x h x w forward gives every CTA at least three items."""
    assert n * h * w >= 3 * 128 * sms(), (n, h, w, sms())


def odd(v):
    return v if v % 2 else v + 1


def work_case(case):
    """(id, config, (n, h, w), kernels) of a TC_CASES entry at a batch large enough for three items per CTA: each side
    made odd (1 x 200 -> 1 x 201), n = ceil(3 * 128 * SMs / (h w)).  The fused R-CNN1 gather is the four-pixel kernel
    exactly when the HR width is a multiple of 4 (forward_impl)."""
    cid, kw, (_, h, w), kernels = case
    h, w = odd(h), odd(w)
    n = -(-3 * 128 * sms() // (h * w))
    s = kw.get("scale", 2)
    if any(k in GATHERS for k in kernels):
        kernels = [k for k in kernels if k not in GATHERS] + [GATHERS[1] if (s * w) % 4 == 0 else GATHERS[0]]
    return cid, kw, (n, h, w), kernels


def batch_one_mismatches(eng, xd, x2d, y):
    """Images of the batch forward `y` (a device tensor) whose own batch-1 forward differs from it in any bit."""
    y1 = torch.empty_like(y)
    for i in range(xd.shape[0]):
        eng.forward(xd[i:i + 1], x2d[i:i + 1], y1[i:i + 1])
    return torch.nonzero((y1 != y).reshape(y.shape[0], -1).any(dim=1)).flatten().tolist()


def report(tag, worst, bad):
    print(tag, "error / bar:", " ".join("%s %.3f" % kv for kv in worst.items()))
    for name, ratio in worst.items():
        if not ratio <= 1.0:
            bad.append((tag, name, ratio))


def merge(worst, ratios):
    for name, ratio in ratios.items():
        worst[name] = max(worst.get(name, 0.0), ratio)


# ------------------------------------------------------------------ every tensor-core planner path, many items ----
@pytest.mark.parametrize("precision", [0, 1], ids=["f16x3", "f16x1"])
@pytest.mark.parametrize("case", TC_CASES, ids=[c[0] for c in TC_CASES])
def test_tensor_core_paths_many_items_per_cta(case, precision):
    cid, kw, (n, h, wd), kernels = work_case(case)
    assert_many_items(n, h, wd)
    assert h % 2 == 1 and wd % 2 == 1          # no patch side above 1 divides either side
    if cid in COLUMN_TILES:
        assert sms() % COLUMN_TILES[cid] != 0
    npl = 2 if precision == 0 else 1
    cfg = O.OracleConfig(**kw)
    w = O.he_init_weights(cfg, seed=0)
    s = cfg.scale
    g = np.random.RandomState(n * 1000 + h * 10 + wd)
    x = (g.rand(n, h, wd, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, s * h, s * wd, 1) * 255).astype(np.float32)
    xd, x2d = torch.from_numpy(x).cuda(), torch.from_numpy(x2).cuda()
    eng = make_engine(kw, w, precision)

    def forward():
        y = eng.forward(xd, x2d)
        torch.cuda.synchronize()
        return y
    _, names = launched_kernels(forward)
    assert_kernels_ran(names, [k.format(P=npl) for k in kernels])
    fused = any(k in GATHERS for k in kernels)
    folded = folded_filter(cfg, w) if fused and npl == 2 else None
    worst, bad = {}, []
    for seg in (0, 1):
        eng.set_option("seg_chunks", seg)
        for fuse in ((1, 0) if fused else (1,)):
            eng.set_option("fuse_last", fuse)
            y = forward().cpu().numpy()
            ratios = isolated_layers(eng, cfg, w, x, x2, y, npl, seg, fused and fuse == 1, device=dev())
            if folded is not None and fuse == 1:   # (reads one partial set of tap planes: the folded launch ran)
                ratios.update({"folded " + k: v for k, v in folded_launch_ratios(eng, cfg, folded, x2, y, seg,
                                                                                 device=dev()).items()})
            merge(worst, ratios)
            for name, ratio in ratios.items():
                if not ratio <= 1.0:
                    bad.append(("seg_chunks=%d fuse_last=%d" % (seg, fuse), name, ratio))
    eng.set_option("seg_chunks", 0)
    eng.set_option("fuse_last", 1)
    print("%s %dx%dx%d error / bar:" % (cid, n, h, wd), " ".join("%s %.3f" % kv for kv in worst.items()))
    mism = batch_one_mismatches(eng, xd, x2d, forward())
    eng.close()
    assert not bad, bad
    assert not mism, ("images differing from their batch-1 forward", mism[:20], len(mism))


# ------------------------------------------------------------------------ bench.py's headline, as bench runs it ----
def bench_inputs(batch, tile, scale):
    gen = torch.Generator().manual_seed(0)
    x = torch.rand(batch, tile, tile, 1, generator=gen) * 255
    x2 = torch.rand(batch, scale * tile, scale * tile, 1, generator=gen) * 255
    return x, x2


def packed_forward(cfg, w, folded, x, x2):
    """fp64 forward, NCHW on x's device, of the function the f16x3 headline evaluates: CNN1 on its fp32 weights, every
    tensor-core layer on its packed operand values (quantise: one power-of-two scale per packed layer, hi + lo), and the
    last upsampler folded with R-CNN1 (`folded` = folded_filter(cfg, w)), its tap planes gathered and x2 added.  Only
    the arithmetic of the kernels is left out, so y minus this is their rounding alone."""
    f = O.feature_filters(cfg)

    def layer(scope, a, wq):
        v = conv(a, wq) + col(w[scope + "/conv_B"], a.device)
        return prelu(v, w["%s/prelu/%s_prelu" % (scope, scope)])
    h = layer("CNN1", x, w["CNN1/conv_W"].astype(np.float64))
    feats = [h]
    for i in range(1, len(f)):
        sc = "CNN%d" % (i + 1)
        feats.append(layer(sc, feats[-1], quantise([w[sc + "/conv_W"]], 2)[0]))
    hc = torch.cat(feats, dim=1)
    del feats
    wa, wb = quantise([w["A1/conv_W"], w["B1/conv_W"]], 2)
    a1, b1 = layer("A1", hc, wa), layer("B1", hc, wb)
    del hc
    b2 = layer("B2", b1, quantise([w["B2/conv_W"]], 2)[0])
    wq, bf = folded
    v = conv(torch.cat([b2, a1], dim=1), wq) + col(bf, x.device)
    m, _, hh, ww = v.shape
    r = cfg.scale
    return gather9(v.reshape(m, r, r, 9, hh, ww).permute(3, 0, 4, 1, 5, 2).reshape(9, m, r * hh, r * ww)) + x2[:, 0]


def output_errors(cfg, w, xd, x2d, y, folded=None):
    """Statistics of y against the fp64 oracle over the batch, formed on the GPU CHUNK images at a time: max and RMS of
    |y - oracle|, each tile's max, and (with `folded`) max and RMS of y against packed_forward and of packed_forward
    against the oracle."""
    params = {k: torch.from_numpy(np.asarray(v, dtype=np.float64)).to(dev()) for k, v in w.items()}
    orc = O.Oracle(cfg, params, torch.float64)
    tile_max, sq, sq_k, sq_p, k_max, p_max = [], 0.0, 0.0, 0.0, 0.0, 0.0
    with torch.no_grad():
        for i0 in range(0, xd.shape[0], CHUNK):
            sl = slice(i0, i0 + CHUNK)
            xc, x2c = xd[sl].double().permute(0, 3, 1, 2), x2d[sl].double().permute(0, 3, 1, 2)
            ref = orc.forward_nchw(xc, x2c, params=params)
            yc = y[sl].double().permute(0, 3, 1, 2)
            e = yc - ref
            tile_max.append(e.abs().amax(dim=(1, 2, 3)))
            sq += float((e * e).sum())
            if folded is not None:
                pk = packed_forward(cfg, w, folded, xc, x2c)
                ek, ep = yc[:, 0] - pk, pk - ref[:, 0]
                sq_k, sq_p = sq_k + float((ek * ek).sum()), sq_p + float((ep * ep).sum())
                k_max, p_max = max(k_max, float(ek.abs().max())), max(p_max, float(ep.abs().max()))
    tile_max = torch.cat(tile_max).cpu().numpy()
    cnt = y.numel()
    out = {"max": float(tile_max.max()), "rms": (sq / cnt) ** 0.5, "tiles": tile_max}
    if folded is not None:
        out.update(kernel_max=k_max, kernel_rms=(sq_k / cnt) ** 0.5, packed_max=p_max, packed_rms=(sq_p / cnt) ** 0.5)
    return out


HEADLINE = [("f16x3-default", 0, 0), ("f16x3-strict", 0, 1), ("f16x1", 1, 0)]


@pytest.mark.parametrize("precision,seg", [c[1:] for c in HEADLINE], ids=[c[0] for c in HEADLINE])
def test_headline_batch(precision, seg):
    """bench.py headline(): the L12 x2 checkpoint on 256 uniform-noise 48 x 48 tiles (bench's generator), forwarded into
    one output buffer until the front of the forward has been replayed as a CUDA graph twice.  f16x3 folds R-CNN1 into
    the Up-PS launch (EPI_D2S_TAPS, checked by the folded-launch reference); f16x1 runs the unfolded EPI_D2S_RDOT
    epilogue, and its y is reported against fp64, not held to a bar (test_gpu_forward.test_fast_mode_is_psnr_neutral).

    y against the fp64 oracle over all 256 tiles, f16x3: the default promotion periods within 1.5e-3, as on the 4 tiles
    of test_gpu_forward.test_l12_stress_noise_tiles; seg_chunks = 1 within STRICT_HEADLINE; both at RMS within
    HEADLINE_RMS.  Plain 1e-3, which the strict setting meets on those 4 tiles, does not hold on all 256.  Measured on an
    H100 SXM (700 W), max / RMS of |y - fp64|: default 8.7e-4 / 9.6e-5 (no tile above 1e-3), strict 2.0e-3 / 1.2e-4
    (73 tiles above 1e-3).  packed_forward splits that error: the packed and folded weights give the same 1.3e-4 /
    2.1e-5 in both settings, and the kernels' rounding is 8.7e-4 / 9.4e-5 at the default periods, 2.0e-3 / 1.2e-4 at
    seg_chunks = 1.  Promoting every 16-channel K slice is less accurate here, not more: it adds into the rounded fp32 sum
    after every K slice, 9 * 13 = 117 promotions in a 196-channel 3 x 3 layer, where the default periods (2 weight tiles there) have
    9 * 4 / 2 = 18 segments of at most 8 truncating k16 steps.  tc_units counts exactly that (121 units of 2^-23 S
    against 29), and every layer stays inside it."""
    model = L12[2]
    w = load_golden_weights(model)
    cfg = O.OracleConfig(**MODEL_FLAGS[model])
    npl = 2 if precision == 0 else 1
    x, x2 = bench_inputs(256, 48, 2)
    n, h, wd = x.shape[:3]
    assert_many_items(n, h, wd)
    xd, x2d = x.cuda(), x2.cuda()
    y = torch.empty_like(x2d)
    eng = make_engine({}, w, precision)
    eng.set_option("seg_chunks", seg)
    eng.forward(xd, x2d, y)
    y_eager = y.cpu().numpy()
    r0 = eng.graph_replays
    replays = 0
    for _ in range(8):
        eng.forward(xd, x2d, y)
        torch.cuda.synchronize()
        assert np.array_equal(y.cpu().numpy(), y_eager), ("a replay differs from the eager forward", eng.graph_replays - r0)
        replays = eng.graph_replays - r0
        if replays >= 2:
            break
    assert replays >= 2, replays
    y_np = y.cpu().numpy()
    ratios = isolated_layers(eng, cfg, w, x.numpy(), x2.numpy(), y_np, npl, seg, True, device=dev(), chunk=CHUNK)
    if npl == 2:          # (folded_launch_ratios reads one partial set of tap planes: the folded launch ran)
        ratios.update({"folded " + k: v for k, v in folded_launch_ratios(eng, cfg, folded_filter(cfg, w), x2.numpy(),
                                                                         y_np, seg, device=dev(), chunk=CHUNK).items()})
    tag = "headline precision=%d seg_chunks=%d" % (precision, seg)
    bad = []
    report(tag, ratios, bad)
    st = output_errors(cfg, w, xd, x2d, y, folded_filter(cfg, w) if npl == 2 else None)
    tiles = np.sort(st["tiles"])[::-1]
    print("%s: |y - oracle(fp64)| over %d tiles: max %.3e, RMS %.3e; tile maxima %s ...; %d tiles above 1e-3"
          % (tag, n, st["max"], st["rms"], " ".join("%.2e" % t for t in tiles[:6]), int((tiles > 1e-3).sum())))
    if npl == 2:
        print("%s: y - packed_forward (kernel rounding) max %.3e RMS %.3e; packed_forward - oracle (weights) max %.3e "
              "RMS %.3e" % (tag, st["kernel_max"], st["kernel_rms"], st["packed_max"], st["packed_rms"]))
    mism = batch_one_mismatches(eng, xd, x2d, y)
    eng.close()
    assert not bad, bad
    if npl == 2:
        tol = TOL_DEFAULT_STRESS if seg == 0 else STRICT_HEADLINE
        assert st["max"] <= tol and st["rms"] <= HEADLINE_RMS, (st["max"], tol, st["rms"], HEADLINE_RMS)
    assert not mism, ("tiles differing from their batch-1 forward", mism[:20], len(mism))


# ------------------------------------------------------------------ the train step's forward at bench's shape ----
class SliceTensors:
    """Captured train-step tensors of one slice of images at a time, as fp64 NCHW on the GPU: each is fetched once per
    slice and only that slice is kept, so host memory stays at one whole tensor at a time."""

    def __init__(self, eng, n, h, wd):
        self.eng, self.shape = eng, (n, h, wd)
        self.sl, self.cache = None, {}

    def __call__(self, name, c, sl):
        if sl != self.sl:
            self.sl, self.cache = sl, {}
        if name not in self.cache:
            self.cache[name] = nchw(self.eng.get_train_tensor(name, self.shape + (c,))[sl], dev())
        return self.cache[name]


def test_train_forward_at_benchmark_train_shape():
    """bench.py's train record: L12 x4, 64 real 48 x 48 patches (y = ground truth), keep 0.8.  Every forward layer and
    y_, the zneg planes and the PReLU slope gradients against their isolated references (test_gpu_train_forward_paths),
    the references formed 16 patches at a time."""
    model = L12[4]
    kw = MODEL_FLAGS[model]
    cfg = O.OracleConfig(**kw)
    wts = load_golden_weights(model)
    keep = 0.8
    x, x2, y = real_patches(4, 64, 48, 48, 24)
    n, h, wd = x.shape[:3]
    assert_many_items(n, h, wd)
    eng, masks = captured_step(kw, wts, "prelu", keep, x, x2, y, FAST)
    planes = SliceTensors(eng, n, h, wd)
    sums, zneg = SlopeSums(), {}

    def pre(scope, z, bz, sl):
        r = zneg_ratio(planes("zneg:" + scope, z.shape[1], sl), z, bz)
        zneg["zneg " + scope] = max(zneg.get("zneg " + scope, 0.0), r)
        g = output_gradient(cfg, scope, lambda name, c: planes(name, c, sl))
        sums.add(scope, after_dropout(g, None if masks is None else nchw(masks[scope][sl], dev()), keep), z, bz)
    yp = eng.get_train_tensor("y_", (n, 4 * h, 4 * wd, 1))
    ratios = isolated_layers(eng, cfg, wts, x, x2, yp, 2, 0, False, masks=masks, keep=keep, pre=pre, device=dev(), chunk=16)
    ratios.update(zneg)
    slopes = sums.ratios(eng, n, h, wd, cfg.scale)
    eng.close()
    print("slope gradient error / sum |g z|:", " ".join("%s %.3g" % (k, v[1]) for k, v in slopes.items()))
    ratios.update({k: v[0] for k, v in slopes.items()})
    bad = []
    report("L12-x4 train 64x48x48", ratios, bad)
    assert not bad, bad


# ------------------------------------------------------------------ bench's depthwise-separable record ----
def test_depthwise_separable_benchmark_shape():
    """bench.py's ds record: the c-DCSCN DS L7 x4 checkpoint on 256 tiles of 48 x 48 (bench's generator seed 3):
    check_depthwise_separable_layers, then the forward repeated into one output buffer as bench times it, bit-identical
    to the first.  The depthwise-separable forward returns before the graph capture of forward_impl, so every repeat is
    eager: graph_replays must not move (should this path ever be captured, the replay check belongs here)."""
    model = "dcscn_L7_F32to8_G1.20_Sc4_NIN_A24_B8_PS_DS_R1F32"
    kw = MODEL_FLAGS[model]

    def repeated(eng, x, x2, y):
        xd, x2d = torch.from_numpy(x).cuda(), torch.from_numpy(x2).cuda()
        yb = torch.empty_like(x2d)
        r0 = eng.graph_replays
        for _ in range(3):
            eng.forward(xd, x2d, yb)
            torch.cuda.synchronize()
            assert np.array_equal(yb.cpu().numpy(), y)
        assert eng.graph_replays == r0, eng.graph_replays - r0
    check_depthwise_separable_layers(kw, load_golden_weights(model), 256, 48, 48, then=repeated, tag="c-DCSCN DS x4 256x48x48")
