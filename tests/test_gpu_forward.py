"""
GPU parity of the forward hot path (run with `-m gpu` on an H100): every call goes through the C-ABI
(helper/engine.py -> libdcscn_b200.so).

Tolerances (north_star: "1e-3 absolute (fp32)"):
  * realistic inputs (Set5 crops, committed golden vectors): max|gpu - fp64 oracle| <= 1e-3.
  * uniform-noise / He-init stress inputs push activations to ~2e3, where ANY fp32 implementation sits up to ~2e-3
    from the exact result (the fp32 CPU oracle itself does).  Two settings are held to two bars there:
      - strict promotion (option seg_chunks = 1: every 16-channel K slice is added to the fp32 sum with round-to-nearest):
        max(1e-3, 1.5 x the fp32 CPU oracle's own error) - on the 4 L12 noise tiles of test_l12_stress_noise_tiles
        plain 1e-3, which does not extend to bench.py's whole 256-tile batch (test_gpu_work_items.py: 2.0e-3 there);
      - the default promotion periods (what bench.py's headline runs): 1.5e-3, and on
        the L12 noise tiles also below 0.75 x the fp32 CPU oracle's error.
    The tensor core truncates its fp32 accumulate on every wgmma; the promotion period trades that error for epilogue
    work (DESIGN.md section 4).  Promoting every K slice is not more accurate in absolute terms: it adds one fp32
    round-to-nearest sum per 16 channels instead of per segment, and on the L12 noise tiles its output lies further from
    fp64 than the default periods' does.
"""
import glob
import os

import numpy as np
import pytest
import torch

import dcscn_oracle as O
from conftest import GOLDEN, MODEL_FLAGS, load_golden_weights

pytestmark = pytest.mark.gpu

TOL = 1e-3


def make_engine(kw, weights, precision=0):
    from helper import engine as E
    eng = E.Engine(E.make_config(precision=precision, **kw))
    eng.set_params(weights)
    return eng


def gpu_forward(eng, x, x2):
    y = eng.forward(torch.from_numpy(x).cuda(), torch.from_numpy(x2).cuda())
    torch.cuda.synchronize()
    return y.cpu().numpy()


TOL_DEFAULT_STRESS = 1.5e-3


def stress_bound(y32, y64):
    return max(TOL, 1.5 * float(np.abs(y32 - y64).max()))


def assert_stress(eng, x, x2, y64, y32):
    """Default promotion periods within 1.5e-3 (or the strict bound if that is larger), strict within the strict bound."""
    y = gpu_forward(eng, x, x2)
    assert np.isfinite(y).all()
    err = float(np.abs(y - y64).max())
    assert err <= max(TOL_DEFAULT_STRESS, stress_bound(y32, y64)), ("default", err)
    eng.set_option("seg_chunks", 1)
    ys = gpu_forward(eng, x, x2)
    eng.set_option("seg_chunks", 0)
    err_s = float(np.abs(ys - y64).max())
    assert err_s <= stress_bound(y32, y64), ("strict", err_s, err)
    return y


SMALL = dict(scale=2, layers=4, filters=40, min_filters=24, filters_decay_gamma=1.5, nin_filters=24, nin_filters2=16)


@pytest.fixture(scope="module")
def small():
    cfg = O.OracleConfig(**SMALL)
    w = O.he_init_weights(cfg, seed=0)
    eng = make_engine(SMALL, w)
    yield cfg, w, eng
    eng.close()


@pytest.mark.parametrize("n,h,w", [(1, 20, 37), (2, 48, 48), (1, 1, 1), (1, 3, 130), (3, 17, 9), (1, 129, 2)])
def test_small_graph_every_layer(small, n, h, w):
    cfg, wts, eng = small
    g = np.random.RandomState(n * 1000 + h * 10 + w)
    x = (g.rand(n, h, w, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, 2 * h, 2 * w, 1) * 255).astype(np.float32)
    y64, inter = O.Oracle(cfg, wts, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64),
                                                           return_intermediates=True)
    y32 = O.Oracle(cfg, wts, torch.float32).forward(x, x2)
    assert_stress(eng, x, x2, y64, y32)
    gpu_forward(eng, x, x2)                      # default setting again: the activations checked below are its own
    for name, ref in inter.items():
        if name == "R-CNN":
            continue
        a = eng.get_activation(name, ref.shape)
        # fp32-level agreement relative to the layer's dynamic range
        assert np.abs(a - ref).max() <= 4e-6 * max(1.0, np.abs(ref).max()) + 1e-4, name


def test_validation_kernels_agree_with_tensor_core_path(small):
    """conv_impl=1 runs the same layers as plain fp32 FMAs on CUDA cores - an independent on-GPU cross-check."""
    cfg, wts, eng = small
    g = np.random.RandomState(7)
    x = (g.rand(2, 33, 21, 1) * 255).astype(np.float32)
    x2 = (g.rand(2, 66, 42, 1) * 255).astype(np.float32)
    y_tc = gpu_forward(eng, x, x2)
    eng.set_option("conv_impl", 1)
    y_ref = gpu_forward(eng, x, x2)
    eng.set_option("conv_impl", 0)
    assert np.abs(y_tc - y_ref).max() <= 2e-3
    y64 = O.Oracle(cfg, wts, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64))
    err_ref = float(np.abs(y_ref - y64).max())
    assert np.abs(y_tc - y64).max() <= max(TOL_DEFAULT_STRESS, 1.5 * err_ref)
    eng.set_option("seg_chunks", 1)
    y_strict = gpu_forward(eng, x, x2)
    eng.set_option("seg_chunks", 0)
    assert np.abs(y_strict - y64).max() <= 1.5 * max(err_ref, 5e-4), (float(np.abs(y_strict - y64).max()), err_ref)


def test_forward_host_matches_device_call_and_plan_cache(small):
    cfg, wts, eng = small
    g = np.random.RandomState(9)
    shapes = [(1, 16, 16), (2, 10, 30), (1, 16, 16), (1, 30, 10)]
    for n, h, w in shapes:
        x = (g.rand(n, h, w, 1) * 255).astype(np.float32)
        x2 = (g.rand(n, 2 * h, 2 * w, 1) * 255).astype(np.float32)
        a = gpu_forward(eng, x, x2)
        b = eng.forward_host(x, x2)
        np.testing.assert_array_equal(a, b)  # same kernels, same order: bit-identical


def golden_cases():
    d = np.load(os.path.join(GOLDEN, "forward_golden.npz"))
    n = len([k for k in d.files if k.endswith("_model")])
    return d, n


@pytest.mark.parametrize("ci", range(12))
def test_golden_vectors(ci):
    """Committed fp64-oracle outputs for Set5 crops through the reference's own checkpoints."""
    d, n = golden_cases()
    assert ci < n
    model = str(d["case%d_model" % ci])
    x, x2, y64 = d["case%d_x" % ci], d["case%d_x2" % ci], d["case%d_y64" % ci]
    eng = make_engine(MODEL_FLAGS[model], load_golden_weights(model))
    y = gpu_forward(eng, np.ascontiguousarray(x), np.ascontiguousarray(x2))
    eng.close()
    err = float(np.abs(y - y64).max())
    assert err <= TOL, (model, err)


DS2 = dict(scale=2, layers=3, filters=12, min_filters=6, filters_decay_gamma=1.5, nin_filters=10, nin_filters2=6,
           pixel_shuffler_filters=1, depthwise_separable=True)


def check_depthwise_separable_layers(kw, w, n, h, wd, then=None, tag=None):
    """Output within 1e-3 of the fp64 oracle, and every layer's activation at fp32 level.  `then(eng, x, x2, y)`, if
    given, runs on the engine before it is closed; with `tag` every check's error / bar is printed under it."""
    cfg = O.OracleConfig(**kw)
    s = kw["scale"]
    g = torch.Generator().manual_seed(3)
    x = (torch.rand(n, h, wd, 1, generator=g) * 255).numpy()
    x2 = (torch.rand(n, s * h, s * wd, 1, generator=g) * 255).numpy()
    y64, inter = O.Oracle(cfg, w, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64),
                                                         return_intermediates=True)
    eng = make_engine(kw, w)
    y = gpu_forward(eng, x, x2)
    ratios = {"y": float(np.abs(y - y64).max()) / TOL}
    assert np.abs(y - y64).max() <= TOL
    for name, ref in inter.items():
        if name == "R-CNN":
            continue
        a = eng.get_activation(name, ref.shape)
        bar = 2e-6 * max(1.0, np.abs(ref).max()) + 1e-4
        ratios[name] = float(np.abs(a - ref).max()) / bar
        assert np.abs(a - ref).max() <= bar, name
    if tag is not None:
        print(tag, "error / bar:", " ".join("%s %.3f" % kv for kv in ratios.items()))
    if then is not None:
        then(eng, x, x2, y)
    eng.close()


def test_depthwise_separable_every_layer():
    """BASELINE configs[4]: the DS c-DCSCN x4 checkpoint (fused depthwise+pointwise CUDA-core kernels)."""
    model = "dcscn_L7_F32to8_G1.20_Sc4_NIN_A24_B8_PS_DS_R1F32"
    check_depthwise_separable_layers(MODEL_FLAGS[model], load_golden_weights(model), 3, 48, 48)


def test_depthwise_separable_odd_hr_width():
    """A He-init x2 depthwise-separable graph on 3 x 17 x 23 tiles: the HR width of 46 is not a multiple of 4, so R-CNN1
    runs on the one-pixel-per-thread kernel instead of the four-pixel one.  The fp32 oracle is 8e-5 from the fp64 one
    on this input, so the 1e-3 bar applies as it does to the checkpoint."""
    check_depthwise_separable_layers(DS2, O.he_init_weights(O.OracleConfig(**DS2), seed=4), 3, 17, 23)


@pytest.mark.parametrize("model", ["dcscn_L12_F196to48_NIN_A64_PS_R1F32", "dcscn_L12_F196to48_Sc4_NIN_A64_PS_R1F32"],
                         ids=["L12x2", "L12x4"])
def test_unfused_last_layer_every_layer(model):
    """Option fuse_last = 0 on the full-width checkpoints: R-CNN1 runs as its own kernel on the materialised Up-PS
    (x2) / Up-PS2 (x4) output, which the fused path never writes.  On a Set5 crop every layer, the pixel-shuffler
    outputs included, matches the fp64 oracle at the fp32-level bar of test_small_graph_every_layer, and the fused and
    unfused outputs are both within 1e-3 of fp64."""
    kw = MODEL_FLAGS[model]
    s = kw.get("scale", 2)
    w = load_golden_weights(model)
    f = sorted(glob.glob(os.path.join(GOLDEN, "data", "set5", "*.png")))[1]
    lr, bic, _ = O.build_inputs_for_evaluate(f, s)
    r0, c0, h, wd = 8, 12, 36, 44
    x = np.ascontiguousarray(lr[r0:r0 + h, c0:c0 + wd].reshape(1, h, wd, 1)).astype(np.float32)
    x2 = np.ascontiguousarray(bic[s * r0:s * (r0 + h), s * c0:s * (c0 + wd)].reshape(1, s * h, s * wd, 1)).astype(np.float32)
    y64, inter = O.Oracle(O.OracleConfig(**kw), w, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64),
                                                                         return_intermediates=True)
    eng = make_engine(kw, w)
    y_fused = gpu_forward(eng, x, x2)
    eng.set_option("fuse_last", 0)
    y = gpu_forward(eng, x, x2)
    assert np.abs(y_fused - y64).max() <= TOL
    assert np.abs(y - y64).max() <= TOL
    bad = []
    for name, ref in inter.items():
        if name == "R-CNN":
            continue
        err = float(np.abs(eng.get_activation(name, ref.shape) - ref).max())
        if not err <= 4e-6 * max(1.0, np.abs(ref).max()) + 1e-4:
            bad.append((name, err, float(np.abs(ref).max())))
    eng.close()
    assert not bad, bad


def test_l12_stress_noise_tiles():
    """BASELINE configs[1] shape: uniform-noise 48x48 tiles through the L12 x2 checkpoint."""
    model = "dcscn_L12_F196to48_NIN_A64_PS_R1F32"
    w = load_golden_weights(model)
    cfg = O.OracleConfig()
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(4, 48, 48, 1, generator=g) * 255).numpy()
    x2 = (torch.rand(4, 96, 96, 1, generator=g) * 255).numpy()
    y64 = O.Oracle(cfg, w, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64))
    y32 = O.Oracle(cfg, w, torch.float32).forward(x, x2)
    err32 = float(np.abs(y32 - y64).max())
    eng = make_engine({}, w)
    y = gpu_forward(eng, x, x2)
    err = float(np.abs(y - y64).max())
    # Default promotion periods (the benchmarked setting): uniform noise drives the activations ~10x beyond natural
    # images, where the fp32 CPU forward itself is ~2.4e-3 from the exact result; the tensor-core path has to stay
    # clearly inside that - two fp32 evaluations cannot agree better than their own rounding noise.
    assert err <= max(TOL, 0.75 * err32), (err, err32)
    # On these 4 tiles the strict setting (every 16-channel K slice promoted to the fp32 RN sum, seg_chunks = 1; bench.py's
    # "strict" record carries its throughput) also meets 1e-3 against the exact (fp64) forward.  That does not hold for
    # the whole 256-tile batch: there the worst tile is 2.0e-3 away (test_gpu_work_items.test_headline_batch).
    eng.set_option("seg_chunks", 1)
    y_strict = gpu_forward(eng, x, x2)
    eng.close()
    err_strict = float(np.abs(y_strict - y64).max())
    assert err_strict <= TOL, err_strict


def test_full_batch_properties():
    """BASELINE.json full size (256 tiles): size-independent properties instead of an oracle run -
    batch invariance (every tile equals its batch-of-1 result bit for bit) and x2 additivity (y - x2 is
    independent of x2, the final tf.add of DCSCN.py:325)."""
    model = "dcscn_L12_F196to48_NIN_A64_PS_R1F32"
    eng = make_engine({}, load_golden_weights(model))
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(256, 48, 48, 1, generator=g) * 255).cuda()
    x2 = (torch.rand(256, 96, 96, 1, generator=g) * 255).cuda()
    y = eng.forward(x, x2).clone()
    for i in (0, 77, 255):
        yi = eng.forward(x[i:i + 1].contiguous(), x2[i:i + 1].contiguous())
        assert torch.equal(yi[0], y[i])
    y0 = eng.forward(x, torch.zeros_like(x2)).clone()
    # y = conv + x2 with one fp32 rounding; y0 = conv + 0 exactly
    assert (y - (y0 + x2)).abs().max().item() == 0.0
    assert torch.isfinite(y).all()
    eng.close()


def test_fast_mode_is_psnr_neutral():
    """f16x1 (single-pass fp16 operands): not 1e-3-exact, but within the 0.01 dB PSNR gate."""
    model = "dcscn_L12_F196to48_NIN_A64_PS_R1F32"
    w = load_golden_weights(model)
    f = sorted(glob.glob(os.path.join(GOLDEN, "data", "set5", "*.png")))[2]
    lr, bic, true_y = O.build_inputs_for_evaluate(f, 2)
    x = lr.reshape(1, *lr.shape).astype(np.float32)
    x2 = bic.reshape(1, *bic.shape).astype(np.float32)
    e3 = make_engine({}, w, precision=0)
    e1 = make_engine({}, w, precision=1)
    y3, y1 = gpu_forward(e3, x, x2), gpu_forward(e1, x, x2)
    e3.close()
    e1.close()
    p3, p1 = O.compute_psnr(true_y, y3[0], 2), O.compute_psnr(true_y, y1[0], 2)
    assert abs(p3 - p1) < 0.01
    assert np.abs(y3 - y1).max() < 1.0


def test_errors_are_loud():
    from helper import engine as E
    with pytest.raises(E.EngineError):
        E.Engine(E.make_config(use_nin=False))
    eng = E.Engine(E.make_config(**SMALL))
    with pytest.raises(E.EngineError):
        eng.set_param("no/such_var", np.zeros(3, np.float32))
    with pytest.raises(E.EngineError):
        eng.set_param("CNN1/conv_B", np.zeros(3, np.float32))  # wrong size
    with pytest.raises(E.EngineError):
        eng.set_option("conv_impl", 7)
    # keys of removed kernel variants are unknown options, not silently ignored
    for key, value in [("cluster", 2), ("kc", 32), ("ds_impl", 1), ("ds_cache", 0), ("gather_impl", 1),
                       ("wgrad_taps", 1), ("host_repack", 1)]:
        with pytest.raises(E.EngineError):
            eng.set_option(key, value)
    eng.close()


def test_cuda_graph_replay_is_bit_identical_and_follows_weight_updates(small):
    """Option "graph": the launches in front of the last kernel are replayed as one CUDA graph once the same input
    pointer came twice in a row.  Replays must equal the eager launches bit for bit, and a graph must never outlive
    what it baked in (weights re-packed with another power-of-two scale, options)."""
    cfg, wts, eng = small
    g = np.random.RandomState(11)
    x = torch.from_numpy((g.rand(2, 40, 56, 1) * 255).astype(np.float32)).cuda()
    x2 = torch.from_numpy((g.rand(2, 80, 112, 1) * 255).astype(np.float32)).cuda()
    eng.set_option("graph", 0)
    la = eng.launch_count
    y_eager = eng.forward(x, x2).cpu().numpy()
    per_forward = eng.launch_count - la
    eng.set_option("graph", 1)
    r0, l0 = eng.graph_replays, eng.launch_count
    ys = [eng.forward(x, x2).cpu().numpy() for _ in range(4)]       # eager, capture + replay, replay, replay
    assert eng.graph_replays - r0 >= 2
    assert eng.launch_count - l0 == 4 * per_forward                 # kernels launched are counted the same, graph or not
    for y in ys:
        assert np.array_equal(y, y_eager)
    # another x2 / y with the same x: the graph stays valid (it does not touch them)
    x2b = x2 * 0.5
    yb = eng.forward(x, x2b).cpu().numpy()
    np.testing.assert_allclose(yb - 0.5 * x2.cpu().numpy(), y_eager - x2.cpu().numpy(), atol=1e-4)
    # new weights (x 3: another power-of-two weight scale in every layer) through the same plan
    w3 = {k: (v * 3.0 if k.endswith("conv_W") else v) for k, v in wts.items()}
    eng.set_params(w3)
    y3 = [eng.forward(x, x2).cpu().numpy() for _ in range(3)]
    eng.set_option("graph", 0)
    y3_eager = eng.forward(x, x2).cpu().numpy()
    eng.set_option("graph", 1)
    for y in y3:
        assert np.array_equal(y, y3_eager)
    assert not np.array_equal(y3_eager, y_eager)
    eng.set_params(wts)
