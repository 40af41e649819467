"""Scale factors above x4 (--scale=5 to 8), the parts that need no GPU: the tiled-inference halo at x5..x8 with the
pixel shuffler and with Up-TCNN, exact and one pixel tight against the fp64 oracle; the Up-TCNN filter gather at K = 9,
12, 13 and 16; the evaluation size rule at x5..x7; the Pillow tables at 1/5..1/8 and back; and the Python layer (model
name, engine config, complexity bookkeeping).  CPU only."""
import numpy as np
import pytest
import torch

import dcscn_oracle as O
import tconv_oracle as T
from conftest import MODEL_FLAGS
from test_tconv_cpu import tile_halo as tconv_tile_halo
from test_tiling_cpu import _core_error, tile_halo

SCALES = (5, 6, 7, 8)
CDCSCN = MODEL_FLAGS["dcscn_L7_F32to8_G1.20_NIN_A24_B8_PS_R1F32"]
DS = MODEL_FLAGS["dcscn_L7_F32to8_G1.20_Sc4_NIN_A24_B8_PS_DS_R1F32"]
SMALL = dict(layers=3, filters=12, min_filters=6, nin_filters=6, nin_filters2=4)


def _window_check(oracle, s, r):
    """The halo reproduces the whole-image fp64 output on an interior core; one pixel less does not."""
    c = 5
    a = r + 4
    size = 2 * a + c
    g = np.random.RandomState(r * 10 + s)
    x = g.rand(1, size, size, 1) * 255
    x2 = g.rand(1, s * size, s * size, 1) * 255
    assert _core_error(oracle, x, x2, s, a, c, r) <= 1e-9
    assert _core_error(oracle, x, x2, s, a, c, r - 1) > 1e-6


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("graph", ["cdcscn", "ds", "cnn5"])
def test_pixel_shuffler_halo_is_exact_and_tight(graph, s):
    """One Up-PS stage of s*s*ps_out columns: the LR stack's reach, Up-PS's own, and ceil(h(k_R) / s) for R-CNN1."""
    kw = {"cdcscn": CDCSCN, "ds": DS, "cnn5": dict(SMALL, cnn_size=5)}[graph]
    cfg = O.OracleConfig(**dict(kw, scale=s))
    r = tile_halo(cfg)
    assert r == {"cdcscn": 10, "ds": 10, "cnn5": 6 + 1 + 2 + 1}[graph]
    _window_check(O.Oracle(cfg, O.he_init_weights(cfg, seed=5), torch.float64), s, r)


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("cnn", [3, 5])
def test_tconv_halo_is_exact_and_tight(s, cnn):
    """Up-TCNN (K = 2s - s%2) and R-CNN1 walked back together reach one LR pixel at every s >= 3."""
    cfg = T.Config(scale=s, **dict(SMALL, cnn_size=cnn))
    r = tconv_tile_halo(cfg)
    assert r == {3: 3 + 1 + 1, 5: 6 + 1 + 1}[cnn]
    _window_check(T.Oracle(cfg, T.random_weights(cfg, seed=5)), s, r)


@pytest.mark.parametrize("s", SCALES)
def test_tconv_filter_size_and_padding(s):
    assert T.ksize(s) == {5: 9, 6: 12, 7: 13, 8: 16}[s]
    assert T.pad_top(s) == {5: 2, 6: 3, 7: 3, 8: 4}[s]
    assert (T.ksize(s) - s) % 2 == 0            # symmetric SAME padding: torch's conv_transpose2d gives s*H exactly


@pytest.mark.parametrize("s", SCALES)
def test_tconv_filter_map_is_a_bijection(s):
    """Every Tconv_W entry appears in the 3x3 LR filter F exactly once, every other entry of F is a structural zero,
    and the inverse gather recovers W bit for bit."""
    c = 3
    k = T.ksize(s)
    idx = T.tconv_filter_index(s, c)
    used = idx[idx >= 0]
    assert np.array_equal(np.sort(used), np.arange(k * k * c * c))
    wt = np.random.RandomState(7 + s).randn(k, k, c, c).astype(np.float32)
    f = T.tconv_filter(wt, s)
    assert f.shape == (3, 3, c, s * s * c)
    assert np.count_nonzero(f[idx < 0]) == 0
    assert np.array_equal(T.tconv_filter_grad(f, s, c), wt)


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("n,c,h,w", [(2, 3, 4, 5), (1, 4, 1, 1), (1, 2, 1, 6)])
def test_gather_conv_equals_scatter_loop_and_conv_transpose(s, n, c, h, w):
    g = np.random.RandomState(s * 10 + h)
    x = g.randn(n, c, h, w)
    wt = g.randn(T.ksize(s), T.ksize(s), c, c)
    ref = T.scatter_reference(x, wt, s)
    got = T.gather_conv(x, wt, s).numpy()
    tor = T.conv_transpose(torch.from_numpy(x), wt, s).numpy()
    assert got.shape == ref.shape == (n, c, s * h, s * w)
    assert np.abs(got - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())
    assert np.abs(tor - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("scale", [5, 6, 7])
def test_eval_size_rule_equals_the_host_resizes(scale):
    from helper import engine as E, utilty as util
    for side in range(scale, 4097, scale):
        (ah, aw), (lh, lw), (bh, bw), _ = E.eval_geometry(side, side + scale - 1, scale, 0)
        assert (ah, aw) == (side, side) and (lh, lw) == (side // scale, side // scale) and (bh, bw) == (side, side)
    for side in range(scale, 700, 7 * scale):
        a = np.zeros((side, side + scale, 1), np.float32)
        lr = util.resize_image_by_pil(a, 1.0 / scale)
        bic = util.resize_image_by_pil(lr, scale)
        _, (lh, lw), (bh, bw), _ = E.eval_geometry(side, side + scale, scale, 0)
        assert lr.shape[:2] == (lh, lw) and bic.shape[:2] == (bh, bw)


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("h,w", [(120, 96), (37 * 8, 53 * 8), (16, 8)])
def test_pillow_tables_down_and_back(s, h, w):
    """The resamplers the device evaluation and crop paths use, against Pillow at 1/s (an antialiased window of up to
    4s + 1 taps) and at s: mode 'F' (the Y of RGB images) and mode 'L' (grayscale files)."""
    from PIL import Image
    from helper import pil_resample as R
    h, w = h // s * s, w // s * s
    rs = np.random.RandomState(s * 1000 + h)
    f = (rs.rand(h, w) * 255).astype(np.float32)
    u = (rs.rand(h, w) * 256).astype(np.uint8)
    u[: max(1, h // 8)] = 255                     # saturated rows and columns overshoot past 0 and 255
    u[:, ::5] = 0
    kk, _ = R.precompute_coeffs(w, w // s)
    assert kk.shape[1] == 4 * s + 1
    for a, resize in ((f, R.resize_float), (u, R.resize_uint8)):
        small = np.asarray(Image.fromarray(a).resize([w // s, h // s], Image.BICUBIC))
        np.testing.assert_array_equal(resize(a, w // s, h // s), small)
        big = np.asarray(Image.fromarray(small).resize([w, h], Image.BICUBIC))
        np.testing.assert_array_equal(resize(small, w, h), big)


# ------------------------------------------------------------------ the Python layer ----

def _flags(tmp_path, argv):
    from helper import args as A
    f = A._Flags()
    for name, (kind, default, help_text) in A.FLAGS._defs.items():
        f._define(name, default, help_text, kind)
    f.parse(["prog"] + argv + ["--checkpoint_dir=" + str(tmp_path / "ckpt"), "--log_filename=" + str(tmp_path / "log.txt"),
                               "--tf_log_dir=" + str(tmp_path / "tf_log"), "--graph_dir=" + str(tmp_path / "graphs"),
                               "--output_dir=" + str(tmp_path / "out")])
    return f


@pytest.mark.parametrize("argv,name", [(["--scale=8"], "dcscn_L12_F196to48_Sc8_NIN_A64_PS_R1F32"),
                                       (["--scale=5", "--pixel_shuffler=false"], "dcscn_L12_F196to48_Sc5_NIN_A64_R1F32")])
def test_model_name_and_engine_config(tmp_path, argv, name):
    import DCSCN
    f = _flags(tmp_path, argv)
    m = DCSCN.SuperResolution(f, model_name=f.model_name)
    assert m.name == name
    cfg = m._engine_config()
    assert cfg.scale == f.scale and cfg.transposed_upsampler == (not f.pixel_shuffler)
    assert m.psnr_calc_border_size == f.scale


def _reference_bookkeeping(cfg, tconv):
    """tf_graph.py's complexity and receptive-field counts for one --scale: conv (k k cin cout), bias (cout) and activator
    (cout) terms at pix_per_input pixels, which only build_transposed_conv changes (to s*s, DCSCN.py:293-311)."""
    table = T.layer_table(cfg) if tconv else O.layer_table(cfg)
    s, pix, cx, rf = cfg.scale, 1, 0, 0
    for scope, k, cin, cout, bias, act in table:
        if scope == "Up-TCNN":
            pix *= s * s
            cx += pix * k * k * cin * cout
            rf += 1
            continue
        cx += pix * (k * k * cin * cout + (cout if bias else 0) + (cout if act else 0))
        rf = k if rf == 0 else rf + k - 1
        if scope == "A1":
            rf -= cfg.cnn_size - 1
    return cx, rf


@pytest.mark.parametrize("tconv", [False, True], ids=["PS", "TCNN"])
def test_complexity_matches_the_reference_at_x8(monkeypatch, tconv):
    import DCSCN
    cfg = (T.Config if tconv else O.OracleConfig)(scale=8)
    table = T.layer_table(cfg) if tconv else O.layer_table(cfg)
    shapes = {}
    for scope, k, cin, cout, bias, act in table:
        if scope == "Up-TCNN":
            shapes[T.TCONV] = (k, k, cin, cout)
            continue
        shapes[scope + "/conv_W"] = (k, k, cin, cout)
        if bias:
            shapes[scope + "/conv_B"] = (cout,)
        if act:
            shapes["%s/prelu/%s_prelu" % (scope, scope)] = (cout,)

    class FakeEngine:
        def __init__(self, config):
            pass

        def param_shapes(self):
            return shapes

    monkeypatch.setattr(DCSCN.eng, "Engine", FakeEngine)
    m = object.__new__(DCSCN.SuperResolution)
    m.workspace_mb, m.layers, m.cnn_size, m.scale = 0, 12, 3, 8
    m._engine_config = lambda: None
    m.build_graph()
    assert (m.complexity, m.receptive_fields) == _reference_bookkeeping(cfg, tconv)
