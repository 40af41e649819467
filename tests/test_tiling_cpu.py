"""Tiled inference (option "workspace_mb"), the parts that need no GPU: the halo formula pinned by the fp64 oracle, and
the --workspace_mb flag's way into the engine.  CPU only."""
import numpy as np
import pytest
import torch

import dcscn_oracle as O
from conftest import MODEL_FLAGS
from helper import args as A

L7 = MODEL_FLAGS["dcscn_L7_F32to8_G1.20_NIN_A24_B8_PS_R1F32"]
CNN5 = dict(scale=2, layers=4, filters=40, min_filters=24, filters_decay_gamma=1.5, nin_filters=24, nin_filters2=16,
            cnn_size=5)
HALO_GRAPHS = {
    "L7x2": L7,
    "L7x3": dict(L7, scale=3),
    "L7x4": dict(L7, scale=4),
    "cnn5": CNN5,
    "DSx4": MODEL_FLAGS["dcscn_L7_F32to8_G1.20_Sc4_NIN_A24_B8_PS_DS_R1F32"],
}


def _ceil_div(a, b):
    return -(-a // b)


def tile_halo(cfg):
    """LR pixels of context a window core needs: the dependency path CNN1 .. CNNL -> B1 (1x1) -> B2 -> Up-PS
    [-> Up-PS2 at 2x] -> R-CNN1 at HR resolution, walked back from an LR core edge (the engine's dcscn_tile_halo)."""
    k = {scope: kk for scope, kk, *_ in O.layer_table(cfg)}
    half = lambda kk: (kk - 1) // 2
    r = sum(half(k["CNN%d" % (i + 1)]) for i in range(cfg.layers))
    r += half(k["B1"]) + half(k["B2"]) + half(k["Up-PS/Up-PS_CNN"])
    hr = half(k["R-CNN1"])
    if cfg.scale == 4:
        r += _ceil_div(half(k["Up-PS2/Up-PS2_CNN"]) + _ceil_div(hr, 2), 2)
    else:
        r += _ceil_div(hr, cfg.scale)
    return r


def test_halo_of_the_shipped_graphs():
    for kw in (dict(), dict(scale=3), dict(scale=4)):
        assert tile_halo(O.OracleConfig(**kw)) == 15
    for name in ("dcscn_L7_F32to8_G1.20_NIN_A24_B8_PS_R1F32", "dcscn_L7_F32to8_G1.20_Sc4_NIN_A24_B8_PS_DS_R1F32"):
        assert tile_halo(O.OracleConfig(**MODEL_FLAGS[name])) == 10


def _core_error(oracle, x, x2, s, a, c, r):
    """max |whole-image output - windowed output| over the c x c core at (a, a), window = core + r pixels each side."""
    y = oracle.forward(x, x2)
    w0, w1 = a - r, a + c + r
    yw = oracle.forward(np.ascontiguousarray(x[:, w0:w1, w0:w1]), np.ascontiguousarray(x2[:, s * w0:s * w1, s * w0:s * w1]))
    core = y[:, s * a:s * (a + c), s * a:s * (a + c)]
    core_w = yw[:, s * r:s * (r + c), s * r:s * (r + c)]
    return float(np.abs(core - core_w).max())


@pytest.mark.parametrize("graph", sorted(HALO_GRAPHS))
def test_halo_is_exact_and_tight(graph):
    """A window with the formula's halo around an interior core reproduces the whole-image fp64 output on that core;
    one pixel less changes some core pixel, so the halo is the smallest that works."""
    cfg = O.OracleConfig(**HALO_GRAPHS[graph])
    s = cfg.scale
    r = tile_halo(cfg)
    c = 5
    a = r + 4                                   # the window stays clear of the image edge on every side
    size = 2 * a + c
    g = np.random.RandomState(r * 10 + s)
    x = g.rand(1, size, size, 1) * 255
    x2 = g.rand(1, s * size, s * size, 1) * 255
    oracle = O.Oracle(cfg, O.he_init_weights(cfg, seed=5), torch.float64)
    assert _core_error(oracle, x, x2, s, a, c, r) <= 1e-9
    assert _core_error(oracle, x, x2, s, a, c, r - 1) > 1e-6


def _fresh_flags(argv):
    f = A._Flags()
    for name, (kind, default, help_text) in A.FLAGS._defs.items():
        f._define(name, default, help_text, kind)
    f.parse(["prog"] + argv)
    return f


def test_workspace_flag_parses_and_defaults_to_zero():
    assert _fresh_flags([]).workspace_mb == 0
    assert _fresh_flags(["--workspace_mb=8192"]).workspace_mb == 8192
    assert _fresh_flags(["--workspace_mb", "512"]).workspace_mb == 512


@pytest.mark.parametrize("value,expect", [(0, []), (8192, [("workspace_mb", 8192)])])
def test_build_graph_sets_the_option_only_when_positive(monkeypatch, value, expect):
    import DCSCN
    calls = []

    class FakeEngine:
        def __init__(self, config):
            pass

        def set_option(self, key, v):
            calls.append((key, v))

        def param_shapes(self):
            return {}

    monkeypatch.setattr(DCSCN.eng, "Engine", FakeEngine)
    m = object.__new__(DCSCN.SuperResolution)
    m.workspace_mb = value
    m.layers, m.cnn_size = 12, 3
    m._engine_config = lambda: None
    m.build_graph()
    assert calls == expect
