"""--pixel_shuffler=false (the Up-TCNN transposed-convolution upsampler), the parts that need no GPU: the identity the
engine computes the layer with (a 3x3 LR convolution with a gathered filter F, then depth_to_space(s)), pinned against
a literal scatter loop of TF's definition and against torch's conv_transpose2d; the exact inverse gather behind the
filter gradient; the tiled-inference halo; and the Python layer (model name, bilinear initial value, flag checks).
CPU only."""
import numpy as np
import pytest
import torch

import dcscn_oracle as O
import tconv_oracle as T
from test_tiling_cpu import _ceil_div, _core_error

SCALES = (2, 3, 4)


def _rand(shape, seed):
    return np.random.RandomState(seed).randn(*shape)


@pytest.mark.parametrize("s", SCALES)
def test_filter_size_and_padding(s):
    assert T.ksize(s) == {2: 4, 3: 5, 4: 8}[s]
    assert T.pad_top(s) == {2: 1, 3: 1, 4: 2}[s]
    assert (T.ksize(s) - s) % 2 == 0            # symmetric SAME padding: torch's conv_transpose2d gives s*H exactly


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("n,c,h,w", [(2, 3, 5, 7), (1, 4, 1, 1), (1, 2, 1, 6), (1, 5, 9, 3)])
def test_gather_conv_equals_scatter_loop(s, n, c, h, w):
    """F-gather 3x3 conv + depth_to_space == TF's scatter definition == torch conv_transpose2d, in fp64."""
    x = _rand((n, c, h, w), 1 + s)
    wt = _rand((T.ksize(s), T.ksize(s), c, c), 2 + s)
    ref = T.scatter_reference(x, wt, s)
    got = T.gather_conv(x, wt, s).numpy()
    tor = T.conv_transpose(torch.from_numpy(x), wt, s).numpy()
    assert got.shape == ref.shape == (n, c, s * h, s * w)
    assert np.abs(got - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())
    assert np.abs(tor - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("s", SCALES)
def test_every_tap_is_used_once(s):
    """(phase, offset) -> tap is a bijection: F holds exactly K^2 C^2 entries of W, each once; the rest are zeros."""
    c = 3
    k = T.ksize(s)
    idx = T.tconv_filter_index(s, c)
    used = idx[idx >= 0]
    assert used.size == k * k * c * c
    assert np.array_equal(np.sort(used), np.arange(k * k * c * c))
    wt = _rand((k, k, c, c), 7).astype(np.float32)
    f = T.tconv_filter(wt, s)
    assert f.shape == (3, 3, c, s * s * c)
    assert np.count_nonzero(f[idx < 0]) == 0
    assert np.array_equal(np.sort(f[idx >= 0]), np.sort(wt.ravel()))
    # the inverse gather recovers W bit for bit
    assert np.array_equal(T.tconv_filter_grad(f, s, c), wt)


@pytest.mark.parametrize("s", SCALES)
def test_filter_gradient_is_the_inverse_gather(s):
    """dL/dW through the transposed convolution == the F gradient of the gathered form, gathered back."""
    c = 2
    k = T.ksize(s)
    x = torch.from_numpy(_rand((1, c, 4, 5), 11))
    g = torch.from_numpy(_rand((1, c, 4 * s, 5 * s), 12))
    w = torch.from_numpy(_rand((k, k, c, c), 13)).requires_grad_(True)
    (T.conv_transpose(x, w, s) * g).sum().backward()
    f = torch.from_numpy(T.tconv_filter(w.detach().numpy(), s)).requires_grad_(True)
    (O.depth_to_space(torch.nn.functional.conv2d(x, f.permute(3, 2, 0, 1), padding=1), s) * g).sum().backward()
    dw = T.tconv_filter_grad(f.grad.numpy(), s, c)
    assert np.abs(dw - w.grad.numpy()).max() <= 1e-12 * np.abs(w.grad.numpy()).max()


SMALL = dict(layers=3, filters=12, min_filters=6, nin_filters=6, nin_filters2=4)


@pytest.mark.parametrize("s", SCALES)
def test_oracle_upsampler_is_the_scatter_loop(s):
    cfg = T.Config(scale=s, **SMALL)
    w = T.random_weights(cfg, seed=s)
    g = np.random.RandomState(s)
    x = g.rand(1, 6, 5, 1) * 255
    x2 = g.rand(1, 6 * s, 5 * s, 1) * 255
    _, inter = T.Oracle(cfg, w).forward(x, x2, return_intermediates=True)
    src = np.concatenate([inter["B2"], inter["A1"]], axis=3).transpose(0, 3, 1, 2)
    ref = T.scatter_reference(src, w[T.TCONV], s).transpose(0, 2, 3, 1)
    assert inter["Up-TCNN"].shape == (1, 6 * s, 5 * s, 10)
    assert np.abs(inter["Up-TCNN"] - ref).max() <= 1e-11 * np.abs(ref).max()


def test_variables_and_l2_set():
    cfg = T.Config(scale=4, **SMALL)
    names = T.variable_names(cfg)
    assert T.TCONV in names and not any(n.startswith("Up-PS") for n in names)
    orc = T.Oracle(cfg, T.random_weights(cfg))
    assert T.TCONV in orc.l2_weight_names()
    ds = T.variable_names(T.Config(scale=2, depthwise_separable=True, **SMALL))
    assert T.TCONV in ds and not any(n.startswith("Up-TCNN/") and n != T.TCONV for n in ds)


def tile_halo(cfg):
    """The engine's dcscn_tile_halo for an Up-TCNN graph: the LR stack's reach, plus the LR pixels that Up-TCNN
    (TF's definition: HR pixel o reads LR pixel i when o = i*s + k - pad_top for a tap k in [0, K)) feeds to the
    HR pixels R-CNN1 reads within h(k_R) of an LR pixel's s x s block."""
    half = lambda kk: (kk - 1) // 2
    k = {scope: kk for scope, kk, *_ in T.layer_table(cfg)}
    r = sum(half(k["CNN%d" % (i + 1)]) for i in range(cfg.layers)) + half(k["B1"]) + half(k["B2"])
    s, hr = cfg.scale, half(k["R-CNN1"])
    reads = [i for o in range(-hr, s + hr) for i in range(-4, 5)
             if any(o == i * s + kk - T.pad_top(s) for kk in range(T.ksize(s)))]
    return r + max(abs(i) for i in reads)


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("cnn", [3, 5])
def test_halo_is_exact_and_tight(s, cnn):
    """A window with the halo around an interior core reproduces the whole-image fp64 output on that core; one pixel
    less changes some core pixel.  With a 3x3 R-CNN1, Up-TCNN and R-CNN1 together reach one LR pixel: each output
    phase of the transposed convolution reads one side of its LR pixel only."""
    cfg = T.Config(scale=s, **dict(SMALL, cnn_size=cnn))
    r = tile_halo(cfg)
    assert r == {3: 3 + 1 + 1, 5: 6 + 1 + {2: 2, 3: 1, 4: 1}[s]}[cnn]
    c = 5
    a = r + 4
    size = 2 * a + c
    g = np.random.RandomState(r * 10 + s)
    x = g.rand(1, size, size, 1) * 255
    x2 = g.rand(1, s * size, s * size, 1) * 255
    oracle = T.Oracle(cfg, T.random_weights(cfg, seed=5))
    assert _core_error(oracle, x, x2, s, a, c, r) <= 1e-9
    assert _core_error(oracle, x, x2, s, a, c, r - 1) > 1e-6


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


def test_flag_constructs_and_names_the_model(tmp_path):
    import DCSCN
    f = _flags(tmp_path, ["--pixel_shuffler=false", "--scale=4"])
    m = DCSCN.SuperResolution(f, model_name=f.model_name)
    assert m.name == "dcscn_L12_F196to48_Sc4_NIN_A64_R1F32"
    cfg = m._engine_config()
    assert cfg.transposed_upsampler == 1
    f = _flags(tmp_path, [])
    assert DCSCN.SuperResolution(f, model_name=f.model_name)._engine_config().transposed_upsampler == 0


@pytest.mark.parametrize("flag", ["--batch_norm=true", "--use_nin=false", "--channels=3", "--reconstruct_layers=2"])
def test_other_flags_are_still_refused(tmp_path, flag):
    import DCSCN
    f = _flags(tmp_path, ["--pixel_shuffler=false", flag])
    with pytest.raises(NotImplementedError):
        DCSCN.SuperResolution(f, model_name=f.model_name)


# utilty.upsample_filter(K) rows: a tent of half-width ceil(K / 2) around the kernel's centre
TENTS = {4: [0.25, 0.75, 0.75, 0.25], 5: [1 / 3, 2 / 3, 1.0, 2 / 3, 1 / 3],
         8: [0.125, 0.375, 0.625, 0.875, 0.875, 0.625, 0.375, 0.125]}


@pytest.mark.parametrize("s", SCALES)
def test_init_is_bilinear_on_the_channel_diagonal(monkeypatch, s):
    import DCSCN
    k, c = T.ksize(s), 5
    shapes = {"B2/conv_W": (3, 3, 4, 4), "B2/conv_B": (4,), T.TCONV: (k, k, c, c), "R-CNN1/conv_W": (3, 3, c, 1)}
    got = {}

    class FakeEngine:
        def param_shapes(self):
            return shapes

        def set_param(self, name, v):
            got[name] = v

        def reset_optimizer(self):
            pass

    m = object.__new__(DCSCN.SuperResolution)
    m.engine, m.initializer, m.weight_dev = FakeEngine(), "he", 0.01
    m.init_all_variables()
    w = got[T.TCONV]
    assert w.dtype == np.float32 and w.shape == (k, k, c, c)
    kern = np.outer(TENTS[k], TENTS[k]).astype(np.float32)
    for i in range(c):
        for j in range(c):
            assert np.array_equal(w[:, :, i, j], kern if i == j else np.zeros_like(kern))
    assert np.allclose(T.bilinear(k), kern)
    assert got["B2/conv_B"].sum() == 0 and got["R-CNN1/conv_W"].std() > 0


def test_complexity_and_receptive_fields(monkeypatch):
    """tf_graph.py:230-233: Up-TCNN multiplies the pixels per input by s*s, costs K*K*C*C per pixel and widens the
    receptive field by one; R-CNN1 then runs at s*s pixels."""
    import DCSCN
    s, k, c = 3, 5, 6
    shapes = {"B2/conv_W": (3, 3, 4, 4), "B2/conv_B": (4,), T.TCONV: (k, k, c, c), "R-CNN1/conv_W": (3, 3, c, 1)}

    class FakeEngine:
        def __init__(self, config):
            pass

        def param_shapes(self):
            return shapes

    monkeypatch.setattr(DCSCN.eng, "Engine", FakeEngine)
    m = object.__new__(DCSCN.SuperResolution)
    m.workspace_mb, m.layers, m.cnn_size, m.scale = 0, 12, 3, s
    m._engine_config = lambda: None
    m.build_graph()
    assert m.complexity == (9 * 16 + 4 + 4) + 9 * k * k * c * c + 9 * 9 * c
    assert m.receptive_fields == 3 + 1 + 2
