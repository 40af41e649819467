"""
Tiled inference under a workspace budget (option "workspace_mb", run with `-m gpu` on an H100).  A forward whose
workspace exceeds the budget runs as batches of overlapping windows; every window core carries dcscn_tile_halo pixels
of context, so the result must equal the whole-image forward of the same handle bit for bit (np.array_equal), for every
graph family, for shapes that split both dimensions, cross images or are narrower than a window, and through every
inference entry point.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import dcscn_oracle as O
from conftest import MODEL_FLAGS, load_golden_weights
from test_tiling_cpu import CNN5, tile_halo

pytestmark = pytest.mark.gpu

MiB = 1 << 20
DS3 = dict(scale=3, layers=3, filters=12, min_filters=6, filters_decay_gamma=1.5, nin_filters=10, nin_filters2=6,
           pixel_shuffler_filters=1, depthwise_separable=True)
GRAPHS = {
    "L12x2": ("dcscn_L12_F196to48_NIN_A64_PS_R1F32", 0),
    "L12x3": ("dcscn_L12_F196to48_Sc3_NIN_A64_PS_R1F32", 0),
    "L12x4": ("dcscn_L12_F196to48_Sc4_NIN_A64_PS_R1F32", 0),
    "L7x2": ("dcscn_L7_F32to8_G1.20_NIN_A24_B8_PS_R1F32", 0),
    "DSx4": ("dcscn_L7_F32to8_G1.20_Sc4_NIN_A24_B8_PS_DS_R1F32", 0),
    "DSx3": ("he:DS3", 0),          # odd HR widths: R-CNN1 on the one-pixel kernel
    "cnn5": ("he:CNN5", 0),
    "L12x2_f16x1": ("dcscn_L12_F196to48_NIN_A64_PS_R1F32", 1),
}
# (n, h, w, LR pixels the budget allows per batch)
SHAPES = {
    "split2d": (1, 97, 131, 6000),
    "images": (3, 40, 57, 5000),
    "strip": (1, 23, 300, 2800),
}
_engines = {}


def graph_kw(graph):
    name, _ = GRAPHS[graph]
    if name == "he:DS3":
        return DS3, O.he_init_weights(O.OracleConfig(**DS3), seed=4)
    if name == "he:CNN5":
        return CNN5, O.he_init_weights(O.OracleConfig(**CNN5), seed=3)
    return {"scale": 2, **MODEL_FLAGS[name]}, load_golden_weights(name)


def new_engine(graph):
    from helper import engine as E
    kw, w = graph_kw(graph)
    eng = E.Engine(E.make_config(precision=GRAPHS[graph][1], **kw))
    eng.set_params(w)
    return eng, kw


def engine(graph):
    """One handle per graph, with its workspace bytes per LR pixel measured on an 8 x 8 forward."""
    if graph not in _engines:
        eng, kw = new_engine(graph)
        s = kw["scale"]
        eng.forward(torch.zeros(1, 8, 8, 1, device="cuda"), torch.zeros(1, 8 * s, 8 * s, 1, device="cuda"))
        torch.cuda.synchronize()
        _engines[graph] = (eng, kw, eng.device_bytes // 64)
    return _engines[graph]


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for eng, _, _ in _engines.values():
        eng.close()
    _engines.clear()


def budget_mb(kw, ws_px, px):
    """A budget (MiB) of about `px` window pixels per batch, staging buffers included."""
    s = kw["scale"]
    return max(1, int(px * (ws_px + 4 * (1 + 2 * s * s)) // MiB))


def inputs(n, h, w, s, seed):
    g = np.random.RandomState(seed)
    return (g.rand(n, h, w, 1) * 255).astype(np.float32), (g.rand(n, s * h, s * w, 1) * 255).astype(np.float32)


def run_entry(eng, entry, x, x2):
    if entry == "forward":
        y = eng.forward(torch.from_numpy(x).cuda(), torch.from_numpy(x2).cuda())
        torch.cuda.synchronize()
        return y.cpu().numpy()
    if entry == "host_bicubic":
        return eng.forward_host(x, None)
    if entry == "ensemble8":
        return eng.forward_ensemble_host(x[0], None, 8)
    if entry == "partial":
        s = eng.config.scale
        h, w = x.shape[1], x.shape[2]
        out = torch.empty((s * h, s * w), dtype=torch.float64, device="cuda")
        xd, x2d = torch.from_numpy(x[0, :, :, 0].copy()).cuda(), torch.from_numpy(x2[0, :, :, 0].copy()).cuda()
        st = torch.cuda.current_stream().cuda_stream
        eng._check(eng.lib.dcscn_forward_ensemble_partial(eng.handle, xd.data_ptr(), x2d.data_ptr(), out.data_ptr(), h, w,
                                                          0b10110101, ctypes.c_void_p(st)))
        torch.cuda.synchronize()
        return out.cpu().numpy()
    raise ValueError(entry)


def tiled_then_whole(eng, mb, entry, x, x2):
    from helper import engine as E
    eng.set_option("workspace_mb", mb)
    l0, r0 = eng.launch_count, eng.graph_replays
    y_tiled = run_entry(eng, entry, x, x2)
    launches, replays = eng.launch_count - l0, eng.graph_replays - r0
    with pytest.raises(E.EngineError) as ei:     # the last forward ran tiled
        eng.get_activation("CNN1", (1,))
    assert "tiled" in str(ei.value)
    eng.set_option("workspace_mb", 0)
    l0 = eng.launch_count
    y_whole = run_entry(eng, entry, x, x2)
    return y_tiled, y_whole, launches, replays, eng.launch_count - l0


@pytest.mark.parametrize("entry", ["forward", "host_bicubic", "ensemble8", "partial"])
@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("graph", sorted(GRAPHS))
def test_tiled_forward_is_bit_identical(graph, shape, entry):
    eng, kw, ws_px = engine(graph)
    n, h, w, px = SHAPES[shape]
    if graph == "DSx3" and shape == "split2d":
        w = 133                                      # HR width 399: odd
    batch_n = n                                      # images of the largest forward of the call
    if entry in ("ensemble8", "partial"):
        n, batch_n = 1, (4 if entry == "ensemble8" else 3)
    s = kw["scale"]
    mb = budget_mb(kw, ws_px, px)
    assert batch_n * h * w * ws_px > mb * MiB, "the image fits the budget: nothing would be tiled"
    x, x2 = inputs(n, h, w, s, seed=h * 7 + w)
    y_tiled, y_whole, launches, replays, launches_whole = tiled_then_whole(eng, mb, entry, x, x2)
    assert y_tiled.shape == y_whole.shape and np.isfinite(y_whole).all()
    assert np.array_equal(y_tiled, y_whole), float(np.abs(y_tiled.astype(np.float64) - y_whole).max())
    if entry == "forward":
        batches = launches // (launches_whole + 2)   # gather + the whole-image launch sequence + stitch per batch
        assert batches * (launches_whole + 2) == launches
        if batches >= 3 and not kw.get("depthwise_separable"):
            assert replays > 0, "full batches never reached the captured-graph path"


def test_tile_halo_matches_the_formula():
    for graph in GRAPHS:
        eng, kw, _ = engine(graph)
        assert eng.tile_halo() == tile_halo(O.OracleConfig(**kw)), graph
    assert engine("L12x2")[0].tile_halo() == 15 and engine("L7x2")[0].tile_halo() == 10


def test_budget_is_kept_and_fitting_images_run_untiled():
    _, kw, ws_px = engine("L12x2")
    mb = budget_mb(kw, ws_px, 6000)
    x, x2 = inputs(1, 97, 131, 2, seed=1)
    tiled, _ = new_engine("L12x2")
    tiled.set_option("workspace_mb", mb)
    y_t = run_entry(tiled, "forward", x, x2)
    assert 0 < tiled.device_bytes <= mb * MiB
    whole, _ = new_engine("L12x2")
    y_w = run_entry(whole, "forward", x, x2)
    assert whole.device_bytes > mb * MiB
    assert np.array_equal(y_t, y_w)
    # an image whose workspace fits runs exactly as without the option
    xs, x2s = inputs(2, 16, 24, 2, seed=2)
    l0 = tiled.launch_count
    y_fit = run_entry(tiled, "forward", xs, x2s)
    fit_launches = tiled.launch_count - l0
    tiled.get_activation("CNN1", (2, 16, 24, 196))     # not tiled: the activations are the image's
    l0 = whole.launch_count
    y_ref = run_entry(whole, "forward", xs, x2s)
    assert fit_launches == whole.launch_count - l0
    assert np.array_equal(y_fit, y_ref)
    tiled.close()
    whole.close()


def test_large_image_without_the_whole_workspace():
    """2048 x 2048 at x2 would need about 32 GB of workspace; at 1 GiB it runs tiled, and a 256 x 256 core of it equals
    the untiled forward of that crop with the halo around it."""
    eng, _ = new_engine("L12x2")
    r = eng.tile_halo()
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.rand(1, 2048, 2048, 1, device="cuda", generator=g) * 255
    x2 = torch.rand(1, 4096, 4096, 1, device="cuda", generator=g) * 255
    eng.set_option("workspace_mb", 1024)
    y = eng.forward(x, x2)
    torch.cuda.synchronize()
    assert eng.device_bytes <= 1024 * MiB
    assert torch.isfinite(y).all()
    a, c = 901, 256
    xc = x[:, a - r:a + c + r, a - r:a + c + r].contiguous()
    x2c = x2[:, 2 * (a - r):2 * (a + c + r), 2 * (a - r):2 * (a + c + r)].contiguous()
    eng.set_option("workspace_mb", 0)
    yc = eng.forward(xc, x2c)
    torch.cuda.synchronize()
    assert torch.equal(yc[:, 2 * r:2 * (r + c), 2 * r:2 * (r + c)], y[:, 2 * a:2 * (a + c), 2 * a:2 * (a + c)])
    eng.close()


def test_timing_covers_every_launch_of_a_tiled_forward():
    eng, kw, ws_px = engine("L7x2")
    x, x2 = inputs(1, 97, 131, 2, seed=3)
    eng.set_option("workspace_mb", budget_mb(kw, ws_px, 3000))
    eng.set_option("timing", 1)
    l0 = eng.launch_count
    run_entry(eng, "forward", x, x2)
    launches = eng.launch_count - l0
    t = eng.timings()
    eng.set_option("timing", 0)
    eng.set_option("workspace_mb", 0)
    assert len(t) == launches and t[0][0] == "tile_gather" and t[-1][0] == "tile_stitch"
    assert sum(name == "tile_gather" for name, _ in t) >= 2 and all(ms >= 0 for _, ms in t)


def test_errors():
    from helper import engine as E
    eng, _, _ = engine("L12x2")
    with pytest.raises(E.EngineError):
        eng.set_option("workspace_mb", -1)
    x, x2 = inputs(1, 97, 131, 2, seed=4)
    eng.set_option("workspace_mb", 1)
    with pytest.raises(E.EngineError) as ei:
        run_entry(eng, "forward", x, x2)
    msg = str(ei.value)
    assert "workspace_mb" in msg and "at least" in msg
    need = int(msg.rsplit("workspace_mb = ", 1)[1].split()[0])
    eng.set_option("workspace_mb", need)
    run_entry(eng, "forward", x, x2)                 # the named minimum is enough
    with pytest.raises(E.EngineError) as ei:
        eng.get_activation("CNN1", (1, 97, 131, 196))
    assert "tiled" in str(ei.value)
    eng.set_option("workspace_mb", 0)
    run_entry(eng, "forward", x, x2)
    eng.get_activation("CNN1", (1, 97, 131, 196))
    assert math.isfinite(eng.tile_halo())
