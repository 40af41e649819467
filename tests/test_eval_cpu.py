"""Evaluation on the device, CPU half: the arithmetic the eval_* kernels (csrc/eval.cuh) perform, restated in numpy
operation by operation, against the host metric (util.compute_psnr_and_ssim / util._ssim_columns), the trim rule of
DCSCN.do + trim_image_as_file, the size rule of the host resizes, and which path SuperResolution takes."""
import glob
import os

import numpy as np
import pytest

from conftest import GOLDEN


def ssim_restated(a, b, params):
    """eval_ssim_kernel: scipy's symmetric correlation loop (acc = v[r] w0, then acc + (v[r - j] + v[r + j]) w_j for
    j = 5 .. 1) on rows 5 .. H - 6 only, whose windows never reach the reflected border, numpy's order for s, and
    the numpy mean of those rows."""
    a = a.astype(np.float64)
    b = b.astype(np.float64)
    h = a.shape[0]
    if h < 11:
        return float("nan")
    w, c1, c2 = params[:6], params[6], params[7]
    rows = np.arange(5, h - 5)

    def filt(v):
        acc = v[rows] * w[0]
        for j in range(5, 0, -1):
            acc = acc + (v[rows - j] + v[rows + j]) * w[j]
        return acc

    ux, uy = filt(a), filt(b)
    exx, eyy, exy = filt(a * a), filt(b * b), filt(a * b)
    uxx, uyy = ux * ux, uy * uy
    vx, vy, vxy = exx - uxx, eyy - uyy, exy - ux * uy
    s = ((2.0 * ux * uy + c1) * (2.0 * vxy + c2)) / ((uxx + uyy + c1) * (vx + vy + c2))
    return float(np.mean(np.ascontiguousarray(s)))


def sse_restated(a, b):
    """eval_sse_kernel: the exact integer sum of squared differences of two integer-valued planes."""
    d = a.astype(np.int64) - b.astype(np.int64)
    return int(np.sum(d * d, dtype=np.uint64)), d.size


def test_impulse_taps_are_scipys_filter():
    from scipy.ndimage import gaussian_filter1d
    from helper import engine as E
    p = E.ssim_params()
    assert p.shape == (8,) and p[6] == (0.01 * 255) ** 2 and p[7] == (0.03 * 255) ** 2
    v = np.random.RandomState(3).rand(40)
    got = gaussian_filter1d(v, 1.5, truncate=3.5, mode="reflect")
    r = 20
    acc = v[r] * p[0]
    for j in range(5, 0, -1):
        acc = acc + (v[r - j] + v[r + j]) * p[j]
    assert acc == got[r]


@pytest.mark.parametrize("height", [11, 12, 301])
@pytest.mark.parametrize("width", [1, 7, 33])
def test_ssim_restatement_equals_host_on_random_planes(height, width):
    from helper import engine as E, utilty as util
    g = np.random.RandomState(height * 100 + width)
    a = g.randint(0, 256, (height, width)).astype(np.float32)
    b = np.clip(a + g.randint(-40, 41, a.shape), 0, 255).astype(np.float32)
    assert ssim_restated(a, b, E.ssim_params()) == util._ssim_columns(a, b)
    assert ssim_restated(a, a, E.ssim_params()) == util._ssim_columns(a, a)


def test_ssim_restatement_short_planes_are_nan():
    from helper import engine as E, utilty as util
    a = np.zeros((10, 9), np.float32)
    assert np.isnan(ssim_restated(a, a, E.ssim_params())) and np.isnan(util._ssim_columns(a, a))


@pytest.mark.parametrize("scale", [2, 3, 4])
def test_metric_restatement_equals_host_on_set14_bicubic(scale):
    """The trimmed truth and bicubic planes of every Set14 image (evaluate_bicubic's inputs), at the default border."""
    from helper import engine as E, loader, utilty as util
    for f in sorted(glob.glob(os.path.join(GOLDEN, "data", "set14", "*.png"))):
        true = util.set_image_alignment(util.load_image(f, print_console=False), scale)
        lr = loader.build_input_image(true, channels=1, scale=scale, alignment=scale, convert_ycbcr=True)
        bic = util.resize_image_by_pil(lr, scale)
        true_y = util.convert_rgb_to_y(true) if true.shape[2] == 3 else true
        want = util.compute_psnr_and_ssim(true_y, bic, border_size=scale)
        a = util.trim_image_as_file(true_y)[scale:-scale, scale:-scale, 0]
        b = util.trim_image_as_file(bic)[scale:-scale, scale:-scale, 0]
        sse, n = sse_restated(a, b)
        assert E.finish_psnr(sse, n, 0) == want[0], f
        assert ssim_restated(a, b, E.ssim_params()) == want[1], f


def trim_restated(y, flips, max_value):
    """eval_trim_kernel: float64 ensemble mean times 255 / max_value in float64, or the fp32 forward output times
    fp32(255 / max_value) in fp32; rint; clip to [0, 255] (NaN kept)."""
    if flips > 1:
        v = y * (255.0 / max_value)
    else:
        v = (y.astype(np.float32) * np.float32(255.0 / max_value)).astype(np.float64)
    r = np.rint(v)
    return np.where(r < 0, 0.0, np.where(r > 255, 255.0, r)).astype(np.float32)


class _ForwardStub:
    """An engine whose forward returns a fixed fp32 output and whose ensemble returns a fixed float64 mean."""

    def __init__(self, y32, y64):
        self.y32, self.y64 = y32, y64

    def forward_host(self, x, x2):
        return self.y32[None]

    def forward_ensemble_host(self, x, x2, flips):
        return self.y64


def _bare_model(engine, max_value, ensemble):
    import DCSCN
    m = DCSCN.SuperResolution.__new__(DCSCN.SuperResolution)
    m.engine, m.max_value, m.self_ensemble, m.scale, m.channels = engine, max_value, ensemble, 2, 1
    m.resampling_method = DCSCN.BICUBIC_METHOD_STRING
    return m


@pytest.mark.parametrize("max_value", [255.0, 1.0, 127.5])
@pytest.mark.parametrize("flips", [1, 8])
def test_trim_rule_equals_do_then_trim_image_as_file(max_value, flips):
    from helper import utilty as util
    g = np.random.RandomState(int(max_value) + flips)
    base = np.concatenate([[np.nan, -0.0, 255.5, 254.5], np.arange(-3, 259) + 0.5, g.uniform(-20, 280, 4000)])[:4264]
    # outputs as the network gives them at this max_value (do multiplies them back by 255 / max_value)
    y32 = (base * (max_value / 255.0)).astype(np.float32).reshape(-1, 4, 1)
    y64 = (base * (max_value / 255.0)).astype(np.float64).reshape(-1, 4, 1)
    m = _bare_model(_ForwardStub(y32, y64), max_value, flips)
    lr = np.zeros((y32.shape[0] // 2, 2, 1), np.float32)
    got = util.trim_image_as_file(m.do(lr, np.zeros(y32.shape, np.float32)))
    want = trim_restated(y64 if flips > 1 else y32, flips, max_value)
    assert got.dtype == want.dtype
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("scale", [2, 3, 4, 8])
def test_size_rule_equals_the_host_resizes(scale):
    from helper import engine as E, utilty as util
    for side in range(scale, 4097, scale):
        (ah, aw), (lh, lw), (bh, bw), _ = E.eval_geometry(side, side + scale - 1, scale, 0)
        assert (ah, aw) == (side, side) and (lh, lw) == (side // scale, side // scale) and (bh, bw) == (side, side)
    for side in range(scale, 700, 7 * scale):    # the shapes Pillow actually produces
        a = np.zeros((side, side + scale, 1), np.float32)
        lr = util.resize_image_by_pil(a, 1.0 / scale)
        bic = util.resize_image_by_pil(lr, scale)
        _, (lh, lw), (bh, bw), _ = E.eval_geometry(side, side + scale, scale, 0)
        assert lr.shape[:2] == (lh, lw) and bic.shape[:2] == (bh, bw)


def test_region_rule():
    from helper import engine as E
    assert E.eval_geometry(40, 50, 2, 0)[3] == (40, 50)
    assert E.eval_geometry(40, 50, 2, -3)[3] == (40, 50)
    assert E.eval_geometry(40, 50, 2, 2)[3] == (36, 46)
    assert E.eval_geometry(40, 50, 2, 30)[3] == (0, 0)
    assert np.isnan(E.finish_psnr(0, 0, 0)) and np.isnan(E.finish_psnr(5, 10, 1)) and E.finish_psnr(0, 10, 0) == np.inf


class _EvalEngine:
    """Records what SuperResolution hands to the device evaluation call."""

    def __init__(self):
        self.stores, self.calls = [], []

    def set_eval_images(self, images):
        self.stores.append([i.shape for i in images])

    def evaluate_image(self, image, flips, max_value, border, bicubic=False):
        self.calls.append((image if isinstance(image, int) else image.shape, flips, max_value, border, bicubic))
        return 30.0, 0.9


def _eval_model(engine):
    m = _bare_model(engine, 255.0, 8)
    m.psnr_calc_border_size = 2
    return m


def test_device_path_selection(monkeypatch):
    import DCSCN
    files = sorted(glob.glob(os.path.join(GOLDEN, "data", "set5", "*.png")))
    eng = _EvalEngine()
    m = _eval_model(eng)
    assert m.do_for_evaluate(files[0]) == (30.0, 0.9)
    assert m.evaluate_bicubic(files[0]) == (30.0, 0.9)
    assert eng.calls[0][1:] == (8, 255.0, 2, False) and eng.calls[1][4] is True
    # an engine without the call, a multi-process job and a non-bicubic resampler keep the host path
    for engine, world, method in ((object(), 1, "bicubic"), (eng, 2, "bicubic"), (eng, 1, "bilinear")):
        m = _eval_model(engine)
        m.resampling_method = method
        monkeypatch.setattr(DCSCN, "_dist_rank_world", lambda w=world: (0, w))
        called = []
        monkeypatch.setattr(m, "_do_for_evaluate_host", lambda f, p=False: called.append(f) or (1.0, 0.5))
        assert m.do_for_evaluate(files[0]) == (1.0, 0.5) and called == files[:1]


def test_evaluate_uploads_the_store_once(tmp_path):
    import shutil
    files = []
    for f in sorted(glob.glob(os.path.join(GOLDEN, "data", "set5", "*.png")))[:3]:
        shutil.copy(f, str(tmp_path))
        files.append(str(tmp_path / os.path.basename(f)))
    eng = _EvalEngine()
    m = _eval_model(eng)
    assert m.evaluate(files) == (30.0, 0.9)
    assert m.evaluate(files) == (30.0, 0.9)
    assert len(eng.stores) == 1 and [c[0] for c in eng.calls] == [0, 1, 2, 0, 1, 2]
    st = os.stat(files[1])
    os.utime(files[1], ns=(st.st_atime_ns, st.st_mtime_ns + 10 ** 9))     # a changed file: the store is rebuilt
    m.evaluate(files)
    assert len(eng.stores) == 2
    m.evaluate(files[:2])
    assert len(eng.stores) == 3
