"""The random-crop data path (loader.DynamicDataSets, reference helper/loader.py:278-355) as the device restates it,
checked on the host: the float64 RGB -> Y order, Pillow's 8-bit bicubic, the crop descriptors and their random draws,
and the SuperResolution glue that sends crops to the engine.  CPU only."""
import os
import random
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, PKG

_Y_FMA_C = r"""
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
/* Y of every 24-bit colour (index r << 16 | g << 8 | b): fma(b, c2, fma(g, c1, r * c0)) + 16, then the plain sum. */
int main(int argc, char** argv) {
  const double c0 = 65.738 / 256.0, c1 = 129.057 / 256.0, c2 = 25.064 / 256.0;
  double* out = malloc(sizeof(double) << 24);
  FILE* f;
  for (int pass = 0; pass < 2; ++pass) {
    for (int i = 0; i < 1 << 24; ++i) {
      const double r = i >> 16, g = (i >> 8) & 255, b = i & 255;
      out[i] = (pass == 0 ? fma(b, c2, fma(g, c1, r * c0)) : r * c0 + g * c1 + b * c2) + 16.0;
    }
    f = fopen(argv[1 + pass], "wb");
    fwrite(out, sizeof(double), 1 << 24, f);
    fclose(f);
  }
  free(out);
  return 0;
}
"""


def all_colours():
    """A 4096 x 4096 RGB image that holds every 24-bit colour once (pixel k has colour k)."""
    k = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(k >> 16) & 255, (k >> 8) & 255, k & 255], axis=-1).astype(np.uint8).reshape(4096, 4096, 3)


def test_rgb_to_y_is_the_fma_chain_for_every_colour(tmp_path):
    """The device forms util.convert_rgb_to_y's float64 Y as fma(b, c2, fma(g, c1, r * c0)) + 16.0: that is what numpy's
    dot (BLAS ddot) gives, for all 2^24 colours, bit for bit."""
    from helper import utilty as util
    src, exe = tmp_path / "y.c", tmp_path / "y"
    src.write_text(_Y_FMA_C)
    subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-o", str(exe), str(src), "-lm"])
    subprocess.check_call([str(exe), str(tmp_path / "fma.bin"), str(tmp_path / "plain.bin")])
    fma = np.fromfile(tmp_path / "fma.bin", dtype=np.float64)
    image = all_colours()
    got = np.concatenate([util.convert_rgb_to_y(image[r:r + 512]).reshape(-1) for r in range(0, 4096, 512)])
    bad = int(np.count_nonzero(got != fma))
    if bad:
        plain = np.fromfile(tmp_path / "plain.bin", dtype=np.float64)
        pytest.fail("numpy's RGB -> Y differs from the fma chain for %d colours (it equals the unfused sum for %d of "
                    "them): this BLAS rounds the dot product differently, so the device's float64 Y no longer matches"
                    % (bad, int(np.count_nonzero((got == plain) & (got != fma)))))


@pytest.mark.parametrize("shape,out", [((48, 48), (24, 24)), ((48, 48), (16, 16)), ((48, 48), (12, 12)),
                                       ((24, 24), (48, 48)), ((16, 16), (48, 48)), ((12, 12), (48, 48)),
                                       ((37, 53), (18, 26)), ((19, 23), (57, 69)), ((1, 9), (3, 27))])
def test_resize_uint8_is_pillow_mode_l_bit_for_bit(shape, out):
    from PIL import Image
    from helper import pil_resample as R
    rs = np.random.RandomState(shape[0] * 100 + out[0])
    a = (rs.rand(*shape) * 256).astype(np.uint8)
    a[: max(1, shape[0] // 8)] = 255                  # saturated rows and columns overshoot past 0 and 255
    a[:, ::5] = 0
    a[-1, ::3] = 255
    ref = np.asarray(Image.fromarray(a).resize([out[1], out[0]], Image.BICUBIC))
    np.testing.assert_array_equal(R.resize_uint8(a, out[1], out[0]), ref)


def dynamic_set(dataset, scale, size):
    from helper import loader
    ds = loader.DynamicDataSets(scale, size)
    ds.set_data_dir(os.path.join(GOLDEN, "data", dataset))
    return ds


@pytest.mark.parametrize("dataset,scale,size", [("set14", 2, 48), ("set14", 4, 64), ("set5", 3, 96), ("set5", 4, 72)])
def test_draw_crop_follows_load_batch_image(dataset, scale, size, capsys):
    """Under the same seed, draw_crop names the crop load_batch_image cuts and leaves `random` in the same state; crops
    stay inside their image and images smaller than one patch are skipped with the reference's message."""
    from helper import utilty as util
    edge = scale * size
    drawn, loaded = dynamic_set(dataset, scale, size), dynamic_set(dataset, scale, size)
    random.seed(11)
    crops = [drawn.draw_crop() for _ in range(30)]
    state = random.getstate()
    random.seed(11)
    for number, top, left, mirror in crops:
        rows, cols = drawn.sizes[number]
        assert rows >= edge and cols >= edge
        assert 0 <= top <= max(rows - edge - 1, 0) and 0 <= left <= max(cols - edge - 1, 0)
        assert mirror in (0, 1)
        x, x2, y = loaded.load_batch_image(255.0)
        image = util.convert_rgb_to_y(util.load_image(drawn.filenames[number], print_console=False))
        want = image[top:top + edge, left:left + edge]
        np.testing.assert_array_equal(y, want[:, ::-1] if mirror else want)
        assert x.shape[:2] == (size, size) and x2.shape[:2] == (edge, edge)
    assert random.getstate() == state
    small = [i for i, (r, c) in enumerate(drawn.sizes) if r < edge or c < edge]
    assert all(c[0] not in small for c in crops)
    out = capsys.readouterr().out
    for i in small:
        assert "Error: %s should have more than %d x %d size." % (drawn.filenames[i], edge, edge) in out


def test_draw_crop_bounds_at_rows_equal_edge():
    """set5/img_002.png is 288 x 288: a 288-pixel crop sits at (0, 0) and draws no position."""
    ds = dynamic_set("set5", 4, 72)
    assert ds.sizes[1] == (288, 288)
    ds.batch_index, ds.index = [1], 0
    random.seed(3)
    assert ds.draw_crop()[:3] == (1, 0, 0)
    state = random.getstate()
    random.seed(3)
    random.randrange(2)                                # the mirror is the only draw
    assert random.getstate() == state


def test_decoded_images_match_the_headers():
    ds = dynamic_set("set14", 2, 48)
    images = ds.decoded_images()
    assert [im.shape[:2] for im in images] == ds.sizes
    assert sorted({im.shape[2] for im in images}) == [1, 3]          # img_003 is mode 'L'


class FakeEngine:
    def __init__(self):
        self.stores, self.steps = [], []

    def set_image_store(self, images):
        self.stores.append(len(images))

    def train_step_crops(self, crops, patch_size, lr, seed, max_value=255.0, apply_update=True):
        self.steps.append((np.array(crops).tolist(), patch_size, lr, seed, max_value))
        return 4.0, 4.0

    def train_step_host(self, *a, **k):
        raise AssertionError("host-buffer step with an engine image store")


def glue_model(engine):
    import DCSCN
    m = object.__new__(DCSCN.SuperResolution)
    m.scale, m.channels, m.resampling_method, m.batch_num, m.max_value = 2, 1, "bicubic", 4, 255.0
    m.lr, m.step = 0.002, 5
    m.engine = engine
    m.load_dynamic_datasets(os.path.join(GOLDEN, "data", "set14"), 24)
    return m


def test_dynamic_set_with_an_engine_uploads_once_and_trains_on_crops():
    eng = FakeEngine()
    m = glue_model(eng)
    random.seed(5)
    m.init_epoch_index()
    m.init_epoch_index()
    assert eng.stores == [m.train.count]                                  # one upload per data set
    m.build_input_batch()
    m.train_batch()
    m.build_input_batch()
    m.train_batch()
    reference = glue_model(None).train
    random.seed(5)
    reference.init_batch_index()
    reference.init_batch_index()
    want = [[list(reference.draw_crop()) for _ in range(4)] for _ in range(2)]
    assert eng.steps == [(want[0], 24, 0.002, 5, 255.0), (want[1], 24, 0.002, 6, 255.0)]
    assert m.training_step == 2 and m.step == 7


def test_dynamic_set_without_an_engine_stays_on_the_host_path():
    m = glue_model(None)
    random.seed(5)
    m.init_epoch_index()
    assert m.batch_crops is None
    m.build_input_batch()
    assert all(x.shape == (24, 24, 1) for x in m.batch_input)
    assert all(y.shape == (48, 48, 1) for y in m.batch_true)
