"""Training data path on the device (SURVEY.md section 8 f3): the grid-patch data set of loader.BatchDataSets
(reference helper/loader.py:70-275) kept as uint8 arrays in HBM, a mini-batch = an index list + one gather launch per
tensor.  Parity: the gathered fp32 tensors equal, bit for bit, what the host path feeds (`load_batch_image` +
np.stack, DCSCN.py:186-190 / :415-420); the indexed train step equals the host-buffer train step on those patches; the
left-right mirror flag equals np.fliplr of the host patches (loader.py:318-319)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

KW = dict(scale=2, layers=3, filters=24, min_filters=16, filters_decay_gamma=1.5, nin_filters=16, nin_filters2=16)


def build_set(scale, size):
    from helper import loader
    ds = loader.BatchDataSets(scale, "unused", size, stride_size=size)
    ds.build_batch(os.path.join(GOLDEN, "data", "set5"))
    assert ds.count > 20
    return ds


def host_batch(ds, idx, max_value=255.0):
    """(x, x2, y) as the host loader feeds patches `idx`, fp32."""
    host = []
    for k in idx:
        ds.batch_index, ds.index = [int(k)], 0          # make the host loader serve exactly patch k
        host.append(ds.load_batch_image(max_value))
    return tuple(np.stack([h[j] for h in host]).astype(np.float32) for j in range(3))


@pytest.mark.parametrize("max_value", [255.0, 1.0])
def test_gather_equals_the_host_loader(max_value):
    import dcscn_oracle as O
    from helper import engine as E
    ds = build_set(2, 24)
    eng = E.Engine(E.make_config(dropout_keep=1.0, **KW))
    eng.set_params(O.he_init_weights(O.OracleConfig(**KW), seed=2))
    eng.set_patch_store(ds.input_images, ds.input_interpolated_images, ds.true_images)
    rs = np.random.RandomState(0)
    idx = rs.randint(0, ds.count, size=13)
    x, x2, y = eng.gather_patches(idx, max_value=max_value)
    hx, hx2, hy = host_batch(ds, idx, max_value)
    np.testing.assert_array_equal(x, hx)
    np.testing.assert_array_equal(x2, hx2)
    np.testing.assert_array_equal(y, hy)
    # mirror flag == np.fliplr of the patch
    mir = rs.randint(0, 2, size=13)
    mx, mx2, my = eng.gather_patches(idx, max_value=max_value, mirror=mir)
    for i in range(13):
        f = (lambda a: a[:, ::-1]) if mir[i] else (lambda a: a)
        np.testing.assert_array_equal(mx[i], f(hx[i]))
        np.testing.assert_array_equal(mx2[i], f(hx2[i]))
        np.testing.assert_array_equal(my[i], f(hy[i]))
    with pytest.raises(E.EngineError):
        eng.gather_patches([ds.count])
    eng.close()


def test_indexed_train_step_equals_the_host_buffer_step():
    import dcscn_oracle as O
    from helper import engine as E
    ds = build_set(2, 16)
    w = O.he_init_weights(O.OracleConfig(**KW), seed=4)
    idx = np.arange(3, 3 + 8) * 2
    out = []
    for mode in ("host", "indexed"):
        eng = E.Engine(E.make_config(dropout_keep=0.8, **KW))
        eng.set_params(w)
        eng.set_patch_store(ds.input_images, ds.input_interpolated_images, ds.true_images)
        if mode == "host":
            x, x2, y = eng.gather_patches(idx)
            res = eng.train_step_host(x, x2, y, lr=1e-3, seed=5)
        else:
            res = eng.train_step_indexed(idx, lr=1e-3, seed=5)
        out.append((res, {n: eng.get_param(n) for n in ("CNN2/conv_W", "A1/conv_B", "R-CNN1/conv_W")}))
        eng.close()
    assert out[0][0] == out[1][0]
    for n in out[0][1]:
        np.testing.assert_allclose(out[0][1][n], out[1][1][n], rtol=0, atol=2e-6)   # fp32 atomics reorder a few sums


@pytest.mark.parametrize("shape,scale", [((3, 48, 48), 2), ((1, 37, 53), 2), ((2, 24, 31), 3), ((1, 20, 22), 4), ((1, 96, 64), 0.5),
                                         ((2, 99, 63), 1 / 3)])
def test_device_bicubic_is_pillow_bit_for_bit(shape, scale):
    """SURVEY.md section 8 f2: `util.resize_image_by_pil` (PIL Image.resize BICUBIC on mode-F images, reference
    helper/utilty.py:211-239) restated on the device - identical bits, up- and down-scaling."""
    import torch
    import dcscn_oracle as O
    from helper import engine as E, utilty as util
    eng = E.Engine(E.make_config(**KW))
    rs = np.random.RandomState(5)
    n, h, w = shape
    a = (rs.rand(n, h, w) * 255).astype(np.float32)
    oh, ow = int(h * scale), int(w * scale)
    got = eng.bicubic_resize(torch.from_numpy(a).cuda(), oh, ow).cpu().numpy()
    for i in range(n):
        ref = util.resize_image_by_pil(a[i].reshape(h, w, 1).astype(np.float64), scale)[:, :, 0]
        assert ref.shape == (oh, ow)
        np.testing.assert_array_equal(got[i], ref)
    eng.close()


def test_set_patch_store_keeps_the_bicubic_tables():
    """Setting the patch store replaces the three patch arrays only: the Pillow tables and the bicubic scratch that an
    earlier device resize cached stay valid, so the same resize after it is still Pillow bit for bit, and each store
    serves its own patches as the host loader does."""
    import torch
    from helper import engine as E, utilty as util
    eng = E.Engine(E.make_config(**KW))
    rs = np.random.RandomState(7)
    n, h, w = 2, 37, 53
    a = (rs.rand(n, h, w) * 255).astype(np.float32)
    ref = np.stack([util.resize_image_by_pil(a[i].reshape(h, w, 1).astype(np.float64), 2)[:, :, 0] for i in range(n)])

    def check_resize():
        np.testing.assert_array_equal(eng.bicubic_resize(torch.from_numpy(a).cuda(), 2 * h, 2 * w).cpu().numpy(), ref)

    check_resize()
    for size in (24, 16):          # the second store replaces the first
        ds = build_set(2, size)
        eng.set_patch_store(ds.input_images, ds.input_interpolated_images, ds.true_images)
        check_resize()
        idx = rs.randint(0, ds.count, size=9)
        for got, want in zip(eng.gather_patches(idx), host_batch(ds, idx)):
            np.testing.assert_array_equal(got, want)
    eng.close()


def test_forward_without_x2_equals_forward_with_pil_bicubic():
    """`SuperResolution.do(image)` without a bicubic argument (sr.py's path, DCSCN.py:551-553): the engine forms x2 in HBM;
    the result must equal the call that is handed Pillow's bicubic, bit for bit, for the plain forward and the ensemble."""
    import dcscn_oracle as O
    from helper import engine as E, utilty as util
    eng = E.Engine(E.make_config(**KW))
    eng.set_params(O.he_init_weights(O.OracleConfig(**KW), seed=6))
    rs = np.random.RandomState(6)
    lr = rs.rand(21, 30, 1) * 255
    bic = util.resize_image_by_pil(lr, 2)
    x = np.ascontiguousarray(lr, np.float32).reshape(1, 21, 30, 1)
    x2 = np.ascontiguousarray(bic, np.float32).reshape(1, 42, 60, 1)
    np.testing.assert_array_equal(eng.forward_host(x, None), eng.forward_host(x, x2))
    np.testing.assert_array_equal(eng.forward_ensemble_host(lr, None, 8), eng.forward_ensemble_host(lr, bic, 8))
    eng.close()
