"""Random-crop training data on the device: the decoded images of loader.DynamicDataSets (reference helper/loader.py:278-355,
the data set of train.py without --build_batch) kept in HBM, a mini-batch = a list of crop descriptors (image, top, left,
mirror).  Parity: the device's fp32 x / x2 / y equal, bit for bit, np.stack(...).astype(np.float32) of the host loader's
load_batch_image under the same seed; the crop step equals the host-buffer step on those tensors."""
import glob
import os
import random
import sys

import numpy as np
import pytest

from conftest import GOLDEN, PKG, ROOT

pytestmark = pytest.mark.gpu

KW = dict(scale=2, layers=3, filters=24, min_filters=16, filters_decay_gamma=1.5, nin_filters=16, nin_filters2=16)
DS_KW = dict(scale=4, layers=7, filters=32, min_filters=8, filters_decay_gamma=1.2, nin_filters=24, nin_filters2=8,
             reconstruct_layers=0, pixel_shuffler_filters=1, depthwise_separable=True)


def dynamic_set(dataset, scale, size):
    from helper import loader
    ds = loader.DynamicDataSets(scale, size)
    ds.set_data_dir(os.path.join(GOLDEN, "data", dataset))
    return ds


def host_and_crops(ds, count, seed, max_value):
    """The host loader's fp32 batch and the descriptors draw_crop names for it, from the same seed."""
    random.seed(seed)
    ds.batch_index = None
    crops = [ds.draw_crop() for _ in range(count)]
    random.seed(seed)
    ds.batch_index = None
    host = [ds.load_batch_image(max_value) for _ in range(count)]
    return crops, tuple(np.stack([h[j] for h in host]).astype(np.float32).reshape(count, *host[0][j].shape[:2], 1)
                        for j in range(3))


def engine(**kw):
    from helper import engine as E
    return E.Engine(E.make_config(**dict(KW, **kw)))


@pytest.mark.parametrize("max_value", [255.0, 1.0])
@pytest.mark.parametrize("dataset,scale,size", [("set14", 2, 32), ("set14", 3, 24), ("set14", 4, 16), ("set5", 4, 72)])
def test_gather_crops_equals_the_host_loader(dataset, scale, size, max_value):
    ds = dynamic_set(dataset, scale, size)
    eng = engine(scale=scale)
    eng.set_image_store(ds.decoded_images())
    crops, host = host_and_crops(ds, 24, seed=scale * 7 + int(max_value), max_value=max_value)
    assert {c[3] for c in crops} == {0, 1}
    if dataset == "set14":
        assert any(ds.filenames[c[0]].endswith("img_003.png") for c in crops)     # mode 'L' beside RGB in one batch
    else:
        assert any(ds.sizes[c[0]] == (scale * size, scale * size) for c in crops)  # rows == edge
    for got, want in zip(eng.gather_crops(crops, size, max_value=max_value), host):
        np.testing.assert_array_equal(got, want)
    eng.close()


@pytest.mark.parametrize("max_value", [255.0, 1.0])
def test_every_rgb_colour_gives_the_host_truth(max_value):
    """A 4096 x 4096 image holding each 24-bit colour once, gathered in 256 crops of 256 x 256 that tile it."""
    from helper import utilty as util
    k = np.arange(1 << 24, dtype=np.uint32)
    image = np.stack([(k >> 16) & 255, (k >> 8) & 255, k & 255], axis=-1).astype(np.uint8).reshape(4096, 4096, 3)
    eng = engine()
    eng.set_image_store([image])
    crops = [(0, 256 * (i // 16), 256 * (i % 16), i % 2) for i in range(256)]
    _, _, y = eng.gather_crops(crops, 128, max_value=max_value)
    truth = util.convert_rgb_to_y(image)
    if max_value != 255:
        truth = np.multiply(truth, max_value / 255.0)
    for i, (_, top, left, mirror) in enumerate(crops):
        want = truth[top:top + 256, left:left + 256]
        np.testing.assert_array_equal(y[i], (want[:, ::-1] if mirror else want).astype(np.float32))
    eng.close()


class _FakeFlagsModel:
    """SuperResolution with only what the data path reads (no checkpoint or log directories)."""

    @staticmethod
    def make(engine_):
        import DCSCN
        m = object.__new__(DCSCN.SuperResolution)
        m.scale, m.channels, m.resampling_method, m.batch_num, m.max_value = 2, 1, "bicubic", 12, 255.0
        m.lr, m.step = 0.002, 0
        m.engine = engine_
        m.load_dynamic_datasets(os.path.join(GOLDEN, "data", "set14"), 32)
        return m


def test_seeded_batches_through_superresolution_equal_the_host_path():
    eng = engine()
    dev, host = _FakeFlagsModel.make(eng), _FakeFlagsModel.make(None)
    for m in (dev, host):
        random.seed(99)
        m.init_epoch_index()
    assert dev.batch_crops is not None and host.batch_crops is None
    for _ in range(3):
        state = random.getstate()
        dev.build_input_batch()
        random.setstate(state)
        host.build_input_batch()
        got = eng.gather_crops(dev.batch_crops, 32)
        want = [np.stack(b).astype(np.float32) for b in (host.batch_input, host.batch_input_bicubic, host.batch_true)]
        for g, w in zip(got, want):
            np.testing.assert_array_equal(g, w)
    eng.close()


@pytest.mark.parametrize("kw", [dict(), DS_KW], ids=["tensor_core", "depthwise_separable"])
def test_crop_step_equals_the_host_buffer_step(kw):
    """The rule of test_indexed_train_step_equals_the_host_buffer_step: losses equal, weights within 2e-6."""
    import dcscn_oracle as O
    cfg = dict(KW, **kw)
    scale, size = cfg["scale"], 64 // cfg["scale"]
    ds = dynamic_set("set14", scale, size)
    crops, _ = host_and_crops(ds, 8, seed=3, max_value=255.0)
    w = O.he_init_weights(O.OracleConfig(**cfg), seed=4)
    out = []
    for mode in ("host", "crops"):
        eng = engine(dropout_keep=0.8, **kw)
        eng.set_params(w)
        eng.set_image_store(ds.decoded_images())
        if mode == "host":
            x, x2, y = eng.gather_crops(crops, size)
            res = eng.train_step_host(x, x2, y, lr=1e-3, seed=5)
        else:
            res = eng.train_step_crops(crops, size, lr=1e-3, seed=5)
        names = [n for n in eng.param_shapes() if n.endswith("conv_W")][:3]
        out.append((res, {n: eng.get_param(n) for n in names}))
        eng.close()
    assert out[0][0] == out[1][0]
    for n in out[0][1]:
        np.testing.assert_allclose(out[0][1][n], out[1][1][n], rtol=0, atol=2e-6)


def test_bad_crops_are_refused_before_any_launch():
    from helper import engine as E
    ds = dynamic_set("set5", 2, 32)
    eng = engine()
    eng.set_image_store(ds.decoded_images())
    rows, cols = ds.sizes[0]
    eng.gather_crops([(0, rows - 64, cols - 64, 1)], 32)               # the last position that fits
    launches = eng.launch_count
    for bad in [(len(ds.sizes), 0, 0, 0), (-1, 0, 0, 0), (0, rows - 63, 0, 0), (0, 0, cols - 63, 0), (0, -1, 0, 0),
                (0, 0, 0, 2)]:
        with pytest.raises(E.EngineError):
            eng.gather_crops([(0, 0, 0, 0), bad], 32)
        with pytest.raises(E.EngineError):
            eng.train_step_crops([bad], 32, lr=1e-3, seed=1)
    assert eng.launch_count == launches
    eng.close()


def test_image_store_keeps_the_bicubic_tables_and_the_patch_store():
    import torch
    from helper import loader
    eng = engine()
    rs = np.random.RandomState(7)
    a = torch.from_numpy((rs.rand(2, 37, 53) * 255).astype(np.float32)).cuda()
    patches = loader.BatchDataSets(2, "unused", 24, stride_size=24)
    patches.build_batch(os.path.join(GOLDEN, "data", "set5"))
    eng.set_patch_store(patches.input_images, patches.input_interpolated_images, patches.true_images)
    idx = rs.randint(0, patches.count, size=9)
    before = (eng.bicubic_resize(a, 74, 106).cpu().numpy(), eng.gather_patches(idx))
    ds = dynamic_set("set14", 2, 32)
    eng.set_image_store(ds.decoded_images())
    crops, host = host_and_crops(ds, 6, seed=1, max_value=255.0)
    for got, want in zip(eng.gather_crops(crops, 32), host):
        np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(eng.bicubic_resize(a, 74, 106).cpu().numpy(), before[0])
    for got, want in zip(eng.gather_patches(idx), before[1]):
        np.testing.assert_array_equal(got, want)
    eng.close()


def test_200_steps_on_random_crops_raise_set5_psnr(tmp_path):
    """test_gpu_convergence.py's bars, trained on random crops of Set14 (--build_batch=false, the default)."""
    from helper import args as A
    import DCSCN
    random.seed(1234)
    np.random.seed(1234)
    f = A._Flags()
    for name, (kind, default, help_text) in A.FLAGS._defs.items():
        f._define(name, default, help_text, kind)
    f.parse(["prog", "--scale=2", "--layers=7", "--filters=32", "--min_filters=8", "--filters_decay_gamma=1.2",
             "--nin_filters=24", "--nin_filters2=8", "--reconstruct_layers=0", "--pixel_shuffler_filters=1",
             "--self_ensemble=1", "--batch_num=20", "--batch_image_size=32", "--build_batch=false",
             "--data_dir=" + os.path.join(GOLDEN, "data"), "--dataset=set14", "--batch_dir=" + str(tmp_path / "batch"),
             "--checkpoint_dir=" + str(tmp_path / "ckpt"), "--log_filename=" + str(tmp_path / "log.txt"),
             "--tf_log_dir=" + str(tmp_path / "tf_log"), "--graph_dir=" + str(tmp_path / "graphs"),
             "--output_dir=" + str(tmp_path / "out")])
    m = DCSCN.SuperResolution(f, model_name=f.model_name)
    m.load_dynamic_datasets(f.data_dir + "/" + f.dataset, f.batch_image_size)
    m.build_graph()
    m.build_optimizer()
    m.build_summary_saver()
    m.init_all_variables()
    m.init_train_step()
    m.init_epoch_index()
    assert m.batch_crops is not None                                  # images live in HBM, mini-batches are crop lists
    test_files = sorted(glob.glob(os.path.join(GOLDEN, "data", "set5", "*.png")))
    curve = [m.evaluate(test_files)[0]]
    losses = []
    for step in range(200):
        m.build_input_batch()
        m.train_batch()
        if (step + 1) % 50 == 0:
            curve.append(m.evaluate(test_files)[0])
            losses.append(m.training_loss_sum / m.training_step)
    print("Set5 PSNR at steps 0/50/100/150/200:", ["%.2f" % p for p in curve], "running mean loss:", ["%.1f" % v for v in losses])
    assert all(np.isfinite(curve))
    assert curve[-1] >= curve[0] + 8.0, curve
    assert curve[-1] >= 28.0, curve
    assert all(b >= a - 1.5 for a, b in zip(curve, curve[1:])), curve
    assert losses[-1] < losses[0]


def _worker(rank, world, port, out_dir, crops):
    sys.path.insert(0, PKG)
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import torch
    import torch.distributed as dist
    import dcscn_oracle as O
    from helper import engine as E
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    eng = E.Engine(E.make_config(device_id=rank, dropout_keep=1.0, **KW))
    eng.set_params(O.he_init_weights(O.OracleConfig(**KW), seed=11))
    eng.set_image_store(dynamic_set("set14", 2, 32).decoded_images())
    eng.train_step_data_parallel(None, None, None, lr=0.002, seed=7, crops=crops[rank::world], patch_size=32)
    np.save(os.path.join(out_dir, "w%d.npy" % rank), eng.get_param("CNN2/conv_W"))
    eng.close()
    dist.destroy_process_group()


def test_two_rank_crop_step_equals_the_whole_batch(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    import dcscn_oracle as O
    crops, _ = host_and_crops(dynamic_set("set14", 2, 32), 8, seed=2, max_value=255.0)
    mp.spawn(_worker, args=(2, 29500 + os.getpid() % 200, str(tmp_path), crops), nprocs=2, join=True)
    eng = engine(dropout_keep=1.0)
    eng.set_params(O.he_init_weights(O.OracleConfig(**KW), seed=11))
    eng.set_image_store(dynamic_set("set14", 2, 32).decoded_images())
    eng.train_step_crops(crops, 32, lr=0.002, seed=7)
    w0, w1 = np.load(tmp_path / "w0.npy"), np.load(tmp_path / "w1.npy")
    np.testing.assert_array_equal(w0, w1)
    assert np.abs(w0 - eng.get_param("CNN2/conv_W")).max() <= 0.05 * 0.002    # as test_gpu_multi.py
    eng.close()
