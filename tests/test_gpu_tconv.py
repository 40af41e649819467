"""
--pixel_shuffler=false on the H100 (run with `-m gpu`): the upsampler is Up-TCNN, one stride-s conv2d_transpose,
which the engine runs as a 3x3 LR conv_tc_kernel layer into s*s*C columns with a gathered filter F (engine.cu
tconv_filter_map), the existing depth_to_space epilogues and, where get_plan's rule allows, the fused R-CNN1.  Its
train step differentiates F with wgrad_tc_kernel and gathers the Tconv_W gradient back (tconv_grad_gather_kernel).

  * forward parity against the fp64 oracle (tconv_oracle.py) with the stress bars of test_gpu_forward.py, fused and
    unfused, at the default and strict promotion periods, x2 / x3 / x4 and the full L12 width;
  * the Up-TCNN layer alone, recomputed in fp64 from the input planes the GPU stored, at the isolated f16x3 / f16x1
    bars of test_gpu_forward_paths.py, and a profiler check of the kernels it reached;
  * a --depthwise_separable graph (Up-TCNN stays dense);
  * tiled forwards, the self-ensemble and CUDA-graph replays bit-identical to the plain forward;
  * every gradient against fp64 autograd with the engine's dropout masks, optimizer steps, a checkpoint round trip,
    200 steps of real patches and the train.py / evaluate.py command lines.
"""
import glob
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import dcscn_oracle as O
import tconv_oracle as T
from conftest import GOLDEN, PKG
from test_gpu_forward import assert_stress, gpu_forward, make_engine, stress_bound
from test_gpu_forward_paths import U23, conv, nchw, pad16, quantise, tc_units
from test_gpu_train import assert_kernels_ran, launched_kernels, oracle_masks

pytestmark = pytest.mark.gpu

TC = dict(transposed_upsampler=True)
SMALL = dict(layers=4, filters=40, min_filters=24, filters_decay_gamma=1.5, nin_filters=32, nin_filters2=16, **TC)
CASES = [
    # id, config, (n, h, w), fused R-CNN1 expected
    ("x2", dict(SMALL, scale=2), (1, 12, 14), True),
    ("x3", dict(SMALL, scale=3), (1, 9, 11), True),
    ("x4", dict(SMALL, scale=4), (1, 9, 11), True),                                   # one stage: 16 C columns
    ("x3-c40", dict(SMALL, scale=3, nin_filters=24), (2, 7, 9), False),               # C = 40: R-CNN1 unfused
    ("L12-x2", dict(scale=2, **TC), (1, 10, 12), True),
    ("L12-x4", dict(scale=4, **TC), (1, 8, 10), True),                                 # 1536 columns
]
# the kernels an Up-TCNN forward may launch: the existing inference kernels, nothing new
FORWARD_KERNELS = ("conv_first3x3_kernel", "conv_first_kernel", "conv_tc_kernel", "conv_last_gather_kernel",
                   "conv_last_gather4_kernel", "conv_last_kernel", "conv_last_direct_kernel")


def oracle_cfg(kw):
    return T.Config(**kw)


def inputs(s, n, h, w, seed=3):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(n, h, w, 1, generator=g) * 255).numpy()
    x2 = (torch.rand(n, s * h, s * w, 1, generator=g) * 255).numpy()
    return x, x2


@pytest.mark.parametrize("kw,shape,fused", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_forward_matches_oracle(kw, shape, fused):
    cfg = oracle_cfg(kw)
    s = cfg.scale
    w = T.random_weights(cfg, seed=0)
    x, x2 = inputs(s, *shape)
    y64, inter = T.Oracle(cfg, w, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64),
                                                          return_intermediates=True)
    y32 = T.Oracle(cfg, w, torch.float32).forward(x, x2)
    eng = make_engine(kw, w)
    _, names = launched_kernels(lambda: gpu_forward(eng, x, x2))
    ours = sorted(n for n in names if "dcscn::" in n)
    assert_kernels_ran(names, ["conv_tc_kernel"])
    assert any("dcscn::conv_last_gather" in n for n in ours) == fused, ours     # the fused R-CNN1's second half
    assert all(any("dcscn::%s" % k in n for k in FORWARD_KERNELS) for n in ours), ours
    assert_stress(eng, x, x2, y64, y32)
    eng.set_option("fuse_last", 0)
    y = gpu_forward(eng, x, x2)
    assert float(np.abs(y - y64).max()) <= max(1.5e-3, stress_bound(y32, y64))
    bad = []
    for name, ref in inter.items():   # the unfused forward materialises every layer, Up-TCNN included
        if name == "R-CNN":
            continue
        err = float(np.abs(eng.get_activation(name, ref.shape) - ref).max())
        if not err <= 4e-6 * max(1.0, np.abs(ref).max()) + 1e-4:
            bad.append((name, err, float(np.abs(ref).max())))
    eng.close()
    assert not bad, bad


@pytest.mark.parametrize("precision", [0, 1], ids=["f16x3", "f16x1"])
@pytest.mark.parametrize("case", ["x2", "x3", "L12-x4"])
def test_up_tcnn_layer_isolated(case, precision):
    """Up-TCNN from the [B2 | A1] planes the GPU stored, in fp64 with F quantised as pack_tc_layer does: the
    tensor-core accumulation bar of a 3x3 layer over the [B2 | A1] pitch plus the epilogue's rounding; the fp32 output
    (EPI_D2S_F32, fuse_last = 0) has no store rounding."""
    kw, shape, _ = {c[0]: c[1:] for c in CASES}[case]
    npl = 2 if precision == 0 else 1
    cfg = oracle_cfg(kw)
    s = cfg.scale
    w = T.random_weights(cfg, seed=0)
    x, x2 = inputs(s, *shape)
    n, h, wd = shape
    c = cfg.nin_filters + cfg.nin_filters2
    pitch = pad16(cfg.nin_filters2) + pad16(cfg.nin_filters)
    eng = make_engine(kw, w, precision)
    eng.set_option("fuse_last", 0)
    (fq,) = quantise([T.tconv_filter(w[T.TCONV], s)], npl)
    worst = 0.0
    for seg in (0, 1):
        eng.set_option("seg_chunks", seg)
        gpu_forward(eng, x, x2)
        a = torch.cat([nchw(eng.get_activation("B2", (n, h, wd, cfg.nin_filters2))),
                       nchw(eng.get_activation("A1", (n, h, wd, cfg.nin_filters)))], dim=1)
        z = O.depth_to_space(conv(a, fq), s)
        sabs = O.depth_to_space(conv(a.abs(), np.abs(fq)), s)
        bar = (tc_units(3, pitch, seg, npl) * U23 * sabs + U23 * sabs).numpy()
        got = nchw(eng.get_activation("Up-TCNN", (n, s * h, s * wd, c))).numpy()
        worst = max(worst, float((np.abs(got - z.numpy()) / (bar + 1e-30)).max()))
    eng.close()
    print("Up-TCNN error / bar: %.3f" % worst)
    assert worst <= 1.0


def test_depthwise_separable_graph_matches_oracle():
    kw = dict(SMALL, scale=2, depthwise_separable=True)
    cfg = oracle_cfg(kw)
    w = T.random_weights(cfg, seed=1)
    x, x2 = inputs(2, 1, 10, 12)
    y64 = T.Oracle(cfg, w, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64))
    y32 = T.Oracle(cfg, w, torch.float32).forward(x, x2)
    eng = make_engine(kw, w)
    _, names = launched_kernels(lambda: gpu_forward(eng, x, x2))
    assert_kernels_ran(names, ["depthwise_planes_kernel", "conv_tc_kernel"])
    assert not [nm for nm in names if "dcscn::ds_" in nm]
    assert "Up-TCNN/depthwise_W" not in eng.param_shapes()
    assert_stress(eng, x, x2, y64, y32)
    eng.close()


@pytest.mark.parametrize("case", ["x3", "L12-x4"])
def test_tiled_ensemble_and_graph_replay_are_bit_identical(case):
    kw, _, _ = {c[0]: c[1:] for c in CASES}[case]
    cfg = oracle_cfg(kw)
    s = cfg.scale
    w = T.random_weights(cfg, seed=2)
    x, x2 = inputs(s, 2, 45, 61, seed=5)
    eng = make_engine(kw, w)
    eng.set_option("graph", 0)
    la = eng.launch_count
    y_whole = gpu_forward(eng, x, x2)
    per_forward = eng.launch_count - la
    px_bytes = eng.device_bytes / float(2 * 45 * 61)
    e_whole = eng.forward_ensemble_host(x[0], x2[0], 8)
    eng.set_option("graph", 1)
    xs, x2s = torch.from_numpy(x).cuda(), torch.from_numpy(x2).cuda()
    r0, l0 = eng.graph_replays, eng.launch_count
    ys = [eng.forward(xs, x2s).cpu().numpy() for _ in range(4)]
    assert eng.graph_replays - r0 >= 2
    assert eng.launch_count - l0 == 4 * per_forward
    for y in ys:
        assert np.array_equal(y, y_whole)
    assert eng.tile_halo() == cfg.layers + 1 + 1
    eng.set_option("workspace_mb", -(-int(px_bytes * 3000) >> 20))
    eng.set_option("timing", 1)
    y_tiled = gpu_forward(eng, x, x2)
    assert sum(nm == "tile_stitch" for nm, _ in eng.timings()) >= 2
    eng.set_option("timing", 0)
    e_tiled = eng.forward_ensemble_host(x[0], x2[0], 8)
    eng.close()
    assert np.array_equal(y_tiled, y_whole)
    assert np.array_equal(e_tiled, e_whole)
    y64 = T.Oracle(cfg, w, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64))
    assert float(np.abs(y_whole - y64).max()) <= 2e-3


TRAIN = dict(layers=3, filters=24, min_filters=16, filters_decay_gamma=1.5, nin_filters=16, nin_filters2=16, **TC)


def setup(kw, keep, n, h, w, seed=0, optimizer="adam"):
    from helper import engine as E
    cfg = oracle_cfg(kw)
    wts = {k: v.astype(np.float64) for k, v in T.random_weights(cfg, seed=seed).items()}
    eng = E.Engine(E.make_config(dropout_keep=keep, optimizer=optimizer, **kw))
    eng.set_params({k: v.astype(np.float32) for k, v in wts.items()})
    g = np.random.RandomState(seed + 1)
    s = cfg.scale
    x = (g.rand(n, h, w, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, s * h, s * w, 1) * 255).astype(np.float32)
    y = np.clip(x2 + g.randn(n, s * h, s * w, 1) * 10, 0, 255).astype(np.float32)
    return cfg, wts, eng, x, x2, y


@pytest.mark.parametrize("kw,shape", [(dict(TRAIN, scale=2), (2, 9, 8)), (dict(TRAIN, scale=3), (2, 8, 7)),
                                      (dict(TRAIN, scale=4), (1, 7, 9)),
                                      (dict(TRAIN, scale=2, depthwise_separable=True), (2, 9, 8))],
                         ids=["x2", "x3", "x4", "ds-x2"])
def test_gradients_match_oracle(kw, shape):
    """Loss and every gradient, Tconv_W included, within 2e-3 of the tensor's max against fp64 autograd."""
    n, h, w = shape
    cfg, wts, eng, x, x2, y = setup(kw, 0.8, n, h, w, seed=5)
    seed = 4321
    (loss, mse), names = launched_kernels(lambda: eng.train_step_host(x, x2, y, lr=0.002, seed=seed, apply_update=False))
    assert_kernels_ran(names, ["wgrad_tc_kernel", "tconv_grad_gather_kernel"])
    masks = oracle_masks(eng, cfg, seed, n, h, w)
    mse_ref, _, grads_ref = T.Oracle(cfg, wts, torch.float64).loss_and_grads(
        x.astype(np.float64), x2.astype(np.float64), y.astype(np.float64), keep_prob=0.8, masks=masks)
    bad = []
    if not mse == pytest.approx(mse_ref, rel=5e-5):
        bad.append(("mse", mse, mse_ref))
    assert T.TCONV in grads_ref
    for name, gref in grads_ref.items():
        err = float(np.abs(eng.get_grad(name) - gref).max())
        if not err <= 2e-3 * np.abs(gref).max() + 1e-7:
            bad.append((name, err, float(np.abs(gref).max())))
    eng.close()
    assert not bad, bad


@pytest.mark.parametrize("optimizer", ["adam", "gd"])
def test_optimizer_steps_follow_oracle(optimizer):
    kw = dict(TRAIN, scale=4)
    n, h, w = 2, 10, 10
    cfg, wts, eng, x, x2, y = setup(kw, 0.8, n, h, w, seed=9, optimizer=optimizer)
    orc = T.Oracle(cfg, wts, torch.float64)
    m = {k: np.zeros_like(v) for k, v in wts.items()}
    v = {k: np.zeros_like(v_) for k, v_ in wts.items()}
    slack = {k: np.zeros_like(v_) for k, v_ in wts.items()}
    lr = 0.002
    for step in range(1, 4):
        seed = 300 + step
        eng.train_step_host(x, x2, y, lr=lr, seed=seed)
        masks = oracle_masks(eng, cfg, seed, n, h, w)
        _, _, grads = orc.loss_and_grads(x.astype(np.float64), x2.astype(np.float64), y.astype(np.float64), keep_prob=0.8,
                                         masks=masks)
        clipped, _ = orc.clip_by_global_norm(grads)
        if optimizer == "adam":
            orc.adam_step(clipped, m, v, step, lr)
        else:
            for name in orc.w:
                orc.w[name] = orc.w[name] - lr * clipped[name]
        for name in wts:
            delta = 2e-3 * np.abs(grads[name]).max()
            slack[name] += np.minimum(2.0, 3.0 * delta / (np.abs(grads[name]) + 1e-300)) if optimizer == "adam" else delta
            tol = 2e-3 * lr * step + lr * slack[name]
            got = eng.get_param(name)
            assert (np.abs(got - orc.w[name]) <= tol).all(), (step, name, float((np.abs(got - orc.w[name]) - tol).max()))
    assert not np.array_equal(eng.get_param(T.TCONV), wts[T.TCONV].astype(np.float32))
    yy = eng.forward_host(x, x2)
    eng.close()
    ref = T.Oracle(cfg, {k: a.astype(np.float64) for k, a in orc.w.items()}, torch.float64).forward(
        x.astype(np.float64), x2.astype(np.float64))
    assert np.abs(yy - ref).max() <= 5e-3


def _model(tmp_path, extra):
    from helper import args as A
    import DCSCN
    f = A._Flags()
    for name, (kind, default, help_text) in A.FLAGS._defs.items():
        f._define(name, default, help_text, kind)
    f.parse(["prog", "--scale=2", "--layers=7", "--filters=32", "--min_filters=8", "--filters_decay_gamma=1.2",
             "--nin_filters=32", "--nin_filters2=16", "--reconstruct_layers=0", "--pixel_shuffler=false",
             "--self_ensemble=1", "--batch_num=20", "--batch_image_size=32", "--build_batch=true",
             "--data_dir=" + os.path.join(GOLDEN, "data"), "--dataset=set14", "--batch_dir=" + str(tmp_path / "batch"),
             "--checkpoint_dir=" + str(tmp_path / "ckpt"), "--log_filename=" + str(tmp_path / "log.txt"),
             "--tf_log_dir=" + str(tmp_path / "tf_log"), "--graph_dir=" + str(tmp_path / "graphs"),
             "--output_dir=" + str(tmp_path / "out")] + extra)
    return f, DCSCN.SuperResolution(f, model_name=f.model_name)


def test_checkpoint_round_trips_tconv_and_its_slots(tmp_path):
    from helper import tf_bundle
    f, m = _model(tmp_path, [])
    m.build_graph()
    m.build_optimizer()
    m.build_summary_saver()
    m.init_all_variables()
    g = np.random.RandomState(0)
    x = (g.rand(4, 16, 16, 1) * 255).astype(np.float32)
    x2 = (g.rand(4, 32, 32, 1) * 255).astype(np.float32)
    for step in range(2):
        m.engine.train_step_host(x, x2, x2 + np.float32(1.0), lr=1e-3, seed=step)
    m.save_model()
    w = m.engine.get_param(T.TCONV)
    slots = [m.engine.get_optimizer_slot(T.TCONV, i) for i in range(2)]
    files = [fn for fn in glob.glob(str(tmp_path / "ckpt" / "*.ckpt.index"))]
    assert files and "_PS_" not in os.path.basename(files[0])
    rd = tf_bundle.BundleReader(files[0][:-len(".index")])
    assert {T.TCONV, T.TCONV + "/Adam", T.TCONV + "/Adam_1"} <= set(rd.keys())
    np.testing.assert_array_equal(rd.get_tensor(T.TCONV), w)
    _, m2 = _model(tmp_path, [])
    m2.build_graph()
    m2.build_optimizer()
    m2.build_summary_saver()
    m2.init_all_variables()
    m2.load_model(restore_optimizer=True)
    np.testing.assert_array_equal(m2.engine.get_param(T.TCONV), w)
    for i in range(2):
        np.testing.assert_array_equal(m2.engine.get_optimizer_slot(T.TCONV, i), slots[i])


def test_200_steps_raise_set5_psnr(tmp_path):
    """200 steps of real Set14 patches from the bilinear-initialised upsampler and He-initialised layers."""
    import random
    random.seed(1234)
    np.random.seed(1234)
    f, m = _model(tmp_path, [])
    m.load_datasets(f.data_dir + "/" + f.dataset, f.batch_dir + "/" + f.dataset, f.batch_image_size, f.stride_size)
    m.build_graph()
    m.build_optimizer()
    m.build_summary_saver()
    m.init_all_variables()
    m.init_train_step()
    m.init_epoch_index()
    test_files = sorted(glob.glob(os.path.join(GOLDEN, "data", "set5", "*.png")))
    curve = [m.evaluate(test_files)[0]]
    for step in range(200):
        m.build_input_batch()
        m.train_batch()
    curve.append(m.evaluate(test_files)[0])
    print("Set5 PSNR before / after 200 steps:", curve)
    assert np.isfinite(curve).all()
    assert curve[-1] >= curve[0] + 3.0 and curve[-1] >= 28.0, curve


def test_train_and_evaluate_cli(tmp_path):
    """train.py --pixel_shuffler=false trains a few steps and saves; evaluate.py with the same flags loads it."""
    from helper import tf_bundle
    ckpt = tmp_path / "ckpt"
    common = ["--scale=3", "--layers=4", "--filters=32", "--min_filters=16", "--pixel_shuffler=false",
              "--self_ensemble=1", "--test_dataset=set5", "--data_dir=" + os.path.join(GOLDEN, "data"),
              "--checkpoint_dir=" + str(ckpt), "--log_filename=" + str(tmp_path / "log.txt"),
              "--tf_log_dir=" + str(tmp_path / "tf_log"), "--graph_dir=" + str(tmp_path / "graphs"),
              "--output_dir=" + str(tmp_path / "out")]
    train = [sys.executable, os.path.join(PKG, "train.py"), "--dataset=set5", "--training_images=16", "--batch_num=8",
             "--batch_image_size=16", "--lr_decay_epoch=1", "--lr_decay=0.01", "--end_lr=1e-5",
             "--batch_dir=" + str(tmp_path / "batch")] + common
    r = subprocess.run(train, cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    index = glob.glob(str(ckpt / "*.ckpt.index"))
    assert index and "_PS" not in os.path.basename(index[0]), os.listdir(str(ckpt))
    rd = tf_bundle.BundleReader(index[0][:-len(".index")])
    assert T.TCONV in rd.keys() and np.isfinite(rd.get_tensor(T.TCONV)).all()
    ev = [sys.executable, os.path.join(PKG, "evaluate.py"), "--save_results=false"] + common
    r = subprocess.run(ev, cwd=str(tmp_path), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    log = open(tmp_path / "log.txt").read()
    found = re.findall(r"Model Average \[set5\] PSNR:([0-9.]+)", log)
    assert found and all(np.isfinite(float(v)) for v in found), log
