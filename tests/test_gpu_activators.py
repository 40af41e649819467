"""--activator on the GPU (helper/tf_graph.py:77-102): forward, gradients and optimizer state of every non-PReLU activator
on tensor-core and depthwise-separable graphs, against the fp64 oracle of tests/activator_oracle.py with the engine's
dropout masks replayed, at the bars of the PReLU tests (test_gpu_forward.py, test_gpu_train.py)."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import activator_oracle as A
import dcscn_oracle as O
from conftest import GOLDEN, PKG
from test_gpu_forward import SMALL, TOL, assert_stress, gpu_forward
from test_gpu_train import DS2, DS4, SMALL as TSMALL, SMALL4 as TSMALL4, launched_kernels

pytestmark = pytest.mark.gpu

ACTS = A.ACTIVATORS[1:]


def engine(kw, w, act, precision=0, keep=0.8):
    from helper import engine as E
    eng = E.Engine(E.make_config(precision=precision, dropout_keep=keep, activator=act, **kw))
    eng.set_params(w)
    return eng


def inputs(cfg, n, h, w, seed):
    g = np.random.RandomState(seed)
    s = cfg.scale
    x = (g.rand(n, h, w, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, s * h, s * w, 1) * 255).astype(np.float32)
    y = np.clip(x2 + g.randn(n, s * h, s * w, 1) * 10, 0, 255).astype(np.float32)
    return x, x2, y


def masks_of(eng, cfg, seed, n, h, w):
    return {scope: np.ascontiguousarray(eng.dropout_mask(scope, seed, n, h, w, cout).transpose(0, 3, 1, 2)).astype(np.float64)
            for scope, k, cin, cout, bias, _ in O.layer_table(cfg) if A.activated(scope)}


@pytest.mark.parametrize("scale", [2, 3, 4])
@pytest.mark.parametrize("act", ACTS)
def test_tensor_core_forward(act, scale):
    """f16x3: the output within the stress bars of the fp64 oracle, fused and unfused, and within 2e-3 of the CUDA-core
    cross-check; f16x1: within the PSNR-neutral bar of the PReLU graph.  Both reach the kernels a PReLU graph of the same
    shape reaches (the activator is a run-time field, not a kernel choice)."""
    kw = dict(SMALL, scale=scale)
    cfg = O.OracleConfig(**kw)
    w = A.he_init_weights(cfg, act, seed=0)
    x, x2, _ = inputs(cfg, 2, 9, 11, seed=scale)
    y64 = A.Oracle(cfg, {k: v.astype(np.float64) for k, v in w.items()}, act).forward(x.astype(np.float64), x2.astype(np.float64))
    y32 = A.Oracle(cfg, w, act, torch.float32).forward(x, x2)
    ours = lambda ns: sorted(n for n in ns if "dcscn::" in n)
    for precision in (0, 1):
        prelu = engine(kw, O.he_init_weights(cfg, seed=0), "prelu", precision)
        _, want = launched_kernels(lambda: gpu_forward(prelu, x, x2))
        prelu.close()
        eng = engine(kw, w, act, precision)
        y, names = launched_kernels(lambda: gpu_forward(eng, x, x2))
        assert ours(names) and ours(names) == ours(want), (ours(names), ours(want))
        if precision == 0:
            y_tc = assert_stress(eng, x, x2, y64, y32)
            eng.set_option("fuse_last", 0)
            assert float(np.abs(gpu_forward(eng, x, x2) - y64).max()) <= TOL
            eng.set_option("fuse_last", 1)
            eng.set_option("conv_impl", 1)
            y_ref = gpu_forward(eng, x, x2)
            assert np.abs(y_tc - y_ref).max() <= 2e-3
        else:
            assert np.abs(y - y64).max() < 1.0
        eng.close()


@pytest.mark.parametrize("kw", [DS2, DS4], ids=["ds-x2", "ds-x4"])
@pytest.mark.parametrize("act", ACTS)
def test_depthwise_separable_forward(act, kw):
    cfg = O.OracleConfig(**kw)
    w = A.he_init_weights(cfg, act, seed=4)
    x, x2, _ = inputs(cfg, 2, 13, 10, seed=3)
    y64, inter = A.Oracle(cfg, {k: v.astype(np.float64) for k, v in w.items()}, act).forward(
        x.astype(np.float64), x2.astype(np.float64), return_intermediates=True)
    eng = engine(kw, w, act)
    y = gpu_forward(eng, x, x2)
    assert float(np.abs(y - y64).max()) <= TOL
    for name, ref in inter.items():
        if name != "R-CNN":
            err = float(np.abs(eng.get_activation(name, ref.shape) - ref).max())
            assert err <= 2e-6 * max(1.0, np.abs(ref).max()) + 1e-4, (name, err)
    eng.close()


@pytest.mark.parametrize("act", ["relu", "selu"])
def test_tiled_forward_is_bit_identical(act):
    kw = dict(SMALL, scale=2)
    cfg = O.OracleConfig(**kw)
    eng = engine(kw, A.he_init_weights(cfg, act, seed=1), act)
    x, x2, _ = inputs(cfg, 1, 97, 131, seed=7)
    whole = eng.forward_host(x, x2)
    eng.set_option("workspace_mb", 2)
    tiled = eng.forward_host(x, x2)
    eng.set_option("workspace_mb", 0)
    assert np.array_equal(whole, tiled)
    eng.close()


def grad_case(kw, act, keep, shape, act_grad_impl=0, zero=False, ds=False):
    cfg = O.OracleConfig(**kw)
    w = {k: v.astype(np.float64) for k, v in A.he_init_weights(cfg, act, seed=0).items()}
    n, h, wd = shape
    x, x2, y = inputs(cfg, n, h, wd, seed=1)
    if zero:                   # zero image and zero biases (the reference's initialisation): every CNN1 z is exactly 0
        x[:] = 0
        for k in w:
            if k.endswith("conv_B"):
                w[k][:] = 0
    eng = engine(kw, {k: v.astype(np.float32) for k, v in w.items()}, act, keep=keep)
    eng.set_option("act_grad_impl", act_grad_impl)
    seed = 1234
    loss, mse = eng.train_step_host(x, x2, y, lr=0.002, seed=seed, apply_update=False)
    masks = masks_of(eng, cfg, seed, n, h, wd) if keep < 1.0 else None
    mse_ref, _, grads_ref = A.Oracle(cfg, w, act).loss_and_grads(x.astype(np.float64), x2.astype(np.float64),
                                                                 y.astype(np.float64), keep_prob=keep, masks=masks)
    assert sorted(grads_ref) == sorted(eng.param_shapes())
    bad = []
    if not mse == pytest.approx(mse_ref, rel=2e-5):
        bad.append(("mse", mse, mse_ref))
    bar = 2e-4 if ds else 2e-3
    for name, gref in grads_ref.items():
        err = float(np.abs(eng.get_grad(name) - gref).max())
        if not err <= bar * np.abs(gref).max() + 1e-7:
            bad.append((name, err, float(np.abs(gref).max())))
    eng.close()
    assert not bad, bad


@pytest.mark.parametrize("impl", [0, 1], ids=["act8", "pair"])
@pytest.mark.parametrize("kw,shape", [(TSMALL, (2, 12, 10)), (TSMALL4, (1, 9, 11))], ids=["x2", "x4"])
@pytest.mark.parametrize("act", ACTS)
def test_gradients_match_oracle(act, kw, shape, impl):
    """keep = 0.8: a derivative taken from the stored (post-dropout) output instead of h = output * keep fails."""
    grad_case(kw, act, 0.8, shape, act_grad_impl=impl)


@pytest.mark.parametrize("act", ACTS)
def test_gradients_at_zero_pre_activation(act):
    """With a zero image and zero biases every CNN1 pre-activation is exactly 0, so CNN1's bias gradient is the sum of
    f'(0) g: 0 for relu, 1 for leaky_relu, lambda for selu (TensorFlow's rules, not torch's)."""
    grad_case(TSMALL, act, 1.0, (2, 12, 10), zero=True)


@pytest.mark.parametrize("kw,shape", [(DS2, (2, 12, 10)), (DS4, (2, 8, 11))], ids=["ds-x2", "ds-x4"])
@pytest.mark.parametrize("act", ACTS)
def test_depthwise_separable_gradients_match_oracle(act, kw, shape):
    grad_case(kw, act, 0.8, shape, ds=True)


@pytest.mark.parametrize("act", ACTS)
def test_adam_steps_and_device_refresh(act):
    """Three Adam steps against the oracle's clip + TF-Adam, then the device-refreshed weights equal a fresh host
    packing of the same parameters (forward output and gradients)."""
    from helper import engine as E
    kw = TSMALL
    cfg = O.OracleConfig(**kw)
    wts = {k: v.astype(np.float64) for k, v in A.he_init_weights(cfg, act, seed=3).items()}
    n, h, w = 2, 12, 14
    x, x2, y = inputs(cfg, n, h, w, seed=4)
    eng = engine(kw, {k: v.astype(np.float32) for k, v in wts.items()}, act)
    orc = A.Oracle(cfg, dict(wts), act)
    m = {k: np.zeros_like(v) for k, v in wts.items()}
    v = {k: np.zeros_like(a) for k, a in wts.items()}
    slack = {k: np.zeros_like(a) for k, a in wts.items()}
    for step in range(1, 4):
        seed = 100 + step
        eng.train_step_host(x, x2, y, lr=0.002, seed=seed)
        _, _, grads = orc.loss_and_grads(x.astype(np.float64), x2.astype(np.float64), y.astype(np.float64), keep_prob=0.8,
                                         masks=masks_of(eng, cfg, seed, n, h, w))
        clipped, _ = orc.clip_by_global_norm(grads)
        orc.adam_step(clipped, m, v, step, 0.002)
        for name in wts:   # the tolerance of test_adam_step_matches_oracle_and_loss_decreases
            delta = 2e-3 * np.abs(grads[name]).max()
            slack[name] += np.minimum(2.0, 3.0 * delta / (np.abs(grads[name]) + 1e-300))
            tol = 2e-3 * 0.002 * step + 0.002 * slack[name]
            assert (np.abs(eng.get_param(name) - orc.w[name]) <= tol).all(), (step, name)
    y_dev = eng.forward_host(x, x2)
    eng.train_step_host(x, x2, y, lr=0.01, seed=99, apply_update=False)
    params = {k: eng.get_param(k) for k in wts}
    grads_dev = {k: eng.get_grad(k) for k in wts}
    fresh = E.Engine(E.make_config(dropout_keep=0.8, activator=act, **kw))
    fresh.set_params(params)
    assert np.abs(y_dev - fresh.forward_host(x, x2)).max() <= 1e-5
    fresh.train_step_host(x, x2, y, lr=0.01, seed=99, apply_update=False)
    for k in wts:
        g = fresh.get_grad(k)
        assert np.abs(g - grads_dev[k]).max() <= 1e-4 * np.abs(g).max() + 1e-9, k
    eng.close()
    fresh.close()


def _flags(argv):
    from helper import args
    f = args._Flags()
    for name, (kind, default, help_text) in args.FLAGS._defs.items():
        f._define(name, default, help_text, kind)
    f.parse(["prog"] + argv)
    return f


def _pngs(root):
    from PIL import Image
    out = {}
    for d, _, files in os.walk(root):
        for fn in files:
            if fn.endswith(".png"):
                out[os.path.relpath(os.path.join(d, fn), root)] = np.asarray(Image.open(os.path.join(d, fn)))
    return out


def test_train_and_evaluate_round_trip(tmp_path):
    """train.py --activator=leaky_relu writes a checkpoint with the reference's variable set and model name.
    evaluate.py --activator=leaky_relu loads it: its logged Set5 average PSNR (printed to 1e-6 dB) and every image it
    saves equal those of an in-process model that loads the same checkpoint.  The same checkpoint read as relu (the same
    variable set) gives another PSNR, so the comparison does see the activator."""
    import glob
    import DCSCN
    from helper import tf_bundle
    graph = ["--scale=2", "--layers=4", "--filters=16", "--min_filters=8", "--nin_filters=8", "--nin_filters2=4",
             "--self_ensemble=1", "--data_dir=" + os.path.join(GOLDEN, "data"), "--checkpoint_dir=" + str(tmp_path / "ckpt"),
             "--tf_log_dir=" + str(tmp_path / "tf_log"), "--graph_dir=" + str(tmp_path / "graphs"), "--test_dataset=set5"]
    leaky = graph + ["--activator=leaky_relu"]
    train = [sys.executable, os.path.join(PKG, "train.py"), "--dataset=set5", "--training_images=16", "--batch_num=8",
             "--batch_image_size=16", "--lr_decay_epoch=1", "--lr_decay=0.01", "--end_lr=1e-5",
             "--batch_dir=" + str(tmp_path / "batch"), "--log_filename=" + str(tmp_path / "train_log.txt"),
             "--output_dir=" + str(tmp_path / "train_out")] + leaky
    r = subprocess.run(train, cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    name = "dcscn_L4_F16to8_NIN_A8_PS_leaky_relu_R1F32"
    rd = tf_bundle.BundleReader(str(tmp_path / "ckpt" / (name + ".ckpt")))
    cfg = O.OracleConfig(layers=4, filters=16, min_filters=8, nin_filters=8, nin_filters2=4)
    trainables = {k for k in rd.keys() if not k.endswith(("/Adam", "/Adam_1")) and "_power" not in k}
    assert trainables == set(A.variable_names(cfg, "leaky_relu"))

    ev = [sys.executable, os.path.join(PKG, "evaluate.py"), "--save_results=true", "--output_dir=" + str(tmp_path / "eval_out"),
          "--log_filename=" + str(tmp_path / "eval_log.txt")] + leaky
    r = subprocess.run(ev, cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    logged = re.search(r"Model Average \[set5\] PSNR:([0-9.]+),", open(tmp_path / "eval_log.txt").read())
    assert logged, open(tmp_path / "eval_log.txt").read()

    files = sorted(glob.glob(os.path.join(GOLDEN, "data", "set5", "*.png")))

    def in_process(act, out):
        m = DCSCN.create(_flags(graph + ["--activator=" + act, "--output_dir=" + str(out),
                                         "--log_filename=" + str(tmp_path / ("inproc_%s.txt" % act))]))
        m.load_model(name)
        psnr = [m.do_for_evaluate_with_output(f, output_directory=str(out))[0] for f in files]
        m.engine.close()
        return "%f" % (sum(psnr) / len(psnr))

    assert in_process("leaky_relu", tmp_path / "inproc_out") == logged.group(1)
    got, want = _pngs(tmp_path / "eval_out"), _pngs(tmp_path / "inproc_out")
    assert sorted(got) == sorted(want) and len(got) >= len(files)
    assert all(np.array_equal(got[k], want[k]) for k in got), [k for k in got if not np.array_equal(got[k], want[k])]
    assert in_process("relu", tmp_path / "relu_out") != logged.group(1)


@pytest.mark.parametrize("act", ["relu", "tanh"])
def test_200_steps_on_real_patches_raise_set5_psnr(tmp_path, act):
    """test_gpu_convergence.py's run with another activator: c-DCSCN x2 from the 'he' initialisation, 200 steps on Set14
    grid patches through the device patch store, Set5 PSNR every 50 steps.  relu starts where PReLU does, at the
    random-weights level (~10 dB), and is held to the PReLU run's bars.  tanh's bounded outputs keep the He-init
    residual small, so its untrained model is already near bicubic (33.3 of bicubic's 33.66 dB on one H100); it must
    climb a further 1 dB, past bicubic, instead of 8."""
    import glob
    import random
    import DCSCN
    random.seed(1234)
    np.random.seed(1234)
    f = _flags(["--scale=2", "--layers=7", "--filters=32", "--min_filters=8", "--filters_decay_gamma=1.2",
                "--nin_filters=24", "--nin_filters2=8", "--reconstruct_layers=0", "--pixel_shuffler_filters=1",
                "--self_ensemble=1", "--batch_num=20", "--batch_image_size=32", "--build_batch=true", "--activator=" + act,
                "--data_dir=" + os.path.join(GOLDEN, "data"), "--dataset=set14", "--batch_dir=" + str(tmp_path / "batch"),
                "--checkpoint_dir=" + str(tmp_path / "ckpt"), "--log_filename=" + str(tmp_path / "log.txt"),
                "--tf_log_dir=" + str(tmp_path / "tf_log"), "--graph_dir=" + str(tmp_path / "graphs"),
                "--output_dir=" + str(tmp_path / "out")])
    m = DCSCN.SuperResolution(f, model_name=f.model_name)
    m.load_datasets(f.data_dir + "/" + f.dataset, f.batch_dir + "/" + f.dataset, f.batch_image_size, f.stride_size)
    m.build_graph()
    assert not any("/prelu/" in n for n in m.engine.param_shapes())
    m.build_optimizer()
    m.build_summary_saver()
    m.init_all_variables()
    m.init_train_step()
    m.init_epoch_index()
    test_files = sorted(glob.glob(os.path.join(GOLDEN, "data", "set5", "*.png")))
    curve = [m.evaluate(test_files)[0]]
    losses = []
    for step in range(200):
        m.build_input_batch()
        m.train_batch()
        if (step + 1) % 50 == 0:
            curve.append(m.evaluate(test_files)[0])
            losses.append(m.training_loss_sum / m.training_step)
    print(act, "Set5 PSNR at steps 0/50/100/150/200:", ["%.2f" % p for p in curve], "running mean loss:",
          ["%.1f" % v for v in losses])
    m.engine.close()
    assert all(np.isfinite(curve))
    assert curve[-1] >= curve[0] + (1.0 if act == "tanh" else 8.0), curve
    assert curve[-1] >= 28.0, curve
    assert all(b >= a - 1.5 for a, b in zip(curve, curve[1:])), curve
    assert losses[-1] < losses[0]
