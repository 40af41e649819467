"""Evaluation on the device: SuperResolution.do_for_evaluate / evaluate_bicubic / evaluate with the luma, the LR and
bicubic inputs, the forward or self-ensemble, the trim and the PSNR / SSIM map formed on the GPU (csrc/eval.cuh,
dcscn_evaluate_image).  Every result is held with == (nan matching nan) to the host path (_do_for_evaluate_host /
_evaluate_bicubic_host: numpy, scipy and Pillow) of the same model."""
import glob
import os
import re
import subprocess
import sys

import numpy as np
import pytest
from PIL import Image

from conftest import GOLDEN, PKG

pytestmark = pytest.mark.gpu

SET5 = sorted(glob.glob(os.path.join(GOLDEN, "data", "set5", "*.png")))
SET14 = sorted(glob.glob(os.path.join(GOLDEN, "data", "set14", "*.png")))
CD = ["--layers=7", "--filters=32", "--min_filters=8", "--filters_decay_gamma=1.2", "--nin_filters=24",
      "--nin_filters2=8", "--reconstruct_layers=0", "--pixel_shuffler_filters=1"]
MODELS = {"L12x2": ["--scale=2"], "L12x3": ["--scale=3"], "L12x4": ["--scale=4"], "c-DCSCNx2": ["--scale=2"] + CD,
          "DSx4": ["--scale=4", "--depthwise_separable=true"] + CD}


def build_model(tmp_path, flag_args, checkpoint=None):
    from helper import args as A
    import DCSCN
    f = A._Flags()
    for name, (kind, default, help_text) in A.FLAGS._defs.items():
        f._define(name, default, help_text, kind)
    f.parse(["prog", "--checkpoint_dir=" + os.path.join(GOLDEN, "models"), "--log_filename=" + str(tmp_path / "log.txt"),
             "--tf_log_dir=" + str(tmp_path / "tf_log"), "--graph_dir=" + str(tmp_path / "graphs"),
             "--output_dir=" + str(tmp_path / "out")] + flag_args)
    m = DCSCN.SuperResolution(f, model_name=f.model_name)
    m.build_graph()
    m.build_summary_saver()
    m.init_all_variables()
    m.load_model(checkpoint or f.load_model_name)
    return m


def same(a, b):
    return all((np.isnan(x) and np.isnan(y)) or x == y for x, y in zip(a, b))


def check_files(m, files, bicubic=False):
    for f in files:
        if bicubic:
            got, want = m.evaluate_bicubic(f), m._evaluate_bicubic_host(f)
        else:
            got, want = m.do_for_evaluate(f), m._do_for_evaluate_host(f)
        assert same(got, want), (f, m.self_ensemble, m.max_value, m.psnr_calc_border_size, got, want)


@pytest.mark.parametrize("model", ["L12x2", "L12x3", "L12x4", "c-DCSCNx2"])
def test_do_for_evaluate_equals_host_on_set5_and_set14(tmp_path, model):
    m = build_model(tmp_path, MODELS[model])
    assert m._device_evaluation()
    for ensemble in (8, 1):
        m.self_ensemble = ensemble
        check_files(m, SET5 + SET14)      # Set14 img_003 is mode 'L'


@pytest.mark.parametrize("ensemble", [1, 8])
def test_max_value_one(tmp_path, ensemble):
    m = build_model(tmp_path, MODELS["c-DCSCNx2"] + ["--max_value=1.0", "--self_ensemble=%d" % ensemble],
                    checkpoint="dcscn_L7_F32to8_G1.20_NIN_A24_B8_PS_R1F32")   # the x2 weights, run at max_value 1
    assert m.max_value == 1.0
    check_files(m, SET5 + SET14[:3])


def test_borders(tmp_path):
    m = build_model(tmp_path, MODELS["c-DCSCNx2"] + ["--self_ensemble=1"])
    for border in (0, 2, 7):
        m.psnr_calc_border_size = border
        check_files(m, SET5[:2] + SET14[2:3])
    # a border that leaves fewer than 11 rows (SSIM nan) of a wide image, and one that leaves nothing (both nan)
    f = [f for f in SET14 if Image.open(f).height < Image.open(f).width][0]
    ah = Image.open(f).height // 2 * 2
    m.psnr_calc_border_size = (ah - 9) // 2
    got = m.do_for_evaluate(f)
    assert np.isnan(got[1]) and np.isfinite(got[0]) and same(got, m._do_for_evaluate_host(f))
    m.psnr_calc_border_size = ah
    with np.errstate(all="ignore"):
        got, want = m.do_for_evaluate(f), m._do_for_evaluate_host(f)
    assert np.isnan(got[0]) and np.isnan(got[1]) and same(got, want)


def test_synthetic_images(tmp_path):
    g = np.random.RandomState(5)
    files = []
    for name, mode, shape in (("rgb", "RGB", (67, 53, 3)), ("rgba", "RGBA", (45, 38, 4)), ("gray", "L", (33, 29)),
                              ("short", "RGB", (13, 41, 3))):
        path = str(tmp_path / (name + ".png"))
        Image.fromarray(g.randint(0, 256, shape).astype(np.uint8), mode).save(path)
        files.append(path)
    pal = str(tmp_path / "palette.png")
    Image.fromarray(g.randint(0, 256, (51, 43, 3)).astype(np.uint8), "RGB").quantize(64).save(pal)
    assert Image.open(pal).mode == "P"
    files.append(pal)
    for model in ("c-DCSCNx2", "L12x3"):
        m = build_model(tmp_path, MODELS[model])
        for ensemble in (1, 8):
            m.self_ensemble = ensemble
            check_files(m, files)
        check_files(m, files, bicubic=True)


def test_evaluate_bicubic_on_set14(tmp_path):
    for model in ("L12x2", "L12x3", "L12x4"):
        check_files(build_model(tmp_path, MODELS[model]), SET14, bicubic=True)


@pytest.mark.parametrize("flags", [["--precision=f16x1"], ["--workspace_mb=32"]], ids=["f16x1", "tiled"])
def test_other_engines(tmp_path, flags):
    from helper import engine as E
    m = build_model(tmp_path, MODELS["L12x2"] + flags)
    for ensemble in (1, 8):
        m.self_ensemble = ensemble
        check_files(m, SET5 + SET14[:4])
    if "tiled" in flags[0] or "workspace" in flags[0]:
        m.do_for_evaluate(SET5[0])
        with pytest.raises(E.EngineError, match="tiled"):      # the forward ran as windows
            m.engine.get_activation("CNN1", (8, 128, 128, 196))


def test_depthwise_separable_checkpoint(tmp_path):
    m = build_model(tmp_path, MODELS["DSx4"])
    for ensemble in (1, 8):
        m.self_ensemble = ensemble
        check_files(m, SET5 + SET14)


def test_evaluate_around_a_train_step(tmp_path):
    from helper import loader
    m = build_model(tmp_path, MODELS["c-DCSCNx2"] + ["--self_ensemble=2"])
    m.build_optimizer()
    ds = loader.DynamicDataSets(2, 24)
    ds.set_data_dir(os.path.join(GOLDEN, "data", "set14"))
    m.engine.set_image_store(ds.decoded_images())
    crops = [(i % len(ds.sizes), 3, 5, i & 1) for i in range(8)]
    before = m.engine.gather_crops(crops, 24)
    uploads = []
    real = m.engine.set_eval_images
    m.engine.set_eval_images = lambda images: uploads.append(len(images)) or real(images)
    files = SET5 + SET14[:3]

    def host_average():      # accumulated as evaluate() does (Python's sum() compensates float rounding)
        total_psnr = total_ssim = 0
        for f in files:
            psnr, ssim = m._do_for_evaluate_host(f)
            total_psnr += psnr
            total_ssim += ssim
        return total_psnr / len(files), total_ssim / len(files)

    first = m.evaluate(files)
    assert first == host_average() and uploads == [len(files)]
    m.engine.train_step_crops(crops, 24, lr=1e-3, seed=1)
    second = m.evaluate(files)
    assert second != first and second == host_average() and uploads == [len(files)]
    for a, b in zip(before, m.engine.gather_crops(crops, 24)):
        np.testing.assert_array_equal(a, b)


def test_device_kernels_run_and_host_metric_does_not(tmp_path, monkeypatch):
    from test_gpu_train import assert_kernels_ran, launched_kernels
    from helper import utilty as util
    m = build_model(tmp_path, MODELS["c-DCSCNx2"] + ["--self_ensemble=8"])
    want = m._do_for_evaluate_host(SET14[2])

    def refuse(*a, **k):
        raise AssertionError("the host SSIM ran on the device path")
    monkeypatch.setattr(util, "_ssim_columns", refuse)
    # In a process that has already run many tests, a trace was seen to miss the first launches after the profiler
    # started, or to hold no kernel at all (the whole GPU suite in one pytest run; test_gpu_train's helper names the
    # second case).  So the image is evaluated twice inside the session, the second call's launches well inside it,
    # and a session that recorded no engine kernel at all, which says nothing about which kernels ran, is repeated
    # up to twice.
    for _ in range(3):
        got, names = launched_kernels(lambda: [m.do_for_evaluate(SET14[2]) for _ in range(2)])
        assert same(got[0], want) and same(got[1], want)
        if any("dcscn::" in n for n in names):
            break
    assert_kernels_ran(names, ["eval_prepare_kernel", "eval_place_kernel", "eval_trim_kernel", "eval_sse_kernel",
                               "eval_ssim_kernel", "pil_resample8_h_kernel", "ensemble_reduce_kernel"])
    m.engine.set_option("timing", 1)
    m.do_for_evaluate(SET5[0])
    steps = [n for n, _ in m.engine.timings()]
    assert steps == ["eval_prepare", "eval_resize", "eval_place", "ensemble", "eval_trim", "eval_sse", "eval_ssim"], steps
    assert all(ms >= 0 for _, ms in m.engine.timings())


def test_evaluate_cli_matches_host_path(tmp_path):
    flags = ["--save_results=false", "--test_dataset=set5", "--data_dir=" + os.path.join(GOLDEN, "data"),
             "--checkpoint_dir=" + os.path.join(GOLDEN, "models"), "--log_filename=" + str(tmp_path / "log.txt"),
             "--tf_log_dir=" + str(tmp_path / "tf_log"), "--graph_dir=" + str(tmp_path / "graphs"),
             "--output_dir=" + str(tmp_path / "out"), "--self_ensemble=8"] + MODELS["c-DCSCNx2"]
    code = "\n".join([
        "import sys",
        "sys.path.insert(0, %r)" % PKG,
        "sys.argv = ['evaluate.py'] + %r" % flags,
        "import evaluate",
        "from helper import utilty as util",
        "made = []",
        "build = evaluate.build_model",
        "evaluate.build_model = lambda: made.append(build()) or made[0]",
        "evaluate.main(['evaluate.py'])",
        "m = made[0]",
        "assert m._device_evaluation()",
        "files = util.get_files_in_directory(evaluate.FLAGS.data_dir + '/set5')",
        "tp = ts = 0",
        "for f in files:",
        "    p, s = m._do_for_evaluate_host(f)",
        "    tp += p",
        "    ts += s",
        "print('HOST PSNR:%f, SSIM:%f' % (tp / len(files), ts / len(files)))",
    ])
    r = subprocess.run([sys.executable, "-c", code], cwd=str(tmp_path), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    logged = re.findall(r"Model Average \[set5\] PSNR:([0-9.]+), SSIM:([0-9.]+)", open(tmp_path / "log.txt").read())
    host = re.findall(r"HOST PSNR:([0-9.]+), SSIM:([0-9.]+)", r.stdout)
    assert logged and host and logged[-1] == host[-1], (logged, host)
