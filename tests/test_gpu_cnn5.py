"""
GPU parity of graphs with 5x5 filters (cnn_size = 5) on the tensor-core path.  A k x k layer reads its k ky taps at row
offsets of TW pixels inside one activation box, so the patch width decides whether the operand descriptors are valid;
the image shapes below make the planner pick 16 x 8, 8 x 16 and 4 x 32 patches.  Bars as in test_gpu_forward.py: the
default promotion periods within max(1.5e-3, 1.5 x the fp32 CPU oracle's error) of the fp64 oracle, the strict setting
within max(1e-3, 1.5 x that error), and the CUDA-core cross-check (conv_impl = 1) within 2e-3.
"""
import numpy as np
import pytest
import torch

import dcscn_oracle as O

pytestmark = pytest.mark.gpu

CNN5 = dict(scale=2, layers=4, filters=40, min_filters=24, filters_decay_gamma=1.5, nin_filters=24, nin_filters2=16,
            cnn_size=5)


@pytest.fixture(scope="module")
def cnn5():
    from helper import engine as E
    cfg = O.OracleConfig(**CNN5)
    w = O.he_init_weights(cfg, seed=3)
    eng = E.Engine(E.make_config(**CNN5))
    eng.set_params(w)
    yield cfg, w, eng
    eng.close()


def run(eng, x, x2):
    y = eng.forward(torch.from_numpy(x).cuda(), torch.from_numpy(x2).cuda())
    torch.cuda.synchronize()
    return y.cpu().numpy()


@pytest.mark.parametrize("n,h,w", [(1, 64, 100), (2, 48, 48), (1, 3, 130)], ids=["tw8", "tw16", "tw32"])
def test_5x5_graph_matches_oracle(cnn5, n, h, w):
    cfg, wts, eng = cnn5
    g = np.random.RandomState(n * 1000 + h * 10 + w)
    x = (g.rand(n, h, w, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, 2 * h, 2 * w, 1) * 255).astype(np.float32)
    y64 = O.Oracle(cfg, wts, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64))
    y32 = O.Oracle(cfg, wts, torch.float32).forward(x, x2)
    err32 = float(np.abs(y32 - y64).max())
    y = run(eng, x, x2)
    assert np.isfinite(y).all()
    err = float(np.abs(y - y64).max())
    assert err <= max(1.5e-3, 1.5 * err32), ("default", err, err32)
    eng.set_option("seg_chunks", 1)
    ys = run(eng, x, x2)
    eng.set_option("seg_chunks", 0)
    err_s = float(np.abs(ys - y64).max())
    assert err_s <= max(1e-3, 1.5 * err32), ("strict", err_s, err32)
    eng.set_option("conv_impl", 1)
    y_ref = run(eng, x, x2)
    eng.set_option("conv_impl", 0)
    assert np.abs(y - y_ref).max() <= 2e-3
