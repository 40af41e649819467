"""GPU parity of the train step (loss, every gradient, global-norm clip, TF-Adam) against the fp64 CPU oracle
(torch autograd of the restated graph, oracle/dcscn_oracle.py).  The oracle replays the engine's dropout masks
(dcscn_dropout_mask), so the comparison is exact up to fp32-level rounding.  Tolerance: 2e-3 of each gradient
tensor's max magnitude (data gradients run on the fp16x3 tensor-core path, filter gradients are fp32 atomics)."""
import numpy as np
import pytest
import torch

import dcscn_oracle as O

pytestmark = pytest.mark.gpu

SMALL = dict(scale=2, layers=3, filters=24, min_filters=16, filters_decay_gamma=1.5, nin_filters=16, nin_filters2=16)
SMALL4 = dict(scale=4, layers=3, filters=20, min_filters=16, filters_decay_gamma=1.5, nin_filters=16, nin_filters2=16)


def setup(kw, keep, n, h, w, seed=0):
    from helper import engine as E
    cfg = O.OracleConfig(**kw)
    wts = {k: v.astype(np.float64) for k, v in O.he_init_weights(cfg, seed=seed).items()}
    eng = E.Engine(E.make_config(dropout_keep=keep, **kw))
    eng.set_params({k: v.astype(np.float32) for k, v in wts.items()})
    g = np.random.RandomState(seed + 1)
    s = cfg.scale
    x = (g.rand(n, h, w, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, s * h, s * w, 1) * 255).astype(np.float32)
    y = np.clip(x2 + g.randn(n, s * h, s * w, 1) * 10, 0, 255).astype(np.float32)
    return cfg, wts, eng, x, x2, y


def oracle_masks(eng, cfg, seed, n, h, w):
    masks = {}
    for scope, k, cin, cout, bias, prelu in O.layer_table(cfg):
        if prelu:
            m = eng.dropout_mask(scope, seed, n, h, w, cout)
            masks[scope] = np.ascontiguousarray(m.transpose(0, 3, 1, 2)).astype(np.float64)
    return masks


@pytest.mark.parametrize("kw,keep,shape", [(SMALL, 1.0, (2, 12, 10)), (SMALL, 0.8, (2, 16, 24)), (SMALL4, 0.8, (1, 9, 11)),
                                           (SMALL, 1.0, (1, 1, 1)), (SMALL4, 1.0, (3, 2, 1)), (SMALL, 0.8, (1, 1, 37)),
                                           (SMALL, 1.0, (2, 33, 3))],
                         ids=["x2-nodrop", "x2-drop", "x4-drop", "x2-1x1", "x4-2x1", "x2-row", "x2-narrow"])
def test_gradients_match_oracle(kw, keep, shape):
    n, h, w = shape
    cfg, wts, eng, x, x2, y = setup(kw, keep, n, h, w)
    seed = 1234
    loss, mse = eng.train_step_host(x, x2, y, lr=0.002, seed=seed, apply_update=False)
    orc = O.Oracle(cfg, wts, torch.float64)
    masks = oracle_masks(eng, cfg, seed, n, h, w) if keep < 1.0 else None
    mse_ref, loss_ref, grads_ref = orc.loss_and_grads(x.astype(np.float64), x2.astype(np.float64), y.astype(np.float64),
                                                      keep_prob=keep, masks=masks)
    assert mse == pytest.approx(mse_ref, rel=2e-5)
    assert loss == pytest.approx(mse_ref, rel=2e-5)          # image_loss == mse (DCSCN.py:346-347)
    norm_ref = np.sqrt(sum(np.sum(v ** 2) for v in grads_ref.values()))
    assert eng.last_grad_norm == pytest.approx(norm_ref, rel=2e-3)
    for name, gref in grads_ref.items():
        g = eng.get_grad(name)
        tol = 2e-3 * np.abs(gref).max() + 1e-7
        assert np.abs(g - gref).max() <= tol, (name, float(np.abs(g - gref).max()), float(np.abs(gref).max()))
    eng.close()


def test_adam_step_matches_oracle_and_loss_decreases():
    n, h, w = 2, 16, 16
    cfg, wts, eng, x, x2, y = setup(SMALL, 0.8, n, h, w, seed=3)
    orc = O.Oracle(cfg, wts, torch.float64)
    m = {k: np.zeros_like(v) for k, v in wts.items()}
    v = {k: np.zeros_like(v_) for k, v_ in wts.items()}
    losses = []
    # Tolerance, derived instead of tuned: test_gradients_match_oracle grants every gradient tensor an absolute error
    # delta = 2e-3 * max|g|.  Adam's update lr_t * m / (sqrt(v) + eps) is ~ lr * sign(g) where |g| >> delta (insensitive to
    # the error) and flips sign - an error of up to 2 lr - where |g| <~ delta; in between its sensitivity to g is O(1/|g|).
    # Allowed error of a weight after t steps: 2e-3 * lr * t  +  lr * sum_s min(2, 3 * delta_s / |g_s|).
    slack = {k: np.zeros_like(v_) for k, v_ in wts.items()}
    for step in range(1, 4):
        seed = 100 + step
        loss, mse = eng.train_step_host(x, x2, y, lr=0.002, seed=seed)
        losses.append(mse)
        masks = oracle_masks(eng, cfg, seed, n, h, w)
        _, _, grads = orc.loss_and_grads(x.astype(np.float64), x2.astype(np.float64), y.astype(np.float64), keep_prob=0.8, masks=masks)
        clipped, _ = orc.clip_by_global_norm(grads)
        orc.adam_step(clipped, m, v, step, 0.002)
        for name in wts:
            delta = 2e-3 * np.abs(grads[name]).max()
            slack[name] += np.minimum(2.0, 3.0 * delta / (np.abs(grads[name]) + 1e-300))
            tol = 2e-3 * 0.002 * step + 0.002 * slack[name]
            got = eng.get_param(name)
            assert (np.abs(got - orc.w[name]) <= tol).all(), (step, name, float((np.abs(got - orc.w[name]) - tol).max()))
    # slots follow the reference's checkpoint convention (<var>/Adam, <var>/Adam_1)
    np.testing.assert_allclose(eng.get_adam_slot("CNN1/conv_W", 0), m["CNN1/conv_W"], rtol=0, atol=3e-3 * np.abs(m["CNN1/conv_W"]).max())
    # the forward pass uses the updated weights (re-packed tensor-core operand images)
    yy = eng.forward_host(x, x2)
    ref = O.Oracle(cfg, {k: a.astype(np.float64) for k, a in orc.w.items()}, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64))
    assert np.abs(yy - ref).max() <= 5e-3
    more = [eng.train_step_host(x, x2, y, lr=0.002, seed=200 + i)[1] for i in range(30)]
    assert np.mean(more[-5:]) < losses[0]
    eng.close()


@pytest.mark.parametrize("kw", [SMALL, SMALL4], ids=["x2", "x4"])
def test_device_refresh_equals_host_repack(kw):
    """After an optimizer step the packed tensor-core weight images (forward layers and dgrad twins), fused bias / PReLU
    vectors and the CNN1 / R-CNN1 filters are refreshed on the device through index maps derived from the host packing
    code.  A fresh engine that packs the same weights on the host must give the same forward output and the same
    gradients (only the power-of-two weight scale may differ, which is exact)."""
    from helper import engine as E
    cfg, wts, eng, x, x2, y = setup(kw, 0.8, 2, 12, 14, seed=3)
    for i in range(4):
        eng.train_step_host(x, x2, y, lr=0.01, seed=50 + i)
    y_dev = eng.forward_host(x, x2)
    eng.train_step_host(x, x2, y, lr=0.01, seed=99, apply_update=False)
    params = {n: eng.get_param(n) for n in wts}
    grads_dev = {n: eng.get_grad(n) for n in wts}
    assert any(np.abs(params[n] - wts[n]).max() > 1e-3 for n in wts)      # the weights did move
    fresh = E.Engine(E.make_config(dropout_keep=0.8, **kw))
    fresh.set_params(params)
    y_host = fresh.forward_host(x, x2)
    fresh.train_step_host(x, x2, y, lr=0.01, seed=99, apply_update=False)
    assert np.abs(y_dev - y_host).max() <= 1e-5
    for n in wts:
        g = fresh.get_grad(n)
        assert np.abs(g - grads_dev[n]).max() <= 1e-4 * np.abs(g).max() + 1e-9, n   # fp32 atomics reorder sums
    eng.close()
    fresh.close()


def test_tensor_core_wgrad_matches_cuda_core_wgrad_full_model():
    """Filter gradients of the full L12 x2 model (196..48 filters, 1301-channel concat, 384-column Up-PS): the wgmma
    wgrad (transposed zero-bordered operands, K-split partial sums) against the straightforward CUDA-core kernel on the
    same planes.  Both accumulate in fp32; 1e-4 of each tensor's max covers the different summation orders."""
    from helper import engine as E, tf_bundle
    import conftest
    wts = conftest.load_golden_weights("dcscn_L12_F196to48_NIN_A64_PS_R1F32")
    g = np.random.RandomState(11)
    n, h, w = 3, 20, 28
    x = (g.rand(n, h, w, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, 2 * h, 2 * w, 1) * 255).astype(np.float32)
    y = np.clip(x2 + g.randn(n, 2 * h, 2 * w, 1) * 10, 0, 255).astype(np.float32)
    grads = []
    for impl in (1, 0):
        eng = E.Engine(E.make_config(scale=2, dropout_keep=0.8))
        eng.set_params(wts)
        eng.set_option("wgrad_impl", impl)
        eng.train_step_host(x, x2, y, lr=0.002, seed=5, apply_update=False)
        grads.append({k: eng.get_grad(k) for k in wts})
        eng.close()
    for k in wts:
        if not k.endswith("conv_W"):
            continue
        ref, got = grads[0][k], grads[1][k]
        assert np.abs(got - ref).max() <= 1e-4 * np.abs(ref).max() + 1e-12, (k, float(np.abs(got - ref).max()), float(np.abs(ref).max()))


def test_activation_gradient_kernels_agree():
    """act_grad_impl 0 (16-byte loads, 8 channels per thread, the default) against 1 (channel pairs): same element-wise
    results, bias / alpha sums in a different order."""
    from helper import engine as E
    import conftest
    wts = conftest.load_golden_weights("dcscn_L12_F196to48_NIN_A64_PS_R1F32")
    g = np.random.RandomState(12)
    n, h, w = 2, 19, 23
    x = (g.rand(n, h, w, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, 2 * h, 2 * w, 1) * 255).astype(np.float32)
    y = np.clip(x2 + g.randn(n, 2 * h, 2 * w, 1) * 10, 0, 255).astype(np.float32)
    grads = []
    for impl in (1, 0):
        eng = E.Engine(E.make_config(scale=2, dropout_keep=0.8))
        eng.set_params(wts)
        eng.set_option("act_grad_impl", impl)
        eng.train_step_host(x, x2, y, lr=0.002, seed=5, apply_update=False)
        grads.append({k: eng.get_grad(k) for k in wts})
        eng.close()
    for k in wts:
        ref, got = grads[0][k], grads[1][k]
        assert np.abs(got - ref).max() <= 2e-5 * np.abs(ref).max() + 1e-12, (k, float(np.abs(got - ref).max()), float(np.abs(ref).max()))


def test_full_size_batch_gradient_is_mean_of_half_batch_gradients():
    """BASELINE configs[3] size (L12 x4, 64 patches of 48x48 -> 192x192), where the CPU oracle would take minutes:
    with dropout off the loss is a mean over patches, so every gradient of the full batch must equal the mean of the
    gradients of its two halves (L2 term included in both)."""
    from helper import engine as E
    import conftest
    wts = conftest.load_golden_weights("dcscn_L12_F196to48_Sc4_NIN_A64_PS_R1F32")
    g = np.random.RandomState(5)
    n = 64
    x = (g.rand(n, 48, 48, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, 192, 192, 1) * 255).astype(np.float32)
    y = np.clip(x2 + g.randn(n, 192, 192, 1) * 10, 0, 255).astype(np.float32)
    eng = E.Engine(E.make_config(scale=4, dropout_keep=1.0))
    eng.set_params(wts)

    def grads(sl):
        loss, mse = eng.train_step_host(x[sl], x2[sl], y[sl], lr=0.002, seed=1, apply_update=False)
        return mse, {k: eng.get_grad(k) for k in wts}

    m_all, g_all = grads(slice(0, n))
    m_a, g_a = grads(slice(0, n // 2))
    m_b, g_b = grads(slice(n // 2, n))
    assert m_all == pytest.approx(0.5 * (m_a + m_b), rel=1e-5)
    for k in wts:
        want = 0.5 * (g_a[k] + g_b[k])
        assert np.abs(g_all[k] - want).max() <= 2e-4 * np.abs(want).max() + 1e-9, (k, float(np.abs(g_all[k] - want).max()), float(np.abs(want).max()))
    eng.close()


def test_full_width_l12_x4_gradients_match_oracle():
    """The flagship train graph at full width (L12, 196..48 filters, 1301-channel concat, two pixel-shuffler stages, the
    reference's own x4 checkpoint) on a batch small enough for the fp64 autograd oracle: loss and EVERY gradient, with
    dropout 0.8 replayed through the engine's masks."""
    from helper import engine as E
    import conftest
    model = "dcscn_L12_F196to48_Sc4_NIN_A64_PS_R1F32"
    cfg = O.OracleConfig(scale=4)
    wts = {k: v.astype(np.float64) for k, v in conftest.load_golden_weights(model).items()}
    n, h, w = 2, 12, 10
    g = np.random.RandomState(21)
    x = (g.rand(n, h, w, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, 4 * h, 4 * w, 1) * 255).astype(np.float32)
    y = np.clip(x2 + g.randn(n, 4 * h, 4 * w, 1) * 10, 0, 255).astype(np.float32)
    eng = E.Engine(E.make_config(scale=4, dropout_keep=0.8))
    eng.set_params({k: v.astype(np.float32) for k, v in wts.items()})
    seed = 77
    loss, mse = eng.train_step_host(x, x2, y, lr=0.002, seed=seed, apply_update=False)
    masks = oracle_masks(eng, cfg, seed, n, h, w)
    mse_ref, loss_ref, grads_ref = O.Oracle(cfg, wts, torch.float64).loss_and_grads(
        x.astype(np.float64), x2.astype(np.float64), y.astype(np.float64), keep_prob=0.8, masks=masks)
    assert mse == pytest.approx(mse_ref, rel=5e-5)
    norm_ref = np.sqrt(sum(np.sum(v ** 2) for v in grads_ref.values()))
    assert eng.last_grad_norm == pytest.approx(norm_ref, rel=2e-3)
    for name, gref in grads_ref.items():
        got = eng.get_grad(name)
        tol = 2e-3 * np.abs(gref).max() + 1e-7
        assert np.abs(got - gref).max() <= tol, (name, float(np.abs(got - gref).max()), float(np.abs(gref).max()))
    eng.close()


def test_l1_loss_gradients_match_oracle():
    """--use_l1_loss (DCSCN.py:342-344): image_loss = mean|y_ - y|, gradient sign(diff) / count; mse is still reported."""
    n, h, w = 2, 12, 10
    cfg, wts, eng, x, x2, y = setup(SMALL, 1.0, n, h, w)
    eng.set_option("l1_loss", 1)
    loss, mse = eng.train_step_host(x, x2, y, lr=0.002, seed=1, apply_update=False)
    orc = O.Oracle(cfg, wts, torch.float64)
    mse_ref, loss_ref, grads_ref = orc.loss_and_grads(x.astype(np.float64), x2.astype(np.float64), y.astype(np.float64),
                                                      keep_prob=1.0, use_l1_loss=True)
    assert mse == pytest.approx(mse_ref, rel=2e-5)
    l2 = cfg.l2_decay * sum(float(np.sum(wts[k] ** 2)) / 2 for k in wts if k.endswith("conv_W"))
    assert loss == pytest.approx(loss_ref - l2, rel=2e-5)       # the engine returns image_loss (what train_batch logs)
    for name, gref in grads_ref.items():
        g = eng.get_grad(name)
        assert np.abs(g - gref).max() <= 2e-3 * np.abs(gref).max() + 1e-7, name
    eng.close()


# ---------------------------------------------------------------- depthwise-separable graphs (tf_graph.py:155-216) ----
DS2 = dict(scale=2, layers=3, filters=12, min_filters=6, filters_decay_gamma=1.5, nin_filters=10, nin_filters2=6,
           pixel_shuffler_filters=1, depthwise_separable=True)
DS4 = dict(scale=4, layers=4, filters=14, min_filters=5, filters_decay_gamma=1.2, nin_filters=9, nin_filters2=7,
           pixel_shuffler_filters=1, depthwise_separable=True)
DS4W = dict(scale=4, layers=3, filters=10, min_filters=6, filters_decay_gamma=1.5, nin_filters=8, nin_filters2=4,
            pixel_shuffler_filters=0, depthwise_separable=True)    # pixel shuffler keeps all 12 channels: R-CNN1 12 -> 1


@pytest.mark.parametrize("kw,keep,shape", [(DS2, 1.0, (2, 9, 7)), (DS2, 0.8, (2, 12, 10)), (DS4, 0.8, (2, 8, 11)),
                                           (DS4, 1.0, (1, 1, 1)), (DS4W, 0.8, (1, 6, 5))],
                         ids=["ds-x2-nodrop", "ds-x2-drop", "ds-x4-drop", "ds-x4-1x1", "ds-x4-wide"])
def test_depthwise_separable_gradients_match_oracle(kw, keep, shape):
    """The train step of --depthwise_separable graphs: loss, mse and EVERY gradient (depthwise_W, pointwise_W, conv_B, PReLU
    slopes, and the dead conv_W whose only gradient is its L2 decay, tf_graph.py:183,212) against fp64 autograd with
    the engine's dropout masks replayed.  All mismatches are reported at once."""
    n, h, w = shape
    cfg, wts, eng, x, x2, y = setup(kw, keep, n, h, w, seed=5)
    seed = 4321
    loss, mse = eng.train_step_host(x, x2, y, lr=0.002, seed=seed, apply_update=False)
    orc = O.Oracle(cfg, wts, torch.float64)
    masks = oracle_masks(eng, cfg, seed, n, h, w) if keep < 1.0 else None
    mse_ref, loss_ref, grads_ref = orc.loss_and_grads(x.astype(np.float64), x2.astype(np.float64), y.astype(np.float64),
                                                      keep_prob=keep, masks=masks)
    bad = []
    if not mse == pytest.approx(mse_ref, rel=2e-5):
        bad.append(("mse", mse, mse_ref))
    for name, gref in grads_ref.items():
        g = eng.get_grad(name)
        tol = 2e-4 * np.abs(gref).max() + 1e-7
        err = float(np.abs(g - gref).max())
        if not err <= tol:
            bad.append((name, err, float(np.abs(gref).max())))
    assert not bad, bad
    # the dead variable: gradient = l2_decay * conv_W exactly
    np.testing.assert_allclose(eng.get_grad("CNN2/conv_W"), cfg.l2_decay * wts["CNN2/conv_W"], rtol=1e-6, atol=1e-12)
    norm_ref = np.sqrt(sum(np.sum(v ** 2) for v in grads_ref.values()))
    assert eng.last_grad_norm == pytest.approx(norm_ref, rel=1e-3)
    eng.close()


def test_depthwise_separable_adam_steps_and_forward_follow():
    """Three optimizer steps of a depthwise-separable graph against the oracle's clip + TF-Adam, then the inference
    kernels (which hold their own filter copies) must see the updated weights, and the loss must go down."""
    n, h, w = 2, 12, 12
    cfg, wts, eng, x, x2, y = setup(DS4, 0.8, n, h, w, seed=9)
    orc = O.Oracle(cfg, wts, torch.float64)
    m = {k: np.zeros_like(v) for k, v in wts.items()}
    v = {k: np.zeros_like(v_) for k, v_ in wts.items()}
    slack = {k: np.zeros_like(v_) for k, v_ in wts.items()}
    first = None
    for step in range(1, 4):
        seed = 300 + step
        loss, mse = eng.train_step_host(x, x2, y, lr=0.002, seed=seed)
        first = mse if first is None else first
        masks = oracle_masks(eng, cfg, seed, n, h, w)
        _, _, grads = orc.loss_and_grads(x.astype(np.float64), x2.astype(np.float64), y.astype(np.float64), keep_prob=0.8, masks=masks)
        clipped, _ = orc.clip_by_global_norm(grads)
        orc.adam_step(clipped, m, v, step, 0.002)
        for name in wts:
            delta = 2e-4 * np.abs(grads[name]).max()
            slack[name] += np.minimum(2.0, 3.0 * delta / (np.abs(grads[name]) + 1e-300))
            tol = 2e-3 * 0.002 * step + 0.002 * slack[name]
            got = eng.get_param(name)
            assert (np.abs(got - orc.w[name]) <= tol).all(), (step, name, float((np.abs(got - orc.w[name]) - tol).max()))
    yy = eng.forward_host(x, x2)
    ref = O.Oracle(cfg, {k: a.astype(np.float64) for k, a in orc.w.items()}, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64))
    assert np.abs(yy - ref).max() <= 5e-3
    more = [eng.train_step_host(x, x2, y, lr=0.002, seed=400 + i)[1] for i in range(40)]
    assert np.mean(more[-5:]) < first
    eng.close()
