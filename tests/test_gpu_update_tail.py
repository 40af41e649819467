"""The part of the train step that runs after the gradients, on the GPU, each piece against a reference formed from the
engine's own inputs:

  * grad_finalize_kernel's L2 decay: the gradient of an engine with l2_decay = 0.5 minus that of the same engine with
    l2_decay = 0, on the same batch and seed, is 0.5 * w on exactly the variables of the reference's self.Weights and 0
    on every other one.  The decayed set comes from the oracles (Oracle.l2_weight_names and the Up-TCNN oracle's), which
    follow tf_graph.py: build_conv and build_depthwise_separable_conv append their conv_W (the dead one, on
    depthwise-separable graphs), build_transposed_conv its Tconv_W.  Biases, slopes and the depthwise / pointwise
    filters are set to random nonzero values, so that a decay applied to them shows;
  * the global norm it sums in fp64: last_grad_norm is fp32 of the root of the sum of squares of the finalized
    gradients;
  * loss_kernel's L1 branch: dY is sign(y_ - y) times fp32(G / count) bit for bit, 0 where y_ == y (tf.abs has
    gradient 0 at 0), and the returned loss is mean |y_ - y|;
  * the data-parallel tail (loss_tail_kernel and apply_gradients_avg) on one GPU: two half-batch steps stand in for two
    ranks, their gradient buffers summed on the host stand in for the all-reduce.

Bars: two engines compute the same raw gradients up to the order of their fp32 atomic sums, 1e-4 of the tensor's
largest magnitude (test_gpu_train.py test_device_refresh_equals_host_repack); the finalized value adds one fp32 rounding.
The optimizer update is held to the bar of tests/test_gpu_optimizers.py."""
import numpy as np
import pytest
import torch

import dcscn_oracle as O
import tconv_oracle as T
from test_gpu_optimizers import adam_rule, rule_errors
from test_gpu_train import DS2, SMALL, setup

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
LAMBDA = 0.5
TCONV = dict(scale=2, layers=4, filters=40, min_filters=24, filters_decay_gamma=1.5, nin_filters=32, nin_filters2=16,
             transposed_upsampler=True)
DS_WIDE = dict(scale=2, layers=3, filters=12, min_filters=6, nin_filters=32, nin_filters2=16, pixel_shuffler_filters=1,
               depthwise_separable=True)      # NIN 48 wide: the dense step on composed filters (test_gpu_ds_wide.py)
L2_CASES = [
    # id, graph, activator
    ("prelu", SMALL, "prelu"),
    ("relu", SMALL, "relu"),                  # no slope variables
    ("tconv", TCONV, "prelu"),                # Up-TCNN/Tconv_W is decayed, and has no conv_W
    ("ds-narrow", DS2, "prelu"),              # the fp32 step; the dead conv_W is decayed, depthwise / pointwise are not
    ("ds-wide", DS_WIDE, "prelu"),
]


def decayed_names(kw):
    """The reference's self.Weights, from the oracles."""
    if kw.get("transposed_upsampler"):
        return set(T.Oracle(T.Config(**kw), {}).l2_weight_names())
    return set(O.Oracle(O.OracleConfig(**kw), {}).l2_weight_names())


def unit_batch(s, n, h, w, seed):
    """Inputs in [0, 1]: gradients small against 0.5 * w, so that the atomics bar stays far below the decay."""
    g = np.random.RandomState(seed)
    x = g.rand(n, h, w, 1).astype(np.float32)
    x2 = g.rand(n, s * h, s * w, 1).astype(np.float32)
    y = np.clip(x2 + g.randn(n, s * h, s * w, 1) * 0.04, 0, 1).astype(np.float32)
    return x, x2, y


@pytest.mark.parametrize("kw,act", [c[1:] for c in L2_CASES], ids=[c[0] for c in L2_CASES])
def test_l2_decay_reaches_exactly_the_reference_weights_and_the_norm_is_the_finalized_one(kw, act):
    from helper import engine as E
    decayed = decayed_names(kw)
    base = T.random_weights(T.Config(**kw), seed=3) if kw.get("transposed_upsampler") else \
        O.he_init_weights(O.OracleConfig(**kw), seed=3)
    r = np.random.RandomState(4)
    engines, weights = [], None
    for l2 in (LAMBDA, 0.0):
        eng = E.Engine(E.make_config(dropout_keep=0.8, l2_decay=l2, activator=act, **kw))
        shapes = eng.param_shapes()
        if weights is None:
            assert decayed <= set(shapes), decayed - set(shapes)
            weights = {n: base[n].astype(np.float32) if n in decayed else
                       (r.uniform(0.05, 0.3, shapes[n]) * np.where(r.rand(*shapes[n]) < 0.5, -1, 1)).astype(np.float32)
                       for n in shapes}
        eng.set_params(weights)
        engines.append(eng)
    s = kw["scale"]
    x, x2, y = unit_batch(s, 2, 10, 12, seed=5)
    grads = []
    for eng in engines:
        eng.train_step_host(x, x2, y, lr=0.0, seed=77, apply_update=False)
        g = {n: eng.get_grad(n) for n in weights}
        grads.append(g)
        # the norm of exactly these finalized gradients: fp64 sum of squares, one rounding of its root to fp32
        want = np.float32(np.sqrt(sum(float(np.sum(v.astype(np.float64) ** 2)) for v in g.values())))
        got = np.float32(eng.last_grad_norm)
        assert abs(float(got) - float(want)) <= 2 * float(np.spacing(want)), (float(got), float(want))
        eng.close()
    bad, worst = [], 0.0
    for n, w in weights.items():
        g_l2, g0 = grads[0][n].astype(np.float64), grads[1][n].astype(np.float64)
        dec = LAMBDA * w.astype(np.float64) if n in decayed else np.zeros(w.shape)
        spread = 1e-4 * np.abs(g0).max()
        assert spread <= 1e-2 * LAMBDA * np.abs(w).max(), (n, spread)      # a missing or extra decay cannot hide in it
        bar = spread + 2 * U * (np.abs(g0) + np.abs(dec)) + 1e-30
        ratio = np.abs(g_l2 - g0 - dec) / bar
        worst = max(worst, float(ratio.max()))
        if not (ratio <= 1).all():
            bad.append((n, n in decayed, float(ratio.max())))
    print("L2 decay: largest error / bar %.3g over %d variables (%d decayed)" % (worst, len(weights), len(decayed)))
    assert not bad, bad


def test_l1_loss_gradient_is_the_sign_times_the_scaled_count_and_zero_where_the_difference_is():
    n, h, w = 2, 10, 12
    cfg, _, eng, x, x2, y = setup(SMALL, 1.0, n, h, w, seed=2)
    shape = y.shape
    eng.set_option("grad_capture", 1)
    eng.train_step_host(x, x2, y, lr=0.0, seed=1, apply_update=False)                 # MSE
    yp = eng.get_train_tensor("y_", shape)
    d = yp - y                                                                        # fp32, as loss_kernel forms it
    dY = eng.get_train_tensor("dY", shape)
    count = d.size
    nz = d != 0
    # the loss scale G is a power of two: read it off the MSE gradient, dY = d * fp32(2 G / count)
    G = 2.0 ** np.round(np.log2(np.median(dY[nz] / d[nz]) * count / 2))
    assert np.array_equal(dY, d * (np.float32(2 * G) / np.float32(count)))
    # y equal to y_ at every 7th pixel: keep 1 and the same seed reproduce y_
    y1 = y.copy().ravel()
    y1[::7] = yp.ravel()[::7]
    y1 = y1.reshape(shape)
    eng.set_option("l1_loss", 1)
    loss, mse = eng.train_step_host(x, x2, y1, lr=0.0, seed=1, apply_update=False)
    assert np.array_equal(eng.get_train_tensor("y_", shape), yp)
    d1 = (yp - y1).astype(np.float32)
    s = np.float32(G) / np.float32(count)
    want = np.where(d1 > 0, s, np.where(d1 < 0, -s, np.float32(0))).astype(np.float32)
    dY1 = eng.get_train_tensor("dY", shape)
    assert np.array_equal(dY1, want)
    assert (dY1.ravel()[::7] == 0).all() and (d1.ravel()[::7] == 0).all()
    assert (dY1.ravel()[1::7] != 0).all()
    l1_ref = np.mean(np.abs(d1.astype(np.float64)))
    assert loss == pytest.approx(l1_ref, rel=1e-6)
    assert mse == pytest.approx(np.mean(d1.astype(np.float64) ** 2), rel=1e-6)
    tail = eng.grad_tensor()[-2:].cpu().numpy()                                       # loss_tail_kernel's pair
    assert np.array_equal(tail, np.array([loss, mse], np.float32))
    eng.close()


@pytest.mark.parametrize("loss_kind", ["mse", "l1"])
def test_one_gpu_data_parallel_tail(loss_kind):
    """Two half-batch steps without update stand in for two ranks; the host sum of their gradient buffers (gradients,
    then {image_loss, mse}) is written back, and apply_gradients_avg(lr, 0.5) must return the mean tail and take the
    fp64 Adam step from the mean gradient and its recomputed norm."""
    from helper import engine as E
    cfg = O.OracleConfig(**SMALL)
    eng = E.Engine(E.make_config(dropout_keep=1.0, clipping_norm=5.0, **SMALL))
    eng.set_params(O.he_init_weights(cfg, seed=11))
    if loss_kind == "l1":
        eng.set_option("l1_loss", 1)
    g = np.random.RandomState(5)
    x = (g.rand(4, 12, 12, 1) * 255).astype(np.float32)
    x2 = (g.rand(4, 24, 24, 1) * 255).astype(np.float32)
    y = (g.rand(4, 24, 24, 1) * 255).astype(np.float32)
    bufs = []
    for half in (slice(0, 2), slice(2, 4)):
        loss, mse = eng.train_step_host(x[half], x2[half], y[half], lr=0.002, seed=7, apply_update=False)
        b = eng.grad_tensor().cpu().numpy().copy()
        assert np.array_equal(b[-2:], np.array([loss, mse], np.float32)), (b[-2:], loss, mse)
        bufs.append(b)
    assert bufs[0][-2] != bufs[0][-1] if loss_kind == "l1" else bufs[0][-2] == bufs[0][-1]
    total = (bufs[0] + bufs[1]).astype(np.float32)
    gt = eng.grad_tensor()
    gt.copy_(torch.from_numpy(total).to(gt.device))
    shapes = eng.param_shapes()
    w0 = {n: eng.get_param(n) for n in shapes}
    s0 = {n: [np.zeros(shapes[n], np.float32), np.zeros(shapes[n], np.float32)] for n in shapes}
    lr = 0.002
    loss, mse = eng.apply_gradients_avg(lr, 0.5)
    torch.cuda.synchronize()
    assert np.float32(loss) == total[-2] * np.float32(0.5) and np.float32(mse) == total[-1] * np.float32(0.5)
    assert eng.adam_step == 1
    gm = total[:-2] * np.float32(0.5)
    norm = np.float32(np.sqrt(np.sum(gm.astype(np.float64) ** 2)))
    assert abs(float(np.float32(eng.last_grad_norm)) - float(norm)) <= 2 * float(np.spacing(norm))
    gc = (gm * (np.float32(5.0) / max(norm, np.float32(5.0)))).astype(np.float32)
    bad, worst = rule_errors("adam", eng, w0, s0, gc, float(np.float32(lr)), adam_rule(1))
    print("%s: largest Adam error / bar %.3f" % (loss_kind, worst))
    eng.close()
    assert not bad, bad[:8]
