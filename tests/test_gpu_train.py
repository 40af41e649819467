"""GPU parity of the train step (loss, every gradient, global-norm clip, TF-Adam) against the fp64 CPU oracle
(torch autograd of the restated graph, oracle/dcscn_oracle.py).  The oracle replays the engine's dropout masks
(dcscn_dropout_mask), so the comparison is exact up to fp32-level rounding.  Tolerance: 2e-3 of each gradient
tensor's max magnitude (data gradients run on the fp16x3 tensor-core path, filter gradients are fp32 atomics)."""
import numpy as np
import pytest
import torch

import dcscn_oracle as O
from conftest import MODEL_FLAGS, load_golden_weights

pytestmark = pytest.mark.gpu

SMALL = dict(scale=2, layers=3, filters=24, min_filters=16, filters_decay_gamma=1.5, nin_filters=16, nin_filters2=16)
SMALL4 = dict(scale=4, layers=3, filters=20, min_filters=16, filters_decay_gamma=1.5, nin_filters=16, nin_filters2=16)
SMALL3 = dict(SMALL, scale=3)
K5 = dict(SMALL, cnn_size=5)
# the shipped c-DCSCN checkpoints: --pixel_shuffler_filters=1, so R-CNN1 reads a single channel (C = 1)
CDCSCN = {2: "dcscn_L7_F32to8_G1.20_NIN_A24_B8_PS_R1F32", 3: "dcscn_L7_F32to8_G1.20_Sc3_NIN_A24_B8_PS_R1F32",
          4: "dcscn_L7_F32to8_G1.20_Sc4_NIN_A24_B8_PS_R1F32"}


def setup(kw, keep, n, h, w, seed=0, weights="he"):
    """`weights` is "he" (He-init with `seed`) or the name of a checkpoint under tests/golden/models, whose MODEL_FLAGS
    then replace `kw`."""
    from helper import engine as E
    if weights != "he":
        kw = MODEL_FLAGS[weights]
    cfg = O.OracleConfig(**kw)
    src = O.he_init_weights(cfg, seed=seed) if weights == "he" else load_golden_weights(weights)
    wts = {k: v.astype(np.float64) for k, v in src.items()}
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


def launched_kernels(fn, attempts=5):
    """Runs fn() under torch.profiler and returns (its result, the names of the CUDA kernels launched meanwhile).  CUPTI
    records every kernel of the process, so the engine's launches from libdcscn_b200.so show up with demangled names
    ("void dcscn::last_wgrad_kernel<9>(dcscn::LastWgradParams)").

    CUPTI now and then hands back a session that lost the kernel records of its first launches: on one H100 about one
    profiled forward in a thousand came back with no kernel at all, and in a process that had run most of the GPU suite
    traces kept every kernel of a forward but its first (conv_first3x3_kernel), or only its last (conv_last_kernel).
    So LEAD_KERNELS kernels of our own run and finish inside the session before fn(), and a trace counts only when it
    holds every one of them and an engine kernel: a trace that lost a leading part of its records loses some of them
    first.  Otherwise fn() runs again (every caller passes a repeatable call: a forward, or a train step with
    apply_update = False); the kernels asserted on are always those of one trace that passed that test."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    for _ in range(attempts):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            lead = torch.zeros(256, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            for _ in range(LEAD_KERNELS):
                lead.bitwise_not_()
            torch.cuda.synchronize()
            out = fn()
            torch.cuda.synchronize()
        events = prof.events()
        names = {e.name for e in events}
        leads = sum(1 for e in events if e.device_type == DeviceType.CUDA and "bitwise_not" in e.name)
        if leads == LEAD_KERNELS and any("dcscn::" in n for n in names):
            break
    return out, names


LEAD_KERNELS = 8


def assert_kernels_ran(names, kernels):
    """Every entry of `kernels` was launched: "foo" matches dcscn::foo( or dcscn::foo< (so last_wgrad_kernel does not
    match last_wgrad_scalar_kernel), "foo<25>" matches that instantiation only."""
    ours = sorted(n for n in names if "dcscn::" in n)
    assert ours, ("the profiler recorded no dcscn:: kernel among %d events: CUPTI did not trace the engine's launches, "
                  "so which kernels a case reaches cannot be checked" % len(names))

    def ran(k):
        pats = ["dcscn::" + k] if "<" in k else ["dcscn::%s(" % k, "dcscn::%s<" % k]
        return any(p in n for n in ours for p in pats)
    missing = [k for k in kernels if not ran(k)]
    assert not missing, ("not launched", missing, ours)


# The fast kernels of the train step, and what each general case must reach instead (train_engine.inc, train_step_impl:
# the selection predicates of CNN1, R-CNN1 forward / filter gradient / data gradient + space_to_depth, x4 space_to_depth).
FAST = ["conv_tc_kernel", "wgrad_tc_kernel", "conv_first3x3_kernel", "first_wgrad_kernel", "conv_last_direct_kernel",
        "last_wgrad_kernel<9>", "last_dgrad_s2d_rows_kernel"]
C1 = ["conv_last_kernel", "last_wgrad_scalar_kernel", "last_dgrad_s2d_kernel"]     # R-CNN1 on one input channel
GENERAL_K = ["conv_first_kernel", "wgrad_kernel", "conv_last_kernel", "last_dgrad_s2d_kernel", "wgrad_tc_kernel"]

GRADIENT_CASES = [
    # id, config, weights, keep, (n, h, w), kernels that must run
    ("x2-nodrop", SMALL, "he", 1.0, (2, 12, 10), FAST),
    ("x2-drop", SMALL, "he", 0.8, (2, 16, 24), FAST),
    ("x4-drop", SMALL4, "he", 0.8, (1, 9, 11), FAST + ["s2d_planes_kernel"]),
    ("x2-1x1", SMALL, "he", 1.0, (1, 1, 1), FAST),
    ("x4-2x1", SMALL4, "he", 1.0, (3, 2, 1), FAST + ["s2d_planes_kernel"]),
    ("x2-row", SMALL, "he", 0.8, (1, 1, 37), FAST),
    ("x2-narrow", SMALL, "he", 1.0, (2, 33, 3), FAST),
    # depth_to_space gradient at r = 3; Up-PS has 9 * 32 = 288 columns: three wgmma column tiles in its filter gradient
    # and a partial last K chunk in its data-gradient twin
    ("x3", SMALL3, "he", 0.8, (2, 9, 11), FAST),
    ("cdcscn-x2", None, CDCSCN[2], 0.8, (2, 12, 10), C1),
    ("cdcscn-x3", None, CDCSCN[3], 0.8, (2, 12, 10), C1),
    ("cdcscn-x4", None, CDCSCN[4], 0.8, (2, 12, 10), C1 + ["s2d_planes_kernel"]),
    # 5x5 everywhere but A1 / B1 / B2: CNN1 stores min(z, 0) from the general kernel, CNN1's filter gradient reads the fp32
    # image, wgmma filter gradients at 25 taps, R-CNN1 C = 32 on the vector branch of the data-gradient kernel
    ("k5-x2", K5, "he", 0.8, (2, 12, 10), GENERAL_K + ["last_wgrad_kernel<25>"]),
    # nin 12 + 8 = 20 channels (not a multiple of 8): per-element space_to_depth and the per-channel data-gradient branch
    ("k5-x4-c20", dict(SMALL4, cnn_size=5, nin_filters=12, nin_filters2=8), "he", 0.8, (1, 9, 7),
     GENERAL_K + ["last_wgrad_kernel<25>", "s2d_planes_kernel"]),
    ("k1-x3", dict(SMALL3, cnn_size=1), "he", 0.8, (2, 8, 9), GENERAL_K + ["last_wgrad_kernel<1>"]),
    # R-CNN1 C = 12: a multiple of 4 but not of 8, still on the vector kernels
    ("ps12-x2", dict(SMALL, pixel_shuffler_filters=12), "he", 0.8, (2, 10, 13), FAST),
    # R-CNN1 C = 144 > 128: general forward and data gradient; Up-PS has 576 columns
    ("ps144-x2", dict(SMALL, nin_filters=96, nin_filters2=48), "he", 0.8, (1, 8, 9),
     ["conv_last_kernel", "last_wgrad_kernel<9>", "last_dgrad_s2d_kernel", "wgrad_tc_kernel"]),
    # CNN1 with 272 filters (n_pad > 256) on the general kernels; CNN2 has a 16-channel partial K chunk (272 = 4 * 64 + 16)
    ("cnn1-272", dict(SMALL, layers=2, filters=272, min_filters=32), "he", 0.8, (1, 8, 8),
     ["conv_first_kernel", "wgrad_kernel", "conv_tc_kernel", "wgrad_tc_kernel"]),
]


@pytest.mark.parametrize("kw,weights,keep,shape,kernels", [c[1:] for c in GRADIENT_CASES], ids=[c[0] for c in GRADIENT_CASES])
def test_gradients_match_oracle(kw, weights, keep, shape, kernels):
    """Loss, mse, global norm and every gradient of one train step against fp64 autograd, on graphs chosen so that each
    kernel the train step can select (fast or general path) runs in at least one case; the profiler trace of the step
    proves it.  All mismatches of a case are reported at once."""
    n, h, w = shape
    cfg, wts, eng, x, x2, y = setup(kw, keep, n, h, w, weights=weights)
    seed = 1234
    (loss, mse), names = launched_kernels(lambda: eng.train_step_host(x, x2, y, lr=0.002, seed=seed, apply_update=False))
    assert_kernels_ran(names, kernels)
    orc = O.Oracle(cfg, wts, torch.float64)
    masks = oracle_masks(eng, cfg, seed, n, h, w) if keep < 1.0 else None
    mse_ref, loss_ref, grads_ref = orc.loss_and_grads(x.astype(np.float64), x2.astype(np.float64), y.astype(np.float64),
                                                      keep_prob=keep, masks=masks)
    bad = []
    if not mse == pytest.approx(mse_ref, rel=2e-5):
        bad.append(("mse", mse, mse_ref))
    if not loss == pytest.approx(mse_ref, rel=2e-5):          # image_loss == mse (DCSCN.py:346-347)
        bad.append(("loss", loss, mse_ref))
    norm_ref = np.sqrt(sum(np.sum(v ** 2) for v in grads_ref.values()))
    if not eng.last_grad_norm == pytest.approx(norm_ref, rel=2e-3):
        bad.append(("grad norm", eng.last_grad_norm, norm_ref))
    for name, gref in grads_ref.items():
        g = eng.get_grad(name)
        tol = 2e-3 * np.abs(gref).max() + 1e-7
        err = float(np.abs(g - gref).max())
        if not err <= tol:
            bad.append((name, err, float(np.abs(gref).max())))
    eng.close()
    assert not bad, bad


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


def test_train_step_refuses_f16x1_and_handle_keeps_working():
    """The train step needs the fp16x3 operand planes of the tensor-core graph: an f16x1 engine refuses it with
    EngineError, and the refusal leaves the handle as it was, so the forward still runs and gives the same output."""
    from helper import engine as E
    cfg = O.OracleConfig(**SMALL)
    wts = O.he_init_weights(cfg, seed=2)
    eng = E.Engine(E.make_config(dropout_keep=0.8, precision=1, **SMALL))
    eng.set_params(wts)
    g = np.random.RandomState(8)
    x = (g.rand(1, 10, 12, 1) * 255).astype(np.float32)
    x2 = (g.rand(1, 20, 24, 1) * 255).astype(np.float32)
    y_before = eng.forward_host(x, x2)
    with pytest.raises(E.EngineError, match="f16x3"):
        eng.train_step_host(x, x2, x2, lr=0.002, seed=1)
    y_after = eng.forward_host(x, x2)
    assert np.array_equal(y_before, y_after)
    ref = O.Oracle(cfg, {k: v.astype(np.float64) for k, v in wts.items()}, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64))
    assert np.abs(y_after - ref).max() < 1.0          # single-pass fp16 operands: the bar of test_fast_mode_is_psnr_neutral
    eng.close()


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


DS3 = dict(scale=3, layers=3, filters=12, min_filters=6, filters_decay_gamma=1.5, nin_filters=10, nin_filters2=6,
           pixel_shuffler_filters=1, depthwise_separable=True)


@pytest.mark.parametrize("kw,keep,shape", [(DS2, 1.0, (2, 9, 7)), (DS2, 0.8, (2, 12, 10)), (DS4, 0.8, (2, 8, 11)),
                                           (DS4, 1.0, (1, 1, 1)), (DS4W, 0.8, (1, 6, 5)), (DS3, 0.8, (2, 7, 9))],
                         ids=["ds-x2-nodrop", "ds-x2-drop", "ds-x4-drop", "ds-x4-1x1", "ds-x4-wide", "ds-x3-oddw"])
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


# ------------------------------------------------------------------------------------------ device refresh ----
def train_tensors(eng, names):
    """{name: fp32 values} of those of `names` the last capture step kept.  dcscn_get_train_tensor refuses a wrong
    element count with "'<name>' has <count> elements", and a name it did not capture with "no tensor": the count of
    each kept tensor is read from the first refusal."""
    import re
    from helper import engine as E
    out = {}
    for name in names:
        try:
            out[name] = eng.get_train_tensor(name, (1,))
        except E.EngineError as e:
            m = re.search(r"has (\d+) elements", str(e))
            if m:
                out[name] = eng.get_train_tensor(name, (int(m.group(1)),))
            else:
                assert "no tensor" in str(e), str(e)
    return out


def scale_exponent(img):
    """pack_tc_layer's power-of-two weight scale of a packed image: 2^floor(log2(16384 / max |w|))."""
    return int(np.floor(np.log2(16384.0 / float(np.abs(img).max()))))


def composed(p, scope):
    """The filter a layer packs: fp32(depthwise * pointwise) on a wide depthwise-separable graph, else its conv_W."""
    if scope + "/depthwise_W" not in p:
        return p[scope + "/conv_W"]
    dw, pw = p[scope + "/depthwise_W"], p[scope + "/pointwise_W"]
    return (dw[:, :, :, :1] * pw[0, 0][None, None]).astype(np.float32)


def folded_image(p, kw, scope):
    """The folded last upsampler's filter as build_fold / fold_kernel form it (tests/test_fold_cpu.py fold32)."""
    from test_fold_cpu import fold32
    wr = composed(p, "R-CNN1")
    c = wr.shape[2]
    if scope == "Up-TCNN":
        import tconv_oracle as T
        w = T.tconv_filter(p["Up-TCNN/Tconv_W"], kw["scale"])
        return fold32(w, np.zeros(w.shape[-1], np.float32), wr, c)[0]
    return fold32(composed(p, scope), p[scope + "/conv_B"], wr, c)[0]


L12 = {2: "dcscn_L12_F196to48_NIN_A64_PS_R1F32", 4: "dcscn_L12_F196to48_Sc4_NIN_A64_PS_R1F32"}
TCONV = dict(layers=4, filters=40, min_filters=24, filters_decay_gamma=1.5, nin_filters=32, nin_filters2=16,
             transposed_upsampler=True)
DS_WIDE = dict(scale=2, layers=3, filters=12, min_filters=6, nin_filters=32, nin_filters2=16, pixel_shuffler_filters=1,
               depthwise_separable=True)
_GC = {c[0]: c for c in GRADIENT_CASES}
REFRESH_CASES = [
    # id, config, weights
    ("x2", SMALL, "he"), ("x4", SMALL4, "he"), ("x3", SMALL3, "he"), ("k5-x2", K5, "he"), ("cdcscn-x3", None, CDCSCN[3]),
    ("L12-x2-fold", None, L12[2]), ("L12-x4-fold", None, L12[4]),                    # the fold on Up-PS / Up-PS2
    ("x8", dict(SMALL, scale=8), "he"),
    ("tconv-x2", dict(TCONV, scale=2), "he"), ("tconv-x3", dict(TCONV, scale=3), "he"),
    ("ds-narrow", DS2, "he"), ("ds-wide", DS_WIDE, "he"),
    ("relu", dict(SMALL, activator="relu"), "he"), ("sigmoid", dict(SMALL, activator="sigmoid"), "he"),
    ("cnn1-272", _GC["cnn1-272"][1], "he"), ("ps144", _GC["ps144-x2"][1], "he"),
]
# the fp32 tensors of the depthwise-separable step (train_ds.inc).  Its atomic kernels (ds_colsum, ds_dpw, ds_ddw) write
# filter gradients only, so every one of these must be bit-identical too.
DS_TENSORS = ("U:", "Z:", "H:", "E:", "dZ:", "dU:", "dH:")


@pytest.mark.parametrize("kw,weights", [c[1:] for c in REFRESH_CASES], ids=[c[0] for c in REFRESH_CASES])
def test_device_refresh_equals_host_repack(kw, weights):
    """After an optimizer step the packed tensor-core weight images (forward layers and dgrad twins, the folded last
    upsampler), fused bias / slope vectors, the CNN1 / R-CNN1 filters and the depthwise-separable filters are refreshed
    on the device (repack_kernel, fold_kernel, gather_params_kernel, ds_compose) through index maps derived from the
    host packing code.  A fresh engine that packs the same weights on the host must compute the same bits.

    The step is gd (no clip, lr 1) from a chosen gradient: every weight moves by a random relative step of at most
    1e-3 and no element grows past its variable's largest magnitude, whose own gradient is 0.  So no image's
    power-of-two scale changes (asserted for the images formed from products: the fold and the composed wide
    depthwise-separable filters), and the device images must equal the host's bit for bit: the forward output and one
    capture step's y_, dY and every dZ / dH plane (non-atomic kernels) are compared with array_equal; the filter
    gradients, summed by fp32 atomics in any order, keep a 1e-4 bar."""
    from helper import engine as E
    import tconv_oracle as T
    if weights != "he":
        kw = MODEL_FLAGS[weights]
    n, h, w = 2, 10, 12
    s = kw["scale"] if "scale" in kw else 2
    ocfg = {k: v for k, v in kw.items() if k not in ("activator", "transposed_upsampler")}
    if weights != "he":
        src = load_golden_weights(weights)
    elif kw.get("transposed_upsampler"):
        src = T.random_weights(T.Config(**ocfg), seed=3)
    else:
        src = O.he_init_weights(O.OracleConfig(**ocfg), seed=3)

    def engine():
        return E.Engine(E.make_config(dropout_keep=0.8, clipping_norm=0.0, optimizer="gd", **kw))
    eng = engine()
    shapes = eng.param_shapes()
    eng.set_params({k: src[k] for k in shapes})
    g = np.random.RandomState(4)
    x = (g.rand(n, h, w, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, s * h, s * w, 1) * 255).astype(np.float32)
    y = np.clip(x2 + g.randn(n, s * h, s * w, 1) * 10, 0, 255).astype(np.float32)
    eng.train_step_host(x, x2, y, lr=0.0, seed=1)                   # first update: host pack, then the refresh maps
    eng.train_step_host(x, x2, y, lr=0.0, seed=2, apply_update=False)
    before = {k: eng.get_param(k) for k in shapes}
    r = np.random.RandomState(5)
    grads = []
    for k in shapes:
        wv = before[k].ravel()
        step = r.uniform(-1e-3, 1e-3, wv.size)
        step = np.where(np.abs(wv) * (1 + 2e-3) > np.abs(wv).max(), -np.abs(step), step)   # never past the largest
        gv = (-wv * step).astype(np.float32)
        gv[np.argmax(np.abs(wv))] = 0.0
        grads.append(gv)
    gflat = np.concatenate(grads)
    gt = eng.grad_tensor()
    gt[:gflat.size] = torch.from_numpy(gflat).to(gt.device)
    eng.apply_gradients(1.0)
    torch.cuda.synchronize()
    after = {k: eng.get_param(k) for k in shapes}
    off = 0
    for k in shapes:
        m = after[k].size
        assert np.array_equal(after[k].ravel(), before[k].ravel() - gflat[off:off + m]), k      # w - 1 * g, one rounding
        assert np.abs(after[k]).max() == np.abs(before[k]).max(), k
        off += m
    assert any(not np.array_equal(after[k], before[k]) for k in shapes)
    for k in shapes:                                            # images formed from products keep their scale too
        if k.endswith("/depthwise_W"):
            sc = k[:-len("/depthwise_W")]
            assert scale_exponent(composed(after, sc)) == scale_exponent(composed(before, sc)), sc
    eng.set_option("grad_capture", 1)
    y_dev = eng.forward_host(x, x2)
    folded = True
    try:
        eng.get_activation("R-CNN1/taps", (1, 9, n, s * h, s * w))
    except E.EngineError:
        folded = False
    if folded:
        up = "Up-TCNN" if kw.get("transposed_upsampler") else ("Up-PS2/Up-PS2_CNN" if s == 4 else "Up-PS/Up-PS_CNN")
        assert scale_exponent(folded_image(after, kw, up)) == scale_exponent(folded_image(before, kw, up))
    eng.train_step_host(x, x2, y, lr=0.0, seed=99, apply_update=False)
    fresh = engine()
    fresh.set_params(after)
    fresh.set_option("grad_capture", 1)
    # a step first makes the fresh handle a training one: a wide depthwise-separable graph then packs its composed
    # filters, as the trained handle does
    fresh.train_step_host(x, x2, y, lr=0.0, seed=99, apply_update=False)
    y_host = fresh.forward_host(x, x2)
    assert np.array_equal(y_dev, y_host), float(np.abs(y_dev - y_host).max())
    scopes = [t[0] for t in O.layer_table(O.OracleConfig(**ocfg))]
    scopes += [sc.split("/")[0] for sc in scopes] + ["A1+B1", "Up-TCNN"]
    prefixes = ("dZ:", "dH:") + (DS_TENSORS if kw.get("depthwise_separable") else ())
    names = ["y_", "dY"] + sorted({p + sc for p in prefixes for sc in scopes})
    got, want = train_tensors(eng, names), train_tensors(fresh, names)
    assert set(got) == set(want)
    assert {"y_", "dY"} <= set(got) and sum(k.startswith("dZ:") for k in got) >= 3, sorted(got)
    differ = [k for k in got if not np.array_equal(got[k], want[k])]
    assert not differ, differ
    for k in shapes:
        gh, gd = fresh.get_grad(k), eng.get_grad(k)
        assert np.abs(gh - gd).max() <= 1e-4 * np.abs(gh).max() + 1e-9, k   # fp32 atomics reorder sums
    print("%d train tensors bit-identical: %s" % (len(got), " ".join(sorted(got))))
    eng.close()
    fresh.close()
