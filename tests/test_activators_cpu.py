"""--activator (helper/tf_graph.py:77-102) on the CPU: the oracle's forward and TensorFlow gradient rules against closed
forms in float64, the checkpoint variable set, the model-name grammar and the flag's error."""
import numpy as np
import pytest
import torch

import activator_oracle as A
import dcscn_oracle as O

LAM, ALPHA = 1.0507009873554805, 1.6732632423543772
Z = np.array([-30.0, -3.0, -1.0, -0.25, -1e-3, 0.0, 1e-3, 0.25, 1.0, 3.0, 30.0])


def closed_form(act, z):
    """(f(z), the derivative TensorFlow's gradient op gives) in float64."""
    if act == "relu":
        return np.maximum(z, 0.0), (z > 0).astype(np.float64)
    if act == "leaky_relu":
        a = float(np.float32(0.1))
        return np.where(z >= 0, z, a * z), np.where(z >= 0, 1.0, a)
    if act == "sigmoid":
        y = 1.0 / (1.0 + np.exp(-z))
        return y, y * (1.0 - y)
    if act == "tanh":
        y = np.tanh(z)
        return y, 1.0 - y * y
    y = np.where(z < 0, LAM * ALPHA * (np.exp(z) - 1.0), LAM * z)
    return y, np.where(z < 0, y + LAM * ALPHA, LAM)


@pytest.mark.parametrize("act", A.ACTIVATORS[1:])
def test_forward_and_gradient_match_closed_forms(act):
    z = torch.tensor(Z, dtype=torch.float64, requires_grad=True)
    y = A.activate(z, act)
    (g,) = torch.autograd.grad(y.sum(), z)
    f, df = closed_form(act, Z)
    np.testing.assert_allclose(y.detach().numpy(), f, rtol=1e-14, atol=1e-15)
    np.testing.assert_allclose(g.numpy(), df, rtol=1e-14, atol=1e-15)


def test_rules_at_zero_and_selu_constants():
    at0 = {}
    for act in A.ACTIVATORS[1:]:
        z = torch.zeros(1, dtype=torch.float64, requires_grad=True)
        (g,) = torch.autograd.grad(A.activate(z, act).sum(), z)
        at0[act] = float(g)
    assert at0["relu"] == 0.0                       # ReluGrad
    assert at0["leaky_relu"] == 1.0                 # Maximum's gradient, x >= y; torch.maximum would give 0.55
    assert at0["selu"] == LAM                       # SeluGrad; F.selu's backward would give lambda * alpha
    assert at0["sigmoid"] == 0.25 and at0["tanh"] == 1.0
    assert A.SELU_SCALE == 1.0507009873554805 and A.SELU_ALPHA == 1.6732632423543772
    z = torch.tensor([-2.0, 1.5], dtype=torch.float64)
    np.testing.assert_allclose(A.activate(z, "selu").numpy(), torch.selu(z).numpy(), rtol=1e-15)


@pytest.mark.parametrize("act", A.ACTIVATORS[1:])
def test_gradients_match_finite_differences_away_from_zero(act):
    cfg = O.OracleConfig(scale=2, layers=3, filters=8, min_filters=6, nin_filters=6, nin_filters2=4)
    w = A.he_init_weights(cfg, act, seed=1)
    w = {k: v.astype(np.float64) for k, v in w.items()}
    g = np.random.RandomState(2)
    x = g.rand(1, 5, 6, 1) * 255
    x2 = g.rand(1, 10, 12, 1) * 255
    y = x2 + g.randn(1, 10, 12, 1)
    orc = A.Oracle(cfg, w, act)
    _, loss, grads = orc.loss_and_grads(x, x2, y)
    assert sorted(grads) == sorted(A.variable_names(cfg, act))
    for name in ("CNN1/conv_B", "B2/conv_B", "A1/conv_W"):
        i = np.unravel_index(np.argmax(np.abs(grads[name])), grads[name].shape)
        eps = 1e-6 * max(1.0, abs(w[name][i]))
        fd = []
        for sgn in (1, -1):
            ww = dict(w)
            ww[name] = w[name].copy()
            ww[name][i] += sgn * eps
            fd.append(A.Oracle(cfg, ww, act).loss_and_grads(x, x2, y)[1])
        num = (fd[0] - fd[1]) / (2 * eps)
        assert num == pytest.approx(grads[name][i], rel=1e-4, abs=1e-9), (name, num, grads[name][i])


@pytest.mark.parametrize("ds", [False, True], ids=["tc", "ds"])
@pytest.mark.parametrize("act", A.ACTIVATORS)
def test_variable_names_follow_the_activator(act, ds):
    cfg = O.OracleConfig(scale=4, layers=4, filters=16, min_filters=8, nin_filters=8, nin_filters2=4, depthwise_separable=ds)
    names = A.variable_names(cfg, act)
    slopes = [n for n in names if "/prelu/" in n]
    if act == "prelu":
        assert names == O.variable_names(cfg)
        assert len(slopes) == 4 + 3 and "B2/prelu/B2_prelu" in slopes
    else:
        assert slopes == [] and len(names) == len(O.variable_names(cfg)) - 7
    assert set(A.he_init_weights(cfg, act)) == set(names)


def _model(argv):
    """A SuperResolution with the flags of `argv`, without its constructor's directories and logging."""
    import DCSCN
    from helper import args
    f = args._Flags()
    for name, (kind, default, help_text) in args.FLAGS._defs.items():
        f._define(name, default, help_text, kind)
    f.parse(["prog"] + argv)
    m = object.__new__(DCSCN.SuperResolution)
    for k in ("layers", "filters", "filters_decay_gamma", "cnn_size", "scale", "use_nin", "nin_filters", "nin_filters2",
              "pixel_shuffler", "max_value", "activator", "batch_norm", "depthwise_separable", "reconstruct_filters",
              "dropout_rate", "pixel_shuffler_filters", "channels", "l2_decay", "clipping_norm", "beta1", "beta2", "epsilon",
              "gpu_device_id", "precision"):
        if hasattr(f, k):
            setattr(m, k, getattr(f, k))
    m.min_filters = min(f.filters, f.min_filters)
    m.reconstruct_layers = max(f.reconstruct_layers, 1)
    m.workspace_mb = 0
    return m


@pytest.mark.parametrize("act", A.ACTIVATORS)
def test_model_name_carries_the_activator(act):
    m = _model(["--activator=" + act])
    want = "dcscn_L12_F196to48_NIN_A64_PS_R1F32" if act == "prelu" else "dcscn_L12_F196to48_NIN_A64_PS_%s_R1F32" % act
    assert m.get_model_name("") == want
    m = _model(["--activator=" + act, "--scale=4", "--depthwise_separable=true"])
    assert m.get_model_name("").endswith(("" if act == "prelu" else "_" + act) + "_DS_R1F32")


def test_unknown_activator_raises_name_error_at_build_graph(monkeypatch):
    import DCSCN
    created = []
    monkeypatch.setattr(DCSCN.eng, "Engine", lambda config: created.append(config))
    m = _model(["--activator=foo"])
    m.precision = "f16x3"
    with pytest.raises(NameError, match="Not implemented activator:foo"):
        m.build_graph()
    assert created == []
    for act, code in (("prelu", 0), ("relu", 1), ("leaky_relu", 2), ("sigmoid", 3), ("tanh", 4), ("selu", 5)):
        m.activator = act
        assert m._engine_config().activator == code
