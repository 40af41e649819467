"""The optimizers without a GPU: the fp64 oracle (tests/optimizer_oracle.py) against torch.optim where torch has the same
rule, rmsprop and adam against their formulas, the checkpoint slot names, and the --optimizer flag handling."""
import numpy as np
import pytest
import torch

import optimizer_oracle as OO
from helper import engine as E
from test_activators_cpu import _model

LR, MU = 0.01, 0.9


def _run_oracle(kind, w0, grads):
    w, slots = w0.copy(), [np.full_like(w0, v) for v in OO.SLOT_INIT[kind]]
    for g in grads:
        w, slots = OO.update(kind, w, g, slots, LR, MU)
    return w, slots


def _grads(seed=0, steps=5, n=200):
    g = np.random.RandomState(seed)
    # magnitudes from 1e-6 to 1e2 and both signs, so that the slot values matter
    return [g.randn(n) * 10.0 ** g.uniform(-6, 2, n) for _ in range(steps)], g.randn(n)


TORCH_TWINS = {
    "gd": lambda p: torch.optim.SGD([p], lr=LR),
    "momentum": lambda p: torch.optim.SGD([p], lr=LR, momentum=MU, dampening=0),
    "adagrad": lambda p: torch.optim.Adagrad([p], lr=LR, initial_accumulator_value=0.1, eps=0),
    "adadelta": lambda p: torch.optim.Adadelta([p], lr=LR, rho=0.95, eps=1e-8),
}


@pytest.mark.parametrize("kind", sorted(TORCH_TWINS))
def test_oracle_matches_torch_optim_in_float64(kind):
    grads, w0 = _grads()
    p = torch.tensor(w0, dtype=torch.float64, requires_grad=True)
    opt = TORCH_TWINS[kind](p)
    for g in grads:
        p.grad = torch.tensor(g, dtype=torch.float64)
        opt.step()
    w, _ = _run_oracle(kind, w0, grads)
    np.testing.assert_allclose(w, p.detach().numpy(), rtol=1e-13, atol=1e-15)


def test_rmsprop_follows_tf_formula_not_torch():
    """TF's RMSProp: ms starts at 1, ms += (g^2 - ms)(1 - rho), mom = mu mom + lr g / sqrt(ms + eps), eps = 1e-10 inside
    the square root.  torch.optim.RMSprop starts its average at 0 and adds eps outside the root: not the same optimizer."""
    grads, w0 = _grads(1)
    w, ms, mom = w0.copy(), np.ones_like(w0), np.zeros_like(w0)
    for g in grads:
        for i in range(w.size):
            ms[i] = ms[i] + (g[i] * g[i] - ms[i]) * (1 - 0.9)
            mom[i] = MU * mom[i] + LR * g[i] / np.sqrt(ms[i] + 1e-10)
            w[i] = w[i] - mom[i]
    got, slots = _run_oracle("rmsprop", w0, grads)
    np.testing.assert_allclose(got, w, rtol=1e-14, atol=1e-15)
    np.testing.assert_allclose(slots[0], ms, rtol=1e-14)
    np.testing.assert_allclose(slots[1], mom, rtol=1e-14, atol=1e-300)
    p = torch.tensor(w0, dtype=torch.float64, requires_grad=True)
    opt = torch.optim.RMSprop([p], lr=LR, alpha=0.9, eps=1e-10, momentum=MU)
    for g in grads:
        p.grad = torch.tensor(g, dtype=torch.float64)
        opt.step()
    assert np.abs(p.detach().numpy() - got).max() > 1e-3


@pytest.mark.parametrize("betas", [(0.9, 0.999, 1e-8), (0.5, 0.9, 1e-3)], ids=["default", "custom"])
def test_adam_follows_oracle_adam_step_and_tf_formula_not_torch(betas):
    """TF's Adam: lr_t = lr sqrt(1 - b2^t) / (1 - b1^t), m = b1 m + (1 - b1) g, v = b2 v + (1 - b2) g^2,
    w -= lr_t m / (sqrt(v) + eps), with eps outside the root and after the bias correction of lr_t.  The oracle's `update`
    must take the steps `Oracle.adam_step` takes (whose t is the update number) and a literal loop takes.
    torch.optim.Adam divides by sqrt(v_hat) + eps: a different optimizer wherever eps matters."""
    import dcscn_oracle as O
    b1, b2, eps = betas
    grads, w0 = _grads(2)
    w, slots = w0.copy(), [np.zeros_like(w0), np.zeros_like(w0)]
    for t, g in enumerate(grads, start=1):
        w, slots = OO.update("adam", w, g, slots, LR, t=t, beta1=b1, beta2=b2, epsilon=eps)
    lw, m, v = w0.copy(), np.zeros_like(w0), np.zeros_like(w0)
    for t, g in enumerate(grads, start=1):
        lr_t = LR * np.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        for i in range(lw.size):
            m[i] = b1 * m[i] + (1 - b1) * g[i]
            v[i] = b2 * v[i] + (1 - b2) * g[i] * g[i]
            lw[i] = lw[i] - lr_t * m[i] / (np.sqrt(v[i]) + eps)
    np.testing.assert_allclose(w, lw, rtol=1e-14, atol=1e-15)
    np.testing.assert_allclose(slots[0], m, rtol=1e-14, atol=1e-300)
    np.testing.assert_allclose(slots[1], v, rtol=1e-14, atol=1e-300)
    orc = O.Oracle(O.OracleConfig(beta1=b1, beta2=b2, epsilon=eps), {"a": w0.copy()}, torch.float64)
    om, ov = {"a": np.zeros_like(w0)}, {"a": np.zeros_like(w0)}
    for t, g in enumerate(grads, start=1):
        orc.adam_step({"a": g}, om, ov, t, LR)
    np.testing.assert_allclose(orc.w["a"], w, rtol=1e-14, atol=1e-15)
    # resuming at update t: the bias correction of the t-th update, not of the first
    w3, _ = OO.update("adam", w0, grads[0], [m, v], LR, t=3, beta1=b1, beta2=b2, epsilon=eps)
    w1, _ = OO.update("adam", w0, grads[0], [m, v], LR, t=1, beta1=b1, beta2=b2, epsilon=eps)
    assert np.abs(w3 - w1).max() > 1e-4 * LR
    p = torch.tensor(w0, dtype=torch.float64, requires_grad=True)
    opt = torch.optim.Adam([p], lr=LR, betas=(b1, b2), eps=eps)
    for g in grads:
        p.grad = torch.tensor(g, dtype=torch.float64)
        opt.step()
    assert np.abs(p.detach().numpy() - w).max() > 1e-6 * LR


def test_adadelta_update_uses_the_old_accum_update():
    w, slots = OO.update("adadelta", np.zeros(1), np.ones(1), [np.zeros(1), np.full(1, 4.0)], lr=1.0)
    acc = 0.05
    u = np.sqrt(4.0 + 1e-8) / np.sqrt(acc + 1e-8)
    assert w[0] == pytest.approx(-u, rel=1e-15)
    assert slots[1][0] == pytest.approx(0.95 * 4.0 + 0.05 * u * u, rel=1e-15)


def test_slot_table_names_and_initial_values():
    assert set(E.OPTIMIZER_SLOTS) == set(E.OPTIMIZERS) == set(OO.KINDS) | {"adam"}
    assert E.OPTIMIZERS["adam"] == 0                        # a zero-filled dcscn_config keeps meaning Adam
    assert E.OPTIMIZER_SLOTS["adam"] == (("/Adam", 0.0), ("/Adam_1", 0.0))
    assert E.OPTIMIZER_SLOTS["gd"] == ()
    assert E.OPTIMIZER_SLOTS["momentum"] == (("/Momentum", 0.0),)
    assert E.OPTIMIZER_SLOTS["adagrad"] == (("/Adagrad", 0.1),)
    assert E.OPTIMIZER_SLOTS["adadelta"] == (("/Adadelta", 0.0), ("/Adadelta_1", 0.0))
    assert E.OPTIMIZER_SLOTS["rmsprop"] == (("/RMSProp", 1.0), ("/RMSProp_1", 0.0))
    for kind in OO.KINDS + ("adam",):
        assert tuple(v for _, v in E.OPTIMIZER_SLOTS[kind]) == OO.SLOT_INIT[kind]
    c = E.make_config(optimizer="rmsprop", momentum=0.5)
    assert (c.optimizer, c.momentum) == (5, 0.5)
    assert (E.make_config().optimizer, E.make_config().momentum) == (0, pytest.approx(0.9))


@pytest.mark.parametrize("kind", ["gd", "momentum", "adadelta", "adagrad", "adam", "rmsprop"])
def test_every_optimizer_flag_is_accepted(kind):
    m = _model(["--optimizer=" + kind, "--momentum=0.7"])
    m.optimizer, m.momentum = kind, 0.7
    m._check_supported()
    c = m._engine_config()
    assert c.optimizer == E.OPTIMIZERS[kind] and c.momentum == pytest.approx(0.7)
    assert m.get_model_name("") == "dcscn_L12_F196to48_NIN_A64_PS_R1F32"      # the optimizer is not part of the name


def test_unknown_optimizer_raises_the_reference_message_at_build_graph(monkeypatch):
    import DCSCN
    created = []
    monkeypatch.setattr(DCSCN.eng, "Engine", lambda config: created.append(config))
    m = _model(["--optimizer=sgd"])
    m.optimizer, m.precision = "sgd", "f16x3"
    with pytest.raises(ValueError, match=r"Optimizer arg should be one of \[gd, adadelta, adagrad, adam, momentum, rmsprop\]\."):
        m.build_graph()
    assert created == []
