"""The optimizers of --optimizer (adam, gd, momentum, adadelta, adagrad, rmsprop) on the GPU, against the fp64 rules of
tests/optimizer_oracle.py.

Isolated kernel parity: the gradient buffer and the slots are set to chosen fp32 values, so the reference starts from the
kernel's own inputs.  The clip scale is formed in fp32 as the kernel forms it; the clipped gradient g = grad * scale is
the one fp32 product both share.  From there every rule is a chain of at most ~12 fp32 operations (adadelta's
accum_update is the longest: two sums, two square roots, a division and three products lead to u, which is then squared).
Each rounds to within u = 2^-24 relative, and no step of any chain cancels (the slot terms are non-negative, or the update
is added to the weight once at the end), so a result's error is at most (number of roundings) * u times the sum of the
magnitudes of the terms that form it.  The bar is 32 u times that sum: the 1-ulp freedom of the fp32 square root of the
fp64 norm sum (its summation order is the device's) is inside it.

Adam (adam_kernel) is held to 16 u, from this count.  The reference takes the kernel's own constants: lr, beta1, beta2 and
epsilon as the fp32 values the config holds (1 - beta is exact in fp32 for beta in [0.5, 1]), and lr_t in fp64 from
them.  With M = beta1 |m| + (1 - beta1) |g|, V = beta2 v + (1 - beta2) g^2 and S = lr_t M / (sqrt(V) + eps):
  m:  two products and a sum, 3 roundings of M (the two terms may cancel), and 1 more from g's clip-scale freedom;
  v:  g * g, two products and a sum, 4 roundings of V (no cancellation), and 2 more from g;
  w:  lr_t rounded once from fp64 (1), m (4), sqrt(v) (1 + half of v's 6 = 4), + eps (1), lr_t * m (1) and the division
      (1): 12 roundings of S, then w - step, 1 rounding of |w| + S.
So every output is within 13 u of its sum of term magnitudes (|w| + S, M, V), which the bar of 16 u covers.  Forming
lr_t in fp32 instead (powf, sqrtf) cancels in 1 - beta2^t: at t = 2 that alone is 56 u of S, so the step cases where S
dominates |w| see it.

End-to-end steps: the gradient of each tensor is within delta = 2e-3 * max|g| of fp64 autograd (2e-4 on depthwise-
separable graphs), the bar test_gradients_match_oracle and test_depthwise_separable_gradients_match_oracle establish;
the global norm is within 2e-3 relative, which moves the clip scale s by as much.  So each clipped gradient element is
within E = s (delta + 2e-3 |g|).  gd and momentum are linear in g: the weight error is lr times the sum of the (momentum-
decayed) E.  adagrad, adadelta and rmsprop are Lipschitz in g with constants read off the slot values (d/dg of
g / sqrt(c + k g^2) is at most 1 / sqrt(c)), and in their slots with constants from the same values; `_propagate` carries
those first-order bounds through the three steps, and the bar is twice that plus the fp32 weight rounding."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import dcscn_oracle as O
import optimizer_oracle as OO
from conftest import GOLDEN, PKG

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
KINDS = OO.KINDS
SMALL = dict(scale=2, layers=3, filters=24, min_filters=16, filters_decay_gamma=1.5, nin_filters=16, nin_filters2=16)
DS4 = dict(scale=4, layers=4, filters=14, min_filters=5, filters_decay_gamma=1.2, nin_filters=9, nin_filters2=7,
           pixel_shuffler_filters=1, depthwise_separable=True)
MU = 0.9


def _engine(kw, kind, keep=0.8, clip=5.0, seed=3, **adam):
    """`adam`: beta1 / beta2 / epsilon of the engine config (make_config's defaults otherwise)."""
    from helper import engine as E
    cfg = O.OracleConfig(**kw)
    wts = {k: v.astype(np.float64) for k, v in O.he_init_weights(cfg, seed=seed).items()}
    eng = E.Engine(E.make_config(dropout_keep=keep, clipping_norm=clip, optimizer=kind, momentum=MU, **kw, **adam))
    eng.set_params({k: v.astype(np.float32) for k, v in wts.items()})
    return cfg, wts, eng


def _batch(cfg, n, h, w, seed):
    g = np.random.RandomState(seed)
    s = cfg.scale
    x = (g.rand(n, h, w, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, s * h, s * w, 1) * 255).astype(np.float32)
    y = np.clip(x2 + g.randn(n, s * h, s * w, 1) * 10, 0, 255).astype(np.float32)
    return x, x2, y


def _terms(kind, w, g, s, lr, **adam):
    """Sum of the magnitudes of the terms forming each output (new w, then each new slot), float64."""
    aw, ag = np.abs(w), np.abs(g)
    if kind == "adam":
        b1, b2 = adam["beta1"], adam["beta2"]
        mm, vv = b1 * np.abs(s[0]) + (1 - b1) * ag, b2 * s[1] + (1 - b2) * g * g
        return [aw + OO.adam_lr(lr, adam["t"], b1, b2) * mm / (np.sqrt(vv) + adam["epsilon"]), mm, vv]
    w1, s1 = OO.update(kind, w, g, s, lr, MU)
    if kind == "gd":
        return [aw + lr * ag]
    if kind == "momentum":
        a = MU * np.abs(s[0]) + ag
        return [aw + lr * a, a]
    if kind == "adagrad":
        return [aw + np.abs(w1 - w), s1[0]]
    if kind == "adadelta":
        return [aw + np.abs(w1 - w), s1[0], s1[1]]                  # both slots: sums of two non-negative terms
    mom = MU * np.abs(s[1]) + np.abs(s1[1] - MU * s[1])               # mu * mom and lr * g / sqrt(ms + eps) may cancel
    return [aw + mom, s1[0], mom]


def rule_errors(kind, eng, w0, s0, gc, lr, rule):
    """Every weight and slot of `eng` after one update of weights w0 and slots s0 (fp32, per variable) with the flat
    clipped fp32 gradient gc, against the fp64 rule at the module docstring's bar (16 u for adam, 32 u for the others).
    `rule`: adam's t / beta1 / beta2 / epsilon.  Returns ([(variable, output, error / bar)] of the violations, the
    largest error / bar)."""
    nu = 16 if kind == "adam" else 32
    shapes = eng.param_shapes()
    off, bad, worst = 0, [], 0.0
    for n in shapes:
        k = int(np.prod(shapes[n]))
        g = gc[off:off + k].reshape(shapes[n]).astype(np.float64)
        off += k
        s = [a.astype(np.float64) for a in s0[n]]
        want = OO.update(kind, w0[n].astype(np.float64), g, s, lr, MU, **rule)
        bars = _terms(kind, w0[n].astype(np.float64), g, s, lr, **rule)
        got = [eng.get_param(n)] + [eng.get_optimizer_slot(n, i) for i in range(len(s))]
        for j, (gv, wv, b) in enumerate(zip(got, [want[0]] + want[1], bars)):
            ratio = np.abs(gv.astype(np.float64) - wv) / (nu * U * b + 1e-44)
            worst = max(worst, float(ratio.max()))
            if not (ratio <= 1).all():
                bad.append((n, j, float(ratio.max())))
    assert off == gc.size
    return bad, worst


def adam_rule(t, beta1=0.9, beta2=0.999, epsilon=1e-8):
    """OO.update's adam arguments for update t of an engine configured with these values: the fp32 values it holds."""
    f32 = lambda a: float(np.float32(a))
    return dict(t=t, beta1=f32(beta1), beta2=f32(beta2), epsilon=f32(epsilon))


ADAM_CFG = dict(beta1=0.5, beta2=0.9, epsilon=1e-3)      # not the defaults: a constant baked into the kernel fails
KERNEL_CASES = ([(k, m, None, {}) for k in KINDS + ("adam",) for m in ("noclip", "clip", "avg")]
                + [("adam", "clip", t, {}) for t in (0, 1, 9, 999, 10 ** 6)] + [("adam", "clip", 1, ADAM_CFG)])


def _kernel_id(c):
    kind, mode, t, adam = c
    return "%s-%s" % (kind, mode) + ("" if t is None else "-t%d" % t) + ("-b0.5-0.9-e1e-3" if adam else "")


@pytest.mark.parametrize("kind,mode,t0,adam", KERNEL_CASES, ids=[_kernel_id(c) for c in KERNEL_CASES])
def test_optimizer_kernel_matches_fp64_rule(kind, mode, t0, adam):
    """One update from chosen gradients and slots: zeros, tiny (1e-20), ordinary and large (1e3) values of both signs
    (Adam's v: of one sign), with clipping off, with clipping that triggers, and through apply_gradients_avg with
    grad_scale = 0.5.  Adam also starts from update counts set through set_adam_step (the checkpoint-resume path: the
    update is then number t0 + 1) and from a non-default beta1 / beta2 / epsilon."""
    cfg, _, eng = _engine(SMALL, kind, clip=0.0 if mode == "noclip" else 5.0, **adam)
    x, x2, y = _batch(cfg, 1, 8, 8, 1)
    eng.train_step_host(x, x2, y, lr=0.01, seed=1, apply_update=False)
    shapes = eng.param_shapes()
    names = list(shapes)
    gt = eng.grad_tensor()
    total = int(gt.numel()) - 2
    r = np.random.RandomState(7)
    mag = np.choose(r.randint(0, 4, total), [np.zeros(total), np.full(total, 1e-20), 10.0 ** r.uniform(-4, 0, total),
                                             10.0 ** r.uniform(2, 3, total)])
    raw = (mag * np.where(r.rand(total) < 0.5, -1.0, 1.0)).astype(np.float32)
    gt[:total] = torch.from_numpy(raw).to(gt.device)
    w0, s0, off = {}, {}, 0
    for n in names:
        k = int(np.prod(shapes[n]))
        w0[n] = eng.get_param(n)
        s0[n] = []
        for i, init in enumerate(OO.SLOT_INIT[kind]):
            if kind == "adam":                                        # m signed, v >= 0, the gradients' magnitudes
                v = np.choose(r.randint(0, 4, k), [np.zeros(k), np.full(k, 1e-20), 10.0 ** r.uniform(-4, 0, k),
                                                   10.0 ** r.uniform(2, 3, k)])
                v = v * np.where(r.rand(k) < 0.5, -1.0, 1.0) if i == 0 else v
            elif (kind, i) in (("momentum", 0), ("rmsprop", 1)):     # signed slots
                v = r.randn(k) * 10.0 ** r.uniform(-4, 0, k)
            else:                                                     # accumulators: positive
                v = 10.0 ** r.uniform(-3, 0, k)
            s0[n].append(v.astype(np.float32).reshape(shapes[n]))
            (eng.set_adam_slot if kind == "adam" else eng.set_optimizer_slot)(n, i, s0[n][i])
        off += k
    assert off == total
    if t0 is not None:
        eng.adam_step = t0
    lr = 0.01
    if mode == "avg":
        eng.apply_gradients_avg(lr, 0.5)
        g32 = raw * np.float32(0.5)
    else:
        eng.apply_gradients(lr)
        g32 = raw
    torch.cuda.synchronize()
    rule = {}
    if kind == "adam":
        assert eng.adam_step == (t0 or 0) + 1
        rule = adam_rule((t0 or 0) + 1, **adam)
        lr = float(np.float32(lr))                                    # the fp32 lr the ABI passes
    scale = np.float32(1.0)
    if mode != "noclip":
        norm = np.float32(np.sqrt(np.sum(g32.astype(np.float64) ** 2)))
        assert norm > 5.0                                             # the clip triggers
        scale = np.float32(5.0) / max(norm, np.float32(5.0))
    gc = (g32 * scale).astype(np.float32)
    bad, worst = rule_errors(kind, eng, w0, s0, gc, lr, rule)
    eng.close()
    print("%s: largest error / bar: %.3f" % (_kernel_id((kind, mode, t0, adam)), worst))
    assert not bad, bad[:8]


def _propagate(kind, st, g, E, lr):
    """First-order bound of the error of weight and slots after one more step, given the oracle's slots before it
    (`st["s"]`), the clipped gradient g and its error bound E.  st carries the slot errors ("ds") and weight error ("dw")."""
    s, ds = st["s"], st["ds"]
    ag = np.abs(g)
    if kind == "gd":
        dstep = lr * E
    elif kind == "momentum":
        ds = [MU * ds[0] + E]
        dstep = lr * ds[0]
    elif kind == "adagrad":
        acc = s[0] + g * g
        dacc = ds[0] + 2 * ag * E + E * E
        dstep = lr * (E / np.sqrt(s[0]) + ag * ds[0] / (2 * acc ** 1.5))
        ds = [dacc]
    elif kind == "adadelta":
        rho, eps = OO.ADADELTA_RHO, OO.ADADELTA_EPS
        acc = rho * s[0] + (1 - rho) * g * g
        dacc = rho * ds[0] + (1 - rho) * (2 * ag * E + E * E)
        su = np.sqrt(s[1] + eps)
        u = su / np.sqrt(acc + eps) * g
        du = su / np.sqrt(rho * s[0] + eps) * E + su * ag * rho * ds[0] / (2 * (acc + eps) ** 1.5) \
            + np.abs(u) * ds[1] / (2 * (s[1] + eps))
        ds = [dacc, rho * ds[1] + (1 - rho) * (2 * np.abs(u) * du + du * du)]
        dstep = lr * du
    else:
        rho, eps = OO.RMSPROP_RHO, OO.RMSPROP_EPS
        ms = rho * s[0] + (1 - rho) * g * g
        dms = rho * ds[0] + (1 - rho) * (2 * ag * E + E * E)
        dmom = MU * ds[1] + lr * (E / np.sqrt(rho * s[0] + eps) + ag * rho * ds[0] / (2 * (ms + eps) ** 1.5))
        ds = [dms, dmom]
        dstep = dmom
    st["ds"] = ds
    st["dw"] = st["dw"] + dstep


@pytest.mark.parametrize("graph", ["tc", "ds"])
@pytest.mark.parametrize("kind", KINDS)
def test_three_steps_match_oracle_and_forward_follows(kind, graph):
    """Three train steps (dropout 0.8, masks replayed) against fp64 autograd + clip + the fp64 rule, on a tensor-core graph
    and a depthwise-separable one; then the forward must use the updated weights."""
    kw, rel = (SMALL, 2e-3) if graph == "tc" else (DS4, 2e-4)
    n, h, w = 2, 12, 12
    cfg, wts, eng = _engine(kw, kind, seed=9)
    x, x2, y = _batch(cfg, n, h, w, 10)
    orc = O.Oracle(cfg, wts, torch.float64)
    slots = OO.init_slots(kind, wts)
    lr = 0.002
    st = {k: {"ds": [np.zeros_like(v) for _ in OO.SLOT_INIT[kind]], "dw": np.zeros_like(v)} for k, v in wts.items()}
    worst = 0.0
    for step in range(1, 4):
        seed = 500 + step
        eng.train_step_host(x, x2, y, lr=lr, seed=seed)
        masks = {}
        for scope, k, cin, cout, bias, act in O.layer_table(cfg):
            if act:
                masks[scope] = np.ascontiguousarray(eng.dropout_mask(scope, seed, n, h, w, cout).transpose(0, 3, 1, 2)).astype(np.float64)
        _, _, grads = orc.loss_and_grads(x.astype(np.float64), x2.astype(np.float64), y.astype(np.float64), keep_prob=0.8, masks=masks)
        clipped, norm = orc.clip_by_global_norm(grads)
        sc = cfg.clipping_norm / max(norm, cfg.clipping_norm)
        for name in wts:
            st[name]["s"] = slots[name]
            E = sc * (rel * np.abs(grads[name]).max() + 2e-3 * np.abs(grads[name]))
            _propagate(kind, st[name], clipped[name], E, lr)
        OO.optimizer_step(orc, kind, clipped, slots, lr, MU)
        for name in wts:
            tol = 2 * st[name]["dw"] + 2e-3 * lr * step + 4 * U * np.abs(orc.w[name]) + 1e-9
            err = np.abs(eng.get_param(name) - orc.w[name])
            worst = max(worst, float((err / tol).max()))
            assert (err <= tol).all(), (step, name, float((err - tol).max()))
    for name in wts:
        for i, sv in enumerate(slots[name]):
            dtol = 2 * st[name]["ds"][i] + 1e-6 * np.abs(sv) + 1e-12
            assert (np.abs(eng.get_optimizer_slot(name, i) - sv) <= dtol).all(), (name, i)
    print("%s/%s: largest weight error / bar over 3 steps: %.3f" % (kind, graph, worst))
    yy = eng.forward_host(x, x2)
    ref = O.Oracle(cfg, {k: a.astype(np.float64) for k, a in orc.w.items()}, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64))
    assert np.abs(yy - ref).max() <= 5e-3
    eng.close()


def test_gd_step_that_shrinks_a_layer_past_its_packed_scale_falls_back_to_the_host_repack():
    """The device refresh keeps each packed layer's power-of-two scale while max |w * scale| stays in [2048, 49152]. A gd
    step with gradient w on Up-PS and lr 31/32 divides that layer by 32, out of the window: the host re-pack takes over,
    and the forward matches fp64 on the new weights and a fresh engine packed from them."""
    from helper import engine as E
    cfg, wts, eng = _engine(SMALL, "gd", keep=1.0, clip=0.0)
    x, x2, y = _batch(cfg, 2, 10, 10, 4)
    eng.train_step_host(x, x2, y, lr=0.0, seed=1)               # first update: host pack, then the device refresh maps
    eng.train_step_host(x, x2, y, lr=0.0, seed=2)               # an update through the device refresh
    eng.train_step_host(x, x2, y, lr=0.0, seed=3, apply_update=False)
    shapes = eng.param_shapes()
    before = {k: eng.get_param(k) for k in shapes}
    target = "Up-PS/Up-PS_CNN/conv_W"
    g = np.concatenate([(before[k] if k == target else np.zeros_like(before[k])).ravel() for k in shapes])
    gt = eng.grad_tensor()
    gt[:g.size] = torch.from_numpy(g).to(gt.device)
    eng.apply_gradients(31 / 32)
    torch.cuda.synchronize()
    after = {k: eng.get_param(k) for k in shapes}
    np.testing.assert_allclose(after[target], before[target] / 32, rtol=2.0 ** -22, atol=0)
    assert all(np.array_equal(after[k], before[k]) for k in shapes if k != target)
    yy = eng.forward_host(x, x2)
    ref = O.Oracle(cfg, {k: v.astype(np.float64) for k, v in after.items()}, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64))
    assert np.abs(yy - ref).max() <= 1e-3
    fresh = E.Engine(E.make_config(dropout_keep=1.0, **SMALL))
    fresh.set_params(after)
    assert np.abs(fresh.forward_host(x, x2) - yy).max() <= 1e-5
    fresh.close()
    eng.close()


GROW_CASES = [("Up-PS", None, "Up-PS/Up-PS_CNN/conv_W"),
              # R-CNN1 itself is an fp32 gather: only the folded upsampler's image (its wmax slot) leaves its window
              ("R-CNN1-folded-L12-x2", "dcscn_L12_F196to48_NIN_A64_PS_R1F32", "R-CNN1/conv_W")]


@pytest.mark.parametrize("weights,target", [c[1:] for c in GROW_CASES], ids=[c[0] for c in GROW_CASES])
def test_gd_step_that_grows_a_layer_past_its_packed_scale_falls_back_to_the_host_repack(weights, target):
    """The other edge of the window: a gd step with gradient -w on one variable and lr 7 multiplies it by 8.  The packed
    scale put max |w * scale| in (8192, 16384]; eight times that is past 49152, and past fp16's 65504, so the old scale
    would pack inf (four times would stay finite where max |w * scale| <= 16376).  The host re-pack takes over: the
    forward matches fp64 on the new weights and a fresh engine packed from them.  Inputs in [0, 1] keep the fp64 bar of
    the shrink test meaningful at the full L12 width."""
    from conftest import MODEL_FLAGS, load_golden_weights
    from helper import engine as E
    kw = SMALL if weights is None else MODEL_FLAGS[weights]
    cfg = O.OracleConfig(**kw)
    w = O.he_init_weights(cfg, seed=3) if weights is None else load_golden_weights(weights)
    eng = E.Engine(E.make_config(dropout_keep=1.0, clipping_norm=0.0, optimizer="gd", **kw))
    eng.set_params(w)
    x, x2, y = (a / np.float32(255) for a in _batch(cfg, 1, 10, 12, 4))
    eng.train_step_host(x, x2, y, lr=0.0, seed=1)               # first update: host pack, then the device refresh maps
    eng.train_step_host(x, x2, y, lr=0.0, seed=2)               # an update through the device refresh
    eng.train_step_host(x, x2, y, lr=0.0, seed=3, apply_update=False)
    shapes = eng.param_shapes()
    before = {k: eng.get_param(k) for k in shapes}
    g = np.concatenate([(-before[k] if k == target else np.zeros_like(before[k])).ravel() for k in shapes])
    gt = eng.grad_tensor()
    gt[:g.size] = torch.from_numpy(g).to(gt.device)
    eng.apply_gradients(7.0)
    torch.cuda.synchronize()
    after = {k: eng.get_param(k) for k in shapes}
    np.testing.assert_allclose(after[target], before[target] * 8, rtol=2.0 ** -22, atol=0)
    assert all(np.array_equal(after[k], before[k]) for k in shapes if k != target)
    yy = eng.forward_host(x, x2)
    assert np.isfinite(yy).all()
    ref = O.Oracle(cfg, {k: v.astype(np.float64) for k, v in after.items()}, torch.float64).forward(x.astype(np.float64), x2.astype(np.float64))
    err = float(np.abs(yy - ref).max())
    fresh = E.Engine(E.make_config(dropout_keep=1.0, **kw))
    fresh.set_params(after)
    err_host = float(np.abs(fresh.forward_host(x, x2) - yy).max())
    fresh.close()
    eng.close()
    print("%s x8: max |y - oracle(fp64)| = %.3e, max |y - fresh host pack| = %.3e" % (target, err, err_host))
    assert err <= 1e-3
    assert err_host <= 1e-5


# ------------------------------------------------------------------------------------------------- checkpoints ----
CD = ["--scale=2", "--layers=7", "--filters=32", "--min_filters=8", "--filters_decay_gamma=1.2", "--nin_filters=24",
      "--nin_filters2=8", "--reconstruct_layers=0", "--pixel_shuffler_filters=1"]


def _model(tmp_path, kind):
    from test_gpu_psnr import build_model
    m = build_model(tmp_path, CD + ["--optimizer=" + kind, "--momentum=0.8"], 1)
    m.checkpoint_dir = str(tmp_path / "ckpt")
    return m


@pytest.mark.parametrize("kind", KINDS)
def test_checkpoint_holds_trainables_and_the_optimizers_slots(tmp_path, kind):
    from helper import engine as E, tf_bundle
    m = _model(tmp_path, kind)
    shapes = m.engine.param_shapes()
    suffixes = [s for s, _ in E.OPTIMIZER_SLOTS[kind]]
    path = os.path.join(m.checkpoint_dir, m.name + ".ckpt")
    m.save_model()                                              # before any step: the initial slot values
    r = tf_bundle.BundleReader(path)
    assert set(r.keys()) == set(shapes) | {v + s for v in shapes for s in suffixes}
    for v in shapes:
        for s, init in E.OPTIMIZER_SLOTS[kind]:
            assert np.array_equal(r.get_tensor(v + s), np.full(shapes[v], init, np.float32)), (v, s)
    g = np.random.RandomState(0)
    x = (g.rand(4, 16, 16, 1) * 255).astype(np.float32)
    x2 = (g.rand(4, 32, 32, 1) * 255).astype(np.float32)
    for i in range(2):
        m.engine.train_step_host(x, x2, x2 + 3, lr=1e-3, seed=i)
    m.save_model()
    r = tf_bundle.BundleReader(path)
    assert set(r.keys()) == set(shapes) | {v + s for v in shapes for s in suffixes}     # no beta powers
    moved = False
    for v in shapes:
        for i, (s, init) in enumerate(E.OPTIMIZER_SLOTS[kind]):
            assert np.array_equal(r.get_tensor(v + s), m.engine.get_optimizer_slot(v, i))
            moved |= not np.array_equal(r.get_tensor(v + s), np.full(shapes[v], init, np.float32))
    assert moved or kind == "gd"
    with pytest.raises(E.EngineError, match="not adam"):
        m.engine.get_adam_slot("CNN1/conv_W", 0)
    for reset in (m.engine.reset_optimizer, m.init_all_variables):
        m.engine.train_step_host(x, x2, x2 + 3, lr=1e-3, seed=5)
        reset()
        assert m.engine.adam_step == 0
        for v in shapes:
            for i, (s, init) in enumerate(E.OPTIMIZER_SLOTS[kind]):
                assert np.array_equal(m.engine.get_optimizer_slot(v, i), np.full(shapes[v], init, np.float32)), (reset, v, s)


@pytest.mark.parametrize("kind", ["momentum", "rmsprop"])
def test_resumed_run_takes_the_uninterrupted_step(tmp_path, kind):
    m = _model(tmp_path, kind)
    shapes = m.engine.param_shapes()
    g = np.random.RandomState(0)
    x = (g.rand(4, 16, 16, 1) * 255).astype(np.float32)
    x2 = (g.rand(4, 32, 32, 1) * 255).astype(np.float32)
    y = (g.rand(4, 32, 32, 1) * 255).astype(np.float32)
    for i in range(3):
        m.engine.train_step_host(x, x2, y, lr=1e-3, seed=i)
    m.save_model()
    m.engine.train_step_host(x, x2, y, lr=1e-3, seed=7)         # the uninterrupted run's 4th step
    want = {v: m.engine.get_param(v) for v in shapes}
    m2 = _model(tmp_path, kind)
    m2.load_model(restore_optimizer=True)
    m2.engine.train_step_host(x, x2, y, lr=1e-3, seed=7)
    for v in shapes:
        assert np.abs(m2.engine.get_param(v) - want[v]).max() <= 1e-5, v
    m3 = _model(tmp_path, kind)                                 # without the slots the step differs
    m3.load_model()
    m3.engine.train_step_host(x, x2, y, lr=1e-3, seed=7)
    assert max(float(np.abs(m3.engine.get_param(v) - want[v]).max()) for v in shapes) > 1e-4


def test_train_cli_with_momentum_writes_momentum_slots(tmp_path):
    from helper import tf_bundle
    ckpt = tmp_path / "ckpt"
    cmd = [sys.executable, os.path.join(PKG, "train.py")] + CD + [
        "--optimizer=momentum", "--self_ensemble=1", "--dataset=set5", "--test_dataset=set5", "--training_images=16",
        "--batch_num=8", "--batch_image_size=16", "--lr_decay_epoch=1", "--lr_decay=0.01", "--end_lr=1e-5",
        "--data_dir=" + os.path.join(GOLDEN, "data"), "--batch_dir=" + str(tmp_path / "batch"),
        "--checkpoint_dir=" + str(ckpt), "--log_filename=" + str(tmp_path / "log.txt"),
        "--tf_log_dir=" + str(tmp_path / "tf_log"), "--graph_dir=" + str(tmp_path / "graphs"),
        "--output_dir=" + str(tmp_path / "out")]
    r = subprocess.run(cmd, cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    log = open(tmp_path / "log.txt").read()
    assert re.search(r"Model Average \[set5\] PSNR:([0-9.]+), SSIM:", log), log
    rd = tf_bundle.BundleReader(str(ckpt / "dcscn_L7_F32to8_G1.20_NIN_A24_B8_PS_R1F32.ckpt"))
    keys = set(rd.keys())
    assert "CNN1/conv_W/Momentum" in keys and "R-CNN1/conv_W/Momentum" in keys
    assert not any(k.endswith(("/Adam", "/Adam_1")) for k in keys) and "beta1_power" not in keys
    assert np.abs(rd.get_tensor("CNN1/conv_W/Momentum")).max() > 0


# ---------------------------------------------------------------------------------------------- data parallel ----
def _dp_worker(rank, world, port, out_dir, kind):
    sys.path.insert(0, PKG)
    sys.path.insert(0, os.path.join(os.path.dirname(PKG), "oracle"))
    import torch.distributed as dist
    import dcscn_oracle as O_
    from helper import engine as E
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    eng = E.Engine(E.make_config(device_id=rank, dropout_keep=1.0, optimizer=kind, **SMALL))
    eng.set_params(O_.he_init_weights(O_.OracleConfig(**SMALL), seed=11))
    g = np.random.RandomState(5)
    x = (g.rand(4, 12, 12, 1) * 255).astype(np.float32)
    x2 = (g.rand(4, 24, 24, 1) * 255).astype(np.float32)
    y = (g.rand(4, 24, 24, 1) * 255).astype(np.float32)
    for step in range(2):
        eng.train_step_data_parallel(np.ascontiguousarray(x[rank::world]), np.ascontiguousarray(x2[rank::world]),
                                     np.ascontiguousarray(y[rank::world]), lr=0.002, seed=7 + step)
    np.save(os.path.join(out_dir, "w%d.npy" % rank), eng.get_param("CNN2/conv_W"))
    eng.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("kind", ["momentum", "rmsprop"])
def test_two_rank_data_parallel_steps_equal_whole_batch(tmp_path, kind):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from helper import engine as E
    port = 29500 + os.getpid() % 200
    mp.spawn(_dp_worker, args=(2, port, str(tmp_path), kind), nprocs=2, join=True)
    eng = E.Engine(E.make_config(dropout_keep=1.0, optimizer=kind, **SMALL))
    eng.set_params(O.he_init_weights(O.OracleConfig(**SMALL), seed=11))
    g = np.random.RandomState(5)
    x = (g.rand(4, 12, 12, 1) * 255).astype(np.float32)
    x2 = (g.rand(4, 24, 24, 1) * 255).astype(np.float32)
    y = (g.rand(4, 24, 24, 1) * 255).astype(np.float32)
    for step in range(2):
        eng.train_step_host(x, x2, y, lr=0.002, seed=7 + step)
    w_single = eng.get_param("CNN2/conv_W")
    w0, w1 = np.load(tmp_path / "w0.npy"), np.load(tmp_path / "w1.npy")
    np.testing.assert_array_equal(w0, w1)                       # replicas stay identical
    step = np.abs(w_single - O.he_init_weights(O.OracleConfig(**SMALL), seed=11)["CNN2/conv_W"]).max()
    assert np.abs(w0 - w_single).max() <= 1e-3 * step + 1e-7    # linear-ish in g: the sum order of the all-reduce
    eng.close()


# ------------------------------------------------------------------------------------------------ convergence ----
def train_200(tmp_path, kind, lr):
    """c-DCSCN x2 from the 'he' initialisation, 200 steps on Set14 grid patches, Set5 PSNR every 50 steps (the protocol of
    test_gpu_convergence.py).  Returns (PSNR curve, running mean losses)."""
    import glob
    import random
    from helper import args as A
    import DCSCN
    random.seed(1234)
    np.random.seed(1234)
    f = A._Flags()
    for name, (k, default, help_text) in A.FLAGS._defs.items():
        f._define(name, default, help_text, k)
    f.parse(["prog"] + CD + ["--optimizer=" + kind, "--initial_lr=%g" % lr,
             "--self_ensemble=1", "--batch_num=20", "--batch_image_size=32", "--build_batch=true",
             "--data_dir=" + os.path.join(GOLDEN, "data"), "--dataset=set14", "--batch_dir=" + str(tmp_path / "batch"),
             "--checkpoint_dir=" + str(tmp_path / "ckpt"), "--log_filename=" + str(tmp_path / "log.txt"),
             "--tf_log_dir=" + str(tmp_path / "tf_log"), "--graph_dir=" + str(tmp_path / "graphs"),
             "--output_dir=" + str(tmp_path / "out")])
    m = DCSCN.SuperResolution(f, model_name=f.model_name)
    m.load_datasets(f.data_dir + "/" + f.dataset, f.batch_dir + "/" + f.dataset, f.batch_image_size, f.stride_size)
    m.build_graph()
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
    m.engine.close()
    return curve, losses


def test_200_momentum_steps_on_real_patches_raise_set5_psnr(tmp_path):
    """At the reference's default lr (0.002) momentum took Set5 from 8.0 to 34.7 dB on one H100; the bar leaves room for
    the random patch order."""
    curve, losses = train_200(tmp_path, "momentum", 0.002)
    print("momentum: Set5 PSNR at steps 0/50/100/150/200:", ["%.2f" % p for p in curve])
    assert all(np.isfinite(curve))
    assert curve[-1] >= curve[0] + 8.0, curve
    assert curve[-1] >= 28.0, curve
    assert losses[-1] < losses[0]
