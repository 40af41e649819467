"""
The train step's own forward, layer by layer, and every activator on the tensor-core path, against the isolated fp64
references of test_gpu_forward_paths.isolated_layers (the forward) and test_gpu_backward_paths.check_step (the
backward): each layer recomputed from the input the GPU itself stored, so each bar follows from one kernel's arithmetic.

The training forward is its own program (train_engine.inc, train_step_impl): every activated epilogue applies dropout
(v fp32(1 / keep), or exactly 0 where dcscn_dropout_mask drops the element) and, for prelu and leaky_relu, stores the fp16
min(z, 0) plane of the pre-dropout z (zneg_value, epilogue.cuh); CNN1 runs conv_first3x3_kernel<true> or
conv_first_kernel with that store; the last layer is never fused; R-CNN1 runs conv_last_direct_kernel or
conv_last_kernel on the materialised pixel-shuffler output.  After a step the engine's activations hold that forward, so
  * every layer is held to the inference f16x3 bars (seg_chunks at its default) with the step's dropout masks, and y_
    to R-CNN1 of the stored pixel-shuffler output plus x2 at the unfused bar;
  * zneg: with B_z the bar of the pre-activation, z < -B_z stores zneg < 0 within half an fp16 ulp of |z| + B_z of z (a
    z in (-2^-24, 0) is stored as -2^-24), z > B_z stores exactly 0, also where dropout zeroed the output;
  * the PReLU slope gradient against sum g z over z < 0 with the isolated z: the fp16 plane adds up to 2^-11 sum |g z|,
    which the bar carries explicitly and the printed error / sum |g z| makes visible.
"""
import math

import numpy as np
import pytest
import torch

import activator_oracle as A
import dcscn_oracle as O
from conftest import MODEL_FLAGS
from test_gpu_backward_paths import L12, Checker, check_step, dev, real_engine, real_patches, release_reference_memory  # noqa: F401
from test_gpu_forward import SMALL, gpu_forward, make_engine
from test_gpu_forward_paths import FIRST3, TC_CASES, isolated_layers, nchw, stored_rounding
from test_gpu_train import FAST, GRADIENT_CASES, SMALL as TSMALL, assert_kernels_ran, launched_kernels, setup

pytestmark = pytest.mark.gpu

U24 = 2.0 ** -24
ACTS = A.ACTIVATORS[1:]
SEED = 1234


def masks_of(eng, cfg, seed, n, h, w):
    return {scope: eng.dropout_mask(scope, seed, n, h, w, cout)
            for scope, k, cin, cout, bias, _ in O.layer_table(cfg) if A.activated(scope)}


def zneg_ratio(zn, z, bz):
    """max err / bar of one layer's min(z, 0) plane `zn` against the isolated pre-activation z (bar bz of the GPU's z),
    all fp64 NCHW tensors on one device (module docstring)."""
    half_ulp = 0.5 * stored_rounding(torch.clamp(z.abs() + bz, max=65504.0), 1)
    tiny = (z < bz) & (z > -(U24 + bz))          # the fp32 z may lie in (-2^-24, 0): stored as -2^-24
    ratio = (zn - z).abs() / (half_ulp + bz + torch.where(tiny, U24, 0.0))
    ratio = torch.where(z > bz, torch.where(zn == 0, 0.0, float("inf")), ratio)
    ratio = torch.where((zn > 0) | ((z < -bz) & (zn >= 0)), float("inf"), ratio)
    return float(ratio.max())


def zneg_ratios(eng, pre, n, h, wd):
    """{zneg <layer>: max err / bar} of the min(z, 0) planes against the isolated pre-activations."""
    return {"zneg " + scope: zneg_ratio(nchw(eng.get_train_tensor("zneg:" + scope, (n, h, wd, z.shape[1])), z.device), z, bz)
            for scope, (z, bz) in pre.items()}


class SlopeSums:
    """Per-channel sums over images of the PReLU slope gradient's reference: sum g z over the isolated z < 0 and its
    bar terms, added one slice of images at a time (add), then compared with the GPU's gradients (ratios)."""

    def __init__(self):
        self.sums = {}

    def add(self, scope, gm, z, bz):
        gz = torch.where(z < 0, gm * z, torch.zeros_like(gm))
        terms = (gz.sum(dim=(0, 2, 3)), gz.abs().sum(dim=(0, 2, 3)), (gm.abs() * (bz + U24) * (z < bz)).sum(dim=(0, 2, 3)))
        old = self.sums.get(scope)
        self.sums[scope] = terms if old is None else tuple(a + b for a, b in zip(old, terms))

    def ratios(self, eng, n, h, wd, scale):
        """{slope <layer>: (max err / bar, max err / (sum |g z| / G))}.  The GPU sums g zneg in fp32 ((npx + 4) 2^-24
        sum |g z|); zneg is the fp32 z (within B_z, and the sign is open where |z| <= B_z) stored in fp16 (2^-11 |z|, or
        -2^-24 for z in (-2^-24, 0))."""
        G = 2.0 ** round(math.log2(n * scale * h * scale * wd / 2.0))
        npx = n * h * wd
        out = {}
        for scope, (sgzs, sgz, extra) in self.sums.items():
            bar = (npx + 4) * U24 * sgz + 2.0 ** -11 * sgz + extra
            ref = sgzs / G
            bar = bar / G + U24 * ref.abs() + 1e-45
            got = torch.from_numpy(eng.get_grad("%s/prelu/%s_prelu" % (scope, scope))).to(sgz.device, torch.float64)
            err = (got - ref).abs()
            out["slope " + scope] = (float((err / bar).max()), float((err / (sgz / G + 1e-45)).max()))
        return out


def slope_ratios(eng, pre, chk, n, h, wd, scale):
    """SlopeSums.ratios of the whole batch, with the output gradients check_step formed."""
    sums = SlopeSums()
    for scope, (z, bz) in pre.items():
        sums.add(scope, chk.gm[scope], z.to(dev()), bz.to(dev()))
    return sums.ratios(eng, n, h, wd, scale)


def captured_step(kw, wts, act, keep, x, x2, y, kernels):
    """(engine, its dropout masks or None) after one captured train step (apply_update = False) that reached
    `kernels`."""
    from helper import engine as E
    cfg = O.OracleConfig(**kw)
    n, h, wd = x.shape[:3]
    eng = E.Engine(E.make_config(dropout_keep=keep, activator=act, **kw))
    eng.set_params({k: v.astype(np.float32) for k, v in wts.items()})
    eng.set_option("grad_capture", 1)
    _, names = launched_kernels(lambda: eng.train_step_host(x, x2, y, lr=0.002, seed=SEED, apply_update=False))
    first = []
    if any(k.startswith("conv_first3x3_kernel") for k in kernels):     # the min(z, 0) store is a template argument
        first = ["conv_first3x3_kernel<%s>" % ("true" if act in ("prelu", "leaky_relu") else "false")]
    assert_kernels_ran(names, kernels + first + ["loss_kernel", "act_grad8_kernel"])
    return eng, (masks_of(eng, cfg, SEED, n, h, wd) if keep < 1.0 else None)


def train_case(kw, wts, act, keep, x, x2, y, kernels, tag):
    """One captured train step (apply_update = False): the kernels it reached, then every forward layer, y_, the zneg
    planes, the PReLU slope gradients and every backward kernel (check_step) against their isolated references.  All
    violations are reported at once."""
    cfg = O.OracleConfig(**kw)
    n, h, wd = x.shape[:3]
    s = cfg.scale
    eng, masks = captured_step(kw, wts, act, keep, x, x2, y, kernels)
    yp = eng.get_train_tensor("y_", (n, s * h, s * wd, 1))
    pre = {}
    ratios = isolated_layers(eng, cfg, wts, x, x2, yp, 2, 0, False, act=act, masks=masks, keep=keep, pre=pre)
    chk = check_step(eng, kw, wts, x, x2, y, keep, SEED, Checker(), act=act)
    if act in ("prelu", "leaky_relu"):
        ratios.update(zneg_ratios(eng, pre, n, h, wd))
    if act == "prelu":
        slopes = slope_ratios(eng, pre, chk, n, h, wd, s)
        print(tag, "slope gradient error / sum |g z|:", " ".join("%s %.3g" % (k, v[1]) for k, v in slopes.items()))
        ratios.update({k: v[0] for k, v in slopes.items()})
    eng.close()
    print(tag, "forward error / bar:", " ".join("%s %.3f" % kv for kv in ratios.items()))
    print(tag, "backward error / bar:", " ".join("%s %.3g" % kv for kv in sorted(chk.worst.items())))
    bad = [(k, v) for k, v in ratios.items() if not v <= 1.0] + chk.bad()
    assert not bad, bad


# ------------------------------------------------------------------------ (1, 2) the train forward, per layer ----
@pytest.mark.parametrize("kw,weights,keep,shape,kernels", [c[1:] for c in GRADIENT_CASES], ids=[c[0] for c in GRADIENT_CASES])
def test_train_forward_isolated(kw, weights, keep, shape, kernels):
    """The GRADIENT_CASES graphs (conv_last_direct vs conv_last, conv_first_kernel, 5 x 5, 1 x 1, c-DCSCN, x3, x4,
    1 x 1 images) on the inputs of test_gpu_train.setup."""
    cfg, wts, eng, x, x2, y = setup(kw, keep, *shape, weights=weights)
    eng.close()
    if weights != "he":
        kw = MODEL_FLAGS[weights]
    train_case(kw, wts, "prelu", keep, x, x2, y, kernels, shape)


def test_train_forward_on_real_patches():
    """The shipped L12 x2 checkpoint on Set5 / Set14 patches, y = ground truth, keep 0.8."""
    kw, wts, eng = real_engine(L12[2], 0.8)
    eng.close()
    x, x2, y = real_patches(2, 6, 32, 32, 37)
    train_case(kw, wts, "prelu", 0.8, x, x2, y, FAST, "L12-x2 real")


# ------------------------------------------------------------------ (3) every activator, inference forward ----
X2R = TC_CASES[0]
FWD_GRAPHS = [("x2", dict(SMALL, scale=2), (2, 9, 11), None), ("x3", dict(SMALL, scale=3), (2, 9, 11), None),
              ("x4", dict(SMALL, scale=4), (1, 9, 11), None), (X2R[0], X2R[1], X2R[2], X2R[3])]


@pytest.mark.parametrize("precision", [0, 1], ids=["f16x3", "f16x1"])
@pytest.mark.parametrize("kw,shape,kernels", [g[1:] for g in FWD_GRAPHS], ids=[g[0] for g in FWD_GRAPHS])
@pytest.mark.parametrize("act", ACTS)
def test_activator_forward_isolated(act, kw, shape, kernels, precision):
    """Every layer of a relu / leaky_relu / sigmoid / tanh / selu graph against its isolated fp64 reference (He-init
    weights of activator_oracle), fused and unfused where the planner fuses R-CNN1."""
    npl = 2 if precision == 0 else 1
    cfg = O.OracleConfig(**kw)
    w = A.he_init_weights(cfg, act, seed=0)
    n, h, wd = shape
    g = np.random.RandomState(n * 1000 + h * 10 + wd)
    x = (g.rand(n, h, wd, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, cfg.scale * h, cfg.scale * wd, 1) * 255).astype(np.float32)
    eng = make_engine(dict(kw, activator=act), w, precision)
    _, names = launched_kernels(lambda: gpu_forward(eng, x, x2))
    want = [k.format(P=npl) for k in kernels] if kernels else [FIRST3, "conv_tc_kernel<%d" % npl]
    assert_kernels_ran(names, want)
    fused = any("conv_last_gather" in k for k in names)
    worst, bad = {}, []
    for fuse in ((1, 0) if fused else (1,)):
        eng.set_option("fuse_last", fuse)
        y = gpu_forward(eng, x, x2)
        for name, ratio in isolated_layers(eng, cfg, w, x, x2, y, npl, 0, fused and fuse == 1, act=act).items():
            worst[name] = max(worst.get(name, 0.0), ratio)
            if not ratio <= 1.0:
                bad.append(("fuse_last=%d" % fuse, name, ratio))
    eng.close()
    print("error / bar:", " ".join("%s %.3f" % kv for kv in worst.items()))
    assert not bad, bad


# ------------------------------------------------------------------------ (4) every activator, train step ----
ACT_STEPS = {c[0]: c for c in GRADIENT_CASES if c[0] in ("x2-drop", "x4-drop")}


@pytest.mark.parametrize("case", ["x2-drop", "x4-drop", "zero"])
@pytest.mark.parametrize("act", ACTS)
def test_activator_train_step_isolated(act, case):
    """The train forward, the zneg planes (leaky_relu) and every backward kernel of a relu / leaky_relu / sigmoid / tanh /
    selu graph.  "zero": keep 1, a zero image and zero biases, so every CNN1 pre-activation is exactly 0 and the
    derivative there is TensorFlow's: 0 for relu, 1 for leaky_relu, lambda for selu."""
    if case == "zero":
        kw, keep, shape, kernels = TSMALL, 1.0, (2, 12, 10), FAST
    else:
        _, kw, _, keep, shape, kernels = ACT_STEPS[case]
    cfg = O.OracleConfig(**kw)
    wts = {k: v.astype(np.float64) for k, v in A.he_init_weights(cfg, act, seed=0).items()}
    n, h, wd = shape
    g = np.random.RandomState(1)
    s = cfg.scale
    x = (g.rand(n, h, wd, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, s * h, s * wd, 1) * 255).astype(np.float32)
    y = np.clip(x2 + g.randn(n, s * h, s * wd, 1) * 10, 0, 255).astype(np.float32)
    if case == "zero":
        x[:] = 0
        for k in wts:
            if k.endswith("conv_B"):
                wts[k][:] = 0
    train_case(kw, wts, act, keep, x, x2, y, kernels, "%s %s" % (act, case))
