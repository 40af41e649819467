"""
Backward parity of every kernel the train step can select, each against an isolated fp64 reference computed from the
values the GPU itself stored (option "grad_capture", dcscn_get_train_tensor; dcscn_get_activation for the forward
planes, which after a train step hold that step's forward after dropout).  No error comes in from the kernels before
the one under test, so each bar follows from that kernel's own arithmetic.  Gradient tensors carry the loss scale
G = grad_scale (a power of two); weights are quantised as pack_tc_layer packs the dgrad twins, each twin at its own
power-of-two scale (quantise, test_gpu_forward_paths.py).  With S = sum |a| |w| of an output's products:

  loss_kernel             dY = fp32(y_ - y) * fp32(2 G / count): 2^-22 |dY|
  last_wgrad_kernel<k*k>, last_wgrad_scalar_kernel, first_wgrad_kernel, wgrad_kernel
                          fp32 sums over the n pixels of the batch: n 2^-24 S
  last_dgrad_s2d[_rows]   k*k fp32 FMAs: k^2 2^-24 S, then the hi / lo store (stored_rounding: 2^-22 |v| + 2^-25)
  s2d_planes_kernel       a copy: bit for bit
  dgrad twins             conv_tc_kernel at K = k^2 cin_pad of the twin: tc_units + 1 (epilogue scale) 2^-23 S, stored
  act_grad[8]_kernel      dZ = (g1 + g2) * mask * fp32(1 / keep) * slope: 4 roundings, 2^-22 |dZ|, stored; bias and
                          slope sums are fp32 over the pixels: (n + 4) 2^-24 sum |terms|.  relu, sigmoid, tanh and selu
                          take f' from h = fp32(stored output * fp32(keep)), the f' of check_step's act_grad in fp64 from
                          that h: relu exact, sigmoid h (1 - h) 2 2^-24 |f'|, tanh 1 - h h 2^-24 (h^2 + |f'|), selu
                          h + lambda alpha 2^-24 |f'|; then one more rounding for the product
  wgrad_tc_kernel         one fp32 wgmma accumulator per (tap, 128 x n_pad tile) and CTA over chunks / ksplit chunks of
                          32 pixels, 6 k16 steps per chunk (a_lo z_hi, a_hi z_lo, a_hi z_hi, each over 2 x 16 pixels).
                          A step aligns its 16 products and the accumulator to the largest exponent and truncates each
                          (one truncation per step, the forward's model, was exceeded 3.4x on real L12 x2 patches, where
                          the long chain keeps |acc| far above a step's products): 6 ceil(chunks / ksplit) 17 2^-23 S;
                          the dropped a_lo z_lo: 2^-22 S; the
                          fixed-order reduce of ksplit partials and the add into dW: (ksplit + 1) 2^-24 S
  grad_finalize_kernel    get_grad = sum / G (exact) + l2 w (conv_W only), rounded once: 2^-24 |g| + 2^-24 |l2 w|
The bars include the 2^-25 absolute floor of the hi / lo planes, which real residuals reach: their small gradients have
subnormal lo planes (and at the extremes subnormal hi planes).
"""
import gc
import glob
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dcscn_oracle as O
from conftest import GOLDEN, MODEL_FLAGS, load_golden_weights
from test_gpu_forward_paths import LEAKY, SELU_SCALE, SELU_SCALE_ALPHA, quantise, tc_units
from test_gpu_train import CDCSCN, GRADIENT_CASES, assert_kernels_ran, launched_kernels, setup

pytestmark = pytest.mark.gpu

U22, U23, U24, U25 = 2.0 ** -22, 2.0 ** -23, 2.0 ** -24, 2.0 ** -25
L12 = {2: "dcscn_L12_F196to48_NIN_A64_PS_R1F32", 3: "dcscn_L12_F196to48_Sc3_NIN_A64_PS_R1F32",
       4: "dcscn_L12_F196to48_Sc4_NIN_A64_PS_R1F32"}


@pytest.fixture(autouse=True)
def release_reference_memory():
    """The fp64 references live in torch's caching allocator (21.5 GB reserved at the benchmark's shape on an H100).  Hand
    them back to the driver after every test, so the tests that follow in the same process - the engines' workspaces and
    the profiler that checks which kernels a case reaches - run with the device as they would on their own."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def pad16(v):
    return (v + 15) // 16 * 16


def cdiv(a, b):
    return -(-a // b)


def dev():
    return torch.device("cuda")


def t64(a):
    """NHWC numpy -> NCHW fp64 on the GPU (the references of the benchmark-size case would take minutes on the CPU)."""
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev(), torch.float64).permute(0, 3, 1, 2)


def hwio(w):
    """HWIO -> OIHW fp64 (torch conv2d weight)."""
    return torch.from_numpy(np.ascontiguousarray(w, dtype=np.float64)).to(dev()).permute(3, 2, 0, 1)


def dgrad(dz, w):
    """Gradient of conv2d(SAME, HWIO w) w.r.t. its input."""
    return F.conv_transpose2d(dz, hwio(w), padding=w.shape[0] // 2)


def wgrad(a, dz, k):
    """Gradient of conv2d(SAME) w.r.t. its HWIO filter: sum_p a[p + off(tap)] dz[p]."""
    g = torch.nn.grad.conv2d_weight(a, (dz.shape[1], a.shape[1], k, k), dz, padding=k // 2)
    return g.permute(2, 3, 1, 0)


def stored(v):
    """stored_rounding(v, 2) of test_gpu_forward_paths.py on GPU tensors: the hi / lo split of an fp32 value."""
    return U22 * v.abs() + U25


def s2d(x, r):
    """space_to_depth (the gradient of depth_to_space, DCR order): channel (i*r + j)*C + c."""
    n, c, h, w = x.shape
    return x.view(n, c, h // r, r, w // r, r).permute(0, 3, 5, 1, 2, 4).reshape(n, r * r * c, h // r, w // r)


def wgrad_tc_chain(sm, n, h, w, k, a_rows, dz_cols):
    """(ceil(chunks / ksplit), ksplit) of run_wgrad_tc (train_engine.inc) for one filter gradient."""
    taps = k * k
    cols16 = pad16(dz_cols)
    n_tiles = cdiv(cols16, 128)
    n_pad = pad16(cdiv(cols16, n_tiles))
    n_groups = cdiv(n_pad, 64)
    m_tiles = cdiv(a_rows, 128)
    chunks = n * cdiv(w, 16) * cdiv(h, 2)
    tap_group = min(taps, min(2, 2 // n_groups))
    tasks = cdiv(taps, tap_group) * m_tiles * n_tiles
    ksplit = max(1, min((2 * sm) // tasks, max(1, chunks // 8)))
    per_split = taps * m_tiles * 128 * n_tiles * n_pad
    while ksplit > 1 and per_split * ksplit > (96 << 20):
        ksplit -= 1
    return cdiv(chunks, ksplit), ksplit


class Checker:
    """Collects max error / bar (and, for filter gradients, the mean signed error / bar) per check."""

    def __init__(self):
        self.worst, self.signed = {}, {}
        self.gm = {}      # per activated layer: the output gradient after dropout, g mask fp32(1 / keep) (check_step)
        self.sums = {}    # per variable: (fp64 sum / G, its accumulation bar / G, L2 term) before finalized (check_step)

    def add(self, name, got, ref, bar, signed=False):
        got = torch.as_tensor(got).to(dev(), torch.float64) if not torch.is_tensor(got) else got.to(dev(), torch.float64)
        err = got - ref
        assert torch.isfinite(got).all(), (name, "inf / NaN")
        self.worst[name] = max(self.worst.get(name, 0.0), float((err.abs() / bar).max()))
        if signed:   # truncation toward zero shows up as an error opposite in sign to the value
            self.signed[name] = float((err * torch.sign(ref) / bar).mean())

    def bad(self):
        return [(k, v) for k, v in self.worst.items() if not v <= 1.0]


def output_gradient(cfg, scope, plane):
    """The gradient reaching the output of activated layer `scope` in a captured train step, before dropout, from the
    step's captured planes: `plane(tensor, channels)` returns "dH:Up-PS" (split into B2 | A1), "dH:B2", "dH:A1+B1" (the
    concatenated CNN outputs) or "dH:CNN<j>" (the gradient CNN<j> passes back to CNN<j-1>) as an fp64 NCHW tensor."""
    f = O.feature_filters(cfg)
    nin2 = cfg.nin_filters2
    if scope in ("A1", "B2"):
        g = plane("dH:Up-PS", cfg.nin_filters + nin2)
        return g[:, nin2:] if scope == "A1" else g[:, :nin2]
    if scope == "B1":
        return plane("dH:B2", nin2)
    j = int(scope[3:])
    offs = np.cumsum([0] + f)
    g = plane("dH:A1+B1", sum(f))[:, offs[j - 1]:offs[j]]
    return g + plane("dH:CNN%d" % (j + 1), f[j - 1]) if j < cfg.layers else g


def after_dropout(g, mask, keep):
    """g mask fp32(1 / keep): the gradient of an activated layer's output before its dropout (`mask` None at keep 1)."""
    return g * (1.0 if mask is None else mask) * float(np.float32(1.0) / np.float32(keep))


def finalized(s, b, dec):
    """get_grad of a variable whose fp32 sum over the batch, over G, is `s` with accumulation bar `b`, plus its L2 term
    `dec`, rounded once: (reference, bar)."""
    ref = s + dec
    return ref, b + U24 * ref.abs() + U24 * dec.abs() + 1e-45


def check_step(eng, kw, w, x, x2, y, keep, seed, chk, get_grad=None, act="prelu", bar_n=None):
    """Every backward kernel of the last train step of `eng` (run with grad_capture = 1, activator `act`) against its
    isolated reference.  `get_grad(name)` returns a variable's gradient as get_grad does (default: eng.get_grad); a wide
    depthwise-separable graph passes its composed filters as the conv_W entries of `w` and reads their gradients from
    "dWc:".  The bars of the filter, bias and slope sums are those of a batch of `bar_n` images (default: this step's):
    a sub-batch of a larger step passes that step's n, and chk.sums then holds its share of the larger step's sums."""
    cfg = O.OracleConfig(**kw)
    n, h, wd = x.shape[:3]
    nb = bar_n or n
    s = cfg.scale
    f = O.feature_filters(cfg)
    L = cfg.layers
    k = cfg.cnn_size
    cps = cfg.nin_filters + cfg.nin_filters2
    ps_out = cfg.pixel_shuffler_filters or cps
    count = n * s * h * s * wd
    G = 2.0 ** round(math.log2(count / 2.0))
    l2 = np.float32(cfg.l2_decay)
    sm = torch.cuda.get_device_properties(0).multi_processor_count

    def T(name, shape):
        return t64(eng.get_train_tensor(name, shape))

    def plane(name, c, r=1):
        return t64(eng.get_activation(name, (n, r * h, r * wd, c)))

    def grad(name):
        return torch.from_numpy((get_grad or eng.get_grad)(name)).to(dev(), torch.float64)

    def finalize(name, ssum, bar_sum):
        """get_grad of a variable whose fp32 sum (scaled by G) is `ssum` with accumulation bar `bar_sum`."""
        wv = torch.from_numpy(w[name].astype(np.float32)).to(dev(), torch.float64)
        dec = float(l2) * wv if name.endswith("conv_W") else torch.zeros_like(wv)
        chk.sums[name] = (ssum / G, bar_sum / G, dec)
        return finalized(ssum / G, bar_sum / G, dec)

    # ---- loss
    yp = t64(eng.get_train_tensor("y_", (n, s * h, s * wd, 1)))
    dY = T("dY", (n, s * h, s * wd, 1))
    ref = (yp - t64(y)) * (2.0 * G / count)
    chk.add("loss_kernel", dY, ref, U22 * ref.abs() + 1e-45)

    # ---- R-CNN1: filter gradient and data gradient (in space_to_depth form)
    up_name, r_last = ("Up-PS2", 2) if s == 4 else ("Up-PS", s)
    hr = plane(up_name, ps_out, s)
    wr = w["R-CNN1/conv_W"]
    kr = wr.shape[0]
    ssum, sabs = wgrad(hr, dY, kr), wgrad(hr.abs(), dY.abs(), kr)
    ref, bar = finalize("R-CNN1/conv_W", ssum, nb * s * h * s * wd * U24 * sabs)
    chk.add("last_wgrad", grad("R-CNN1/conv_W"), ref, bar, signed=True)
    v = s2d(dgrad(dY, wr), r_last)
    sv = s2d(dgrad(dY.abs(), np.abs(wr)), r_last)
    lh, lw = (2 * h, 2 * wd) if s == 4 else (h, wd)
    dz_last = T("dZ:Up-PS2" if s == 4 else "dZ:Up-PS", (n, lh, lw, r_last * r_last * ps_out))
    chk.add("last_dgrad_s2d", dz_last, v, kr * kr * U24 * sv + stored(v))

    def twin(name, dz, wq, cin_pad, kk):
        """A dgrad twin through conv_tc_kernel: (reference, bar) of its output."""
        v = dgrad(dz, wq)
        sv = dgrad(dz.abs(), np.abs(wq))
        return v, (tc_units(kk, cin_pad, 0, 2) + 1) * U23 * sv + stored(v)

    def wgrad_tc(name, a, dz, kk, a_rows, dz_cols, hh, ww):
        cpc, ksplit = wgrad_tc_chain(sm, nb, hh, ww, kk, a_rows, dz_cols)
        ssum, sabs = wgrad(a, dz, kk), wgrad(a.abs(), dz.abs(), kk)
        return finalize(name, ssum, ((6 * cpc) * 17 * U23 + U22 + (ksplit + 1) * U24) * sabs)

    def conv_b(name, dz):
        ref, bar = finalize(name, dz.sum(dim=(0, 2, 3)), (dz[0, 0].numel() * nb + 4) * U24 * dz.abs().sum(dim=(0, 2, 3)))
        chk.add("bias sums", grad(name), ref, bar)

    # ---- pixel shuffler(s)
    b1w, a1w = pad16(cfg.nin_filters2), pad16(cfg.nin_filters)
    nin_in = torch.cat([plane("B2", cfg.nin_filters2), plane("A1", cfg.nin_filters)], dim=1)
    if s == 4:
        sc = "Up-PS2/Up-PS2_CNN"
        a_up = plane("Up-PS", cps, 2)
        ref, bar = wgrad_tc(sc + "/conv_W", a_up, dz_last, k, cps, 4 * ps_out, 2 * h, 2 * wd)
        chk.add("wgrad_tc Up-PS2", grad(sc + "/conv_W"), ref, bar, signed=True)
        conv_b(sc + "/conv_B", dz_last)
        (wq,) = quantise([w[sc + "/conv_W"]], 2)
        v, bar = twin("Up-PS2", dz_last, wq, pad16(4 * ps_out), k)
        dmid = T("dH:Up-PS2", (n, 2 * h, 2 * wd, cps))
        chk.add("dgrad twin Up-PS2", dmid, v, bar)
        dz_up = T("dZ:Up-PS", (n, h, wd, 4 * cps))
        chk.add("s2d_planes (exact)", dz_up, s2d(dmid, 2), torch.full_like(dz_up, 1e-300))
        up_cols = 4 * cps
    else:
        dz_up = dz_last
        up_cols = s * s * ps_out
    sc = "Up-PS/Up-PS_CNN"
    ref, bar = wgrad_tc(sc + "/conv_W", nin_in, dz_up, k, b1w + cfg.nin_filters, up_cols, h, wd)
    chk.add("wgrad_tc Up-PS", grad(sc + "/conv_W"), ref, bar, signed=True)
    conv_b(sc + "/conv_B", dz_up)
    (wq,) = quantise([w[sc + "/conv_W"]], 2)
    v, bar = twin("Up-PS", dz_up, wq, pad16(up_cols), k)
    dnin = T("dH:Up-PS", (n, h, wd, cps))
    chk.add("dgrad twin Up-PS", dnin, v, bar)

    # ---- activation gradients
    captured = {}     # the captured planes output_gradient reads, as they are fetched below

    def act_grad(scope, c):
        g = output_gradient(cfg, scope, lambda name, _: captured[name])
        gm = after_dropout(g, t64(eng.dropout_mask(scope, seed, n, h, wd, c).astype(np.float32)) if keep < 1.0 else None,
                           keep)
        chk.gm[scope] = gm
        got = T("dZ:" + scope, (n, h, wd, c))
        if act in ("prelu", "leaky_relu"):    # the slope below zero, decided by the min(z, 0) plane
            zn = T("zneg:" + scope, (n, h, wd, c))
            neg = zn < 0
            if act == "prelu":
                slope = torch.from_numpy(w["%s/prelu/%s_prelu" % (scope, scope)].astype(np.float32)).to(dev(), torch.float64).view(1, -1, 1, 1)
            else:
                slope = LEAKY
            dz = torch.where(neg, gm * slope, gm)
            bar = 4 * U24 * dz.abs()
        else:   # f'(h) at h = fp32(stored * fp32(keep)) of the GPU's own stored output (act_deriv_from_output)
            hv = (torch.from_numpy(eng.get_activation(scope, (n, h, wd, c))).to(dev()) * torch.tensor(np.float32(keep), device=dev()))
            hv = hv.permute(0, 3, 1, 2).double()
            if act == "relu":
                d, dbar = (hv > 0).double(), 0.0
            elif act == "sigmoid":      # h * (1 - h): two roundings
                d = hv * (1 - hv)
                dbar = 2 * U24 * d.abs()
            elif act == "tanh":         # 1 - h * h: the square's rounding, then the cancellation's
                d = 1 - hv * hv
                dbar = U24 * hv * hv + U24 * d.abs()
            else:                       # selu: h + kSeluScaleAlpha below zero, kSeluScale (exact) above
                d = torch.where(hv < 0, hv + SELU_SCALE_ALPHA, torch.full_like(hv, SELU_SCALE))
                dbar = U24 * (hv < 0).double() * d.abs()
            dz = gm * d
            bar = (4 if act == "relu" else 5) * U24 * dz.abs() + gm.abs() * dbar
        chk.add("act_grad dZ", got, dz, bar + stored(dz))
        conv_b(scope + "/conv_B", dz)
        if act == "prelu":
            term = torch.where(neg, gm * zn, torch.zeros_like(gm))
            pn = "%s/prelu/%s_prelu" % (scope, scope)
            ref, bar = finalize(pn, term.sum(dim=(0, 2, 3)), (nb * h * wd + 4) * U24 * term.abs().sum(dim=(0, 2, 3)))
            chk.add("act_grad slope sums", grad(pn), ref, bar)
        return got

    nin2 = cfg.nin_filters2
    captured["dH:Up-PS"] = dnin
    dz_a1 = act_grad("A1", cfg.nin_filters)
    dz_b2 = act_grad("B2", nin2)
    b1 = plane("B1", nin2)
    ref, bar = wgrad_tc("B2/conv_W", b1, dz_b2, 3, nin2, nin2, h, wd)
    chk.add("wgrad_tc B2", grad("B2/conv_W"), ref, bar, signed=True)
    (wq,) = quantise([w["B2/conv_W"]], 2)
    v, bar = twin("B2", dz_b2, wq, b1w, 3)
    db1 = T("dH:B2", (n, h, wd, nin2))
    chk.add("dgrad twin B2", db1, v, bar)
    captured["dH:B2"] = db1
    dz_b1 = act_grad("B1", nin2)
    feats = [plane("CNN%d" % (i + 1), f[i]) for i in range(L)]
    concat = torch.cat(feats, dim=1)
    feat_pitch = sum(pad16(c) for c in f)
    for nm, dz, cols in (("A1", dz_a1, cfg.nin_filters), ("B1", dz_b1, nin2)):
        # one GEMM over [A1 | B1] columns (a1_w + b1_w wide), A rows = concat positions
        ref, bar = wgrad_tc(nm + "/conv_W", concat, dz, 1, feat_pitch, a1w + b1w, h, wd)
        chk.add("wgrad_tc A1+B1", grad(nm + "/conv_W"), ref, bar, signed=True)
    wa, wb = quantise([w["A1/conv_W"], w["B1/conv_W"]], 2)
    v, bar = twin("A1+B1", torch.cat([dz_a1, dz_b1], dim=1), np.concatenate([wa, wb], axis=3), a1w + b1w, 1)
    dcat = T("dH:A1+B1", (n, h, wd, sum(f)))
    chk.add("dgrad twin A1+B1", dcat, v, bar)
    captured["dH:A1+B1"] = dcat

    # ---- feature-extraction stack
    for i in range(L - 1, -1, -1):
        sc = "CNN%d" % (i + 1)
        dz = act_grad(sc, f[i])
        if i == 0:
            a = t64(x)
            ssum, sabs = wgrad(a, dz, k), wgrad(a.abs(), dz.abs(), k)
            ref, bar = finalize(sc + "/conv_W", ssum, nb * h * wd * U24 * sabs)
            chk.add("first_wgrad / wgrad (CNN1)", grad(sc + "/conv_W"), ref, bar, signed=True)
        else:
            ref, bar = wgrad_tc(sc + "/conv_W", feats[i - 1], dz, k, f[i - 1], f[i], h, wd)
            chk.add("wgrad_tc CNN", grad(sc + "/conv_W"), ref, bar, signed=True)
            (wq,) = quantise([w[sc + "/conv_W"]], 2)
            v, bar = twin(sc, dz, wq, pad16(f[i]), k)
            captured["dH:" + sc] = T("dH:" + sc, (n, h, wd, f[i - 1]))
            chk.add("dgrad twin CNN", captured["dH:" + sc], v, bar)
    return chk


def capture_step(eng, x, x2, y, keep, seed):
    eng.set_option("grad_capture", 1)
    return eng.train_step_host(x, x2, y, lr=0.002, seed=seed, apply_update=False)


def report(tag, chk):
    print(tag, "error / bar:", " ".join("%s %.3g" % kv for kv in sorted(chk.worst.items())))
    if chk.signed:
        print(tag, "mean signed error / bar:", " ".join("%s %+.3g" % kv for kv in sorted(chk.signed.items())))


# ------------------------------------------------------------------------------------------- (a) every kernel ----
@pytest.mark.parametrize("kw,weights,keep,shape,kernels", [c[1:] for c in GRADIENT_CASES], ids=[c[0] for c in GRADIENT_CASES])
def test_backward_kernels_isolated(kw, weights, keep, shape, kernels):
    """The GRADIENT_CASES graphs of test_gpu_train.py (each reaches the kernels listed there, profiler-checked): every
    backward kernel of the step against its isolated fp64 reference and bar.  All violations reported at once."""
    n, h, wd = shape
    cfg, wts, eng, x, x2, y = setup(kw, keep, n, h, wd, weights=weights)
    if weights != "he":
        kw = MODEL_FLAGS[weights]
    seed = 1234
    eng.set_option("grad_capture", 1)
    _, names = launched_kernels(lambda: eng.train_step_host(x, x2, y, lr=0.002, seed=seed, apply_update=False))
    assert_kernels_ran(names, kernels + ["loss_kernel", "act_grad8_kernel", "grad_finalize_kernel"])
    chk = check_step(eng, kw, wts, x, x2, y, keep, seed, Checker())
    report(shape, chk)
    eng.close()
    assert not chk.bad(), chk.bad()


def test_channel_pair_activation_gradient_isolated():
    """act_grad_kernel (option act_grad_impl = 1) under the same element-wise and sum bars."""
    kw = GRADIENT_CASES[1][1]
    cfg, wts, eng, x, x2, y = setup(kw, 0.8, 2, 16, 24)
    eng.set_option("act_grad_impl", 1)
    eng.set_option("grad_capture", 1)
    _, names = launched_kernels(lambda: eng.train_step_host(x, x2, y, lr=0.002, seed=7, apply_update=False))
    assert_kernels_ran(names, ["act_grad_kernel"])
    chk = check_step(eng, kw, wts, x, x2, y, 0.8, 7, Checker())
    report("act_grad_impl=1", chk)
    eng.close()
    assert not chk.bad(), chk.bad()


def test_cuda_core_wgrad_isolated():
    """wgrad_kernel for every filter gradient (option wgrad_impl = 1): its fp32 sums stay under the wgmma bars."""
    kw = GRADIENT_CASES[1][1]
    cfg, wts, eng, x, x2, y = setup(kw, 0.8, 2, 16, 24)
    eng.set_option("wgrad_impl", 1)
    eng.set_option("grad_capture", 1)
    _, names = launched_kernels(lambda: eng.train_step_host(x, x2, y, lr=0.002, seed=7, apply_update=False))
    assert_kernels_ran(names, ["wgrad_kernel"])
    chk = check_step(eng, kw, wts, x, x2, y, 0.8, 7, Checker())
    report("wgrad_impl=1", chk)
    eng.close()
    assert not chk.bad(), chk.bad()


# ------------------------------------------------------------------------------------------- (b) real patches ----
def real_patches(scale, n, ph, pw, step):
    """n LR / bicubic / ground-truth patches of ph x pw LR pixels, cut at matching positions from the Set5 and Set14
    evaluation inputs (build_inputs_for_evaluate) every `step` LR pixels."""
    xs, x2s, ys = [], [], []
    files = sorted(glob.glob(os.path.join(GOLDEN, "data", "set5", "*.png"))) + \
        sorted(glob.glob(os.path.join(GOLDEN, "data", "set14", "*.png")))
    for fn in files:
        inp, bic, true = O.build_inputs_for_evaluate(fn, scale)
        for y0 in range(0, inp.shape[0] - ph + 1, step):
            for x0 in range(0, inp.shape[1] - pw + 1, step):
                xs.append(inp[y0:y0 + ph, x0:x0 + pw])
                x2s.append(bic[scale * y0:scale * (y0 + ph), scale * x0:scale * (x0 + pw)])
                ys.append(true[scale * y0:scale * (y0 + ph), scale * x0:scale * (x0 + pw)])
                if len(xs) == n:
                    return tuple(np.ascontiguousarray(np.stack(a).reshape(len(a), *a[0].shape[:2], 1), dtype=np.float32)
                                 for a in (xs, x2s, ys))
    raise AssertionError("not enough patches")


def real_engine(model, keep):
    from helper import engine as E
    kw = MODEL_FLAGS[model]
    wts = load_golden_weights(model)
    eng = E.Engine(E.make_config(dropout_keep=keep, **kw))
    eng.set_params(wts)
    return kw, wts, eng


@pytest.mark.parametrize("model", [L12[2], L12[3], L12[4], CDCSCN[4]], ids=["L12-x2", "L12-x3", "L12-x4", "cdcscn-x4"])
def test_backward_kernels_on_real_patches(model):
    """Shipped checkpoints on Set5 / Set14 patches with y = ground truth and keep 0.8: the gradient magnitudes training
    sees, where many lo planes (and some hi planes) of the small gradients are subnormal."""
    kw, wts, eng = real_engine(model, 0.8)
    x, x2, y = real_patches(kw.get("scale", 2), 6, 32, 32, 37)
    capture_step(eng, x, x2, y, 0.8, 99)
    chk = check_step(eng, kw, wts, x, x2, y, 0.8, 99, Checker())
    report(model, chk)
    eng.close()
    assert not chk.bad(), chk.bad()


# ------------------------------------------------------------------------------------ (c) the benchmark's shape ----
def test_backward_kernels_at_benchmark_train_shape():
    """L12 x4 on 64 real patches of 48 x 48 (bench.py's train record): every filter gradient against fp64 sum A dZ over
    the captured planes, and every other kernel of the step.  The mean signed error / bar of each wgmma filter gradient is
    printed: truncation toward zero would show as a negative mean."""
    kw, wts, eng = real_engine(L12[4], 0.8)
    x, x2, y = real_patches(4, 64, 48, 48, 24)
    capture_step(eng, x, x2, y, 0.8, 5)
    chk = check_step(eng, kw, wts, x, x2, y, 0.8, 5, Checker())
    report("L12-x4 64x48x48", chk)
    eng.close()
    assert not chk.bad(), chk.bad()


# ----------------------------------------------------------------------------------------- (d) residual extremes ----
@pytest.mark.parametrize("residual", [1e-3, 255.0], ids=["tiny", "large"])
def test_backward_kernels_at_residual_extremes(residual):
    """y = y_ +- residual around a first forward (keep 1): with 1e-3 most gradient planes are subnormal, with 255 the
    gradients are as large as a residual can make them.  No inf / NaN, and every bar (floors included) holds."""
    kw, wts, eng = real_engine(CDCSCN[2], 1.0)
    x, x2, _ = real_patches(2, 4, 24, 24, 29)
    yp = eng.forward_host(x, x2)
    sign = np.where(np.random.RandomState(3).rand(*yp.shape) < 0.5, -1.0, 1.0).astype(np.float32)
    y = (yp + sign * np.float32(residual)).astype(np.float32)
    capture_step(eng, x, x2, y, 1.0, 11)
    for name in wts:
        assert np.isfinite(eng.get_grad(name)).all(), name
    chk = check_step(eng, kw, wts, x, x2, y, 1.0, 11, Checker())
    report("residual %g" % residual, chk)
    eng.close()
    assert not chk.bad(), chk.bad()


# ------------------------------------------------------------------------------------------- (e) z -> 0- edge ----
def test_prelu_slope_for_pre_activations_just_below_zero():
    """A zero image with CNN1 biases of -1e-9 makes every CNN1 pre-activation -1e-9, which fp16 rounds to -0.  TensorFlow
    takes slope alpha for every z < 0, so dZ = g alpha and d alpha = sum g z; the min(z, 0) plane keeps the sign at
    -2^-24, moving d alpha by at most 2^-24 sum |g|."""
    from helper import engine as E
    kw = GRADIENT_CASES[1][1]
    cfg = O.OracleConfig(**kw)
    wts = O.he_init_weights(cfg, seed=0)
    wts["CNN1/conv_B"] = np.full_like(wts["CNN1/conv_B"], -1e-9)
    eng = E.Engine(E.make_config(dropout_keep=0.8, **kw))
    eng.set_params(wts)
    n, h, wd = 2, 12, 10
    x = np.zeros((n, h, wd, 1), np.float32)
    x2 = np.zeros((n, 2 * h, 2 * wd, 1), np.float32)
    y = np.random.RandomState(4).rand(n, 2 * h, 2 * wd, 1).astype(np.float32) * 255
    capture_step(eng, x, x2, y, 0.8, 21)
    c = cfg.filters
    assert (eng.get_train_tensor("zneg:CNN1", (n, h, wd, c)) < 0).all()
    g = eng.get_train_tensor("dH:A1+B1", (n, h, wd, sum(O.feature_filters(cfg))))[..., :c].astype(np.float64) + \
        eng.get_train_tensor("dH:CNN2", (n, h, wd, c)).astype(np.float64)
    gm = g * eng.dropout_mask("CNN1", 21, n, h, wd, c) * float(np.float32(1) / np.float32(0.8))
    alpha = wts["CNN1/prelu/CNN1_prelu"].astype(np.float64)
    dz = eng.get_train_tensor("dZ:CNN1", (n, h, wd, c))
    np.testing.assert_allclose(dz, gm * alpha, rtol=2 ** -20, atol=2 ** -24)
    G = 2.0 ** round(math.log2(n * 4 * h * wd / 2.0))
    want = (gm * -1e-9).sum(axis=(0, 1, 2)) / G
    slack = U24 * np.abs(gm).sum(axis=(0, 1, 2)) / G
    got = eng.get_grad("CNN1/prelu/CNN1_prelu")
    assert (np.abs(got - want) <= slack * 1.01 + 1e-30).all(), (got, want, slack)
    assert (got * want > 0).all() | (want == 0).all()
    eng.close()
