"""
Backward parity of the depthwise-separable train steps, kernel by kernel, each against an isolated fp64 reference
computed (with torch, on the GPU) from the tensors the GPU itself stored (option "grad_capture", dcscn_get_train_tensor).

The narrow step (train_ds.inc, kernels in train_ds.cuh) is fp32 throughout and has no loss scale.  With u = 2^-24 and
S = sum |a| |w| over an output's products:

  ds_dw_fwd_kernel     U = depthwise(input, dw): a chain of k^2 FMAs, k^2 u S
  ds_pw_fwd_kernel     Z = b + U . pw: cin FMAs from the bias, (cin + 1) u (S + |b|);  H = f(Z) mask fp32(1 / keep)
                       (depth_to_space scattered; + x2 on R-CNN1) from the captured Z: bit for bit for linear layers,
                       3 u |h| for prelu / relu / leaky_relu (slope product, dropout), 6 u |h| for sigmoid / tanh / selu
                       (libdevice curve within 4 u), 2 u |h| for the x2 add
  loss_kernel          dY = fp32(y_ - y) fp32(2 / count): 2^-22 |dY|
  ds_act_bwd_kernel    dZ, E from the layer's output gradient, Z, the dropout mask and the slope: a fixed sequence of fp32
                       products that torch float32 reproduces, so bit for bit for prelu / relu / leaky_relu; for sigmoid,
                       tanh and selu f' is formed from the fp32 h (within dh = 4 u |h|, + 2^-126 for sigmoid, whose
                       1 / (1 + expf(-z)) is 0 once expf overflows): |gm| (|df'/dh| dh + 3 u |f'|) + u |dZ|
  ds_colsum_kernel     bias and slope gradients, fp32 sums over the pixels: (npx + 4) u sum |terms|
  ds_dpw_kernel        d pw = sum_px U dZ: one FMA chain per block over its px_per_block pixels, then one atomicAdd per
                       block: (px_per_block + blocks) u S (restated launch arithmetic, cs_launch)
  ds_du_kernel         dU = dZ . pw^T: cout FMAs, cout u S
  ds_ddw_kernel        d dw = sum_px input[px + t] dU[px]: each lane chains ceil(px_per_block / lanes) pixels, the lanes are
                       summed in order, then one atomicAdd per block: (ceil(ppb / lanes) + lanes + blocks) u S (ddw_launch)
  ds_dx_kernel         the transposed depthwise of dU, k^2 FMAs, written or added to the gradient buffer at the layer's
                       input.  Checked per writer against the buffer the previous writer left (B1 writes the concat
                       gradient, A1 adds, CNNi+1 adds to CNNi's channels): k^2 u S, + u |v| where it adds
  grad_finalize_kernel the dead conv_W's gradient is l2 conv_W rounded once; depthwise_W, pointwise_W, conv_B and the
                       slopes get no decay: the sums above plus one rounding, u |g|

Every rounding may also land in the subnormal range, where it moves a value by up to 2^-150 whatever its size: each
chain's bar adds 2^-150 per rounding (gradients of saturated sigmoid layers reach it).

The wide step (the tensor-core train step on composed filters) is checked by test_gpu_backward_paths.check_step with
the composed filters in place of conv_W and their gradients read from "dWc:"; ds_compose_kernel must equal numpy's
float32 product bit for bit and ds_decompose_kernel (fp64 sums) must be within one fp32 rounding of the fp64 chain rule.
"""
import gc
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import activator_oracle as A
import dcscn_oracle as O
from conftest import MODEL_FLAGS, load_golden_weights
from test_gpu_backward_paths import Checker, check_step, dev, real_patches, report, s2d
from test_gpu_train import DS2, DS3, DS4, DS4W, assert_kernels_ran, launched_kernels, setup, \
    test_depthwise_separable_gradients_match_oracle

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TINY = 1e-300
SUB = 2.0 ** -150        # the most one fp32 rounding into the subnormal range can move a value
MIN_NORMAL = 2.0 ** -126
CDS = "dcscn_L7_F32to8_G1.20_Sc4_NIN_A24_B8_PS_DS_R1F32"
NARROW = ["ds_dw_fwd_kernel", "ds_pw_fwd_kernel", "loss_kernel", "ds_act_bwd_kernel", "ds_colsum_kernel", "ds_dpw_kernel",
          "ds_du_kernel", "ds_ddw_kernel", "ds_dx_kernel", "grad_finalize_kernel"]
WIDE = ["ds_compose_kernel", "ds_decompose_kernel"]
# graphs that ds_tile_fits sends to the narrow kernels with a layer wider than the train kernels once took:
# the c-DCSCN shape at x3 with the reference's default pixel-shuffler width (Up-PS 32 -> 288 columns), and a 12-layer
# stack of 32 filters whose A1 / B1 read 384 concat channels
UPPS288 = dict(depthwise_separable=True, scale=3, layers=7, filters=32, min_filters=8, filters_decay_gamma=1.2,
               nin_filters=24, nin_filters2=8, pixel_shuffler_filters=0, reconstruct_layers=0)
A1B1_384 = dict(depthwise_separable=True, layers=12, filters=32, min_filters=32, nin_filters=24, nin_filters2=8)


@pytest.fixture(autouse=True)
def release_reference_memory():
    """Hand the fp64 references' memory back to the driver after every test (see test_gpu_backward_paths.py)."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def cdiv(a, b):
    return -(-a // b)


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def cs_launch(npx, sm):
    """(px_per_block, blocks) of ds_colsum_kernel and ds_dpw_kernel (train_step_ds_impl: cs_ppb, cs_grid)."""
    blocks = max(1, min(cdiv(npx, 512), sm * 8))
    ppb = cdiv(npx, blocks)
    return ppb, cdiv(npx, ppb)


def ddw_launch(npx, cin, sm):
    """(px_per_block, lanes, blocks) of ds_ddw_kernel (train_step_ds_impl)."""
    cpb = 1
    while cpb < cin and cpb < 256:
        cpb <<= 1
    lanes = 256 // cpb
    want = max(1, min(cdiv(npx, 64 * lanes), sm * 8))
    ppb = cdiv(npx, want)
    return ppb, lanes, cdiv(npx, ppb)


def nchw(a, dtype=torch.float64):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev()).permute(0, 3, 1, 2).to(dtype)


def vec(a, dtype=torch.float64):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev()).to(dtype)


def ds_layers(cfg, n, h, w):
    """The layer table of train_step_ds_impl in forward order: scope -> (k, cin, cout, activated, bias, (H, W) of the
    input, input, output-gradient source, depth_to_space r, previous writer of the input-gradient buffer)."""
    L, s = cfg.layers, cfg.scale
    f = O.feature_filters(cfg)
    off = np.cumsum([0] + f)
    nb, na = cfg.nin_filters2, cfg.nin_filters
    up = ["Up-PS/Up-PS_CNN", "Up-PS2/Up-PS2_CNN"] if s == 4 else ["Up-PS/Up-PS_CNN"]
    out = {}
    tab = {e[0]: e for e in O.layer_table(cfg)}

    def put(scope, res, src, gout, r=0, prev=None):
        _, k, cin, cout, bias, act = tab[scope]
        out[scope] = dict(k=k, cin=cin, cout=cout, act=act, bias=bias, res=res, src=src, gout=gout, r=r, prev=prev)

    for i in range(L):
        gout = ("dH:CNN%d" % (i + 2), None) if i < L - 1 else ("dH:A1", (off[i], off[i + 1]))
        prev = ("dH:A1", (off[i - 1], off[i])) if i > 0 else None
        put("CNN%d" % (i + 1), (h, w), "x" if i == 0 else "CNN%d" % i, gout, prev=prev)
    put("A1", (h, w), "concat", ("dH:" + up[0], (nb, nb + na)), prev=("dH:B1", None))
    put("B1", (h, w), "concat", ("dH:B2", None))
    put("B2", (h, w), "B1", ("dH:" + up[0], (0, nb)))
    if s == 4:
        put(up[0], (h, w), "nin", ("dH:" + up[1], None), r=2)
        put(up[1], (2 * h, 2 * w), up[0], ("dH:R-CNN1", None), r=2)
    else:
        put(up[0], (h, w), "nin", ("dH:R-CNN1", None), r=s)
    put("R-CNN1", (s * h, s * w), up[-1], ("dY", None))
    return out


def depthwise_w(dw):
    """[k, k, c, 1] -> torch grouped-conv weight [c, 1, k, k] (fp64)."""
    return vec(dw).permute(2, 3, 0, 1).contiguous()


def act_eval(act, z, alpha):
    """f(z) in fp64 with the kernels' fp32 constants."""
    if act == "prelu":
        return torch.where(z > 0, z, alpha.view(1, -1, 1, 1) * z)
    if act == "relu":
        return torch.clamp_min(z, 0.0)
    if act == "leaky_relu":
        return torch.where(z > 0, z, A.LEAKY * z)
    if act == "sigmoid":
        return 1.0 / (1.0 + torch.exp(-z))
    if act == "tanh":
        return torch.tanh(z)
    return torch.where(z < 0, float(np.float32(1.7580993408473766)) * torch.expm1(z), float(np.float32(1.0507009873554805)) * z)


def act_deriv(act, z):
    """(f'(z), |d f' / d h| at h = f(z)) in fp64 for sigmoid, tanh and selu."""
    h = act_eval(act, z, None)
    if act == "sigmoid":
        return h * (1 - h), (1 - 2 * h).abs()
    if act == "tanh":
        return 1 - h * h, 2 * h.abs()
    sa, lam = float(np.float32(1.7580993408473766)), float(np.float32(1.0507009873554805))
    neg = h < 0
    return torch.where(neg, h + sa, torch.full_like(h, lam)), neg.to(h.dtype)


def check_ds_step(eng, cfg, wts, act, x, x2, y, keep, seed, chk):
    """Every kernel of the last narrow depthwise-separable train step of `eng` (run with grad_capture = 1).  Returns
    {kernel: most blocks any of its launches had} from the restated launch arithmetic."""
    n, h, w = x.shape[:3]
    s = cfg.scale
    count = n * s * h * s * w
    sm = sm_count()
    l2 = np.float32(cfg.l2_decay)
    tab = ds_layers(cfg, n, h, w)
    blocks = {"ds_colsum_kernel": 0, "ds_dpw_kernel": 0, "ds_ddw_kernel": 0}
    f = O.feature_filters(cfg)
    cps = cfg.nin_filters + cfg.nin_filters2
    ps_out = cfg.pixel_shuffler_filters or cps

    cache = {}

    def T(name, nhw, c, dtype=torch.float64):
        key = (name, dtype)
        if key not in cache:
            cache[key] = nchw(eng.get_train_tensor(name, (n,) + tuple(nhw) + (c,)), dtype)
        return cache[key]

    def grad(name):
        return vec(eng.get_grad(name))

    def wv(name):
        return vec(wts[name])

    def src_of(scope):
        e = tab[scope]
        name = e["src"]
        if name == "x":
            return nchw(x)
        if name == "concat":
            return torch.cat([T("H:CNN%d" % (i + 1), (h, w), f[i]) for i in range(cfg.layers)], dim=1)
        if name == "nin":
            return torch.cat([T("H:B2", (h, w), cfg.nin_filters2), T("H:A1", (h, w), cfg.nin_filters)], dim=1)
        if name.startswith("Up-PS"):
            r = tab[name]["r"]
            hh, ww = tab[name]["res"]
            c = tab[name]["cout"] // (r * r)
            return T("H:" + name, (r * hh, r * ww), c)
        return T("H:" + name, (h, w), tab[name]["cout"])

    def out_grad(scope, dtype):
        """The layer's output gradient in its column order (space_to_depth of a depth_to_space output)."""
        e = tab[scope]
        name, sl = e["gout"]
        hh, ww = e["res"]
        r = e["r"]
        if name == "dY":
            g = T("dY", (hh, ww), 1, dtype)
        else:
            cons = name[3:]
            ce = tab[cons]
            g = T(name, ce["res"], ce["cin"], dtype)
        if sl is not None:
            g = g[:, sl[0]:sl[1]]
        return s2d(g, r) if r else g

    def finalize(name, ssum, bar_sum, decay=False):
        dec = float(l2) * wv(name) if decay else torch.zeros_like(ssum)
        ref = ssum + dec
        return ref, bar_sum + U * ref.abs() + U * dec.abs() + TINY

    # ---- loss
    yp = T("y_", (s * h, s * w), 1)
    dY = T("dY", (s * h, s * w), 1)
    ref = (yp - nchw(y)) * (2.0 / count)
    chk.add("loss_kernel", dY, ref, 2.0 ** -22 * ref.abs() + TINY)

    for scope, e in tab.items():
        k, cin, cout = e["k"], e["cin"], e["cout"]
        hh, ww = e["res"]
        npx = n * hh * ww
        dwt, pw = depthwise_w(wts[scope + "/depthwise_W"]), wv(scope + "/pointwise_W")[0, 0]
        inp = src_of(scope)
        activated = e["act"]
        a_name = "%s/prelu/%s_prelu" % (scope, scope.split("/")[-1])
        alpha = wv(a_name) if activated and act == "prelu" else None

        # ---- forward: depthwise, pointwise (+ bias, activation, dropout, depth_to_space, x2)
        Uc = T("U:" + scope, (hh, ww), cin)
        ref = F.conv2d(inp, dwt, padding=k // 2, groups=cin)
        sabs = F.conv2d(inp.abs(), dwt.abs(), padding=k // 2, groups=cin)
        chk.add("ds_dw_fwd_kernel", Uc, ref, k * k * (U * sabs + SUB))
        Z = T("Z:" + scope, (hh, ww), cout)
        b = wv(scope + "/conv_B").view(1, -1, 1, 1) if e["bias"] else torch.zeros(1, cout, 1, 1, device=dev(), dtype=torch.float64)
        ref = torch.einsum("nchw,cd->ndhw", Uc, pw) + b
        sabs = torch.einsum("nchw,cd->ndhw", Uc.abs(), pw.abs()) + b.abs()
        chk.add("ds_pw_fwd_kernel Z", Z, ref, (cin + 1) * (U * sabs + SUB))
        mask = 1.0
        if activated and keep < 1.0:
            mask = nchw(eng.dropout_mask(scope, seed, n, hh, ww, cout).astype(np.float32))
        inv_keep = float(np.float32(1.0) / np.float32(keep))
        if activated:
            hv = act_eval(act, Z, alpha) * mask * (inv_keep if keep < 1.0 else 1.0)
            hbar = (6 if act in ("sigmoid", "tanh", "selu") else 3) * (U * hv.abs() + SUB)
            if act == "sigmoid":   # 1 / (1 + expf(-z)) is 0 once expf overflows (z < -88): h < 2^-126 there
                hbar = hbar + MIN_NORMAL
        else:
            hv, hbar = Z, torch.zeros_like(Z)
        if scope == "R-CNN1":
            hv = hv + nchw(x2)
            chk.add("ds_pw_fwd_kernel H", yp, hv, 2 * U * hv.abs() + TINY)
        else:
            if e["r"]:
                hv, hbar = O.depth_to_space(hv, e["r"]), O.depth_to_space(hbar, e["r"])
            Hc = T("H:" + scope, (hv.shape[2], hv.shape[3]), hv.shape[1])
            chk.add("ds_pw_fwd_kernel H", Hc, hv, hbar + TINY)

        # ---- activation gradient (bit for bit where the kernel's arithmetic is a fixed sequence of fp32 products)
        g32 = out_grad(scope, torch.float32)
        dZ32 = T("dZ:" + scope, (hh, ww), cout, torch.float32)
        dZ = dZ32.double()
        if not activated:
            chk.add("ds_act_bwd_kernel", dZ, g32.double(), TINY)
        else:
            z32 = T("Z:" + scope, (hh, ww), cout, torch.float32)
            gm = g32
            if keep < 1.0:
                gm = torch.where(mask > 0, g32 * torch.tensor(np.float32(inv_keep), device=dev()), torch.zeros_like(g32))
            if act in ("prelu", "relu", "leaky_relu"):
                if act == "prelu":
                    a32 = alpha.float().view(1, -1, 1, 1)
                    ref = torch.where(z32 > 0, gm, a32 * gm)
                    E = T("E:" + scope, (hh, ww), cout)
                    chk.add("ds_act_bwd_kernel E", E, (gm * torch.clamp_max(z32, 0.0)).double(), TINY)
                elif act == "relu":
                    ref = gm * (z32 > 0).float()
                else:
                    ref = torch.where(z32 < 0, torch.tensor(np.float32(0.1), device=dev()) * gm, gm)
                chk.add("ds_act_bwd_kernel", dZ, ref.double(), TINY)
            else:
                d, dd = act_deriv(act, z32.double())
                hval = act_eval(act, z32.double(), None)
                ref = gm.double() * d
                dh = 4 * U * hval.abs() + (MIN_NORMAL if act == "sigmoid" else SUB)
                bar = gm.double().abs() * (dd * dh + 3 * U * d.abs()) + U * ref.abs() + 4 * SUB
                chk.add("ds_act_bwd_kernel", dZ, ref, bar)
        # the dead conv_W: only its L2 decay
        wc = wts[scope + "/conv_W"]
        want = vec(l2 * wc)
        chk.add("grad_finalize_kernel conv_W", grad(scope + "/conv_W"), want, U * want.abs() + TINY)

        # ---- bias / slope sums
        ppb, nblk = cs_launch(npx, sm)
        if e["bias"]:
            ref, bar = finalize(scope + "/conv_B", dZ.sum(dim=(0, 2, 3)), (npx + 4) * U * dZ.abs().sum(dim=(0, 2, 3)))
            chk.add("ds_colsum_kernel bias", grad(scope + "/conv_B"), ref, bar)
            blocks["ds_colsum_kernel"] = max(blocks["ds_colsum_kernel"], nblk)
        if alpha is not None:
            E = T("E:" + scope, (hh, ww), cout)
            ref, bar = finalize(a_name, E.sum(dim=(0, 2, 3)), (npx + 4) * U * E.abs().sum(dim=(0, 2, 3)))
            chk.add("ds_colsum_kernel slope", grad(a_name), ref, bar)

        # ---- pointwise filter gradient
        ssum = torch.einsum("nchw,ndhw->cd", Uc, dZ)
        sabs = torch.einsum("nchw,ndhw->cd", Uc.abs(), dZ.abs())
        ref, bar = finalize(scope + "/pointwise_W", ssum, (ppb + nblk) * U * sabs)
        chk.add("ds_dpw_kernel", grad(scope + "/pointwise_W")[0, 0], ref, bar)
        blocks["ds_dpw_kernel"] = max(blocks["ds_dpw_kernel"], nblk)

        # ---- gradient at the depthwise output
        dU = T("dU:" + scope, (hh, ww), cin)
        ref = torch.einsum("ndhw,cd->nchw", dZ, pw)
        sabs = torch.einsum("ndhw,cd->nchw", dZ.abs(), pw.abs())
        chk.add("ds_du_kernel", dU, ref, cout * (U * sabs + SUB))

        # ---- depthwise filter gradient
        ppb, lanes, nblk = ddw_launch(npx, cin, sm)
        ssum = torch.nn.grad.conv2d_weight(inp, (cin, 1, k, k), dU, padding=k // 2, groups=cin)
        sabs = torch.nn.grad.conv2d_weight(inp.abs(), (cin, 1, k, k), dU.abs(), padding=k // 2, groups=cin)
        ref, bar = finalize(scope + "/depthwise_W", ssum.permute(2, 3, 0, 1), (cdiv(ppb, lanes) + lanes + nblk) * U * sabs.permute(2, 3, 0, 1))
        chk.add("ds_ddw_kernel", grad(scope + "/depthwise_W"), ref, bar)
        blocks["ds_ddw_kernel"] = max(blocks["ds_ddw_kernel"], nblk)

        # ---- gradient at the layer's input (written, or added to what the previous writer left)
        if scope == "CNN1":
            continue
        v = F.conv_transpose2d(dU, dwt, padding=k // 2, groups=cin)
        sv = F.conv_transpose2d(dU.abs(), dwt.abs(), padding=k // 2, groups=cin)
        bar = k * k * (U * sv + SUB)
        if e["prev"] is not None:
            pname, sl = e["prev"]
            pe = tab[pname[3:]]
            prev = T(pname, pe["res"], pe["cin"])
            if sl is not None:
                prev = prev[:, sl[0]:sl[1]]
            v = prev + v
            bar = bar + U * v.abs() + SUB
        got = T("dH:" + scope, (hh, ww), cin)
        chk.add("ds_dx_kernel", got, v, bar + TINY)
    return blocks


def run_case(cfg_kw, wts, x, x2, y, keep, seed, act="prelu", tag="", extra=None):
    """One captured narrow step under the profiler: every kernel of NARROW reached, every bar held.  `extra(eng)` runs
    on the engine after the checks."""
    from helper import engine as E
    eng = E.Engine(E.make_config(dropout_keep=keep, activator=act, **cfg_kw))
    eng.set_params({k: v.astype(np.float32) for k, v in wts.items()})
    eng.set_option("grad_capture", 1)
    _, names = launched_kernels(lambda: eng.train_step_host(x, x2, y, lr=0.002, seed=seed, apply_update=False))
    assert_kernels_ran(names, NARROW)
    wide = sorted(n for n in names if "conv_tc_kernel" in n or "wgrad_tc_kernel" in n)
    assert not wide, wide
    chk = Checker()
    blocks = check_ds_step(eng, O.OracleConfig(**cfg_kw), wts, act, x, x2, y, keep, seed, chk)
    report(tag, chk)
    print(tag, "most blocks:", blocks)
    if extra is not None:
        extra(eng)
    eng.close()
    assert not chk.bad(), chk.bad()
    return blocks


def he_case(kw, keep, shape, seed=5, act="prelu"):
    cfg, wts, eng, x, x2, y = setup(kw, keep, *shape, seed=seed)
    eng.close()
    if act != "prelu":
        wts = {k: v for k, v in wts.items() if k in set(A.variable_names(cfg, act))}
    return wts, x, x2, y


# ------------------------------------------------------------------------------- (a) the graphs of test_gpu_train ----
DS_CASES = [("ds-x2-nodrop", DS2, 1.0, (2, 9, 7)), ("ds-x2-drop", DS2, 0.8, (2, 12, 10)), ("ds-x4-drop", DS4, 0.8, (2, 8, 11)),
            ("ds-x4-1x1", DS4, 1.0, (1, 1, 1)), ("ds-x4-wide", DS4W, 0.8, (1, 6, 5)), ("ds-x3-oddw", DS3, 0.8, (2, 7, 9))]


@pytest.mark.parametrize("kw,keep,shape", [c[1:] for c in DS_CASES], ids=[c[0] for c in DS_CASES])
def test_ds_kernels_isolated(kw, keep, shape):
    wts, x, x2, y = he_case(kw, keep, shape)
    run_case(kw, wts, x, x2, y, keep, 4321, tag=str(shape))


# ----------------------------------------------------------------------------------------- (b) other activators ----
@pytest.mark.parametrize("act", ["relu", "leaky_relu", "sigmoid", "tanh", "selu"])
@pytest.mark.parametrize("kw,shape", [(DS2, (2, 12, 10)), (DS4, (2, 8, 11))], ids=["x2", "x4"])
def test_ds_kernels_isolated_activators(kw, shape, act):
    wts, x, x2, y = he_case(kw, 0.8, shape, act=act)
    run_case(kw, wts, x, x2, y, 0.8, 77, act=act, tag=act)


# --------------------------------------------------------------------------- (c), (d) the shipped DS checkpoint ----
def cds():
    return MODEL_FLAGS[CDS], {k: v.astype(np.float32) for k, v in load_golden_weights(CDS).items()}


def test_ds_kernels_on_real_patches():
    """The shipped c-DCSCN x4 depthwise-separable checkpoint on Set5 / Set14 patches, y = ground truth, keep 0.8."""
    kw, wts = cds()
    x, x2, y = real_patches(4, 6, 32, 32, 37)
    run_case(kw, wts, x, x2, y, 0.8, 99, tag="cdcscn-ds real")


def test_ds_kernels_at_benchmark_train_shape():
    """The same checkpoint on 64 real 48 x 48 patches at x4 (2.36 M HR pixels): every reduction kernel runs on many
    blocks, whose partial sums meet in atomicAdds."""
    kw, wts = cds()
    x, x2, y = real_patches(4, 64, 48, 48, 24)
    blocks = run_case(kw, wts, x, x2, y, 0.8, 5, tag="cdcscn-ds 64x48x48")
    for kname in ("ds_colsum_kernel", "ds_dpw_kernel", "ds_ddw_kernel"):
        assert blocks[kname] >= 64, (kname, blocks)


# ------------------------------------------------------------------------------------- (e) residual extremes ----
@pytest.mark.parametrize("residual", [1e-3, 255.0], ids=["tiny", "large"])
def test_ds_kernels_at_residual_extremes(residual):
    from helper import engine as E
    kw, wts = cds()
    x, x2, _ = real_patches(4, 4, 24, 24, 29)
    eng = E.Engine(E.make_config(dropout_keep=1.0, **kw))
    eng.set_params(wts)
    yp = eng.forward_host(x, x2)
    eng.close()
    sign = np.where(np.random.RandomState(3).rand(*yp.shape) < 0.5, -1.0, 1.0).astype(np.float32)
    y = (yp + sign * np.float32(residual)).astype(np.float32)
    run_case(kw, wts, x, x2, y, 1.0, 11, tag="residual %g" % residual)


# ------------------------------------------------------------------------------------ (f) odd-sized images ----
def test_ds_kernels_on_odd_images_across_block_borders():
    """5 images of 13 x 23 LR pixels at x4 with the checkpoint's weights: the reduction blocks' pixel ranges start and
    end inside images and on their border rows.  Image 2 is black and CNN1 has zero biases, so CNN1's pre-activations
    there are exactly 0, where the PReLU gradient takes the slope (z > 0 is false)."""
    kw, wts = cds()
    wts = dict(wts, **{"CNN1/conv_B": np.zeros_like(wts["CNN1/conv_B"])})
    n, h, w = 5, 13, 23
    g = np.random.RandomState(17)
    x = (g.rand(n, h, w, 1) * 255).astype(np.float32)
    x[2] = 0.0
    x2 = np.repeat(np.repeat(x, 4, axis=1), 4, axis=2)
    y = np.clip(x2 + g.randn(*x2.shape) * 10, 0, 255).astype(np.float32)
    sm = sm_count()
    for r in (1, 2, 4):   # LR, 2x and 4x layers: every block edge lies inside an image row
        ppb, nblk = cs_launch(n * r * h * r * w, sm)
        assert nblk > 1 and ppb % (r * w) != 0, (r, ppb)

    def zero_z(eng):
        z = eng.get_train_tensor("Z:CNN1", (n, h, w, 32))
        assert (z[2, 1:-1, 1:-1] == 0).all()
    blocks = run_case(kw, wts, x, x2, y, 0.8, 31, tag="odd 5x13x23", extra=zero_z)
    for kname in ("ds_colsum_kernel", "ds_dpw_kernel", "ds_ddw_kernel"):
        assert blocks[kname] > 1, (kname, blocks)


# ------------------------------------------------------------------ (g) graphs the train kernels once refused ----
WIDE_NARROW = [("upps-288", UPPS288, (2, 9, 11)), ("a1b1-384", A1B1_384, (2, 10, 9))]


@pytest.mark.parametrize("kw,shape", [c[1:] for c in WIDE_NARROW], ids=[c[0] for c in WIDE_NARROW])
def test_wide_layers_of_narrow_graphs_isolated(kw, shape):
    wts, x, x2, y = he_case(kw, 0.8, shape)
    run_case(kw, wts, x, x2, y, 0.8, 4321, tag=str(kw.get("scale", 2)))


@pytest.mark.parametrize("kw,shape", [c[1:] for c in WIDE_NARROW], ids=[c[0] for c in WIDE_NARROW])
def test_wide_layers_of_narrow_graphs_match_oracle(kw, shape):
    """End to end against fp64 autograd, with the bars of test_depthwise_separable_gradients_match_oracle."""
    test_depthwise_separable_gradients_match_oracle(kw, 0.8, shape)


# ------------------------------------------------------------------------------------ (h) wide DS graphs ----
def test_wide_ds_chain_rule_isolated():
    """L8 F96: the dense step's kernels on the composed filters (check_step), ds_compose_kernel bit for bit and
    ds_decompose_kernel within one fp32 rounding of the fp64 chain rule from the captured composed gradients."""
    kw = dict(depthwise_separable=True, layers=8, filters=96)
    n, h, w = 1, 12, 14
    keep, seed = 0.8, 1234
    cfg, wts, eng, x, x2, y = setup(kw, keep, n, h, w)
    eng.set_option("grad_capture", 1)
    _, names = launched_kernels(lambda: eng.train_step_host(x, x2, y, lr=0.002, seed=seed, apply_update=False))
    assert_kernels_ran(names, WIDE + ["conv_tc_kernel", "wgrad_tc_kernel", "loss_kernel", "grad_finalize_kernel"])
    count = n * cfg.scale ** 2 * h * w
    G = 2.0 ** round(math.log2(count / 2.0))
    l2 = float(np.float32(cfg.l2_decay))
    w32 = {k: v.astype(np.float32) for k, v in wts.items()}
    comp, dwc = {}, {}
    bad = []
    for scope, k, cin, cout, bias, act in O.layer_table(cfg):
        want = w32[scope + "/depthwise_W"][:, :, :, 0][:, :, :, None] * w32[scope + "/pointwise_W"][0, 0][None, None]
        got = eng.get_train_tensor("Wc:" + scope, (k, k, cin, cout))
        if not np.array_equal(got, want.astype(np.float32)):
            bad.append(("ds_compose_kernel", scope))
        comp[scope + "/conv_W"] = got.astype(np.float64)
        dwc[scope] = eng.get_train_tensor("dWc:" + scope, (k, k, cin, cout)).astype(np.float64)
    assert not bad, bad
    wc = dict(wts, **comp)

    def get_grad(name):
        if name.endswith("/conv_W"):
            return dwc[name[:-7]] / G + l2 * comp[name]
        return eng.get_grad(name)

    chk = check_step(eng, kw, wc, x, x2, y, keep, seed, Checker(), get_grad=get_grad)
    for scope, k, cin, cout, bias, act in O.layer_table(cfg):
        gc_ = torch.from_numpy(dwc[scope]).to(dev())
        dw = vec(wts[scope + "/depthwise_W"])[:, :, :, 0]
        pw = vec(wts[scope + "/pointwise_W"])[0, 0]
        ref = (gc_ * pw).sum(dim=3) / G
        sabs = (gc_.abs() * pw.abs()).sum(dim=3) / G
        chk.add("ds_decompose_kernel dw", vec(eng.get_grad(scope + "/depthwise_W"))[:, :, :, 0], ref,
                U * ref.abs() + cout * 2.0 ** -53 * sabs + TINY)
        ref = (gc_ * dw[:, :, :, None]).sum(dim=(0, 1)) / G
        sabs = (gc_.abs() * dw.abs()[:, :, :, None]).sum(dim=(0, 1)) / G
        chk.add("ds_decompose_kernel pw", vec(eng.get_grad(scope + "/pointwise_W"))[0, 0], ref,
                U * ref.abs() + k * k * 2.0 ** -53 * sabs + TINY)
        dead = vec(np.float32(cfg.l2_decay) * w32[scope + "/conv_W"])
        chk.add("grad_finalize_kernel conv_W", vec(eng.get_grad(scope + "/conv_W")), dead, U * dead.abs() + TINY)
    report("wide L8F96", chk)
    eng.close()
    assert not chk.bad(), chk.bad()
