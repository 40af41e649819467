"""
A long-lived engine computes what a fresh one does (run with `-m gpu` on an H100).  train.py and evaluate.py keep one
handle for a whole run: it interleaves train steps with evaluation on whole images of many sizes, self-ensembles,
tiled forwards and batches of other shapes, and keeps grow-only workspaces, per-(n, h, w) launch plans and CUDA graphs,
buffers that several layers share (dzl / dtmp at pitch maxw) and the tiled, ensemble, evaluation and crop stores.

Every test builds two engines the same way, A and B, and runs the same main line on both.  A also runs distractors
between the main-line operations; B never does.  At every main-line point A's results must equal B's:
  * forward outputs, the loss, y_, dY and every captured dZ / dH / zneg plane (and the fp32 tensors of the
    depthwise-separable step) bit for bit;
  * every gradient within 1e-4 of its tensor's max (fp32 atomics reorder sums, as in
    test_device_refresh_equals_host_repack) and finite;
  * after an update from the same gradient buffer: every weight, optimizer slot and the update count bit for bit.
B's main line is pinned to fp64 once per family (check_step / isolated_layers on B's captured planes, or fp64 autograd
where those do not apply), so bit identity carries that guarantee over to A.

  1. non-finite history in training: steps whose planes overflow (target +-1e30, NaN / Inf pixels, input x 1e6);
  2. non-finite history in inference: f16x3 / f16x1, fused / unfused R-CNN1, tiled forwards, the self-ensemble and
     evaluate_image, and a training engine;
  3. shape and mode history: workspace regrowth, other shapes and batch sizes, graph capture and replay at one input
     pointer, ensembles, tiled forwards, evaluation, bicubic resize, the crop and patch stores and option switches.

The dgrad twins read their sources over pad16(C) channels, and act_grad8_kernel zeroes a result's pad channels only up
to 8 ceil(C / 8), so channels 8 ceil(C / 8) .. pad16(C) - 1 of the shared plane dzl keep a wider layer's dZ from the
step before (CNN2 of L12 reads channels 168-175, which CNN1 wrote).  That history cannot leak: every fp16 plane is
written through split_f16 / split_f16x2, which clamp to +-65504 (NaN becomes -65504, lo then 0), so a stale channel is
always finite and meets a zero weight row as an exact 0.  Test 1 pins that on the L12 widths.
"""
import numpy as np
import pytest
import torch

import dcscn_oracle as O
import tconv_oracle as T
from conftest import MODEL_FLAGS
from test_gpu_backward_paths import Checker, check_step, real_engine, real_patches, report
from test_gpu_ds_wide import TRAIN_CASES as DS_WIDE_CASES
from test_gpu_forward_paths import isolated_layers
from test_gpu_tconv import TRAIN as TCONV, setup as tconv_setup
from test_gpu_train import (DS3, GRADIENT_CASES, L12, SMALL, assert_kernels_ran, launched_kernels, oracle_masks, setup,
                            train_tensors)

pytestmark = pytest.mark.gpu

GRAD_REL = 1e-4        # fp32 atomics: the bar of test_device_refresh_equals_host_repack
LR = 0.002


# ------------------------------------------------------------------------------------------------ comparisons ----
def capture_names(kw):
    """Every tensor name a train step of graph `kw` can capture (train_tensors drops the ones it did not keep)."""
    ocfg = {k: v for k, v in kw.items() if k not in ("activator", "transposed_upsampler")}
    scopes = [t[0] for t in O.layer_table(O.OracleConfig(**ocfg))]
    scopes += [sc.split("/")[0] for sc in scopes] + ["A1+B1", "Up-TCNN"]
    prefixes = ("dZ:", "dH:", "zneg:", "Wc:")          # not "dWc:": filter gradients, summed by fp32 atomics
    if kw.get("depthwise_separable"):
        prefixes += ("U:", "Z:", "H:", "E:", "dU:")
    return ["y_", "dY"] + sorted({p + sc for p in prefixes for sc in scopes})


class Pair:
    """Engines A (with history) and B (main line only) and the record of what was compared."""

    def __init__(self, a, b, kw):
        self.a, self.b, self.kw = a, b, kw
        self.shapes = a.param_shapes()
        self.names = capture_names(kw)
        self.distractors = []
        self.compared = set()
        self.points = 0

    def close(self):
        self.a.close()
        self.b.close()

    def distract(self, name, fn):
        """Runs fn(A) and records its name."""
        out = fn(self.a)
        torch.cuda.synchronize()
        self.distractors.append(name)
        return out

    def same(self, tag, fn):
        """fn(engine) on B and then on A: results equal bit for bit (arrays, floats or tuples of them)."""
        rb = fn(self.b)
        ra = fn(self.a)
        torch.cuda.synchronize()
        eq = _bit_equal(ra, rb)
        assert eq, (tag, "A differs from B after distractors", self.distractors)
        self.points += 1
        self.compared.add(tag)
        return rb

    def step(self, tag, x, x2, y, seed):
        """One captured main-line train step (no update) on both: loss, every captured tensor bit for bit, every gradient
        within GRAD_REL of its max and finite."""
        from helper import engine as E
        lb = self.b.train_step_host(x, x2, y, lr=LR, seed=seed, apply_update=False)
        la = self.a.train_step_host(x, x2, y, lr=LR, seed=seed, apply_update=False)
        assert _bit_equal(la, lb), (tag, "loss", la, lb, self.distractors)
        try:                                      # sigmoid graphs and the fp32 ds step keep no min(z, 0) planes
            self.b.get_train_tensor("zneg:CNN1", (1,))
        except E.EngineError as e:
            if "keeps no min(z, 0)" in str(e):
                self.names = [k for k in self.names if not k.startswith("zneg:")]
        assert np.isfinite(lb).all(), (tag, lb)
        ta, tb = train_tensors(self.a, self.names), train_tensors(self.b, self.names)
        assert set(ta) == set(tb), (tag, sorted(set(ta) ^ set(tb)))
        assert sum(k.startswith("dZ:") for k in tb) >= 3 and {"y_", "dY"} <= set(tb), sorted(tb)
        differ = [k for k in tb if not np.array_equal(ta[k], tb[k])]
        assert not differ, (tag, "tensors differ", differ, self.distractors)
        bad = []
        for k in self.shapes:
            ga, gb = self.a.get_grad(k), self.b.get_grad(k)
            if not (np.isfinite(ga).all() and np.isfinite(gb).all()):
                bad.append((k, "non-finite", int((~np.isfinite(ga)).sum()), int((~np.isfinite(gb)).sum())))
            elif not np.abs(ga - gb).max() <= GRAD_REL * np.abs(gb).max() + 1e-9:
                bad.append((k, float(np.abs(ga - gb).max()), float(np.abs(gb).max())))
        assert not bad, (tag, "gradients", bad, self.distractors)
        self.points += 1
        self.compared.update(["loss"] + sorted(tb) + ["grad:" + k for k in self.shapes])
        return lb

    def update(self, tag):
        """The same optimizer update on both: B's gradient buffer takes A's (the two differ only by fp32 atomic order, which
        step() bounds), then apply_gradients on each.  Weights, every optimizer slot and the update count bit for bit."""
        ga, gb = self.a.grad_tensor(), self.b.grad_tensor()
        gb.copy_(ga)
        torch.cuda.synchronize()
        self.a.apply_gradients(LR)
        self.b.apply_gradients(LR)
        torch.cuda.synchronize()
        assert self.a.adam_step == self.b.adam_step >= 1
        differ = [k for k in self.shapes if not np.array_equal(self.a.get_param(k), self.b.get_param(k))]
        for s in range(self.b.optimizer_slot_count):
            differ += ["slot%d:%s" % (s, k) for k in self.shapes
                       if not np.array_equal(self.a.get_optimizer_slot(k, s), self.b.get_optimizer_slot(k, s))]
        assert not differ, (tag, "update differs", differ, self.distractors)
        self.points += 1
        self.compared.update(["weights", "optimizer slots", "update count"])

    def params(self):
        return {k: self.b.get_param(k).astype(np.float64) for k in self.shapes}

    def summary(self, tag):
        grads = sum(k.startswith("grad:") for k in self.compared)
        rest = sorted(k for k in self.compared if not k.startswith("grad:"))
        print("%s: distractors on A: %s" % (tag, ", ".join(self.distractors)))
        print("%s: %d comparison points; compared bit for bit: %s; gradients of %d variables" %
              (tag, self.points, " ".join(rest), grads))


def _bit_equal(a, b):
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_bit_equal(u, v) for u, v in zip(a, b))
    if isinstance(a, torch.Tensor):
        a, b = a.cpu().numpy(), b.cpu().numpy()
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()      # NaN payloads and -0 included


# --------------------------------------------------------------------------------- 1. non-finite train history ----
def overflow_steps(pair, x, x2, y, seed):
    """Distractor steps on A without update whose planes overflow; returns their losses (at least one non-finite)."""
    g = np.random.RandomState(seed)
    sign = np.where(g.rand(*y.shape) < 0.5, -1.0, 1.0).astype(np.float32)
    xbad = bad_pixels(x, seed)
    losses = [
        pair.distract("step y=+-1e30", lambda e: e.train_step_host(x, x2, sign * np.float32(1e30), lr=LR, seed=seed + 1,
                                                                     apply_update=False)),
        pair.distract("step NaN/Inf pixels", lambda e: e.train_step_host(xbad, x2, y, lr=LR, seed=seed + 2,
                                                                           apply_update=False)),
        pair.distract("step x*1e6", lambda e: e.train_step_host(x * np.float32(1e6), x2 * np.float32(1e6), y, lr=LR,
                                                                  seed=seed + 3, apply_update=False)),
    ]
    print("distractor losses:", losses)
    assert not np.isfinite(losses).all(), losses
    return losses


def family(case):
    """(kw, make_engine(), x, x2, y, keep, pin) of one family of test 1.  pin(eng, w, x, x2, y, keep, seed) checks the
    last captured step of `eng`, run at weights `w`, against fp64."""
    gc = {c[0]: c for c in GRADIENT_CASES}

    def pin_isolated(act="prelu"):
        def pin(eng, kw, w, x, x2, y, keep, seed):
            kw = {k: v for k, v in kw.items() if k != "activator"}
            chk = check_step(eng, kw, w, x, x2, y, keep, seed, Checker(), act=act)
            report(case, chk)
            assert not chk.bad(), chk.bad()
        return pin

    def pin_autograd(oracle, bar):
        def pin(eng, kw, w, x, x2, y, keep, seed):
            cfg = oracle(kw)
            n, h, wd = x.shape[:3]
            masks = oracle_masks(eng, cfg, seed, n, h, wd) if keep < 1.0 else None
            orc = (T.Oracle if oracle is tconv_cfg else O.Oracle)(cfg, w, torch.float64)
            _, _, grads = orc.loss_and_grads(x.astype(np.float64), x2.astype(np.float64), y.astype(np.float64),
                                             keep_prob=keep, masks=masks)
            worst = 0.0
            for name, gref in grads.items():
                ratio = float(np.abs(eng.get_grad(name) - gref).max()) / (bar * np.abs(gref).max() + 1e-7)
                worst = max(worst, ratio)
                assert ratio <= 1.0, (name, ratio)
            print(case, "gradients against fp64 autograd: worst error / bar %.3f" % worst)
        return pin

    if case.startswith("L12"):
        model = L12[int(case[-1])]

        def make():
            return real_engine(model, 0.8)[2]
        kw = MODEL_FLAGS[model]
        x, x2, y = real_patches(kw.get("scale", 2), 4, 24, 24, 37)
        return kw, make, x, x2, y, 0.8, pin_isolated()
    if case in gc:
        _, kw, weights, keep, shape, _ = gc[case]
        if weights != "he":
            kw = MODEL_FLAGS[weights]

        def make():
            return setup(kw, keep, *shape, weights=weights)[2]
        _, _, e, x, x2, y = setup(kw, keep, *shape, weights=weights)
        e.close()
        return kw, make, x, x2, y, keep, pin_isolated()
    if case in ("x8", "sigmoid"):
        kw = dict(SMALL, scale=8) if case == "x8" else dict(SMALL, activator="sigmoid")
        shape = (1, 6, 7) if case == "x8" else (2, 12, 10)
        kw_o = {k: v for k, v in kw.items() if k != "activator"}

        def make():
            from helper import engine as E
            cfg = O.OracleConfig(**kw_o)
            e = E.Engine(E.make_config(dropout_keep=0.8, **kw))
            e.set_params(O.he_init_weights(cfg, seed=0))
            return e
        _, _, e, x, x2, y = setup(kw_o, 0.8, *shape)
        e.close()
        return kw, make, x, x2, y, 0.8, pin_isolated(kw.get("activator", "prelu"))
    if case == "ds-narrow":
        def make():
            return setup(DS3, 0.8, 2, 7, 9, seed=5)[2]
        _, _, e, x, x2, y = setup(DS3, 0.8, 2, 7, 9, seed=5)
        e.close()
        return DS3, make, x, x2, y, 0.8, pin_autograd(lambda kw: O.OracleConfig(**kw), 2e-4)
    if case == "ds-wide":
        _, kw, shape = DS_WIDE_CASES[0]

        def make():
            return setup(kw, 0.8, *shape, seed=5)[2]
        _, _, e, x, x2, y = setup(kw, 0.8, *shape, seed=5)
        e.close()
        return kw, make, x, x2, y, 0.8, pin_autograd(lambda kw: O.OracleConfig(**kw), 2e-3)
    if case == "tconv":
        kw = dict(TCONV, scale=2)

        def make():
            return tconv_setup(kw, 0.8, 2, 9, 8, seed=5)[2]
        _, _, e, x, x2, y = tconv_setup(kw, 0.8, 2, 9, 8, seed=5)
        e.close()
        return kw, make, x, x2, y, 0.8, pin_autograd(tconv_cfg, 2e-3)
    raise ValueError(case)


def tconv_cfg(kw):
    return T.Config(**{k: v for k, v in kw.items() if k != "transposed_upsampler"})


TRAIN_FAMILIES = ["L12-x2", "L12-x4"] + [c[0] for c in GRADIENT_CASES] + ["ds-narrow", "ds-wide", "tconv", "x8",
                                                                           "sigmoid"]


@pytest.mark.parametrize("case", TRAIN_FAMILIES)
def test_train_step_after_non_finite_steps(case):
    """Warm-up step and update on both; on A three steps whose planes overflow (no update); then a main-line step, an
    update and a forward on both.  Every plane a later step reads over a padded channel extent (the dgrad twins' sources
    dzl / dzlast / dzup / dzb2 / dza1b1, the forward's feat / b1 / nin / mid, the fp32 ds_* buffers) must not carry the
    bad step into the next one."""
    kw, make, x, x2, y, keep, pin = family(case)
    pair = Pair(make(), make(), kw)
    for e in (pair.a, pair.b):
        e.set_option("grad_capture", 1)
    w = pair.params()
    pair.step("warm-up", x, x2, y, seed=11)
    pin(pair.b, kw, w, x, x2, y, keep, 11)
    pair.update("warm-up")
    overflow_steps(pair, x, x2, y, seed=31)
    pair.step("after overflow", x, x2, y, seed=12)
    pair.update("after overflow")
    pair.same("forward", lambda e: e.forward_host(x, x2))
    pair.summary(case)
    pair.close()


# ------------------------------------------------------------------------------ 2. non-finite inference history ----
INFER_CASES = [
    # id, precision (0 f16x3, 1 f16x1), fuse_last, workspace_mb, training engine
    ("f16x3-fused", 0, 1, 0, False),
    ("f16x1-fused", 1, 1, 0, False),
    ("f16x3-unfused", 0, 0, 0, False),
    ("f16x1-unfused", 1, 0, 0, False),
    ("f16x3-tiled", 0, 1, 1, False),
    ("f16x1-tiled", 1, 1, 1, False),
    ("train-engine", 0, 1, 0, True),
]


def bad_pixels(x, seed):
    xb = x.copy()
    flat = xb.reshape(-1)
    pos = np.random.RandomState(seed).permutation(flat.size)[:max(1, flat.size // 9)]   # a 1 x 1 image: its one pixel
    flat[pos[0::3]] = np.nan
    flat[pos[1::3]] = np.inf
    flat[pos[2::3]] = -np.inf
    return xb


@pytest.mark.parametrize("precision,fuse,mb,train", [c[1:] for c in INFER_CASES], ids=[c[0] for c in INFER_CASES])
def test_inference_after_non_finite_inputs(precision, fuse, mb, train):
    """Main line: a forward, an 8-flip self-ensemble and evaluate_image.  Distractors on A: forwards on NaN / Inf pixels and
    on inputs x 1e6, a self-ensemble of a NaN image and (training engine) train steps whose planes overflow.  The tiled
    cases run the main forward as batches of windows (workspace_mb = 1)."""
    from helper import engine as E
    kw = SMALL
    cfg = O.OracleConfig(**kw)
    w = O.he_init_weights(cfg, seed=0)
    npl = 2 if precision == 0 else 1

    def make():
        e = E.Engine(E.make_config(precision=precision, dropout_keep=0.8, **kw))
        e.set_params(w)
        e.set_option("fuse_last", fuse)
        if mb:
            e.set_option("workspace_mb", mb)
        return e
    pair = Pair(make(), make(), kw)
    g = np.random.RandomState(7)
    n, h, wd = (2, 96, 100) if mb else (2, 20, 22)
    x = (g.rand(n, h, wd, 1) * 255).astype(np.float32)
    x2 = (g.rand(n, 2 * h, 2 * wd, 1) * 255).astype(np.float32)
    img = (g.rand(61, 74, 1) * 255).astype(np.uint8)
    tx, tx2 = x[:, :12, :10].copy(), x2[:, :24, :20].copy()
    ty = np.clip(tx2 + g.randn(*tx2.shape).astype(np.float32) * 10, 0, 255).astype(np.float32)
    if train:
        pair.same("warm-up step", lambda e: e.train_step_host(tx, tx2, ty, lr=LR, seed=3, apply_update=False))
    y, names = launched_kernels(lambda: pair.b.forward_host(x, x2))
    assert_kernels_ran(names, ["tile_gather_kernel", "tile_stitch_kernel"] if mb else
                       ["conv_last_gather4_kernel" if fuse else "conv_last_kernel"])
    if not mb:   # B's main-line forward against the isolated per-layer fp64 references
        ratios = isolated_layers(pair.b, cfg, w, x, x2, y, npl, 0, fuse == 1)
        print("B forward, error / bar:", " ".join("%s %.3f" % kv for kv in ratios.items()))
        assert max(ratios.values()) <= 1.0, ratios
    pair.distract("forward NaN/Inf pixels", lambda e: e.forward_host(bad_pixels(x, 1), x2))
    pair.same("forward", lambda e: e.forward_host(x, x2))
    pair.distract("forward x*1e6", lambda e: e.forward_host(x * np.float32(1e6), x2 * np.float32(1e6)))
    if train:
        pair.distract("step NaN/Inf pixels", lambda e: e.train_step_host(bad_pixels(tx, 2), tx2, ty, lr=LR, seed=4,
                                                                          apply_update=False))
        pair.distract("step y=1e30", lambda e: e.train_step_host(tx, tx2, ty * np.float32(1e30), lr=LR, seed=5,
                                                                  apply_update=False))
    pair.same("forward", lambda e: e.forward_host(x, x2))
    pair.distract("ensemble NaN image", lambda e: e.forward_ensemble_host(bad_pixels(x[0, :30, :40], 3), None, 8))
    pair.same("ensemble-8", lambda e: e.forward_ensemble_host(x[0, :30, :40], None, 8))
    pair.distract("forward NaN/Inf pixels", lambda e: e.forward_host(bad_pixels(x, 4), bad_pixels(x2, 5)))
    pair.same("evaluate_image", lambda e: e.evaluate_image(img, 1, 255.0, 2))
    pair.distract("ensemble x*1e6", lambda e: e.forward_ensemble_host(x[1, :30, :40] * np.float32(1e6), None, 4))
    pair.same("evaluate_image-8", lambda e: e.evaluate_image(img, 8, 255.0, 0))
    pair.same("forward", lambda e: e.forward_host(x, x2))
    pair.summary("inference")
    pair.close()


# -------------------------------------------------------------------------------- 3. shape and mode history ----
def test_results_do_not_depend_on_shape_and_mode_history():
    """SMALL x2 at keep 0.8.  Between main-line operations (a captured train step and update, forwards at one shape and at
    one device input pointer, an 8-flip ensemble, evaluate_image) A grows its workspace, runs other shapes and batch
    sizes, a 1 x 1 image and an HR width that is not a multiple of 4 (gather vs gather4), builds and replays a graph at a
    pointer and writes new contents there, runs ensembles, a tiled forward and then workspace_mb = 0, evaluations,
    bicubic resizes, the crop and patch stores with steps at other seeds and patch sizes, and sets and restores every
    option.  A profiler trace shows once that the distractors reached the paths they name."""
    from helper import engine as E
    kw = SMALL
    cfg = O.OracleConfig(**kw)
    w = O.he_init_weights(cfg, seed=0)

    def make():
        e = E.Engine(E.make_config(dropout_keep=0.8, **kw))
        e.set_params(w)
        e.set_option("grad_capture", 1)
        return e
    pair = Pair(make(), make(), kw)
    a = pair.a
    g = np.random.RandomState(9)

    def inputs(n, h, wd):
        x = (g.rand(n, h, wd, 1) * 255).astype(np.float32)
        x2 = (g.rand(n, 2 * h, 2 * wd, 1) * 255).astype(np.float32)
        return x, x2
    x, x2 = inputs(2, 16, 20)                     # HR width 40: conv_last_gather4_kernel
    y = np.clip(x2 + g.randn(*x2.shape).astype(np.float32) * 10, 0, 255).astype(np.float32)
    xs, x2s = x[:, :12, :10].copy(), x2[:, :24, :20].copy()
    ys = y[:, :24, :20].copy()
    img = (g.rand(53, 66, 1) * 255).astype(np.uint8)
    dx = torch.from_numpy(x).cuda()               # the main line's device input pointers, one per engine
    dx2 = torch.from_numpy(x2).cuda()
    ptr = {id(pair.a): (dx.clone(), dx2.clone()), id(pair.b): (dx.clone(), dx2.clone())}

    def device_forward(e):
        px, px2 = ptr[id(e)]
        return e.forward(px, px2).cpu().numpy()

    main = [
        ("forward", lambda: pair.same("forward", lambda e: e.forward_host(x, x2))),
        ("device forward", lambda: pair.same("device forward", device_forward)),
        ("ensemble-8", lambda: pair.same("ensemble-8", lambda e: e.forward_ensemble_host(x[0], x2[0], 8))),
        ("evaluate_image", lambda: pair.same("evaluate_image", lambda e: e.evaluate_image(img, 1, 255.0, 2))),
        ("step", lambda: (pair.step("step", xs, x2s, ys, seed=21), pair.update("step"))),
    ]

    # ---- distractors (on A only)
    big = inputs(3, 70, 90)
    def grow(e):
        before = e.device_bytes
        e.forward_host(*big)
        assert e.device_bytes > before, (before, e.device_bytes)

    def shapes(e):
        for shp in [(1, 5, 7), (4, 3, 9), (3, 16, 20), (1, 1, 1)]:
            e.forward_host(*inputs(*shp))

    odd = inputs(1, 9, 11)                        # HR width 22: conv_last_gather_kernel
    gx, gx2 = (torch.from_numpy(v).cuda() for v in inputs(2, 16, 20))

    def graph(e):
        before = e.graph_replays
        for _ in range(3):                        # eager, capture, replay
            e.forward(gx, gx2)
        gx.copy_(torch.from_numpy(inputs(2, 16, 20)[0]))     # new contents at the same pointer
        e.forward(gx, gx2)
        torch.cuda.synchronize()
        assert e.graph_replays >= before + 3, (before, e.graph_replays)

    def main_pointer_new_contents(e):             # A's own main-line pointer: other contents, then the main contents back
        px, px2 = ptr[id(e)]
        px.copy_(torch.from_numpy(bad_pixels(x, 6)))
        e.forward(px, px2)
        e.forward(px, px2)
        px.copy_(dx)

    def tiled(e):
        e.set_option("workspace_mb", 1)
        e.forward_host(*big)
        e.set_option("workspace_mb", 0)

    def evaluate(e):
        e.evaluate_image((g.rand(37, 41, 1) * 255).astype(np.uint8), 8, 255.0, 0)
        e.evaluate_image((g.rand(90, 31, 1) * 255).astype(np.uint8), 1, 1.0, 4, bicubic=True)

    def bicubic(e):
        e.bicubic_resize(torch.from_numpy(g.rand(2, 13, 17).astype(np.float32)).cuda(), 40, 33)

    def crops(e):
        e.set_image_store([(g.rand(60, 70, 1) * 255).astype(np.uint8), (g.rand(40, 44, 3) * 255).astype(np.uint8)])
        c = [(0, 3, 5, 0), (1, 10, 2, 1), (0, 20, 30, 1)]
        e.gather_crops(c, 8)
        e.train_step_crops(c, 8, lr=LR, seed=77, apply_update=False)

    def patches(e):
        pg = np.random.RandomState(3)
        e.set_patch_store((pg.rand(6, 7, 9, 1) * 255).astype(np.uint8), (pg.rand(6, 14, 18, 1) * 255).astype(np.uint8),
                          (pg.rand(6, 14, 18, 1) * 255).astype(np.uint8))
        e.train_step_indexed([0, 3, 5], lr=LR, seed=78, mirror=[0, 1, 0], apply_update=False)
        e.train_step_host(*inputs(3, 9, 13), inputs(3, 9, 13)[1], lr=LR, seed=79, apply_update=False)

    def options(e):
        for key, value, restore in [("fuse_last", 0, 1), ("seg_chunks", 1, 0), ("graph", 0, 1), ("conv_impl", 1, 0)]:
            e.set_option(key, value)
            e.forward_host(x, x2)
            e.forward_host(x, x2)
            e.set_option(key, restore)
        for key in ("act_grad_impl", "wgrad_impl"):
            e.set_option(key, 1)
            e.train_step_host(xs, x2s, ys, lr=LR, seed=80, apply_update=False)
            e.set_option(key, 0)

    distractors = [("grow workspace", grow), ("other shapes, batch sizes, 1x1", shapes),
                   ("HR width 22 (gather)", lambda e: e.forward_host(*odd)), ("graph capture + replay + new contents", graph),
                   ("main pointer, other contents", main_pointer_new_contents), ("forward_host", lambda e: e.forward_host(*odd)),
                   ("ensemble-8 other image", lambda e: e.forward_ensemble_host(odd[0][0], None, 8)),
                   ("tiled forward, then workspace_mb=0", tiled), ("evaluate_image", evaluate), ("bicubic_resize", bicubic),
                   ("crop store: gather + step", crops), ("patch store: indexed step + other patch size", patches),
                   ("options set and restored", options), ("grow workspace again", lambda e: e.forward_host(*inputs(2, 90, 97)))]

    # once, under the profiler: the distractors reach what they name
    _, names = launched_kernels(lambda: (tiled(a), a.forward_host(*odd), crops(a), patches(a)))
    assert_kernels_ran(names, ["tile_gather_kernel", "tile_stitch_kernel", "conv_last_gather_kernel", "crop_gather_kernel",
                               "patch_gather_kernel", "act_grad8_kernel"])
    pair.distractors.append("profiled: tiled, HR width 22, crop store, patch store")
    # B's main line pinned to fp64: its first step (every backward kernel) and its forward at the updated weights
    pair.step("step", xs, x2s, ys, seed=21)
    chk = check_step(pair.b, kw, w, xs, x2s, ys, 0.8, 21, Checker())
    report("B step", chk)
    assert not chk.bad(), chk.bad()
    pair.update("step")
    yb = pair.same("forward", lambda e: e.forward_host(x, x2))
    ratios = isolated_layers(pair.b, cfg, pair.params(), x, x2, yb, 2, 0, True)
    print("B forward, error / bar:", " ".join("%s %.3f" % kv for kv in ratios.items()))
    assert max(ratios.values()) <= 1.0, ratios
    for op in main:
        op[1]()
    for i, (dname, fn) in enumerate(distractors):
        pair.distract(dname, fn)
        main[i % len(main)][1]()
    for op in main:
        op[1]()
    pair.summary("shape / mode history")
    pair.close()
