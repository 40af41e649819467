"""Same-process bit-identity A/B of two builds of the C-ABI library: for each graph of a config matrix, both builds run a
forward, then (f16x3 only) two train steps with dropout, and every tensor the ABI can read back must be byte-identical:
the output, every named activation, every parameter, gradient and optimizer slot, every dcscn_get_train_tensor name
(zneg: included) and every dropout mask.  Refusals must carry the same message.  The train step accumulates filter,
bias and slope gradients with atomics, so their last bits (and what the optimizer makes of them) vary from run to run of
one build: build A runs twice, B is compared with A on every tensor A's two runs agree on, and the ones that vary are
listed.  A difference in a gradient, parameter or optimizer slot, or anything of the second step, is only meaningful
when it is not downstream of such a sum (two runs can round a sum alike by chance).
usage: python scripts/ab_tensors.py <libA.so> <libB.so>"""
import os
import re
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "dcscn-super-resolution_b200"))
from helper import engine as E  # noqa: E402

C7 = dict(layers=7, filters=32, min_filters=8, filters_decay_gamma=1.2, nin_filters=24, nin_filters2=8,
          reconstruct_layers=0, pixel_shuffler_filters=1)
CONFIGS = [   # id, make_config arguments, trains
    ("L12 x2 f16x3", dict(), True),
    ("L12 x2 f16x1", dict(precision=E.PRECISION_F16X1), False),
    ("L12 x4", dict(scale=4), True),
    ("L12 x3", dict(scale=3), True),
    ("L12 Up-TCNN x2", dict(transposed_upsampler=True), True),
    ("L12 cnn_size 5", dict(cnn_size=5), True),
    ("c-DCSCN DS x4 (narrow)", dict(C7, scale=4, depthwise_separable=True), True),
    ("DS wide x2", dict(layers=4, filters=40, min_filters=24, filters_decay_gamma=1.5, nin_filters=24, nin_filters2=16,
                        depthwise_separable=True), True),
    ("L12 x2 relu", dict(activator="relu"), True),
    ("L12 x2 sigmoid", dict(activator="sigmoid"), True),
]
N, H, W = 4, 20, 24
SEEDS = (11, 12)


def weights(shapes):
    rng = np.random.default_rng(0)
    out = {}
    for name, shape in sorted(shapes.items()):
        if name.endswith("_prelu"):
            out[name] = 0.1 + 0.05 * rng.standard_normal(shape)
        elif name.endswith("/conv_B"):
            out[name] = 0.01 * rng.standard_normal(shape)
        else:
            fan_in = int(np.prod(shape[:-1])) if len(shape) > 1 else 1
            out[name] = rng.standard_normal(shape) * np.sqrt(2.0 / max(fan_in, 1))
    return {k: v.astype(np.float32) for k, v in out.items()}


SIZE = re.compile(r"(?:has|expected) (\d+) elements")


def read(call, name, dtype=np.float32):
    """(bytes, None) of a named tensor, or (None, message) when the ABI refuses it.  The element count is read off the
    size check's message (a zero-element request)."""
    empty = np.empty(0, dtype)
    try:
        call(name, empty)
    except E.EngineError as e:
        m = SIZE.search(str(e))
        if not m:
            return None, str(e)
        a = np.empty(int(m.group(1)), empty.dtype)
        call(name, a)
        return a.view(np.uint8).copy(), None
    return empty.view(np.uint8).copy(), None


def collect(path, kw, trains):
    E._lib = None
    E.load_library(path)
    eng = E.Engine(E.make_config(**kw))
    eng.set_params(weights(eng.param_shapes()))
    lib, hd = eng.lib, eng.handle
    s = eng.config.scale
    g = torch.Generator().manual_seed(1)
    x = (torch.rand(N, H, W, 1, generator=g) * 255).cuda()
    x2 = (torch.rand(N, s * H, s * W, 1, generator=g) * 255).cuda()
    y = (torch.rand(N, s * H, s * W, 1, generator=g) * 255).cuda()
    out = {}
    scopes = [l for l in eng.param_shapes() if l.endswith("/conv_W") or l.endswith("/Tconv_W")]
    scopes = sorted({n.rsplit("/", 1)[0] for n in scopes})
    short = ["CNN%d" % (i + 1) for i in range(eng.config.layers + 1)] + ["A1", "B1", "B2", "Up-PS", "Up-PS2", "Up-TCNN"]
    fp = lambda a: a.ctypes.data_as(E.ctypes.POINTER(E.ctypes.c_float))  # noqa: E731
    act = lambda nm, a: eng._check(lib.dcscn_get_activation(hd, nm.encode(), fp(a), a.size))  # noqa: E731

    def activations(tag):
        for nm in short + ["R-CNN1/taps"]:
            out["%s act %s" % (tag, nm)] = read(act, nm)

    yo = torch.empty_like(x2)
    eng.forward(x, x2, yo)
    torch.cuda.synchronize()
    out["forward y"] = (yo.cpu().numpy().view(np.uint8).copy(), None)
    activations("forward")
    if not trains:
        return out
    eng.set_option("grad_capture", 1)
    tt = lambda nm, a: eng._check(lib.dcscn_get_train_tensor(hd, nm.encode(), fp(a), a.size))  # noqa: E731
    names = ["y_", "dY"] + [p + l for p in ("dZ:", "dH:", "zneg:") for l in short + ["A1+B1"]]
    names += [p + l for p in ("U:", "Z:", "H:", "E:", "dU:", "dZ:", "dH:", "Wc:", "dWc:") for l in scopes]

    def mask(nm, a):
        eng._check(lib.dcscn_dropout_mask(hd, nm.encode(), seed, N, H, W,
                                          a.ctypes.data_as(E.ctypes.POINTER(E.ctypes.c_uint8)), a.size))
    for k, seed in enumerate(SEEDS):
        loss, mse = eng.train_step(x, x2, y, 1e-3, seed)
        torch.cuda.synchronize()
        tag = "step%d " % k
        out[tag + "loss"] = (np.array([loss, mse], np.float32).view(np.uint8), None)
        for nm in names:
            out[tag + "train " + nm] = read(tt, nm)
        for nm in short:
            out[tag + "mask " + nm] = read(mask, nm, np.uint8)
        for nm in eng.param_shapes():
            out[tag + "param " + nm] = (eng.get_param(nm).view(np.uint8).copy(), None)
            out[tag + "grad " + nm] = (eng.get_grad(nm).view(np.uint8).copy(), None)
            for sl in range(eng.optimizer_slot_count):
                out[tag + "slot%d %s" % (sl, nm)] = (eng.get_optimizer_slot(nm, sl).view(np.uint8).copy(), None)
    activations("train")
    eng.close()
    return out


def main():
    paths = [os.path.abspath(p) for p in sys.argv[1:3]]
    print("A = %s\nB = %s" % tuple(paths))
    print("card: %s" % torch.cuda.get_device_name(0))
    def same(u, v):
        return u[1] == v[1] and (u[0] is None) == (v[0] is None) and (u[0] is None or np.array_equal(u[0], v[0]))

    bad = 0
    for cid, kw, trains in CONFIGS:
        a, b, a2 = (collect(p, kw, trains) for p in (paths[0], paths[1], paths[0]))
        keys = sorted(set(a) | set(b))
        if set(a) != set(b):
            print("%s: the builds read different tensor sets" % cid)
            bad += 1
            continue
        stable = [k for k in keys if same(a[k], a2[k])]
        diff = [k for k in stable if not same(a[k], b[k])]
        read_ok = sum(1 for k in stable if a[k][0] is not None)
        print("%-24s %4d tensors equal in A's two runs: %s; %3d refusals; %3d vary run to run in A" % (
            cid, read_ok, "B IDENTICAL" if not diff else "B DIFFERS: " + ", ".join(diff), len(stable) - read_ok,
            len(keys) - len(stable)))
        print("    varying in A: " + ", ".join(k for k in keys if k not in stable))
        bad += len(diff)
    print("ALL IDENTICAL" if bad == 0 else "%d differences" % bad)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
