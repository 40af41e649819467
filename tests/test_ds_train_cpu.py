"""CPU checks of the depthwise-separable train step's coverage and limits (no GPU needed).

* Every depthwise-separable train kernel in the built library (nm -C) is named by a case of
  test_gpu_ds_backward_paths.py, so a new one cannot ship without an isolated backward check.
* Every graph that ds_tile_fits (engine.cu) sends to the fp32 CUDA-core kernels also passes train_step_ds_impl's width
  check: the layer shapes the predicate accepts are restated here from the source's constants and scanned."""
import os
import re
import subprocess

import dcscn_oracle as O
from conftest import PKG
from test_gpu_ds_backward_paths import A1B1_384, NARROW, UPPS288, WIDE

CSRC = os.path.join(PKG, "csrc")
INFERENCE_DS = {"ds_tile_kernel", "ds_single_kernel", "ds_single4_kernel", "ds_act_kernel"}


def test_every_ds_train_kernel_has_a_backward_case():
    lib = os.path.join(CSRC, "libdcscn_b200.so")
    syms = subprocess.run(["nm", "-C", lib], check=True, capture_output=True, text=True).stdout
    built = set(re.findall(r"dcscn::(ds_[a-z0-9_]+_kernel)[(<]", syms)) - INFERENCE_DS
    assert {"ds_dpw_kernel", "ds_ddw_kernel", "ds_compose_kernel", "ds_decompose_kernel"} <= built, sorted(built)
    assert not sorted(built - set(NARROW + WIDE)), sorted(built - set(NARROW + WIDE))


def constants(fname):
    src = open(os.path.join(CSRC, fname)).read()
    return {k: eval(v) for k, v in re.findall(r"constexpr int (k\w+) = ([0-9 */+]+);", src)}


DT = constants("conv_ds_tile.cuh")
DP = constants("train_ds.cuh")


def ds_tile_launch_smem(k, cin, cout):
    """engine.cu ds_tile_launch_smem."""
    cols = ((cout + 3) & ~3) if cout < 32 else 32
    tcols = 4 if cols <= 4 else 8 if cols <= 8 else 16 if cols <= 16 else 24 if cols <= 24 else 32
    in_px = (DT["kDtT"] + 2) * DT["kDtS"] if k == 3 else DT["kDtThreads"]
    cache = DT["kDtThreads"] * DT["kDtCP"] if (k == 3 and cout > 32 and cin <= DT["kDtCC"]) else 0
    return (in_px * DT["kDtCP"] + cin * tcols + k * k * cin + cache) * 4


def ds_tile_accepts(k, cin, cout):
    return k in (1, 3) and not (cout > 32 and cin > DT["kDtCC"]) and ds_tile_launch_smem(k, cin, cout) <= 200 * 1024


def ds_tile_fits(cfg):
    """engine.cu ds_tile_fits for a pixel-shuffler graph."""
    T = sum((f + 3) & ~3 for f in O.feature_filters(cfg))
    cps = cfg.nin_filters + cfg.nin_filters2
    if cps > 32 or not ds_tile_accepts(1, T, cps):
        return False
    for scope, k, cin, cout, _, _ in O.layer_table(cfg):
        if scope in ("A1", "B1"):
            continue
        if cin == 1 and cout == 1:
            if k not in (1, 3):
                return False
        elif not ds_tile_accepts(k, cin, cout):
            return False
    return True


def train_accepts(k, cin, cout):
    """train_step_ds_impl: a 1x1 or 3x3 filter, and ds_dpw_kernel stages at least one pixel in 48 KB."""
    w = cin + min(cout, DP["kDsDpwCols"])
    return k in (1, 3) and min(DP["kDsDpwSmemFloats"] // w, DP["kDsDpwChunk"]) >= 1


def test_every_layer_ds_tile_accepts_trains():
    # the launch size depends on cout only through its 4-column group up to 32 and whether cout > 32
    couts = list(range(1, 34)) + [64, 256, 257, 288, 1 << 20]
    widest = 0
    for k in (1, 3):
        for cout in couts:
            for cin in range(1, 20000):
                if ds_tile_accepts(k, cin, cout):
                    widest = max(widest, cin)
                    assert train_accepts(k, cin, cout), (k, cin, cout)
    assert 1000 < widest < DP["kDsDpwSmemFloats"] - DP["kDsDpwCols"], widest
    # A1 / B1 are admitted through the fused A1 | B1 launch: cps <= 32 columns over T <= the same widest input
    for T in range(1, 20000, 4):
        for cps in range(2, 33):
            if ds_tile_accepts(1, T, cps):
                assert train_accepts(1, T, cps - 1), (T, cps)


def test_graphs_once_refused_are_narrow():
    """The two graph families of test_gpu_ds_backward_paths.py (g) run inference on the fp32 kernels, and each has a
    layer beyond the width check the train step used to make (cin, cout <= 256, cin + cout <= 380)."""
    for kw in (UPPS288, A1B1_384):
        cfg = O.OracleConfig(**kw)
        assert ds_tile_fits(cfg), kw
        assert any(cin > 256 or cout > 256 or cin + cout > 380 for _, _, cin, cout, _, _ in O.layer_table(cfg)), kw
