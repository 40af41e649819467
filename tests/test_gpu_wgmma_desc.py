"""Which wgmma descriptor reads a SWIZZLE_128B operand that starts part-way into a swizzle atom (csrc/conv_tc.cuh).

conv_tc_kernel loads one activation box of (TW + k - 1) x (TH + k - 1) pixels per 64-channel chunk and reads tap
(kx, ky) at a start kx + ky * W_box rows into it, with a stride of W_box rows between the operand's 8-row groups.  A
shift of one row is 128 bytes, not a whole 1024-byte swizzle atom.  tests/wgmma_desc_probe.cu TMA-loads such a box with
the kernel's tensor-map settings and runs wgmma.m64n16k16 on it at r = 0 ... 7 rows in and W_box = 10, 12, 16, 18,
with base_offset = 0 and with base_offset = (start >> 7) & 7, against the same wgmma on an aligned tile that TMA
loaded at the shifted origin.

Established on an H100 80GB HBM3: the swizzle is a function of the shared-memory address itself, as TMA writes it, so
base_offset = 0 reads the right rows at every start and every stride tried (W_box = 10 included, whose stride is not
a multiple of 1024 bytes), and the (start >> 7) & 7 form reads wrong values whenever that is not 0.  conv_tc_kernel
therefore uses base_offset = 0 (make_smem_desc) for its chunk boxes."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
W_BOXES = [10, 12, 16, 18]

# Runs in a child process, so that the probe library (and its own CUDA runtime) never loads into the test process,
# whose later tests trace the engine's kernels with the profiler.  argv: library, output .npz
CHILD = """
import ctypes, sys
import numpy as np
lib = ctypes.CDLL(sys.argv[1])
lib.wgmma_desc_probe.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_float)]
res = {}
for w_box in %r:
    out = np.zeros((8, 3, 64, 16), np.float32)
    for r in range(8):
        rc = lib.wgmma_desc_probe(w_box, r, out[r].ctypes.data_as(ctypes.POINTER(ctypes.c_float)))
        assert rc == 0, (w_box, r, rc)
    res["w%%d" %% w_box] = out
np.savez(sys.argv[2], **res)
""" % (W_BOXES,)


def nvcc():
    if os.environ.get("NVCC"):
        return os.environ["NVCC"]
    found = shutil.which("nvcc")
    if found:
        return found
    from torch.utils.cpp_extension import CUDA_HOME
    return os.path.join(CUDA_HOME or "/usr/local/cuda", "bin", "nvcc")


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    """{W_box: [r][form][64][16]}: form 0 base_offset 0, 1 base_offset (start >> 7) & 7, 2 the aligned reference."""
    d = tmp_path_factory.mktemp("wgmma_desc")
    so, out = str(d / "wgmma_desc_probe.so"), str(d / "probe.npz")
    subprocess.check_call([nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-Xcompiler",
                           "-fPIC", "-shared", "-o", so, os.path.join(HERE, "wgmma_desc_probe.cu")])
    subprocess.check_call([sys.executable, "-c", CHILD, so, out])
    with np.load(out) as f:
        return {w: f["w%d" % w] for w in W_BOXES}


@pytest.mark.parametrize("w_box", W_BOXES)
def test_unaligned_start_reads_by_address(probe, w_box):
    for r in range(8):
        zero, addr, ref = probe[w_box][r]
        assert np.abs(ref).max() > 0
        # base_offset = 0: bit for bit what the aligned tile gives
        assert np.array_equal(zero, ref), "W_box=%d r=%d: base_offset 0 misreads" % (w_box, r)
        # base_offset = (start >> 7) & 7 is not the rule: it misreads as soon as it is not 0
        if r:
            assert not np.array_equal(addr, ref), "W_box=%d r=%d" % (w_box, r)
