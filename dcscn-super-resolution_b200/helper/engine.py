"""
ctypes binding of the C-ABI in include/dcscn_b200.h (libdcscn_b200.so, built from csrc/).

This is what stands where `self.sess.run(...)` stood in the reference
(DCSCN.py:420, :565, :575): PyTorch tensors are only the device containers whose
raw pointers are handed to the library.  There is NO CPU fallback: if the shared
library is missing or no H100 is present, construction raises.
"""

import ctypes
import math
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# DCSCN_B200_LIB points the binding at another build of the same C-ABI (kernel A/B runs); default: the in-tree library
LIB_PATH = os.environ.get("DCSCN_B200_LIB") or os.path.join(os.path.dirname(_HERE), "csrc", "libdcscn_b200.so")

PRECISION_F16X3 = 0
PRECISION_F16X1 = 1

# DCSCN_ACTIVATOR_* (--activator)
ACTIVATORS = {"prelu": 0, "relu": 1, "leaky_relu": 2, "sigmoid": 3, "tanh": 4, "selu": 5}

# DCSCN_OPTIMIZER_* (--optimizer)
OPTIMIZERS = {"adam": 0, "gd": 1, "momentum": 2, "adadelta": 3, "adagrad": 4, "rmsprop": 5}
# Checkpoint suffix of each slot, in the engine's slot order, as TF's slot creator names them ("<var>/<Name>", then
# "<var>/<Name>_1"), and the value the slot starts at.
OPTIMIZER_SLOTS = {
    "adam": (("/Adam", 0.0), ("/Adam_1", 0.0)),
    "gd": (),
    "momentum": (("/Momentum", 0.0),),
    "adadelta": (("/Adadelta", 0.0), ("/Adadelta_1", 0.0)),
    "adagrad": (("/Adagrad", 0.1),),
    "rmsprop": (("/RMSProp", 1.0), ("/RMSProp_1", 0.0)),
}


class DcscnConfig(ctypes.Structure):
    """Mirror of `struct dcscn_config` (include/dcscn_b200.h)."""
    _fields_ = [
        ("struct_size", ctypes.c_int32),
        ("scale", ctypes.c_int32),
        ("layers", ctypes.c_int32),
        ("filters", ctypes.c_int32),
        ("min_filters", ctypes.c_int32),
        ("filters_decay_gamma", ctypes.c_float),
        ("use_nin", ctypes.c_int32),
        ("nin_filters", ctypes.c_int32),
        ("nin_filters2", ctypes.c_int32),
        ("cnn_size", ctypes.c_int32),
        ("reconstruct_layers", ctypes.c_int32),
        ("reconstruct_filters", ctypes.c_int32),
        ("pixel_shuffler_filters", ctypes.c_int32),
        ("depthwise_separable", ctypes.c_int32),
        ("channels", ctypes.c_int32),
        ("dropout_keep", ctypes.c_float),
        ("l2_decay", ctypes.c_float),
        ("clipping_norm", ctypes.c_float),
        ("beta1", ctypes.c_float),
        ("beta2", ctypes.c_float),
        ("epsilon", ctypes.c_float),
        ("device_id", ctypes.c_int32),
        ("precision", ctypes.c_int32),
        ("activator", ctypes.c_int32),
        ("optimizer", ctypes.c_int32),
        ("momentum", ctypes.c_float),
        ("transposed_upsampler", ctypes.c_int32),
    ]


EXPORTED_SYMBOLS = [
    "dcscn_create", "dcscn_destroy", "dcscn_last_error", "dcscn_num_params", "dcscn_param_info",
    "dcscn_set_param", "dcscn_get_param", "dcscn_forward", "dcscn_forward_host", "dcscn_bicubic_resize", "dcscn_forward_ensemble", "dcscn_forward_ensemble_host", "dcscn_forward_ensemble_partial", "dcscn_get_activation",
    "dcscn_set_option", "dcscn_get_timings", "dcscn_launch_count", "dcscn_device_bytes",
    "dcscn_train_step", "dcscn_train_step_host", "dcscn_get_grad", "dcscn_get_adam_slot", "dcscn_set_adam_slot", "dcscn_get_adam_step",
    "dcscn_set_adam_step", "dcscn_last_grad_norm",
    "dcscn_patch_store_set", "dcscn_train_step_indexed", "dcscn_patch_gather", "dcscn_dropout_mask", "dcscn_grad_buffer", "dcscn_apply_gradients", "dcscn_apply_gradients_avg", "dcscn_reset_optimizer", "dcscn_graph_replays",
    "dcscn_tile_halo", "dcscn_optimizer_slot_count", "dcscn_get_optimizer_slot", "dcscn_set_optimizer_slot",
    "dcscn_get_train_tensor", "dcscn_image_store_set", "dcscn_train_step_crops", "dcscn_crop_gather",
    "dcscn_eval_store_set", "dcscn_evaluate_image",
]

_lib = None


class EngineError(RuntimeError):
    pass


def load_library(path=None):
    """dlopen the C-ABI library; raises EngineError (never falls back) when it is missing."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    path = path or LIB_PATH
    if not os.path.isfile(path):
        raise EngineError("CUDA extension %s not found - build it with `python __graft_entry__.py` "
                          "(or `make -C dcscn-super-resolution_b200/csrc`); there is no CPU fallback" % path)
    lib = ctypes.CDLL(path)
    vp, ci, c64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
    fp = ctypes.POINTER(ctypes.c_float)
    lib.dcscn_last_error.restype = ctypes.c_char_p
    lib.dcscn_create.argtypes = [ctypes.POINTER(DcscnConfig), ctypes.POINTER(vp)]
    lib.dcscn_destroy.argtypes = [vp]
    lib.dcscn_num_params.argtypes = [vp]
    lib.dcscn_param_info.argtypes = [vp, ci, ctypes.c_char_p, ci, ctypes.POINTER(c64), ctypes.POINTER(ci)]
    lib.dcscn_set_param.argtypes = [vp, ctypes.c_char_p, fp, c64]
    lib.dcscn_get_param.argtypes = [vp, ctypes.c_char_p, fp, c64]
    lib.dcscn_forward.argtypes = [vp, vp, vp, vp, ci, ci, ci, vp]
    lib.dcscn_forward_host.argtypes = [vp, vp, vp, vp, ci, ci, ci]
    lib.dcscn_bicubic_resize.argtypes = [vp, vp, vp, ci, ci, ci, ci, ci, vp]
    lib.dcscn_forward_ensemble.argtypes = [vp, vp, vp, vp, ci, ci, ci, vp]
    lib.dcscn_forward_ensemble_host.argtypes = [vp, vp, vp, vp, ci, ci, ci]
    lib.dcscn_forward_ensemble_partial.argtypes = [vp, vp, vp, vp, ci, ci, ci, vp]
    lib.dcscn_get_activation.argtypes = [vp, ctypes.c_char_p, fp, c64]
    lib.dcscn_get_train_tensor.argtypes = [vp, ctypes.c_char_p, fp, c64]
    lib.dcscn_set_option.argtypes = [vp, ctypes.c_char_p, c64]
    lib.dcscn_get_timings.argtypes = [vp, fp, ci, ctypes.POINTER(ci), ctypes.c_char_p, ci]
    u32, cf = ctypes.c_uint32, ctypes.c_float
    lib.dcscn_train_step.argtypes = [vp, vp, vp, vp, ci, ci, ci, cf, u32, ci, fp, fp, vp]
    lib.dcscn_train_step_host.argtypes = [vp, vp, vp, vp, ci, ci, ci, cf, u32, ci, fp, fp]
    lib.dcscn_get_grad.argtypes = [vp, ctypes.c_char_p, fp, c64]
    lib.dcscn_get_adam_slot.argtypes = [vp, ctypes.c_char_p, ci, fp, c64]
    lib.dcscn_set_adam_slot.argtypes = [vp, ctypes.c_char_p, ci, fp, c64]
    lib.dcscn_get_adam_step.argtypes = [vp, ctypes.POINTER(c64)]
    lib.dcscn_set_adam_step.argtypes = [vp, c64]
    lib.dcscn_last_grad_norm.argtypes = [vp]
    lib.dcscn_last_grad_norm.restype = cf
    lib.dcscn_dropout_mask.argtypes = [vp, ctypes.c_char_p, u32, ci, ci, ci, ctypes.POINTER(ctypes.c_uint8), c64]
    lib.dcscn_grad_buffer.argtypes = [vp, ctypes.POINTER(fp), ctypes.POINTER(c64)]
    lib.dcscn_apply_gradients.argtypes = [vp, cf, vp]
    lib.dcscn_reset_optimizer.argtypes = [vp]
    i32p = ctypes.POINTER(ctypes.c_int32)
    lib.dcscn_patch_store_set.argtypes = [vp, vp, vp, vp, c64, ci, ci]
    lib.dcscn_train_step_indexed.argtypes = [vp, i32p, ci, cf, cf, u32, ci, fp, fp]
    lib.dcscn_patch_gather.argtypes = [vp, i32p, ci, cf, vp, vp, vp]
    lib.dcscn_apply_gradients_avg.argtypes = [vp, cf, cf, fp, fp, vp]
    c64p = ctypes.POINTER(c64)
    lib.dcscn_image_store_set.argtypes = [vp, vp, c64, c64p, i32p, i32p, i32p, ci]
    lib.dcscn_train_step_crops.argtypes = [vp, i32p, ci, ci, cf, cf, u32, ci, fp, fp]
    lib.dcscn_crop_gather.argtypes = [vp, i32p, ci, ci, cf, vp, vp, vp]
    u64p = ctypes.POINTER(ctypes.c_uint64)
    lib.dcscn_eval_store_set.argtypes = [vp, vp, c64, c64p, i32p, i32p, i32p, ci]
    lib.dcscn_evaluate_image.argtypes = [vp, ci, vp, ci, ci, ci, ci, ci, ci, ctypes.c_double, ci, vp, u64p, c64p, c64p, vp, c64]
    lib.dcscn_launch_count.argtypes = [vp]
    lib.dcscn_launch_count.restype = c64
    lib.dcscn_device_bytes.argtypes = [vp]
    lib.dcscn_device_bytes.restype = c64
    lib.dcscn_graph_replays.argtypes = [vp]
    lib.dcscn_graph_replays.restype = c64
    lib.dcscn_tile_halo.argtypes = [vp, ctypes.POINTER(ci)]
    lib.dcscn_optimizer_slot_count.argtypes = [vp]
    lib.dcscn_get_optimizer_slot.argtypes = [vp, ctypes.c_char_p, ci, fp, c64]
    lib.dcscn_set_optimizer_slot.argtypes = [vp, ctypes.c_char_p, ci, fp, c64]
    _lib = lib
    return lib


def make_config(scale=2, layers=12, filters=196, min_filters=48, filters_decay_gamma=1.5, use_nin=True,
                nin_filters=64, nin_filters2=32, cnn_size=3, reconstruct_layers=1, reconstruct_filters=32,
                pixel_shuffler_filters=0, depthwise_separable=False, channels=1, dropout_keep=0.8,
                l2_decay=0.0001, clipping_norm=5.0, beta1=0.9, beta2=0.999, epsilon=1e-8, device_id=0,
                precision=PRECISION_F16X3, activator="prelu", optimizer="adam", momentum=0.9,
                transposed_upsampler=False):
    """`transposed_upsampler`: --pixel_shuffler=false (the Up-TCNN conv2d_transpose instead of Up-PS)."""
    c = DcscnConfig()
    c.struct_size = ctypes.sizeof(DcscnConfig)
    c.scale, c.layers, c.filters, c.min_filters = scale, layers, filters, min_filters
    c.filters_decay_gamma = filters_decay_gamma
    c.use_nin, c.nin_filters, c.nin_filters2, c.cnn_size = int(use_nin), nin_filters, nin_filters2, cnn_size
    c.reconstruct_layers, c.reconstruct_filters = reconstruct_layers, reconstruct_filters
    c.pixel_shuffler_filters, c.depthwise_separable, c.channels = pixel_shuffler_filters, int(depthwise_separable), channels
    c.dropout_keep, c.l2_decay, c.clipping_norm = dropout_keep, l2_decay, clipping_norm
    c.beta1, c.beta2, c.epsilon = beta1, beta2, epsilon
    c.device_id, c.precision = device_id, precision
    c.activator = ACTIVATORS[activator]
    c.optimizer, c.momentum = OPTIMIZERS[optimizer], momentum
    c.transposed_upsampler = int(transposed_upsampler)
    return c


def eval_geometry(height, width, scale, border):
    """Sizes of one evaluated image as the host forms them (DCSCN._evaluation_set, util.compute_psnr_and_ssim): the
    aligned ground truth (util.set_image_alignment), the LR input (util.resize_image_by_pil by 1.0 / scale), its bicubic
    up-scale and the region left after shaving `border` pixels from each side (border > 0 only).
    Returns (ah, aw), (lh, lw), (bh, bw), (rh, rw)."""
    ah, aw = height // scale * scale, width // scale * scale
    lh, lw = int(ah * (1.0 / scale)), int(aw * (1.0 / scale))
    bh, bw = int(lh * scale), int(lw * scale)
    b = border if border > 0 else 0
    return (ah, aw), (lh, lw), (bh, bw), (max(ah - 2 * b, 0), max(aw - 2 * b, 0))


_SSIM_PARAMS = None


def ssim_params():
    """{w0 .. w5, c1, c2} of util._ssim_columns: scipy's gaussian_filter1d(sigma 1.5, truncate 3.5) taps, read off the
    filter's response to a unit impulse (so they are scipy's own numbers), and the constants (0.01 * 255)^2,
    (0.03 * 255)^2."""
    global _SSIM_PARAMS
    if _SSIM_PARAMS is None:
        from scipy.ndimage import gaussian_filter1d
        impulse = np.zeros(11)
        impulse[5] = 1.0
        taps = gaussian_filter1d(impulse, 1.5, axis=0, truncate=3.5, mode="reflect")
        _SSIM_PARAMS = np.ascontiguousarray(np.concatenate([taps[5:], [(0.01 * 255) ** 2, (0.03 * 255) ** 2]]))
    return _SSIM_PARAMS


def finish_psnr(sse, pixels, nan_pixels):
    """util.compute_psnr_and_ssim's PSNR from the exact squared-error sum: err = sse / n, 10 log10(255^2 / err), inf at
    err = 0; nan for an empty region or a NaN output pixel (as np.mean gives)."""
    if nan_pixels or pixels == 0:
        return float("nan")
    err = float(sse) / pixels
    return float("inf") if err == 0 else 10.0 * math.log10(255.0 * 255.0 / err)


class Engine:
    """One DCSCN graph instance on one GPU."""

    def __init__(self, config):
        self.lib = load_library()
        self.config = config
        self.handle = ctypes.c_void_p()
        self._check(self.lib.dcscn_create(ctypes.byref(config), ctypes.byref(self.handle)))

    def _check(self, rc):
        if rc != 0:
            raise EngineError(self.lib.dcscn_last_error().decode("utf-8", "replace"))

    def close(self):
        if self.handle:
            self.lib.dcscn_destroy(self.handle)
            self.handle = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- variables ----
    def param_shapes(self):
        out = {}
        buf = ctypes.create_string_buffer(256)
        dims = (ctypes.c_int64 * 4)()
        nd = ctypes.c_int()
        for i in range(self.lib.dcscn_num_params(self.handle)):
            self._check(self.lib.dcscn_param_info(self.handle, i, buf, 256, dims, ctypes.byref(nd)))
            out[buf.value.decode()] = tuple(int(dims[k]) for k in range(nd.value))
        return out

    def set_param(self, name, array):
        a = np.ascontiguousarray(array, dtype=np.float32)
        self._check(self.lib.dcscn_set_param(self.handle, name.encode(), a.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                                             a.size))

    def get_param(self, name):
        shape = self.param_shapes()[name]
        a = np.empty(shape, dtype=np.float32)
        self._check(self.lib.dcscn_get_param(self.handle, name.encode(), a.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                                             a.size))
        return a

    def set_params(self, weights):
        shapes = self.param_shapes()
        for name, shape in shapes.items():
            if name not in weights:
                raise EngineError("checkpoint has no variable '%s'" % name)
            w = np.asarray(weights[name])
            if tuple(w.shape) != tuple(shape):
                raise EngineError("variable '%s': checkpoint shape %s != graph shape %s" % (name, w.shape, shape))
            self.set_param(name, w)

    # ---- compute ----
    def forward(self, x, x2, y=None, stream=None):
        """x [n,h,w,1], x2 [n,s*h,s*w,1]: contiguous fp32 CUDA torch tensors.  Asynchronous."""
        import torch
        n, h, w = int(x.shape[0]), int(x.shape[1]), int(x.shape[2])
        s = self.config.scale
        assert x.is_cuda and x2.is_cuda and x.dtype == torch.float32 and x2.dtype == torch.float32
        assert x.is_contiguous() and x2.is_contiguous()
        assert tuple(x2.shape[:3]) == (n, s * h, s * w), "x2 must be [n, scale*h, scale*w, 1]"
        if y is None:
            y = torch.empty((n, s * h, s * w, 1), dtype=torch.float32, device=x.device)
        st = stream if stream is not None else torch.cuda.current_stream(x.device).cuda_stream
        self._check(self.lib.dcscn_forward(self.handle, x.data_ptr(), x2.data_ptr(), y.data_ptr(), n, h, w,
                                           ctypes.c_void_p(st)))
        return y

    def forward_host(self, x, x2, y=None):
        """numpy (or pinned torch CPU) fp32 arrays in, numpy out; H2D + forward + D2H, synchronous.  With x2 = None the
        bicubic up-scale of x (util.resize_image_by_pil, bit-exact) is formed on the device and only x is copied."""
        xa = _host_array(x)
        n, h, w = xa.shape[0], xa.shape[1], xa.shape[2]
        s = self.config.scale
        x2p = None
        if x2 is not None:
            x2a = _host_array(x2)
            assert tuple(x2a.shape[:3]) == (n, s * h, s * w)
            x2p = x2a.ctypes.data
        if y is None:
            y = np.empty((n, s * h, s * w, 1), dtype=np.float32)
        ya = _host_array(y)
        self._check(self.lib.dcscn_forward_host(self.handle, xa.ctypes.data, x2p, ya.ctypes.data, n, h, w))
        return y

    def bicubic_resize(self, src, out_height, out_width, out=None, stream=None):
        """Pillow's bicubic `Image.resize` of float images on the device: src [n,h,w] fp32 CUDA tensor -> [n,oh,ow]."""
        import torch
        n, h, w = int(src.shape[0]), int(src.shape[1]), int(src.shape[2])
        assert src.is_cuda and src.dtype == torch.float32 and src.is_contiguous()
        if out is None:
            out = torch.empty((n, int(out_height), int(out_width)), dtype=torch.float32, device=src.device)
        st = stream if stream is not None else torch.cuda.current_stream(src.device).cuda_stream
        self._check(self.lib.dcscn_bicubic_resize(self.handle, src.data_ptr(), out.data_ptr(), n, h, w, int(out_height),
                                                  int(out_width), ctypes.c_void_p(st)))
        return out

    def forward_ensemble_host(self, x, x2, flips):
        """Self-ensemble of one image on the device (DCSCN.py:547-586): x [h,w,(1)], x2 [s*h,s*w,(1)] float32 ->
        float64 [s*h, s*w, 1] mean of the inverse-transformed outputs of the first `flips` transforms."""
        xa = np.ascontiguousarray(x, dtype=np.float32)
        h, w = xa.shape[:2]
        s = int(self.config.scale)
        x2p = None                      # None: the device forms the bicubic up-scale of x itself (bit-exact Pillow)
        if x2 is not None:
            x2a = np.ascontiguousarray(x2, dtype=np.float32)
            if x2a.shape[:2] != (s * h, s * w):
                raise ValueError("x2 must be [%d,%d], got %s" % (s * h, s * w, x2a.shape[:2]))
            x2p = x2a.ctypes.data
        y = np.empty((s * h, s * w, 1), dtype=np.float64)
        self._check(self.lib.dcscn_forward_ensemble_host(self.handle, xa.ctypes.data, x2p, y.ctypes.data, h, w, int(flips)))
        return y

    def forward_ensemble(self, x, x2, flips, out=None, stream=None):
        """Device-resident self-ensemble of one image: x [h,w] / x2 [s*h,s*w] fp32 CUDA tensors -> float64 [s*h,s*w]."""
        import torch
        h, w = int(x.shape[0]), int(x.shape[1])
        s = int(self.config.scale)
        if out is None:
            out = torch.empty((s * h, s * w), dtype=torch.float64, device=x.device)
        st = stream if stream is not None else torch.cuda.current_stream(x.device).cuda_stream
        self._check(self.lib.dcscn_forward_ensemble(self.handle, x.data_ptr(), x2.data_ptr(), out.data_ptr(), h, w, int(flips),
                                                    ctypes.c_void_p(st)))
        return out

    def forward_ensemble_sharded(self, x, x2, flips, out=None):
        """The same ensemble with the transforms spread over the ranks of the current torch.distributed job (rank r
        takes transforms r, r + world, ...): every rank runs its share as batched forwards, writes the float64 SUM of
        its inverse-transformed outputs, ONE all-reduce (NCCL sum over NVLink) combines them and the mean is taken.
        Every rank returns the full result.  x / x2: the SAME image on every rank (fp32 CUDA tensors)."""
        import torch
        import torch.distributed as dist
        rank, world = (dist.get_rank(), dist.get_world_size()) if dist.is_available() and dist.is_initialized() else (0, 1)
        h, w = int(x.shape[0]), int(x.shape[1])
        s = int(self.config.scale)
        if out is None:
            out = torch.empty((s * h, s * w), dtype=torch.float64, device=x.device)
        mask = 0
        for t in range(rank, int(flips), world):
            mask |= 1 << t
        st = torch.cuda.current_stream(x.device).cuda_stream
        if mask:
            self._check(self.lib.dcscn_forward_ensemble_partial(self.handle, x.data_ptr(), x2.data_ptr(), out.data_ptr(), h, w,
                                                                mask, ctypes.c_void_p(st)))
        else:
            out.zero_()          # more ranks than transforms: this rank contributes nothing
        if world > 1:
            dist.all_reduce(out, op=dist.ReduceOp.SUM)
        out.div_(float(flips))
        return out

    # ---- training patches resident in HBM ----
    def set_patch_store(self, lr_u8, bicubic_u8, true_u8):
        """uint8 patch arrays [count, ph, pw(, 1)] / [count, s*ph, s*pw(, 1)] -> device memory, once per data set."""
        a = [np.ascontiguousarray(v, dtype=np.uint8) for v in (lr_u8, bicubic_u8, true_u8)]
        count, ph, pw = a[0].shape[:3]
        s = int(self.config.scale)
        if a[1].shape[:3] != (count, s * ph, s * pw) or a[2].shape[:3] != (count, s * ph, s * pw):
            raise ValueError("patch arrays do not match: %s %s %s at scale %d" % (a[0].shape, a[1].shape, a[2].shape, s))
        self._check(self.lib.dcscn_patch_store_set(self.handle, a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data, count, ph, pw))
        self._patch_shape = (ph, pw)

    @staticmethod
    def _index_array(indices, mirror=None):
        idx = np.ascontiguousarray(indices, dtype=np.int64)
        if mirror is not None:
            idx = idx | (np.asarray(mirror, dtype=np.int64).astype(bool).astype(np.int64) << 31)
        return np.ascontiguousarray(idx.astype(np.uint32).view(np.int32))

    def train_step_indexed(self, indices, lr, seed, max_value=255.0, mirror=None, apply_update=True):
        """One optimisation step on the patches `indices` of the device store; returns (image_loss, mse)."""
        idx = self._index_array(indices, mirror)
        loss, mse = ctypes.c_float(), ctypes.c_float()
        self._check(self.lib.dcscn_train_step_indexed(self.handle, idx.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), int(idx.size),
                                                      float(max_value), float(lr), int(seed) & 0xFFFFFFFF,
                                                      int(bool(apply_update)), ctypes.byref(loss), ctypes.byref(mse)))
        return float(loss.value), float(mse.value)

    def gather_patches(self, indices, max_value=255.0, mirror=None):
        """The fp32 mini-batch tensors (x, x2, y) the indexed step feeds the network, copied back to the host."""
        idx = self._index_array(indices, mirror)
        ph, pw = self._patch_shape
        s = int(self.config.scale)
        n = int(idx.size)
        x = np.empty((n, ph, pw, 1), np.float32)
        x2 = np.empty((n, s * ph, s * pw, 1), np.float32)
        y = np.empty((n, s * ph, s * pw, 1), np.float32)
        self._check(self.lib.dcscn_patch_gather(self.handle, idx.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), n, float(max_value),
                                                x.ctypes.data, x2.ctypes.data, y.ctypes.data))
        return x, x2, y

    # ---- random-crop training data: decoded images resident in HBM ----
    def set_image_store(self, images):
        """Decoded uint8 images [h, w, 3] (RGB) or [h, w(, 1)] (mode 'L'), as util.load_image returns them -> device
        memory, once per data set.  A crop (image, top, left, mirror) of train_step_crops / gather_crops names image i of
        this list."""
        arrays = [np.ascontiguousarray(np.atleast_3d(a), dtype=np.uint8) for a in images]
        shapes = np.array([a.shape for a in arrays], dtype=np.int64).reshape(-1, 3)
        sizes = np.array([a.size for a in arrays], dtype=np.int64)
        offsets = np.ascontiguousarray(np.concatenate([[0], np.cumsum(sizes)[:-1]]), dtype=np.int64)
        pixels = np.concatenate([a.reshape(-1) for a in arrays]) if arrays else np.zeros(0, np.uint8)
        heights, widths, channels = (np.ascontiguousarray(shapes[:, k], dtype=np.int32) for k in range(3))
        i32 = ctypes.POINTER(ctypes.c_int32)
        self._check(self.lib.dcscn_image_store_set(self.handle, pixels.ctypes.data, int(pixels.size),
                                                   offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                                   heights.ctypes.data_as(i32), widths.ctypes.data_as(i32),
                                                   channels.ctypes.data_as(i32), len(arrays)))

    @staticmethod
    def _crop_array(crops):
        c = np.ascontiguousarray(np.asarray(crops, dtype=np.int64).reshape(-1, 4))
        if c.size and (c.min() < -2 ** 31 or c.max() >= 2 ** 31):
            raise EngineError("crop descriptor out of the int32 range")
        return np.ascontiguousarray(c.astype(np.int32))

    def train_step_crops(self, crops, patch_size, lr, seed, max_value=255.0, apply_update=True):
        """One optimisation step on the crops (image, top, left, mirror) of the device image store, each
        scale * patch_size pixels square; returns (image_loss, mse)."""
        c = self._crop_array(crops)
        loss, mse = ctypes.c_float(), ctypes.c_float()
        self._check(self.lib.dcscn_train_step_crops(self.handle, c.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), len(c),
                                                    int(patch_size), float(max_value), float(lr), int(seed) & 0xFFFFFFFF,
                                                    int(bool(apply_update)), ctypes.byref(loss), ctypes.byref(mse)))
        return float(loss.value), float(mse.value)

    def gather_crops(self, crops, patch_size, max_value=255.0):
        """The fp32 mini-batch tensors (x, x2, y) the crop step feeds the network, copied back to the host."""
        c = self._crop_array(crops)
        n, p, e = len(c), int(patch_size), int(patch_size) * int(self.config.scale)
        x = np.empty((n, p, p, 1), np.float32)
        x2 = np.empty((n, e, e, 1), np.float32)
        y = np.empty((n, e, e, 1), np.float32)
        self._check(self.lib.dcscn_crop_gather(self.handle, c.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), n, p,
                                               float(max_value), x.ctypes.data, x2.ctypes.data, y.ctypes.data))
        return x, x2, y

    # ---- evaluation: test images resident in HBM, inputs and metric formed on the device ----
    @staticmethod
    def _pack_images(images):
        arrays = [np.ascontiguousarray(np.atleast_3d(a), dtype=np.uint8) for a in images]
        shapes = np.array([a.shape for a in arrays], dtype=np.int64).reshape(-1, 3)
        sizes = np.array([a.size for a in arrays], dtype=np.int64)
        offsets = np.ascontiguousarray(np.concatenate([[0], np.cumsum(sizes)[:-1]]), dtype=np.int64)
        pixels = np.concatenate([a.reshape(-1) for a in arrays]) if arrays else np.zeros(0, np.uint8)
        heights, widths, channels = (np.ascontiguousarray(shapes[:, k], dtype=np.int32) for k in range(3))
        return pixels, offsets, heights, widths, channels

    def set_eval_images(self, images):
        """Decoded uint8 test images [h, w, 3] (RGB) or [h, w(, 1)] (mode 'L'), as util.load_image returns them -> the
        device evaluation store, once per test set.  evaluate_image(i, ...) evaluates image i of this list.  The training
        stores are not touched."""
        pixels, offsets, heights, widths, channels = self._pack_images(images)
        i32 = ctypes.POINTER(ctypes.c_int32)
        self._check(self.lib.dcscn_eval_store_set(self.handle, pixels.ctypes.data, int(pixels.size),
                                                  offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)),
                                                  heights.ctypes.data_as(i32), widths.ctypes.data_as(i32),
                                                  channels.ctypes.data_as(i32), len(heights)))
        self._eval_shapes = [tuple(int(v) for v in t) for t in zip(heights, widths, channels)]

    def evaluate_image(self, image, flips, max_value, border, bicubic=False):
        """(PSNR, SSIM) of one test image, equal to the host's DCSCN.do_for_evaluate (or evaluate_bicubic with bicubic=True)
        at self_ensemble = flips: image i of the evaluation store (an int) or a decoded uint8 image (util.load_image).
        The device forms the luma, the LR / bicubic inputs, the forward or self-ensemble, the trimmed output, the exact
        squared-error sum and the SSIM map; the host finishes PSNR and the numpy mean of the map."""
        s = int(self.config.scale)
        if isinstance(image, (int, np.integer)):
            index, ptr, a = int(image), None, None
            if not 0 <= index < len(getattr(self, "_eval_shapes", ())):
                raise EngineError("evaluate_image: no image %d in the evaluation store" % index)
            h, w, c = self._eval_shapes[index]
        else:
            a = np.atleast_3d(np.asarray(image))
            if a.dtype != np.uint8:
                raise EngineError("evaluate_image: a decoded uint8 image is expected, got %s" % a.dtype)
            a = np.ascontiguousarray(a)
            index, ptr = -1, a.ctypes.data
            h, w, c = a.shape
        _, (lh, lw), _, (rh, rw) = eval_geometry(h, w, s, border)
        rows = rh - 10 if rh >= 11 else 0
        ssim_map = np.empty((rows, rw), np.float64)
        sse, pixels, nans = ctypes.c_uint64(), ctypes.c_int64(), ctypes.c_int64()
        params = ssim_params()
        self._check(self.lib.dcscn_evaluate_image(self.handle, index, ptr, h, w, c, lh, lw, 0 if bicubic else max(int(flips), 1),
                                                  float(max_value), int(border), params.ctypes.data, ctypes.byref(sse),
                                                  ctypes.byref(pixels), ctypes.byref(nans), ssim_map.ctypes.data,
                                                  int(ssim_map.size)))
        psnr = finish_psnr(int(sse.value), int(pixels.value), int(nans.value))
        # the host's np.mean(s[5:-5, :]) of a contiguous slice of this shape: the same reduction, bit for bit
        ssim = float(np.mean(ssim_map)) if rows > 0 and rw > 0 else float("nan")
        return psnr, ssim

    def train_step_host(self, x, x2, y, lr, seed, apply_update=True):
        """One optimisation step on host fp32 arrays x [n,h,w,1], x2 / y [n,sh,sw,1]; returns (image_loss, mse)."""
        xa, x2a, ya = _host_array(x), _host_array(x2), _host_array(y)
        n, h, w = xa.shape[0], xa.shape[1], xa.shape[2]
        s = self.config.scale
        assert tuple(x2a.shape[:3]) == (n, s * h, s * w) and tuple(ya.shape[:3]) == (n, s * h, s * w)
        loss, mse = ctypes.c_float(), ctypes.c_float()
        self._check(self.lib.dcscn_train_step_host(self.handle, xa.ctypes.data, x2a.ctypes.data, ya.ctypes.data, n, h, w,
                                                   float(lr), int(seed) & 0xFFFFFFFF, int(bool(apply_update)),
                                                   ctypes.byref(loss), ctypes.byref(mse)))
        return float(loss.value), float(mse.value)

    def train_step(self, x, x2, y, lr, seed, apply_update=True, stream=None):
        """Same with contiguous fp32 CUDA torch tensors."""
        import torch
        n, h, w = int(x.shape[0]), int(x.shape[1]), int(x.shape[2])
        assert x.is_cuda and x2.is_cuda and y.is_cuda and x.is_contiguous() and x2.is_contiguous() and y.is_contiguous()
        st = stream if stream is not None else torch.cuda.current_stream(x.device).cuda_stream
        loss, mse = ctypes.c_float(), ctypes.c_float()
        self._check(self.lib.dcscn_train_step(self.handle, x.data_ptr(), x2.data_ptr(), y.data_ptr(), n, h, w, float(lr),
                                              int(seed) & 0xFFFFFFFF, int(bool(apply_update)), ctypes.byref(loss),
                                              ctypes.byref(mse), ctypes.c_void_p(st)))
        return float(loss.value), float(mse.value)

    def grad_tensor(self):
        """Zero-copy torch view of the flat device gradient buffer (for torch.distributed.all_reduce over NCCL)."""
        import torch
        ptr, cnt = ctypes.POINTER(ctypes.c_float)(), ctypes.c_int64()
        self._check(self.lib.dcscn_grad_buffer(self.handle, ctypes.byref(ptr), ctypes.byref(cnt)))

        class _Buf:
            __cuda_array_interface__ = {"shape": (int(cnt.value),), "typestr": "<f4", "version": 2,
                                        "data": (ctypes.cast(ptr, ctypes.c_void_p).value, False)}
        return torch.as_tensor(_Buf(), device="cuda:%d" % self.config.device_id)

    def apply_gradients(self, lr, stream=None):
        import torch
        st = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        self._check(self.lib.dcscn_apply_gradients(self.handle, float(lr), ctypes.c_void_p(st)))

    def apply_gradients_avg(self, lr, grad_scale, stream=None):
        """After the all-reduce(sum) of `grad_tensor()`: scale to the mean, clip + Adam; returns (image_loss, mse) means."""
        import torch
        st = stream if stream is not None else torch.cuda.current_stream().cuda_stream
        loss, mse = ctypes.c_float(), ctypes.c_float()
        self._check(self.lib.dcscn_apply_gradients_avg(self.handle, float(lr), float(grad_scale), ctypes.byref(loss),
                                                       ctypes.byref(mse), ctypes.c_void_p(st)))
        return float(loss.value), float(mse.value)

    def train_step_data_parallel(self, x, x2, y, lr, seed, indices=None, max_value=255.0, crops=None, patch_size=None):
        """One optimisation step with the mini-batch sharded over the ranks of the current torch.distributed job (equal
        shards): local gradients -> ONE flat all-reduce carrying [gradients | loss | mse] -> identical mean, clip and
        Adam on every rank.  Returns the job-wide (image_loss, mse).  With `indices` the rank's shard is taken from the
        device patch store, with `crops` (and `patch_size`) from the device image store (x, x2, y ignored)."""
        import torch.distributed as dist
        if crops is not None:
            loss, mse = self.train_step_crops(crops, patch_size, lr, seed, max_value=max_value, apply_update=False)
        elif indices is not None:
            loss, mse = self.train_step_indexed(indices, lr, seed, max_value=max_value, apply_update=False)
        else:
            fn = self.train_step if hasattr(x, "is_cuda") and x.is_cuda else self.train_step_host
            loss, mse = fn(x, x2, y, lr, seed, apply_update=False)
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            g = self.grad_tensor()
            dist.all_reduce(g, op=dist.ReduceOp.SUM)
            return self.apply_gradients_avg(lr, 1.0 / dist.get_world_size())
        self.apply_gradients(lr)
        return loss, mse

    def get_grad(self, name):
        a = np.empty(self.param_shapes()[name], dtype=np.float32)
        self._check(self.lib.dcscn_get_grad(self.handle, name.encode(), a.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), a.size))
        return a

    def get_adam_slot(self, name, slot):
        a = np.empty(self.param_shapes()[name], dtype=np.float32)
        self._check(self.lib.dcscn_get_adam_slot(self.handle, name.encode(), slot,
                                                 a.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), a.size))
        return a

    def set_adam_slot(self, name, slot, value):
        a = np.ascontiguousarray(value, dtype=np.float32)
        self._check(self.lib.dcscn_set_adam_slot(self.handle, name.encode(), slot,
                                                 a.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), a.size))

    @property
    def optimizer_slot_count(self):
        return int(self.lib.dcscn_optimizer_slot_count(self.handle))

    def get_optimizer_slot(self, name, slot):
        """Slot `slot` of the configured optimizer (order of OPTIMIZER_SLOTS); its initial value before any step."""
        a = np.empty(self.param_shapes()[name], dtype=np.float32)
        self._check(self.lib.dcscn_get_optimizer_slot(self.handle, name.encode(), slot,
                                                      a.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), a.size))
        return a

    def set_optimizer_slot(self, name, slot, value):
        a = np.ascontiguousarray(value, dtype=np.float32)
        self._check(self.lib.dcscn_set_optimizer_slot(self.handle, name.encode(), slot,
                                                      a.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), a.size))

    @property
    def adam_step(self):
        """Number of optimizer updates applied so far (TF stores beta^(t+1) as beta1_power / beta2_power)."""
        t = ctypes.c_int64()
        self._check(self.lib.dcscn_get_adam_step(self.handle, ctypes.byref(t)))
        return int(t.value)

    @adam_step.setter
    def adam_step(self, t):
        self._check(self.lib.dcscn_set_adam_step(self.handle, int(t)))

    def reset_optimizer(self):
        """Optimizer slots back to their initial values and update count to 0 (what re-running the initializer does in
        the reference)."""
        self._check(self.lib.dcscn_reset_optimizer(self.handle))

    @property
    def last_grad_norm(self):
        return float(self.lib.dcscn_last_grad_norm(self.handle))

    def dropout_mask(self, tensor, seed, n, h, w, channels):
        a = np.empty((n, h, w, channels), dtype=np.uint8)
        self._check(self.lib.dcscn_dropout_mask(self.handle, tensor.encode(), int(seed) & 0xFFFFFFFF, n, h, w,
                                                a.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), a.size))
        return a

    def get_activation(self, tensor, shape):
        a = np.empty(shape, dtype=np.float32)
        self._check(self.lib.dcscn_get_activation(self.handle, tensor.encode(),
                                                  a.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), a.size))
        return a

    def get_train_tensor(self, name, shape):
        """A tensor of the last train step (dcscn_get_train_tensor: "y_", "dY", "dZ:<layer>", "dH:<layer>",
        "zneg:<layer>"; "Wc:" / "dWc:<layer>" on wide depthwise-separable graphs; "U:", "Z:", "H:", "E:", "dU:<layer>"
        on the fp32 depthwise-separable step) as fp32 of `shape`; all but "zneg:" need set_option("grad_capture", 1)
        before the step."""
        a = np.empty(shape, dtype=np.float32)
        self._check(self.lib.dcscn_get_train_tensor(self.handle, name.encode(),
                                                    a.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), a.size))
        return a

    def set_option(self, key, value):
        self._check(self.lib.dcscn_set_option(self.handle, key.encode(), int(value)))

    def tile_halo(self):
        """LR pixels of context around each window core of a tiled forward (option "workspace_mb")."""
        r = ctypes.c_int()
        self._check(self.lib.dcscn_tile_halo(self.handle, ctypes.byref(r)))
        return int(r.value)

    def timings(self):
        """[(launch name, ms)] of the last forward, or of the steps of the last evaluate_image call when that came
        after it (needs set_option("timing", 1) before it)."""
        cap = 64
        while True:   # a tiled forward has one sequence of launches per batch of windows
            ms = (ctypes.c_float * cap)()
            cnt = ctypes.c_int()
            names = ctypes.create_string_buffer(32 * cap)
            self._check(self.lib.dcscn_get_timings(self.handle, ms, cap, ctypes.byref(cnt), names, 32 * cap))
            if cnt.value <= cap:
                break
            cap = cnt.value
        return list(zip(names.value.decode().split(","), [float(ms[i]) for i in range(cnt.value)]))

    @property
    def launch_count(self):
        return int(self.lib.dcscn_launch_count(self.handle))

    @property
    def graph_replays(self):
        return int(self.lib.dcscn_graph_replays(self.handle))

    @property
    def device_bytes(self):
        return int(self.lib.dcscn_device_bytes(self.handle))


def _host_array(a):
    if isinstance(a, np.ndarray):
        assert a.dtype == np.float32 and a.flags["C_CONTIGUOUS"]
        return a
    # torch CPU tensor (possibly pinned): share memory
    return a.numpy()
