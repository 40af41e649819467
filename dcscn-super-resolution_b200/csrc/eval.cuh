#pragma once
// Evaluation of one test image on the device: what DCSCN._evaluation_set -> do(lr, bicubic) -> util.compute_psnr_and_ssim
// compute on the host (reference DCSCN.py:672-703, helper/utilty.py:509-536), bit for bit.  The engine chains these
// kernels with the Pillow resamplers of conv_aux.cuh and the forward / self-ensemble (engine.cu dcscn_evaluate_image).
#include <cstdint>

#include "conv_aux.cuh"

namespace dcscn {

// One decoded uint8 image: `channels` = 3 (RGB, interleaved) or 1 (mode 'L'), rows of `width * channels` bytes.
struct EvalImage {
  const uint8_t* pixels;
  int height, width, channels;
};

// The top-left ah x aw pixels of the image (util.set_image_alignment).  An RGB pixel becomes util.convert_rgb_to_y's
// float64 Y (the FMA chain of crop_gather_kernel): fp32(Y) is the mode-'F' resampler input and the truth is
// clip(rint(Y), 0, 255) of the float64 Y (trim_image_as_file).  A mode-'L' pixel feeds the 8-bit resampler as is and
// is its own truth.
__global__ void __launch_bounds__(256) eval_prepare_kernel(const EvalImage im, int ah, int aw, float* __restrict__ truth,
                                                           float* __restrict__ f_in, uint8_t* __restrict__ l_in) {
  const long long total = (long long)ah * aw;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(idx / aw), x = (int)(idx - (long long)y * aw);
    const uint8_t* p = im.pixels + ((long long)y * im.width + x) * im.channels;
    if (im.channels == 3) {
      const double v = __dadd_rn(__fma_rn((double)__ldg(p + 2), DCSCN_Y_B,
                                          __fma_rn((double)__ldg(p + 1), DCSCN_Y_G, __dmul_rn((double)__ldg(p), DCSCN_Y_R))),
                                 16.0);
      const double r = rint(v);
      truth[idx] = (float)(r < 0.0 ? 0.0 : (r > 255.0 ? 255.0 : r));
      f_in[idx] = (float)v;
    } else {
      const uint8_t v = __ldg(p);
      truth[idx] = (float)v;
      l_in[idx] = v;
    }
  }
}

// The network inputs of `do` (DCSCN.py:547-586): `np.multiply(image, max_value / 255.0)` of a mode-'F' (fp32) resize is
// an fp32 product with fp32(scale), of a mode-'L' (uint8) one a float64 product rounded to fp32 at the feed.  scale is
// exactly 1 at max_value 255, where the host skips the multiply.
__global__ void __launch_bounds__(256) eval_place_kernel(const float* __restrict__ f_src, const uint8_t* __restrict__ l_src,
                                                         float* __restrict__ out, long long total, double scale) {
  const float fscale = (float)scale;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x)
    out[idx] = l_src ? (float)__dmul_rn((double)__ldg(l_src + idx), scale) : __fmul_rn(__ldg(f_src + idx), fscale);
}

// trim_image_as_file of the evaluated output: clip(rint(v), 0, 255), NaN kept (np.clip passes it through).  Exactly one
// source is set:
//   y64  the float64 self-ensemble mean; v = y64 * (255 / max_value) in float64 (do with self_ensemble > 1);
//   y32  an fp32 plane; v = y32 * fp32(255 / max_value) in fp32 (do with self_ensemble = 1: numpy multiplies the fp32
//        forward output by a Python float in fp32), or the mode-'F' bicubic up-scale with back = 1 (evaluate_bicubic);
//   y8   the mode-'L' bicubic up-scale (evaluate_bicubic), already an integer.
// back = 1 at max_value 255, where the host skips the multiply.
__global__ void __launch_bounds__(256) eval_trim_kernel(const double* __restrict__ y64, const float* __restrict__ y32,
                                                        const uint8_t* __restrict__ y8, float* __restrict__ out, long long total,
                                                        double back) {
  const float fback = (float)back;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    double v;
    if (y64) v = __dmul_rn(__ldg(y64 + idx), back);
    else if (y32) v = (double)__fmul_rn(__ldg(y32 + idx), fback);
    else v = (double)__ldg(y8 + idx);
    const double r = rint(v);                  // rint of an fp32 value is the fp32 rint (np.rint on float32)
    out[idx] = (float)(r < 0.0 ? 0.0 : (r > 255.0 ? 255.0 : r));
  }
}

// PSNR numerator: sum of (truth - out)^2 over the hs x ws region at (b, b) of the [.. x pitch] planes, as an exact
// integer (the planes hold integers 0..255), and the number of NaN output pixels in the region.  acc[0] += sse,
// acc[1] += NaN count.
__global__ void __launch_bounds__(256) eval_sse_kernel(const float* __restrict__ truth, const float* __restrict__ out, int pitch,
                                                       int b, int hs, int ws, unsigned long long* __restrict__ acc) {
  const long long total = (long long)hs * ws;
  unsigned long long sse = 0, nan = 0;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(idx / ws), x = (int)(idx - (long long)y * ws);
    const long long o = (long long)(b + y) * pitch + b + x;
    const float a = __ldg(truth + o), v = __ldg(out + o);
    if (v != v) {
      ++nan;
    } else {
      const long long d = (long long)a - (long long)v;
      sse += (unsigned long long)(d * d);
    }
  }
  for (int off = 16; off > 0; off >>= 1) {
    sse += __shfl_down_sync(0xffffffffu, sse, off);
    nan += __shfl_down_sync(0xffffffffu, nan, off);
  }
  __shared__ unsigned long long part[2][8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { part[0][warp] = sse; part[1][warp] = nan; }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long s = 0, n = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { s += part[0][w]; n += part[1][w]; }
    if (s) atomicAdd(acc, s);
    if (n) atomicAdd(acc + 1, n);
  }
}

// SSIM weights and constants: w[0..5] the centre and side taps of scipy's gaussian_filter1d(sigma 1.5, truncate 3.5),
// c1 = (0.01 * 255)^2, c2 = (0.03 * 255)^2 - all taken from the host.
struct EvalSsim {
  double w[6];
  double c1, c2;
};

// scipy's symmetric NI_Correlate1D loop at row r of a column: acc = v[r] w0, then acc += (v[r - j] + v[r + j]) w_j for
// j = 5 .. 1.  Only rows 5 .. hs - 6 are evaluated, so the window never reaches the reflected border.
template <typename F>
__device__ __forceinline__ double eval_gauss(const EvalSsim& p, F v) {
  double acc = __dmul_rn(v(0), p.w[0]);
#pragma unroll
  for (int j = 5; j >= 1; --j) acc = __dadd_rn(acc, __dmul_rn(__dadd_rn(v(-j), v(j)), p.w[j]));
  return acc;
}

// util._ssim_columns: each column of the hs x ws region at (b, b) is a 1-D signal along the rows; map row i (i = 0 ..
// hs - 11) is row 5 + i of the SSIM map s, in numpy's operation order, nothing contracted into an FMA.
__global__ void __launch_bounds__(256) eval_ssim_kernel(const float* __restrict__ truth, const float* __restrict__ out, int pitch,
                                                        int b, int hs, int ws, const EvalSsim p, double* __restrict__ map) {
  const long long total = (long long)(hs - 10) * ws;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(idx / ws), x = (int)(idx - (long long)i * ws);
    const float* ta = truth + (long long)(b + 5 + i) * pitch + b + x;
    const float* tb = out + (long long)(b + 5 + i) * pitch + b + x;
    auto a = [&](int k) { return (double)__ldg(ta + (long long)k * pitch); };
    auto c = [&](int k) { return (double)__ldg(tb + (long long)k * pitch); };
    const double ux = eval_gauss(p, a);
    const double uy = eval_gauss(p, c);
    const double exx = eval_gauss(p, [&](int k) { const double v = a(k); return __dmul_rn(v, v); });
    const double eyy = eval_gauss(p, [&](int k) { const double v = c(k); return __dmul_rn(v, v); });
    const double exy = eval_gauss(p, [&](int k) { return __dmul_rn(a(k), c(k)); });
    const double uxx = __dmul_rn(ux, ux), uyy = __dmul_rn(uy, uy);
    const double vx = __dsub_rn(exx, uxx);
    const double vy = __dsub_rn(eyy, uyy);
    const double vxy = __dsub_rn(exy, __dmul_rn(ux, uy));
    const double num = __dmul_rn(__dadd_rn(__dmul_rn(__dmul_rn(2.0, ux), uy), p.c1), __dadd_rn(__dmul_rn(2.0, vxy), p.c2));
    const double den = __dmul_rn(__dadd_rn(__dadd_rn(uxx, uyy), p.c1), __dadd_rn(__dadd_rn(vx, vy), p.c2));
    map[idx] = __ddiv_rn(num, den);
  }
}

}  // namespace dcscn
