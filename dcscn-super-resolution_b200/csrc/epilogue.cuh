// Fused convolution epilogue shared by the tensor-core kernel and the CUDA-core validation kernel:
//   acc * out_scale + bias  -> PReLU -> [inverted dropout] -> store
// replacing the reference's un-fused  tf.add(bias) / PReLU / tf.nn.dropout / tf.concat /
// tf.depth_to_space  ops (helper/tf_graph.py:109, :89-94, :130, :248; DCSCN.py:259,281).
#pragma once
#include "common.h"

namespace dcscn {

__device__ __forceinline__ void split_f16(float v, __half& hi, __half& lo) {
  // fp16 saturates at 65504; DCSCN activations live in 0..~1e3 (inputs are 0..255 luma).
  v = fminf(fmaxf(v, -65504.f), 65504.f);
  hi = __float2half_rn(v);
  lo = __float2half_rn(v - __half2float(hi));
}

// Counter-based keep mask for inverted dropout (tf.nn.dropout, tf_graph.py:130).
__host__ __device__ __forceinline__ uint32_t dropout_hash(uint32_t seed, uint32_t layer, uint64_t idx) {
  uint64_t z = idx + 0x9E3779B97F4A7C15ull * (uint64_t)(seed + 1) + ((uint64_t)layer << 40);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z = z ^ (z >> 31);
  return (uint32_t)(z >> 32);
}
__host__ __device__ __forceinline__ bool dropout_keep(uint32_t seed, uint32_t layer, uint64_t idx, float keep_prob) {
  // 24-bit uniform in [0,1)
  return (float)(dropout_hash(seed, layer, idx) >> 8) * (1.0f / 16777216.0f) < keep_prob;
}

// TensorFlow's selu constants: lambda and lambda * alpha (tf.nn.selu, SeluGrad).
constexpr float kSeluScale = 1.0507009873554805f;
constexpr float kSeluScaleAlpha = 1.7580993408473766f;
constexpr float kLeakySlope = 0.1f;   // build_activator's leaky_relu_alpha (tf_graph.py:77)

// sigmoid, tanh or selu of z in fp32 with the accurate libdevice functions (the build has no --use_fast_math).
__device__ __forceinline__ float act_curve(int act, float z) {
  if (act == ACT_SIGMOID) return 1.0f / (1.0f + expf(-z));
  if (act == ACT_TANH) return tanhf(z);
  return z < 0.f ? kSeluScaleAlpha * expm1f(z) : kSeluScale * z;
}

// The same as an out-of-line call: inlined at every epilogue site, the libdevice code grew conv_tc_kernel enough to
// slow the PReLU graph by 4 % (bench.py headline), with unchanged registers.
__device__ __noinline__ float act_curve_call(int act, float z) { return act_curve(act, z); }

// f(z) of an activated layer; `a` is the slope below zero of prelu / relu / leaky_relu.
__device__ __forceinline__ float act_apply(int act, float z, float a) {
  return act >= ACT_SIGMOID ? act_curve(act, z) : (z > 0.f ? z : a * z);
}

// f'(z) of relu, sigmoid, tanh and selu from the output h = f(z), the rule of TensorFlow's ReluGrad, SigmoidGrad,
// TanhGrad and SeluGrad: relu' = [h > 0] (0 at z = 0), selu' = lambda at z = 0.
__device__ __forceinline__ float act_deriv_from_output(int act, float h) {
  if (act == ACT_RELU) return h > 0.f ? 1.f : 0.f;
  if (act == ACT_SIGMOID) return h * (1.f - h);
  if (act == ACT_TANH) return 1.f - h * h;
  return h < 0.f ? h + kSeluScaleAlpha : kSeluScale;
}

// min(z, 0) as the PReLU / leaky_relu backward reads it from its fp16 plane.  A z in (-2^-24, 0) would round to -0 there
// and take slope 1 (TensorFlow takes alpha for every z < 0), so it is stored as -2^-24, the smallest fp16 subnormal:
// the sign survives and d alpha = sum g * z moves by at most 2^-24 |g| per such element.
__device__ __forceinline__ float zneg_value(float t) { return t < 0.f ? fminf(fmaxf(t, -65504.f), -0x1p-24f) : 0.f; }

__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
  return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}

// A lane's 16 fp16 channels of one plane as two 16-byte stores (sm_90 has no 32-byte global store).  `dst` must be
// 16-byte aligned (16-channel slots).
__device__ __forceinline__ void store_words8(void* dst, const uint32_t (&w)[8]) {
  uint4* q = reinterpret_cast<uint4*>(dst);
  q[0] = make_uint4(w[0], w[1], w[2], w[3]);
  q[1] = make_uint4(w[4], w[5], w[6], w[7]);
}

// Two values at once: one packed conversion (cvt.rn.f16x2.f32 -> F2FP.PACK_AB) per plane instead of two scalar F2F, which
// issue at a fraction of the ALU rate - the epilogues convert 2 x 16 values per 16-column chunk.  Same results as split_f16.
__device__ __forceinline__ void split_f16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
  a = fminf(fmaxf(a, -65504.f), 65504.f);
  b = fminf(fmaxf(b, -65504.f), 65504.f);
  const __half2 h = __floats2half2_rn(a, b);               // .x (low half) = a
  const float2 f = __half22float2(h);
  const __half2 l = __floats2half2_rn(a - f.x, b - f.y);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

__device__ __forceinline__ void split_planes16(const float (&v)[16], uint32_t (&ph)[8], uint32_t (&pl)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) split_f16x2(v[2 * i], v[2 * i + 1], ph[i], pl[i]);
}

__device__ __forceinline__ void store_planes16(__half* dst_hi, __half* dst_lo, size_t off, const float (&v)[16]) {
  uint32_t ph[8], pl[8];
  split_planes16(v, ph, pl);
  store_words8(dst_hi + off, ph);
  if (dst_lo != nullptr) store_words8(dst_lo + off, pl);
}

// acc * out_scale + bias -> activation -> [inverted dropout] of 16 consecutive GEMM columns starting at `cg`; zn = fp16
// pairs of min(z, 0), only formed when `want_zneg`.  `bias` / `alpha` are e.bias / e.alpha, read through the read-only
// cache, or (kSmemBias) plain loads from copies in shared memory or, where the rings leave no room for those, from
// e.bias / e.alpha.
template <bool kSmemBias>
__device__ __forceinline__ void epilogue_values16(const EpiParams& e, const float* bias, const float* alpha,
                                                  const ConvGeom& g, int n_total, int img, int y, int x, int cg,
                                                  const float (&acc)[16], float (&v)[16], uint32_t (&zn)[8],
                                                  bool want_zneg) {
  const float4* b4 = reinterpret_cast<const float4*>(bias + cg);
  const float4* a4 = reinterpret_cast<const float4*>(alpha + cg);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float4 b = kSmemBias ? b4[q] : __ldg(b4 + q);
    float4 a = kSmemBias ? a4[q] : __ldg(a4 + q);
    float t0 = fmaf(acc[4 * q + 0], e.out_scale, b.x);
    float t1 = fmaf(acc[4 * q + 1], e.out_scale, b.y);
    float t2 = fmaf(acc[4 * q + 2], e.out_scale, b.z);
    float t3 = fmaf(acc[4 * q + 3], e.out_scale, b.w);
    v[4 * q + 0] = t0 > 0.f ? t0 : a.x * t0;
    v[4 * q + 1] = t1 > 0.f ? t1 : a.y * t1;
    v[4 * q + 2] = t2 > 0.f ? t2 : a.z * t2;
    v[4 * q + 3] = t3 > 0.f ? t3 : a.w * t3;
    if (want_zneg) {
      const __half2 z01 = __floats2half2_rn(zneg_value(t0), zneg_value(t1));
      const __half2 z23 = __floats2half2_rn(zneg_value(t2), zneg_value(t3));
      zn[2 * q] = *reinterpret_cast<const uint32_t*>(&z01);
      zn[2 * q + 1] = *reinterpret_cast<const uint32_t*>(&z23);
    }
  }
  if (e.act >= ACT_SIGMOID) {   // these layers carry slope 1, so v == z here; an out-of-line call keeps the code small
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = act_curve_call(e.act, v[i]);
  }
  if (e.keep_prob < 1.0f) {
    const float inv_keep = 1.0f / e.keep_prob;
    const uint64_t base = ((uint64_t)((size_t)img * g.H + y) * g.W + x) * (uint64_t)(e.drop_ntotal ? e.drop_ntotal : n_total) + cg;
#pragma unroll
    for (int i = 0; i < 16; ++i)
      v[i] = dropout_keep(e.drop_seed, e.drop_layer, base + i, e.keep_prob) ? v[i] * inv_keep : 0.f;
  }
}

// One output pixel (img, y, x) of the LR grid, 16 consecutive GEMM columns starting at `cg`.  kSmemBias: the bias and
// slopes come from `bias` / `alpha` (conv_tc_kernel's epilogue warps: shared-memory copies when p.bias_smem).
template <bool kSmemBias = false>
__device__ __forceinline__ void epilogue_store16(const EpiParams& e, const ConvGeom& g, int n_total, int img, int y,
                                                 int x, int cg, const float (&acc)[16], const float* bias = nullptr,
                                                 const float* alpha = nullptr) {
  float v[16];
  uint32_t zn[8];      // fp16 pairs of min(z, 0), only formed when a training segment asks for them
  const bool want_zneg = e.mode == EPI_PLANES && (e.seg[0].dst_zneg != nullptr || (e.num_seg > 1 && e.seg[1].dst_zneg != nullptr));
  epilogue_values16<kSmemBias>(e, kSmemBias ? bias : e.bias, kSmemBias ? alpha : e.alpha, g, n_total, img, y, x, cg,
                               acc, v, zn, want_zneg);

  if (e.mode == EPI_PLANES) {
#pragma unroll
    for (int s = 0; s < kMaxSegments; ++s) {
      if (s < e.num_seg && cg >= e.seg[s].col_begin && cg < e.seg[s].col_end) {
        size_t off = ((size_t)((size_t)img * g.H + y) * g.W + x) * e.seg[s].pitch + (cg - e.seg[s].col_begin);
        store_planes16(e.seg[s].dst_hi, e.seg[s].dst_lo, off, v);
        if (e.seg[s].dst_zneg != nullptr) store_words8(e.seg[s].dst_zneg + off, zn);
      }
    }
    return;
  }

  // depth_to_space, DCR order: column = (i*r + j)*cout + c  ->  (y*r + i, x*r + j, c)   (tf_graph.py:248)
  const int r = e.d2s_r;
  const int co = e.d2s_cout;
  const int HR_H = g.H * r, HR_W = g.W * r;
  if ((co & 15) == 0) {
    if (cg >= e.n_valid) return;
    const int ij = cg / co, c = cg - ij * co;
    const int i = ij / r, j = ij - i * r;
    const size_t pix = (size_t)((size_t)img * HR_H + (y * r + i)) * HR_W + (x * r + j);
    if (e.mode == EPI_D2S_F32) {
      float4* d = reinterpret_cast<float4*>(e.dst_f32 + pix * e.d2s_pitch + c);
#pragma unroll
      for (int q = 0; q < 4; ++q) d[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    } else {
      store_planes16(e.seg[0].dst_hi, e.seg[0].dst_lo, pix * e.seg[0].pitch + c, v);
    }
  } else {
    // narrow pixel-shuffler outputs (c-DCSCN: pixel_shuffler_filters = 1): element-wise scatter
#pragma unroll
    for (int t = 0; t < 16; ++t) {
      const int col = cg + t;
      if (col >= e.n_valid) continue;
      const int ij = col / co, c = col - ij * co;
      const int i = ij / r, j = ij - i * r;
      const size_t pix = (size_t)((size_t)img * HR_H + (y * r + i)) * HR_W + (x * r + j);
      if (e.mode == EPI_D2S_F32) {
        e.dst_f32[pix * e.d2s_pitch + c] = v[t];
      } else {
        __half hi, lo;
        split_f16(v[t], hi, lo);
        e.seg[0].dst_hi[pix * e.seg[0].pitch + c] = hi;
        if (e.seg[0].dst_lo != nullptr) e.seg[0].dst_lo[pix * e.seg[0].pitch + c] = lo;
      }
    }
  }
}

// EPI_D2S_RDOT: 16 linear (bias only) columns of one sub-pixel -> accumulate the 9 per-tap dot products of the final
// cout=1 convolution (R-CNN1, DCSCN.py:318-323) so that only `taps` floats per HR pixel ever reach HBM.
__device__ __forceinline__ void rdot_accumulate16(const EpiParams& e, const float* w_smem, int cg, int c,
                                                  const float (&acc)[16], float (&v)[9]) {
  float t[16];
  const float4* b4 = reinterpret_cast<const float4*>(e.bias + cg);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float4 b = __ldg(b4 + q);
    t[4 * q + 0] = fmaf(acc[4 * q + 0], e.out_scale, b.x);
    t[4 * q + 1] = fmaf(acc[4 * q + 1], e.out_scale, b.y);
    t[4 * q + 2] = fmaf(acc[4 * q + 2], e.out_scale, b.z);
    t[4 * q + 3] = fmaf(acc[4 * q + 3], e.out_scale, b.w);
  }
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    if (tap < e.rdot_taps) {
      // filter taps staged in shared memory: every lane reads the same address (broadcast, one wavefront)
      const float4* w4 = reinterpret_cast<const float4*>(w_smem + tap * e.d2s_cout + c);
      // The 16 products are summed on their own and added to the running value once: one long fmaf chain over all the
      // channels of a sub-pixel (96 with the 192-column tiles) lets the rounding error of a partial sum of magnitude ~1e3
      // accumulate 96 times - on the uniform-noise tiles that alone was ~1e-3 of output error.
      float s = 0.f;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float4 w = w4[q];
        s = fmaf(t[4 * q + 0], w.x, s);
        s = fmaf(t[4 * q + 1], w.y, s);
        s = fmaf(t[4 * q + 2], w.z, s);
        s = fmaf(t[4 * q + 3], w.w, s);
      }
      v[tap] += s;
    }
  }
}

__device__ __forceinline__ void rdot_flush(const EpiParams& e, const ConvGeom& g, int img, int y, int x, int ij,
                                           int part, float (&v)[9]) {
  const int r = e.d2s_r;
  const int i = ij / r, j = ij - i * r;
  const size_t HR_H = (size_t)g.H * r, HR_W = (size_t)g.W * r;
  const size_t plane = (size_t)g.n_img * HR_H * HR_W;
  const size_t pix = ((size_t)img * HR_H + (size_t)(y * r + i)) * HR_W + (size_t)(x * r + j);
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    if (tap < e.rdot_taps) e.rdot_out[(size_t)(part * e.rdot_taps + tap) * plane + pix] = v[tap];
    v[tap] = 0.f;
  }
}
__device__ __forceinline__ void rdot_flush(const EpiParams& e, const ConvGeom& g, int img, int y, int x, int ij,
                                           float (&v)[9]) {
  rdot_flush(e, g, img, y, x, ij, 0, v);
}

// EPI_D2S_TAPS: 16 linear (bias only) columns of the folded last upsampler, column ij * taps + t = R-CNN1 tap t of
// sub-pixel ij, stored element-wise into the tap-planar layout rdot_flush writes (one partial set).
__device__ __forceinline__ void taps_store16(const EpiParams& e, const ConvGeom& g, int img, int y, int x, int cg,
                                             const float (&acc)[16]) {
  const int r = e.d2s_r, taps = e.rdot_taps;
  const size_t HR_H = (size_t)g.H * r, HR_W = (size_t)g.W * r;
  const size_t plane = (size_t)g.n_img * HR_H * HR_W;
  const float4* b4 = reinterpret_cast<const float4*>(e.bias + cg);
  // column cg + t is tap `tap` of sub-pixel (i, j): stepped from column to column instead of divided out of each
  int tap = cg % taps, i = cg / taps / r, j = cg / taps % r;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 b = __ldg(b4 + q);
    const float bq[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int col = cg + 4 * q + u;
      if (col >= e.n_valid) return;
      const size_t pix = ((size_t)img * HR_H + (size_t)(y * r + i)) * HR_W + (size_t)(x * r + j);
      e.rdot_out[(size_t)tap * plane + pix] = fmaf(acc[4 * q + u], e.out_scale, bq[u]);
      if (++tap == taps) {
        tap = 0;
        if (++j == r) { j = 0; ++i; }
      }
    }
  }
}

}  // namespace dcscn
