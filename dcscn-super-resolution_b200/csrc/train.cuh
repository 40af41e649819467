// Backward pass + optimizer kernels of the DCSCN train step (reference: DCSCN.py:334-413 `build_optimizer` /
// `add_optimizer_op`, i.e. what `sess.run(self.training_optimizer)` executed: tf.gradients of
// mse + l2_decay * sum(l2_loss(W)), tf.clip_by_global_norm, tf.train.AdamOptimizer).
//
// Split of the work:
//   * data gradients (dgrad) of every 3x3 / 1x1 layer run on the SAME wgmma implicit-GEMM kernels as the forward
//     pass (conv_tc*.cuh) with the filters transposed and spatially flipped - no extra MMA code;
//   * filter gradients (wgrad) of those layers run on wgmma too, with MN-major operands read straight from the NHWC
//     planes (wgrad_tc.cuh); `wgrad_kernel` below is the CUDA-core version kept as the cross-check (option wgrad_impl);
//   * everything else is in this file, on CUDA cores, laid out so a warp touches whole 128-byte lines: loss / output
//     gradient, R-CNN1 forward / backward fused with the depth_to_space gradient (= space_to_depth), CNN1's filter
//     gradient, PReLU + dropout gradients with the per-channel bias / alpha reductions, the fused L2-decay + global
//     norm + Adam update over one flat parameter buffer, and the device-side refresh of the packed weight images.
//   All activation-sized gradients are kept in the fp16 hi/lo plane format of the forward pass, multiplied by a
//   power-of-two `grad_scale` (loss scaling) so they sit in fp16's normal range; the scale is removed when the filter
//   gradients are finalised.
#pragma once
#include "common.h"
#include "epilogue.cuh"

namespace dcscn {

__device__ __forceinline__ float load_planes(const __half* hi, const __half* lo, size_t i) {
  float v = __half2float(hi[i]);
  if (lo != nullptr) v += __half2float(lo[i]);
  return v;
}
__device__ __forceinline__ void store_planes(__half* hi, __half* lo, size_t i, float v) {
  __half h, l;
  split_f16(v, h, l);
  hi[i] = h;
  if (lo != nullptr) lo[i] = l;
}

// ------------------------------------------------------------------------------------------------ loss ----
// diff = y_ - y; mse = mean(diff^2) (DCSCN.py:340-347).  image_loss = mse, or mean|diff| with --use_l1_loss
// (DCSCN.py:342-344).  dY = d image_loss / d y_ * grad_scale: diff * dscale (dscale = 2 * grad_scale / count), or
// sign(diff) * dscale (dscale = grad_scale / count) for the L1 loss.
struct LossParams {
  const float* y_pred;
  const float* y_true;
  float* dY;
  size_t count;
  float dscale;
  double* sq_sum;      // sum of diff^2
  double* abs_sum;     // sum of |diff|
  int l1;
};

__global__ void __launch_bounds__(256) loss_kernel(const LossParams p) {
  double acc = 0.0, acc1 = 0.0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.count; i += (size_t)gridDim.x * blockDim.x) {
    const float d = p.y_pred[i] - p.y_true[i];
    p.dY[i] = p.l1 ? (d > 0.f ? p.dscale : (d < 0.f ? -p.dscale : 0.f)) : d * p.dscale;   // tf.abs has gradient sign(x)
    acc += (double)d * (double)d;
    acc1 += (double)fabsf(d);
  }
  __shared__ double s[256], s1[256];
  s[threadIdx.x] = acc;
  s1[threadIdx.x] = acc1;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      s[threadIdx.x] += s[threadIdx.x + o];
      s1[threadIdx.x] += s1[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    atomicAdd(p.sq_sum, s[0]);
    atomicAdd(p.abs_sum, s1[0]);
  }
}

// --------------------------------------------------------------------------------------- R-CNN1 backward ----
// forward: out[q] = sum_tap sum_c w[tap][c] * hr[q + off(tap)][c]  (+ x2).
// (a) dW[tap][c] = sum_q hr[q + off(tap)][c] * dY[q]
struct LastWgradParams {
  int n_img, H, W, ksz, C, pitch;
  const float* hr;     // [N,H,W,pitch]
  const float* dY;     // [N,H,W]
  float* dW;           // [taps][C]
  int px_per_block;
};

// Thread = (pixel slot, channel quad): hr[q'][4 channels] is one 16-byte load and meets the up to k*k values
// dY[q' - off(tap)]; k*k x 4 accumulators per thread, reduced over the block's pixel slots in shared memory, one atomic
// per (tap, channel) per CTA.  Needs C % 4 == 0 and pitch % 4 == 0 (else `last_wgrad_scalar_kernel`).
constexpr int kLastWgMaxTaps = 25;
template <int TAPS>
__global__ void __launch_bounds__(256) last_wgrad_kernel(const LastWgradParams p) {
  extern __shared__ float s_red[];                 // [slots][TAPS][C]
  constexpr int KS = TAPS == 9 ? 3 : (TAPS == 25 ? 5 : 1), half = KS >> 1;
  const int quads = p.C >> 2;                      // threads per pixel
  const int slots = blockDim.x / quads;            // pixels in flight per CTA
  const int cq = threadIdx.x % quads, slot = threadIdx.x / quads;
  const long long total = (long long)p.n_img * p.H * p.W;
  const long long q0 = (long long)blockIdx.x * p.px_per_block;
  const long long q1 = q0 + p.px_per_block < total ? q0 + p.px_per_block : total;
  float acc[TAPS][4];
#pragma unroll
  for (int t = 0; t < TAPS; ++t) acc[t][0] = acc[t][1] = acc[t][2] = acc[t][3] = 0.f;
  if (slot < slots) {
    long long q = q0 + slot;
    int x = (int)(q % p.W), y = (int)((q / p.W) % p.H);
    for (; q < q1; q += slots) {
      const float4 hv = __ldg(reinterpret_cast<const float4*>(p.hr + q * p.pitch) + cq);
#pragma unroll
      for (int t = 0; t < TAPS; ++t) {
        const int dy = t / KS - half, dx = t % KS - half;   // hr[q] is the (dy,dx) neighbour of pixel q - off
        const int yy = y - dy, xx = x - dx;
        if (yy >= 0 && yy < p.H && xx >= 0 && xx < p.W) {
          const float d = __ldg(p.dY + q - ((long long)dy * p.W + dx));
          acc[t][0] = fmaf(hv.x, d, acc[t][0]);
          acc[t][1] = fmaf(hv.y, d, acc[t][1]);
          acc[t][2] = fmaf(hv.z, d, acc[t][2]);
          acc[t][3] = fmaf(hv.w, d, acc[t][3]);
        }
      }
      x += slots;
      while (x >= p.W) {
        x -= p.W;
        if (++y == p.H) y = 0;
      }
    }
#pragma unroll
    for (int t = 0; t < TAPS; ++t)
#pragma unroll
      for (int i = 0; i < 4; ++i) s_red[((size_t)slot * TAPS + t) * p.C + 4 * cq + i] = acc[t][i];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < TAPS * p.C; i += blockDim.x) {
    float sum = 0.f;
    for (int r = 0; r < slots; ++r) sum += s_red[(size_t)r * TAPS * p.C + i];
    atomicAdd(p.dW + i, sum);
  }
}

__global__ void __launch_bounds__(256) last_wgrad_scalar_kernel(const LastWgradParams p) {
  const int taps = p.ksz * p.ksz, half = p.ksz >> 1;
  const size_t total = (size_t)p.n_img * p.H * p.W;
  const size_t q0 = (size_t)blockIdx.x * p.px_per_block;
  const size_t q1 = q0 + p.px_per_block < total ? q0 + p.px_per_block : total;
  for (int tc = threadIdx.x; tc < taps * p.C; tc += blockDim.x) {
    const int tap = tc / p.C, c = tc - tap * p.C;
    const int dy = tap / p.ksz - half, dx = tap % p.ksz - half;
    float acc = 0.f;
    for (size_t q = q0; q < q1; ++q) {
      const int x = (int)(q % p.W), y = (int)((q / p.W) % p.H);
      const int yy = y + dy, xx = x + dx;
      if (yy < 0 || yy >= p.H || xx < 0 || xx >= p.W) continue;
      acc = fmaf(__ldg(p.hr + (q + (ptrdiff_t)dy * p.W + dx) * p.pitch + c), __ldg(p.dY + q), acc);
    }
    atomicAdd(p.dW + tc, acc);
  }
}

// (b) d hr[q][c] = sum_tap w[tap][c] * dY[q - off(tap)], written straight into the space_to_depth layout that is the
//     gradient of tf.depth_to_space (tf_graph.py:248): dZ[lr pixel][(i*r + j)*C + c] = d hr[(y*r+i, x*r+j)][c],
//     as fp16 hi/lo planes (input of the Up-PS dgrad / wgrad).
struct LastDgradParams {
  int n_img, H, W;     // LR-side resolution of the layer that feeds depth_to_space
  int r, C, ksz;
  const float* w;      // [taps][C]
  const float* dY;     // [N, r*H, r*W]
  __half* dz_hi;       // [N,H,W,pitch]
  __half* dz_lo;
  int pitch;
};

// Thread = (HR pixel, 8-channel group): the pixel's k*k dY neighbours are loaded (shared by the lanes of the pixel),
// 8 channels are k*k FMAs each against the filter in shared memory and leave as one 16-byte store per plane, so a warp
// writes whole lines of the LR pixel's (i*r + j)*C + c column block.  Other channel counts: one thread per pixel.
__global__ void __launch_bounds__(256) last_dgrad_s2d_kernel(const LastDgradParams p) {
  extern __shared__ float s_w[];                   // [taps][C]
  const int taps = p.ksz * p.ksz, half = p.ksz >> 1;
  for (int i = threadIdx.x; i < taps * p.C; i += blockDim.x) s_w[i] = __ldg(p.w + i);
  __syncthreads();
  const int HH = p.H * p.r, WW = p.W * p.r;
  const bool vec = (p.C & 7) == 0 && (p.pitch & 7) == 0;
  const int groups = vec ? p.C >> 3 : 1;
  const size_t total = (size_t)p.n_img * HH * WW * groups;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    // 32-bit index math (the launcher guarantees fewer than 2^32 elements; 64-bit divisions dominate otherwise)
    const unsigned i32 = (unsigned)idx;
    const unsigned Q32 = i32 / (unsigned)groups;
    const int g = (int)(i32 - Q32 * (unsigned)groups);
    const unsigned R32 = Q32 / (unsigned)WW;
    const int X = (int)(Q32 - R32 * (unsigned)WW), Y = (int)(R32 % (unsigned)HH);
    const size_t img = R32 / (unsigned)HH;
    float dy[kLastWgMaxTaps];
#pragma unroll
    for (int t = 0; t < kLastWgMaxTaps; ++t) {
      dy[t] = 0.f;
      if (t < taps) {
        const int yy = Y - (t / p.ksz - half), xx = X - (t % p.ksz - half);
        if (yy >= 0 && yy < HH && xx >= 0 && xx < WW) dy[t] = __ldg(p.dY + (img * HH + yy) * WW + xx);
      }
    }
    const int y = Y / p.r, i = Y - y * p.r, x = X / p.r, j = X - x * p.r;
    const size_t o = ((img * p.H + y) * p.W + x) * p.pitch + (size_t)(i * p.r + j) * p.C;
    if (vec) {
      const int c = 8 * g;
      uint32_t ph[4], pl[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float a0 = 0.f, a1 = 0.f;
#pragma unroll
        for (int t = 0; t < kLastWgMaxTaps; ++t)
          if (t < taps) {
            const float2 w2 = *reinterpret_cast<const float2*>(s_w + t * p.C + c + 2 * k);
            a0 = fmaf(w2.x, dy[t], a0);
            a1 = fmaf(w2.y, dy[t], a1);
          }
        split_f16x2(a0, a1, ph[k], pl[k]);
      }
      *reinterpret_cast<uint4*>(p.dz_hi + o + c) = make_uint4(ph[0], ph[1], ph[2], ph[3]);
      if (p.dz_lo != nullptr) *reinterpret_cast<uint4*>(p.dz_lo + o + c) = make_uint4(pl[0], pl[1], pl[2], pl[3]);
      continue;
    }
    for (int c = 0; c < p.C; ++c) {
      float a0 = 0.f;
#pragma unroll
      for (int t = 0; t < kLastWgMaxTaps; ++t)
        if (t < taps) a0 = fmaf(s_w[t * p.C + c], dy[t], a0);
      store_planes(p.dz_hi, p.dz_lo, o + c, a0);
    }
  }
}

// Row-walking form of the same kernel for 3x3 filters and C % 4 == 0, C <= 128 (the reference's R-CNN1): lane = channel
// quad with its 9 x 4 filter values in registers, a warp walks a run of HR pixels of one image row with a sliding 3x3
// window of dY (three broadcast loads per pixel, no index divisions in the loop) and writes 8 bytes per plane per lane:
// a pixel's C channels leave as one contiguous run of the LR pixel's (i*r + j)*C column block.
constexpr int kDgradRun = 32;
__global__ void __launch_bounds__(256) last_dgrad_s2d_rows_kernel(const LastDgradParams p) {
  const int lane = threadIdx.x & 31, quads = p.C >> 2;
  const bool active = lane < quads;
  float4 w[9];                                     // scalar loads: p.w points into the flat parameter buffer (4-byte aligned)
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const float* wt = p.w + t * p.C + 4 * lane;
    w[t] = active ? make_float4(__ldg(wt), __ldg(wt + 1), __ldg(wt + 2), __ldg(wt + 3)) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const int HH = p.H * p.r, WW = p.W * p.r;
  const int segs = (WW + kDgradRun - 1) / kDgradRun;    // runs never cross an image row
  const long long runs = (long long)p.n_img * HH * segs;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long run = warp0; run < runs; run += nwarps) {
    const long long row = run / segs;                 // img * HH + Y
    const int xs = (int)(run - row * segs) * kDgradRun;
    const int xe = xs + kDgradRun < WW ? xs + kDgradRun : WW;
    const int Y = (int)(row % HH);
    const long long img = row / HH;
    const bool up = Y > 0, dn = Y + 1 < HH;
    const float* rowp = p.dY + row * WW;
    // d hr[q] = sum_tap w[tap] * dY[q - off(tap)]: window columns X+1, X, X-1 pair with filter columns dx = -1, 0, +1
    auto load_col = [&](int XX, float (&col)[3]) {
      const bool in = XX >= 0 && XX < WW;
      const float* c = rowp + (XX < 0 ? 0 : XX);
      col[0] = (in && up) ? __ldg(c - WW) : 0.f;
      col[1] = in ? __ldg(c) : 0.f;
      col[2] = (in && dn) ? __ldg(c + WW) : 0.f;
    };
    float l[3], m[3], r3[3];                        // dY columns X-1, X, X+1 (rows Y-1, Y, Y+1)
    load_col(xs - 1, l);
    load_col(xs, m);
    const int y = Y / p.r, i = Y - y * p.r;
    const size_t orow = ((size_t)img * p.H + y) * p.W;
#pragma unroll 4
    for (int X = xs; X < xe; ++X) {
      load_col(X + 1, r3);
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
      for (int rr = 0; rr < 3; ++rr) {
        // filter row ky = 2 - rr pairs with dY row Y + (rr - 1): tap (dy, dx) meets dY[Y - dy][X - dx]
        const float4 wl = w[3 * (2 - rr) + 2], wm = w[3 * (2 - rr) + 1], wr = w[3 * (2 - rr) + 0];
        a0 = fmaf(wl.x, l[rr], fmaf(wm.x, m[rr], fmaf(wr.x, r3[rr], a0)));
        a1 = fmaf(wl.y, l[rr], fmaf(wm.y, m[rr], fmaf(wr.y, r3[rr], a1)));
        a2 = fmaf(wl.z, l[rr], fmaf(wm.z, m[rr], fmaf(wr.z, r3[rr], a2)));
        a3 = fmaf(wl.w, l[rr], fmaf(wm.w, m[rr], fmaf(wr.w, r3[rr], a3)));
      }
      if (active) {
        const int x = X / p.r, j = X - x * p.r;
        const size_t o = (orow + x) * p.pitch + (size_t)(i * p.r + j) * p.C + 4 * lane;
        uint32_t h01, l01, h23, l23;
        split_f16x2(a0, a1, h01, l01);
        split_f16x2(a2, a3, h23, l23);
        *reinterpret_cast<uint2*>(p.dz_hi + o) = make_uint2(h01, h23);
        if (p.dz_lo != nullptr) *reinterpret_cast<uint2*>(p.dz_lo + o) = make_uint2(l01, l23);
      }
#pragma unroll
      for (int rr = 0; rr < 3; ++rr) {
        l[rr] = m[rr];
        m[rr] = r3[rr];
      }
    }
  }
}

// space_to_depth of a plane tensor (gradient of the first depth_to_space of the x4 graph, DCSCN.py:298-301).
struct S2dParams {
  int n_img, H, W, r, C;   // LR-side size; src is [N, r*H, r*W, src_pitch]
  const __half *src_hi, *src_lo;
  int src_pitch;
  __half *dst_hi, *dst_lo;
  int dst_pitch;
};

__global__ void __launch_bounds__(256) s2d_planes_kernel(const S2dParams p) {
  const int rr = p.r * p.r;
  if ((p.C & 7) == 0 && (p.src_pitch & 7) == 0 && (p.dst_pitch & 7) == 0) {   // 16-byte moves of 8 channels
    const int g8 = p.C >> 3;
    const size_t total = (size_t)p.n_img * p.H * p.W * rr * g8;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
      const unsigned i32 = (unsigned)idx;           // < 2^32 elements (launcher)
      const unsigned r1 = i32 / (unsigned)g8;
      const int g = (int)(i32 - r1 * (unsigned)g8);
      const unsigned pix32 = r1 / (unsigned)rr;
      const int ij = (int)(r1 - pix32 * (unsigned)rr);
      const size_t pix = pix32;
      const int i = ij / p.r, j = ij - i * p.r;
      const unsigned row32 = pix32 / (unsigned)p.W;
      const int x = (int)(pix32 - row32 * (unsigned)p.W), y = (int)(row32 % (unsigned)p.H);
      const size_t img = row32 / (unsigned)p.H;
      const size_t s = ((img * p.H * p.r + (size_t)(y * p.r + i)) * (p.W * p.r) + (size_t)(x * p.r + j)) * p.src_pitch + 8 * g;
      const size_t d = pix * p.dst_pitch + (size_t)ij * p.C + 8 * g;
      *reinterpret_cast<uint4*>(p.dst_hi + d) = __ldg(reinterpret_cast<const uint4*>(p.src_hi + s));
      if (p.dst_lo != nullptr) *reinterpret_cast<uint4*>(p.dst_lo + d) = __ldg(reinterpret_cast<const uint4*>(p.src_lo + s));
    }
    return;
  }
  const int cols = rr * p.C;
  const size_t total = (size_t)p.n_img * p.H * p.W * cols;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int col = (int)(idx % cols);
    const size_t pix = idx / cols;
    const int x = (int)(pix % p.W), y = (int)((pix / p.W) % p.H), img = (int)(pix / ((size_t)p.W * p.H));
    const int ij = col / p.C, c = col - ij * p.C, i = ij / p.r, j = ij - i * p.r;
    const size_t s = (((size_t)img * p.H * p.r + (size_t)(y * p.r + i)) * (p.W * p.r) + (size_t)(x * p.r + j)) * p.src_pitch + c;
    const size_t d = pix * p.dst_pitch + col;
    p.dst_hi[d] = p.src_hi[s];
    if (p.dst_lo != nullptr) p.dst_lo[d] = p.src_lo[s];
  }
}

// -------------------------------------------------------------- PReLU + dropout gradient, bias / alpha sums ----
// out = dropout(f(z)) (tf_graph.py:126-130).  g = dL/d out (sum of up to two plane tensors), dh = g * keepmask/keep.
//   prelu:       dZ = dh * (z < 0 ? alpha : 1)      dalpha = sum dh * min(z, 0)        (from the min(z, 0) plane)
//   leaky_relu:  dZ = dh * (z < 0 ? 0.1f : 1)       (from the min(z, 0) plane: slope 1 at z = 0, like Maximum's gradient)
//   relu, sigmoid, tanh, selu: dZ = dh * f'(z) from the stored forward output y = h / keep of a kept element,
//                h = y * keep, as TensorFlow's ReluGrad / SigmoidGrad / TanhGrad / SeluGrad take it from h
//   db = sum dZ.  Layers without activation (act == ACT_NONE): dZ = g.
struct ActGradParams {
  size_t pixels;
  int C;                 // logical channels
  int n_total;           // padded GEMM width used by the forward dropout hash
  int col0;              // first column of this tensor inside that GEMM (A1+B1 fusion)
  const __half *g1_hi, *g1_lo; int g1_pitch;   // gradient source 1 (already offset to channel 0 of this tensor)
  const __half *g2_hi, *g2_lo; int g2_pitch;   // optional source 2 (nullptr: none)
  const __half* zneg; int zneg_pitch;          // min(z, 0) of the forward pre-activation (EpiSegment::dst_zneg), fp16
  const __half *y_hi, *y_lo; int y_pitch;      // the layer's stored forward output (relu, sigmoid, tanh, selu)
  int act;               // Activation
  const float* alpha;    // [C] PReLU slope (prelu only)
  float keep;
  uint32_t seed, layer;
  __half *dz_hi, *dz_lo; int dz_pitch;         // result planes (pad channels must stay zero)
  float* dbias;          // [C] accumulators (scaled by grad_scale) or nullptr
  float* dalpha;         // [C] or nullptr (prelu only)
  int px_per_block;
};

// blockDim = (channel pairs rounded up to a warp multiple, pixel rows): a thread keeps its channel pair and strides
// over the block's pixels (half2 loads, two pixels in flight); bias / alpha sums are reduced over the rows in shared
// memory, one atomic per channel per CTA.
__device__ __forceinline__ float2 load_planes2(const __half* hi, const __half* lo, size_t i) {
  float2 v = __half22float2(*reinterpret_cast<const __half2*>(hi + i));
  if (lo != nullptr) {
    const float2 l = __half22float2(*reinterpret_cast<const __half2*>(lo + i));
    v.x += l.x;
    v.y += l.y;
  }
  return v;
}

__global__ void __launch_bounds__(256) act_grad_kernel(const ActGradParams p) {
  extern __shared__ float s_sum[];                 // [2][rows][2 * PP]
  const int PP = blockDim.x, R = blockDim.y;
  const size_t q0 = (size_t)blockIdx.x * p.px_per_block;
  const size_t q1 = q0 + p.px_per_block < p.pixels ? q0 + p.px_per_block : p.pixels;
  const float inv_keep = 1.0f / p.keep;
  const int c = 2 * threadIdx.x;
  const bool v0 = c < p.C, v1 = c + 1 < p.C;
  const bool by_zneg = p.act == ACT_PRELU || p.act == ACT_LEAKY_RELU;
  float a0 = kLeakySlope, a1 = kLeakySlope;
  if (p.alpha) {
    if (v0) a0 = __ldg(p.alpha + c);
    if (v1) a1 = __ldg(p.alpha + c + 1);
  }
  float sb0 = 0.f, sb1 = 0.f, sa0 = 0.f, sa1 = 0.f;
  if (v0) {
#pragma unroll 2
    for (size_t q = q0 + threadIdx.y; q < q1; q += R) {
      float2 g = load_planes2(p.g1_hi, p.g1_lo, q * p.g1_pitch + c);
      if (p.g2_hi != nullptr) {
        const float2 g2 = load_planes2(p.g2_hi, p.g2_lo, q * p.g2_pitch + c);
        g.x += g2.x;
        g.y += g2.y;
      }
      float2 dz = g;
      if (p.act != ACT_NONE && p.keep < 1.0f) {
        const uint64_t e = (uint64_t)q * (uint64_t)p.n_total + p.col0 + c;
        g.x = dropout_keep(p.seed, p.layer, e, p.keep) ? g.x * inv_keep : 0.f;
        g.y = dropout_keep(p.seed, p.layer, e + 1, p.keep) ? g.y * inv_keep : 0.f;
      }
      if (by_zneg) {
        // PReLU backward from the pre-activation itself: z < 0 -> dz = g * alpha and d alpha += g * z.  (Deciding by the
        // sign of the OUTPUT is wrong for alpha <= 0 - alpha * z is then >= 0 - and shipped checkpoints have many
        // negative slopes; recovering z as output / alpha also breaks down as alpha -> 0.)
        const float2 zn = __half22float2(*reinterpret_cast<const __half2*>(p.zneg + q * p.zneg_pitch + c));
        dz = g;
        if (zn.x < 0.f) {
          sa0 = fmaf(g.x, zn.x, sa0);
          dz.x = g.x * a0;
        }
        if (zn.y < 0.f) {
          sa1 = fmaf(g.y, zn.y, sa1);
          dz.y = g.y * a1;
        }
      } else if (p.act != ACT_NONE) {
        const float2 y = load_planes2(p.y_hi, p.y_lo, q * p.y_pitch + c);
        dz.x = g.x * act_deriv_from_output(p.act, y.x * p.keep);
        dz.y = g.y * act_deriv_from_output(p.act, y.y * p.keep);
      }
      if (!v1) dz.y = 0.f;                          // pad channels of the result stay zero
      sb0 += dz.x;
      sb1 += dz.y;
      __half h0, l0, h1, l1;
      split_f16(dz.x, h0, l0);
      split_f16(dz.y, h1, l1);
      *reinterpret_cast<__half2*>(p.dz_hi + q * p.dz_pitch + c) = __halves2half2(h0, h1);
      if (p.dz_lo != nullptr) *reinterpret_cast<__half2*>(p.dz_lo + q * p.dz_pitch + c) = __halves2half2(l0, l1);
    }
  }
  if (p.dbias == nullptr && p.dalpha == nullptr) return;
  float* sb = s_sum;
  float* sa = s_sum + (size_t)R * 2 * PP;
  sb[(size_t)threadIdx.y * 2 * PP + c] = sb0;
  sb[(size_t)threadIdx.y * 2 * PP + c + 1] = sb1;
  sa[(size_t)threadIdx.y * 2 * PP + c] = sa0;
  sa[(size_t)threadIdx.y * 2 * PP + c + 1] = sa1;
  __syncthreads();
  for (int i = threadIdx.y * PP + threadIdx.x; i < 2 * PP; i += PP * R) {
    if (i >= p.C) continue;
    float tb = 0.f, ta = 0.f;
    for (int r = 0; r < R; ++r) {
      tb += sb[(size_t)r * 2 * PP + i];
      ta += sa[(size_t)r * 2 * PP + i];
    }
    if (p.dbias != nullptr) atomicAdd(p.dbias + i, tb);
    if (p.dalpha != nullptr) atomicAdd(p.dalpha + i, ta);
  }
}

// Same operation, 8 channels per thread with 16-byte loads / stores (all planes 16-byte aligned, which the 16-channel
// slot layout guarantees): the pair version above moved 4 bytes per thread and instruction and reached ~2 TB/s; this
// kernel is the default, the pair version the fallback for unaligned views.
__device__ __forceinline__ void unpack8(const uint4 v, float (&f)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __half22float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

__global__ void __launch_bounds__(256) act_grad8_kernel(const ActGradParams p) {
  extern __shared__ float s_sum[];                 // [2][rows][8 * TX]
  const int TX = blockDim.x, R = blockDim.y;
  const size_t q0 = (size_t)blockIdx.x * p.px_per_block;
  const size_t q1 = q0 + p.px_per_block < p.pixels ? q0 + p.px_per_block : p.pixels;
  const float inv_keep = 1.0f / p.keep;
  const int c = 8 * threadIdx.x;
  float a[8], sb[8], sa[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    a[i] = (p.alpha != nullptr && c + i < p.C) ? __ldg(p.alpha + c + i) : kLeakySlope;
    sb[i] = 0.f;
    sa[i] = 0.f;
  }
  if (c < p.C) {
#pragma unroll 2
    for (size_t q = q0 + threadIdx.y; q < q1; q += R) {
      float g[8], t[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(p.g1_hi + q * p.g1_pitch + c)), g);
      if (p.g1_lo != nullptr) {
        unpack8(__ldg(reinterpret_cast<const uint4*>(p.g1_lo + q * p.g1_pitch + c)), t);
#pragma unroll
        for (int i = 0; i < 8; ++i) g[i] += t[i];
      }
      if (p.g2_hi != nullptr) {
        float u[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(p.g2_hi + q * p.g2_pitch + c)), u);
        if (p.g2_lo != nullptr) {
          unpack8(__ldg(reinterpret_cast<const uint4*>(p.g2_lo + q * p.g2_pitch + c)), t);
#pragma unroll
          for (int i = 0; i < 8; ++i) u[i] += t[i];
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) g[i] += u[i];          // same association as the pair kernel: (g1h + g1l) + (g2h + g2l)
      }
      float dz[8];
      if (p.act == ACT_PRELU || p.act == ACT_LEAKY_RELU) {
        float zn[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(p.zneg + q * p.zneg_pitch + c)), zn);
        const uint64_t e = (uint64_t)q * (uint64_t)p.n_total + p.col0 + c;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float gi = g[i];
          if (p.keep < 1.0f) gi = dropout_keep(p.seed, p.layer, e + i, p.keep) ? gi * inv_keep : 0.f;
          dz[i] = gi;
          if (zn[i] < 0.f) {                               // PReLU backward from the pre-activation (see above)
            sa[i] = fmaf(gi, zn[i], sa[i]);
            dz[i] = gi * a[i];
          }
        }
      } else if (p.act != ACT_NONE) {                      // derivative from the stored output (see above)
        float y[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(p.y_hi + q * p.y_pitch + c)), y);
        if (p.y_lo != nullptr) {
          unpack8(__ldg(reinterpret_cast<const uint4*>(p.y_lo + q * p.y_pitch + c)), t);
#pragma unroll
          for (int i = 0; i < 8; ++i) y[i] += t[i];
        }
        const uint64_t e = (uint64_t)q * (uint64_t)p.n_total + p.col0 + c;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          float gi = g[i];
          if (p.keep < 1.0f) gi = dropout_keep(p.seed, p.layer, e + i, p.keep) ? gi * inv_keep : 0.f;
          dz[i] = gi * act_deriv_from_output(p.act, y[i] * p.keep);
        }
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) dz[i] = g[i];
      }
      uint32_t ph[4], pl[4];
#pragma unroll
      for (int i = 0; i < 8; i += 2) {
        if (c + i >= p.C) dz[i] = 0.f;                     // pad channels of the result stay zero
        if (c + i + 1 >= p.C) dz[i + 1] = 0.f;
        sb[i] += dz[i];
        sb[i + 1] += dz[i + 1];
        split_f16x2(dz[i], dz[i + 1], ph[i >> 1], pl[i >> 1]);
      }
      *reinterpret_cast<uint4*>(p.dz_hi + q * p.dz_pitch + c) = make_uint4(ph[0], ph[1], ph[2], ph[3]);
      if (p.dz_lo != nullptr) *reinterpret_cast<uint4*>(p.dz_lo + q * p.dz_pitch + c) = make_uint4(pl[0], pl[1], pl[2], pl[3]);
    }
  }
  if (p.dbias == nullptr && p.dalpha == nullptr) return;
  float* s_b = s_sum;
  float* s_a = s_sum + (size_t)R * 8 * TX;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    s_b[(size_t)threadIdx.y * 8 * TX + c + i] = sb[i];
    s_a[(size_t)threadIdx.y * 8 * TX + c + i] = sa[i];
  }
  __syncthreads();
  for (int i = threadIdx.y * TX + threadIdx.x; i < 8 * TX; i += TX * R) {
    if (i >= p.C) continue;
    float tb = 0.f, ta = 0.f;
    for (int r = 0; r < R; ++r) {
      tb += s_b[(size_t)r * 8 * TX + i];
      ta += s_a[(size_t)r * 8 * TX + i];
    }
    if (p.dbias != nullptr) atomicAdd(p.dbias + i, tb);
    if (p.dalpha != nullptr) atomicAdd(p.dalpha + i, ta);
  }
}

// --------------------------------------------------------------------------------------------- wgrad ----
// dW[tap][ci][co] += sum_p A[p + off(tap)][pos(ci)] * dZ[p][co]   (gradient of tf.nn.conv2d w.r.t. the HWIO filter)
// One CTA: one tap, a 64 x 64 (ci x co) tile, a range of image rows; 256 threads, 4 x 4 register micro-tile each,
// operands staged through shared memory as fp32 in chunks of 32 pixels.
struct WgradParams {
  int n_img, H, W, ksz, cin, cout;
  const __half *a_hi, *a_lo;   // input activation planes (nullptr when a_f32 is used)
  const float* a_f32;          // fp32 input (CNN1: the LR image, cin == 1)
  int a_pitch;
  const int* in_map;           // [cin] channel position inside the input buffer, or nullptr (identity)
  const __half *dz_hi, *dz_lo; // output-gradient planes [pixels][dz_pitch]
  int dz_pitch;
  float* dW;                   // [taps][cin][cout] fp32, accumulated with atomics
  int rows_per_block;          // image rows (of the N*H row space) per CTA
};

constexpr int kWgTile = 64, kWgPix = 32;

__global__ void __launch_bounds__(256) wgrad_kernel(const WgradParams p) {
  __shared__ float sA[kWgPix][kWgTile + 1];
  __shared__ float sZ[kWgPix][kWgTile + 1];
  const int taps = p.ksz * p.ksz, half = p.ksz >> 1;
  const int ci_tiles = (p.cin + kWgTile - 1) / kWgTile, co_tiles = (p.cout + kWgTile - 1) / kWgTile;
  int b = blockIdx.x;
  const int co_t = b % co_tiles; b /= co_tiles;
  const int ci_t = b % ci_tiles; b /= ci_tiles;
  const int tap = b % taps; b /= taps;
  const int row0 = b * p.rows_per_block;
  const int total_rows = p.n_img * p.H;
  const int row1 = row0 + p.rows_per_block < total_rows ? row0 + p.rows_per_block : total_rows;
  const int dy = tap / p.ksz - half, dx = tap % p.ksz - half;
  const int ci0 = ci_t * kWgTile, co0 = co_t * kWgTile;
  const int tci = (threadIdx.x >> 4) * 4, tco = (threadIdx.x & 15) * 4;   // 16 x 16 threads, 4 x 4 each
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int row = row0; row < row1; ++row) {
    const int y = row % p.H, img = row / p.H;
    const int yy = y + dy;
    if (yy < 0 || yy >= p.H) continue;   // warp-uniform (whole CTA)
    for (int x0 = 0; x0 < p.W; x0 += kWgPix) {
      __syncthreads();
      for (int i = threadIdx.x; i < kWgPix * kWgTile; i += blockDim.x) {
        const int c = i % kWgTile, px = i / kWgTile;
        const int x = x0 + px, xx = x + dx;
        float va = 0.f, vz = 0.f;
        if (x < p.W) {
          const size_t q = ((size_t)img * p.H + y) * p.W + x;
          if (co0 + c < p.cout) vz = load_planes(p.dz_hi, p.dz_lo, q * p.dz_pitch + co0 + c);
          if (xx >= 0 && xx < p.W && ci0 + c < p.cin) {
            const size_t qa = ((size_t)img * p.H + yy) * p.W + xx;
            const int pos = p.in_map ? __ldg(p.in_map + ci0 + c) : ci0 + c;
            va = p.a_f32 ? __ldg(p.a_f32 + qa * p.a_pitch + pos) : load_planes(p.a_hi, p.a_lo, qa * p.a_pitch + pos);
          }
        }
        sA[px][c] = va;
        sZ[px][c] = vz;
      }
      __syncthreads();
#pragma unroll 4
      for (int px = 0; px < kWgPix; ++px) {
        float a[4], z[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = sA[px][tci + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) z[j] = sZ[px][tco + j];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], z[j], acc[i][j]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int ci = ci0 + tci + i, co = co0 + tco + j;
      if (ci < p.cin && co < p.cout && acc[i][j] != 0.f) atomicAdd(p.dW + ((size_t)tap * p.cin + ci) * p.cout + co, acc[i][j]);
    }
}

// cin == 1 (CNN1: the input is the fp32 LR image): dW[tap][0][co] = sum_q x[q + off(tap)] * dZ[q][co].  One thread per
// output channel x pixel row; dZ[q][co] is loaded once and meets the k*k neighbours of x (broadcast loads).
struct FirstWgradParams {
  int n_img, H, W, ksz, cout;
  const float* x;               // [N,H,W]
  const __half *dz_hi, *dz_lo;  // [pixels][dz_pitch]
  int dz_pitch;
  float* dW;                    // [taps][1][cout]
  int px_per_block;
};

__global__ void __launch_bounds__(256) first_wgrad_kernel(const FirstWgradParams p) {
  // Thread = one output channel (all warps walk the SAME pixel run of the CTA, each with its own 32 channels); the 3x3
  // neighbourhood of x slides along the row (three broadcast loads per pixel, no divisions in the loop); k*k partial
  // sums per thread, one atomic per (tap, channel) per CTA.  Only ksz == 3 takes this path.
  const int c = threadIdx.x;
  const bool active = c < p.cout;
  const long long total = (long long)p.n_img * p.H * p.W;
  const long long q0 = (long long)blockIdx.x * p.px_per_block;
  const long long q1 = q0 + p.px_per_block < total ? q0 + p.px_per_block : total;
  if (q0 >= total) return;
  const int W = p.W, H = p.H;
  int x = (int)(q0 % W), y = (int)((q0 / W) % H);
  float acc[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) acc[t] = 0.f;
  float l[3], m[3], r3[3];
  auto load_col = [&](long long q, int xx, float (&col)[3]) {
#pragma unroll
    for (int rr = 0; rr < 3; ++rr) {
      const int yy = y + rr - 1;
      col[rr] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? __ldg(p.x + q + (long long)(rr - 1) * W + (xx - x)) : 0.f;
    }
  };
  load_col(q0, x - 1, l);
  load_col(q0, x, m);
  for (long long q = q0; q < q1; ++q) {
    load_col(q, x + 1, r3);
    const float zv = active ? load_planes(p.dz_hi, p.dz_lo, (size_t)q * p.dz_pitch + c) : 0.f;
#pragma unroll
    for (int rr = 0; rr < 3; ++rr) {               // tap (dy, dx) = (rr - 1, -1 | 0 | +1) meets x[q + off]
      acc[3 * rr + 0] = fmaf(zv, l[rr], acc[3 * rr + 0]);
      acc[3 * rr + 1] = fmaf(zv, m[rr], acc[3 * rr + 1]);
      acc[3 * rr + 2] = fmaf(zv, r3[rr], acc[3 * rr + 2]);
    }
    if (++x == W) {
      x = 0;
      if (++y == H) y = 0;
      if (q + 1 < q1) {
#pragma unroll
        for (int rr = 0; rr < 3; ++rr) l[rr] = 0.f;
        load_col(q + 1, 0, m);
      }
    } else {
#pragma unroll
      for (int rr = 0; rr < 3; ++rr) {
        l[rr] = m[rr];
        m[rr] = r3[rr];
      }
    }
  }
  if (active) {
#pragma unroll
    for (int t = 0; t < 9; ++t) atomicAdd(p.dW + (size_t)t * p.cout + c, acc[t]);
  }
}

// per-channel sum of a plane tensor (bias gradient of layers without activation)
struct ColSumParams {
  size_t pixels; int C; const __half *hi, *lo; int pitch; float* out; int px_per_block;
};
__global__ void __launch_bounds__(256) colsum_kernel(const ColSumParams p) {
  // blockDim = (8-channel lanes, pixel rows); 16-byte loads, per-thread partial sums reduced over the rows in smem.
  // Needs pitch % 8 == 0 (true for every plane tensor: pitches are multiples of 16).
  extern __shared__ float s_cs[];                  // [rows][8 * lanes]
  const int CP = blockDim.x, R = blockDim.y;
  const size_t q0 = (size_t)blockIdx.x * p.px_per_block;
  const size_t q1 = q0 + p.px_per_block < p.pixels ? q0 + p.px_per_block : p.pixels;
  for (int c0 = 0; c0 < p.C; c0 += 8 * CP) {
    const int c = c0 + 8 * threadIdx.x;
    float sum[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) sum[i] = 0.f;
    if (c < p.C) {
#pragma unroll 2
      for (size_t q = q0 + threadIdx.y; q < q1; q += R) {
        const uint4 vh = __ldg(reinterpret_cast<const uint4*>(p.hi + q * p.pitch + c));
        const uint4 vl = p.lo ? __ldg(reinterpret_cast<const uint4*>(p.lo + q * p.pitch + c)) : make_uint4(0, 0, 0, 0);
        const uint32_t hh[4] = {vh.x, vh.y, vh.z, vh.w}, ll[4] = {vl.x, vl.y, vl.z, vl.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&hh[i]));
          const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&ll[i]));
          sum[2 * i] += a.x + b.x;
          sum[2 * i + 1] += a.y + b.y;
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 8; ++i) s_cs[threadIdx.y * 8 * CP + 8 * threadIdx.x + i] = sum[i];
    __syncthreads();
    for (int i = threadIdx.y * CP + threadIdx.x; i < 8 * CP; i += CP * R) {
      if (c0 + i >= p.C) continue;
      float tot = 0.f;
      for (int r = 0; r < R; ++r) tot += s_cs[r * 8 * CP + i];
      atomicAdd(p.out + c0 + i, tot);
    }
  }
}

// ------------------------------------------------------------------------------- clip + Adam (flat buffers) ----
// g = grad / grad_scale (+ l2_decay * w for conv filters: d/dw of l2_decay * sum(w^2)/2, DCSCN.py:350-351);
// norm^2 over ALL trainables (tf.clip_by_global_norm, DCSCN.py:407).
struct GradFinalizeParams {
  float* grad; const float* w; const uint8_t* is_filter; size_t count; float inv_scale; float l2_decay; double* norm_sq;
};
__global__ void __launch_bounds__(256) grad_finalize_kernel(const GradFinalizeParams p) {
  double acc = 0.0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.count; i += (size_t)gridDim.x * blockDim.x) {
    float g = p.grad[i] * p.inv_scale;
    if (p.is_filter[i]) g = fmaf(p.l2_decay, p.w[i], g);
    p.grad[i] = g;
    acc += (double)g * (double)g;
  }
  __shared__ double s[256];
  s[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) atomicAdd(p.norm_sq, s[0]);
}

// Data-parallel training: this rank's image_loss and mse as two extra floats behind the flat gradient buffer, so that ONE
// all-reduce carries gradients and both scalars.  scal = {sum diff^2, -, sum |diff|}.
__global__ void loss_tail_kernel(const double* scal, double inv_count, int l1_loss, float* tail) {
  const double mse = scal[0] * inv_count;
  tail[0] = (float)(l1_loss ? scal[2] * inv_count : mse);
  tail[1] = (float)mse;
}

// tf.train.AdamOptimizer (DCSCN.py:388): m = b1*m + (1-b1)*g; v = b2*v + (1-b2)*g*g; w -= lr_t * m / (sqrt(v) + eps),
// lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t) (host), g = clipped gradient = g * clip / max(norm, clip).
struct AdamParams {
  float* w; float* m; float* v; const float* grad; size_t count;
  const double* norm_sq; float clip; float lr_t, beta1, beta2, eps;
};
__global__ void __launch_bounds__(256) adam_kernel(const AdamParams p) {
  float cscale = 1.f;
  if (p.clip > 0.f) {
    const float norm = (float)sqrt(*p.norm_sq);
    cscale = p.clip / fmaxf(norm, p.clip);
  }
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.count; i += (size_t)gridDim.x * blockDim.x) {
    const float g = p.grad[i] * cscale;
    const float m = p.beta1 * p.m[i] + (1.f - p.beta1) * g;
    const float v = p.beta2 * p.v[i] + (1.f - p.beta2) * g * g;
    p.m[i] = m;
    p.v[i] = v;
    p.w[i] -= p.lr_t * m / (sqrtf(v) + p.eps);
  }
}

// The other TF1 optimizers of add_optimizer_op (DCSCN.py:380-391) at TF's defaults, on the same clipped gradient; the
// update rules and slot orders are documented at DCSCN_OPTIMIZER_* (include/dcscn_b200.h).  One instantiation per
// optimizer, so each reads and writes only its own slots: s0 is slot 0, s1 slot 1.
struct OptimizerParams {
  float* w; float* s0; float* s1; const float* grad; size_t count;
  const double* norm_sq; float clip; float lr, momentum;
};
template <int OPT>
__global__ void __launch_bounds__(256) optimizer_kernel(const OptimizerParams p) {
  float cscale = 1.f;
  if (p.clip > 0.f) {
    const float norm = (float)sqrt(*p.norm_sq);
    cscale = p.clip / fmaxf(norm, p.clip);
  }
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.count; i += (size_t)gridDim.x * blockDim.x) {
    const float g = p.grad[i] * cscale;
    if constexpr (OPT == DCSCN_OPTIMIZER_GD) {
      p.w[i] -= p.lr * g;
    } else if constexpr (OPT == DCSCN_OPTIMIZER_MOMENTUM) {
      const float a = p.momentum * p.s0[i] + g;
      p.s0[i] = a;
      p.w[i] -= p.lr * a;
    } else if constexpr (OPT == DCSCN_OPTIMIZER_ADAGRAD) {
      const float acc = p.s0[i] + g * g;
      p.s0[i] = acc;
      p.w[i] -= p.lr * g / sqrtf(acc);
    } else if constexpr (OPT == DCSCN_OPTIMIZER_ADADELTA) {
      constexpr float rho = 0.95f, eps = 1e-8f;
      const float acc = rho * p.s0[i] + (1.f - rho) * g * g;
      const float acc_u = p.s1[i];
      const float u = sqrtf(acc_u + eps) / sqrtf(acc + eps) * g;
      p.s0[i] = acc;
      p.s1[i] = rho * acc_u + (1.f - rho) * u * u;
      p.w[i] -= p.lr * u;
    } else if constexpr (OPT == DCSCN_OPTIMIZER_RMSPROP) {
      constexpr float rho = 0.9f, eps = 1e-10f;
      const float ms = p.s0[i] + (g * g - p.s0[i]) * (1.f - rho);
      const float mom = p.momentum * p.s1[i] + p.lr * g / sqrtf(ms + eps);
      p.s0[i] = ms;
      p.s1[i] = mom;
      p.w[i] -= mom;
    }
  }
}


// ---- device-side refresh of the packed operand images after an optimizer step -------------------------------------
// dst = operand image (hi plane block, then lo plane block, per [n_tile][tap][chunk]); map[i] = flat
// index into the fp32 master weights behind hi-plane element i (-1 = structural zero).  Also records max |w * scale|
// so the host can tell when the power-of-two scale has to be re-chosen.
struct RepackParams {
  const float* w;
  const int* map;
  __half* dst;
  unsigned long long n;
  int half_elems;     // elements of one plane block
  float wscale;
  unsigned* wmax;     // float bits (values are non-negative, so unsigned order == float order)
};

__global__ void __launch_bounds__(256) repack_kernel(const RepackParams p) {
  float m = 0.f;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const int idx = __ldg(p.map + i);
    const float v = idx >= 0 ? __ldg(p.w + idx) * p.wscale : 0.f;
    m = fmaxf(m, fabsf(v));
    const __half hi = __float2half_rn(v);
    const __half lo = __float2half_rn(v - __half2float(hi));
    const unsigned long long blk = i / (unsigned)p.half_elems, pos = i - blk * (unsigned)p.half_elems;
    p.dst[blk * 2ull * p.half_elems + pos] = hi;
    p.dst[blk * 2ull * p.half_elems + p.half_elems + pos] = lo;
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(p.wmax, __float_as_uint(m));
}

// The folded last upsampler (engine.cu build_fold) from the master weights:
//   wf[r][ij * 9 + t] = sum_c W[r][ij * C + c] w_r[t][c]  for the filter rows r = (tap, ci),
//   bf[ij * 9 + t]    = sum_c b[ij * C + c] w_r[t][c]
// exact fp32 products added in fp64, c ascending, rounded once: the bits fold_dot gives on the host.  The maps hold
// each W / w_r / b element's index in the master weights (-1 = structural zero).
struct FoldParams {
  const float* w;
  const int* wu_map;   // [rows][sub * C]
  const int* wr_map;   // [9][C]
  const int* bu_map;   // [sub * C]
  int rows, sub, C;
  float* wf;           // [rows][sub * 9], read by repack_kernel through the folded layer's image map
  float* bf;           // [sub * 9], the folded layer's bias
};

__global__ void __launch_bounds__(256) fold_kernel(const FoldParams p) {
  const int cols = p.sub * 9;
  const long long n = (long long)(p.rows + 1) * cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(i % cols);
    const long long r = i / cols;
    const int ij = col / 9, t = col - ij * 9;
    const int* am = (r < p.rows ? p.wu_map + (size_t)r * p.sub * p.C : p.bu_map) + (size_t)ij * p.C;
    const int* wm = p.wr_map + (size_t)t * p.C;
    double s = 0.0;
    for (int c = 0; c < p.C; ++c) {
      const int ia = __ldg(am + c), iw = __ldg(wm + c);
      const float a = ia >= 0 ? __ldg(p.w + ia) : 0.f;
      const float b = iw >= 0 ? __ldg(p.w + iw) : 0.f;
      s += (double)a * (double)b;   // the product is exact in fp64, so a fused multiply-add gives the same sum
    }
    if (r < p.rows) p.wf[i] = (float)s;
    else p.bf[col] = (float)s;
  }
}

__global__ void __launch_bounds__(256) gather_params_kernel(const float* __restrict__ w, const int* __restrict__ map,
                                                            float* __restrict__ dst, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const int idx = map[i];
    if (idx >= 0) dst[i] = w[idx];
  }
}

// Up-TCNN (--pixel_shuffler=false): dW[i] = dF[src[i]], the gradient of Tconv_W from that of its 3x3 LR form F.  Each
// Tconv_W element is exactly one entry of F (engine.cu tconv_filter_map), so the gather is exact.
__global__ void __launch_bounds__(256) tconv_grad_gather_kernel(const float* __restrict__ dF, const int* __restrict__ src,
                                                                float* __restrict__ dW, int n) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dW[i] = dF[src[i]];
}

// ---- wide depthwise-separable graphs: the dense train step on composed filters ----
// One tf.nn.separable_conv2d layer's variables inside the flat parameter vectors: depthwise [taps][cin], pointwise
// [cin][cout] and the layer's conv_W slot [taps][cin][cout], which holds the composed filter / its gradient.
struct DsComposeParams {
  int taps, cin, cout;
  size_t dw, pw, wc;     // offsets into the flat vectors
};

// wc[t][ci][co] = dw[t][ci] * pw[ci][co] (one fp32 product, as the host packing forms it).
__global__ void __launch_bounds__(256) ds_compose_kernel(const float* __restrict__ w, float* __restrict__ wc,
                                                         const DsComposeParams p) {
  const long long n = (long long)p.taps * p.cin * p.cout;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(i % p.cout);
    const long long tc = i / p.cout;               // t * cin + ci
    const int ci = (int)(tc % p.cin);
    wc[p.wc + i] = w[p.dw + tc] * w[p.pw + (size_t)ci * p.cout + co];
  }
}

// The chain rule through the composition, from the composed filter's gradient gc[t][ci][co]:
//   d dw[t][ci] = sum_co gc[t][ci][co] pw[ci][co],   d pw[ci][co] = sum_t gc[t][ci][co] dw[t][ci]
// (fp64 sums); written into g, whose depthwise / pointwise slots nothing else of the dense step touches.
__global__ void __launch_bounds__(256) ds_decompose_kernel(const float* __restrict__ w, const float* __restrict__ gc,
                                                           float* __restrict__ g, const DsComposeParams p) {
  const long long ndw = (long long)p.taps * p.cin, n = ndw + (long long)p.cin * p.cout;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    double s = 0.0;
    if (i < ndw) {
      const int ci = (int)(i % p.cin);
      for (int co = 0; co < p.cout; ++co)
        s += (double)gc[p.wc + (size_t)i * p.cout + co] * (double)w[p.pw + (size_t)ci * p.cout + co];
      g[p.dw + i] = (float)s;
    } else {
      const long long j = i - ndw;                 // ci * cout + co
      const int ci = (int)(j / p.cout);
      for (int t = 0; t < p.taps; ++t)
        s += (double)gc[p.wc + ((size_t)t * p.cin + ci) * p.cout + (j % p.cout)] * (double)w[p.dw + (size_t)t * p.cin + ci];
      g[p.pw + j] = (float)s;
    }
  }
}

}  // namespace dcscn
