// Depthwise-separable DCSCN layers (reference: helper/tf_graph.py:155-216 `depthwise_separable_conv2d` /
// `build_depthwise_separable_conv`, i.e. tf.nn.separable_conv2d: depthwise k x k with channel multiplier 1 and no
// bias, then pointwise 1x1, then +bias, then PReLU; used for EVERY layer of a `--depthwise_separable` graph incl. the
// 1x1 A1/B1 (a per-channel scale) and R-CNN1).
//
// These graphs are tiny (c-DCSCN: <= 131 channels, 14,240 MAC per LR pixel at x4): a 131 x 24 contraction per pixel
// does not fill a tensor-core tile, so every layer is one kernel on CUDA cores over fp32 NHWC activations, and the
// depthwise value never leaves registers.  The layout keeps every thread issuing FMAs:
//   * one CTA = a 16 x 16 pixel tile (3x3 layers) or 256 consecutive pixels (1x1 layers), ONE PIXEL PER THREAD;
//   * the input tile (+1 halo, 32-channel chunks) is staged with 16-byte coalesced loads into shared memory with an odd
//     channel pitch (33) and a row stride of 24 pixels, so that the 4 x 8 pixel block of a warp reads 32 distinct banks
//     for every tap (lane -> (row, col) of the block; row offsets 0, 24, 48, 72 pixels = banks 0, 24, 16, 8);
//   * a thread forms the depthwise value of its pixel and channel c in registers (9 LDS + 9 FMA) and immediately
//     contracts it against the pointwise row W[c][0..cout_t) read as broadcast LDS.128 - up to 32 accumulators per
//     thread, no second pass over shared memory, no idle threads;
//   * layers with more than 32 output columns (Up-PS: 32 -> 128) loop over groups of 32 columns on the staged tile;
//   * two destinations (the fused A1 | B1 1x1 layer writes its A1 columns to the [B2 | A1] buffer and its B1 columns
//     to the B1 buffer), depth_to_space scatter and the final + x2 are epilogue variants;
//   * R-CNN1 (1 -> 1 channel at HR resolution) has kernels of its own: four pixels of a row per thread
//     (ds_single4_kernel), or one pixel per thread where the row width or the alignment does not allow four.
// fp32 throughout (CUDA cores): the contraction depth is <= 140 and the layers are HBM / issue bound, not FLOP bound.
#pragma once
#include <cstdint>
#include "epilogue.cuh"

namespace dcscn {

struct DsTileParams {
  int n_img, H, W;
  int cin, cout;
  const float* src;          // [N,H,W,src_pitch], offset to the first input channel
  int src_pitch;
  const float* dw;           // [k*k][cin] depthwise taps, or null = identity (scale folded into pw)
  const float* pw;           // [cin][cout]
  const float* bias;         // [cout] or null
  const float* alpha;        // [cout] or null
  float* dst;                // columns [0, split) (all columns when split == 0)
  int dst_pitch, dst_off;
  int split;                 // 0, or first column that goes to dst2
  float* dst2;
  int dst2_pitch, dst2_off;
  int d2s_r, d2s_cout;       // depth_to_space scatter (DCR) into dst [N, r*H, r*W, dst_pitch]
  const float* add;          // + x2 on channel 0 (cout == 1)
  int tiles_x, tiles_y;      // 3x3: 16 x 16 tiles per image
};

constexpr int kDtThreads = 256;
constexpr int kDtT = 16;                 // tile edge (3x3 layers)
constexpr int kDtS = 24;                 // shared-memory row stride in pixels (>= 18; 24 spreads a warp's 4 rows over banks)
constexpr int kDtCC = 32;                // channels per staged chunk
constexpr int kDtCP = 33;                // channel pitch of a staged pixel (odd: pixel index = bank offset)

// Layers with several column groups (cout > 32: the pixel shufflers) and a single input chunk keep each thread's depthwise
// values in a private shared-memory row after the first group instead of recomputing them (9 + 9 shared loads per value).
inline bool ds_tile_caches_depthwise(int ksz, int cin, int cout) { return ksz == 3 && cout > 32 && cin <= kDtCC; }

inline size_t ds_tile_smem_bytes(int ksz, int cin, int cout) {
  const int cols = cout < 32 ? ((cout + 3) & ~3) : 32;
  const size_t in_px = ksz == 3 ? (size_t)(kDtT + 2) * kDtS : (size_t)kDtThreads;
  const size_t cache = ds_tile_caches_depthwise(ksz, cin, cout) ? (size_t)kDtThreads * kDtCP : 0;
  return (in_px * kDtCP + (size_t)cin * cols + (size_t)ksz * ksz * cin + cache) * sizeof(float);
}

template <int KSZ, int CG4>
__global__ void __launch_bounds__(kDtThreads) ds_tile_kernel(const DsTileParams p) {
  extern __shared__ float4 s_raw4[];
  constexpr int kk = KSZ * KSZ;
  constexpr int COLS = 4 * CG4;                                    // output columns per pass
  constexpr int IN_PX = KSZ == 3 ? (kDtT + 2) * kDtS : kDtThreads;
  float* s_in = reinterpret_cast<float*>(s_raw4);                  // [IN_PX][kDtCP]
  float* s_pw = s_in + IN_PX * kDtCP;                              // [cin][COLS]  (current column group)
  float* s_dw = s_pw + p.cin * COLS;                               // [kk][cin]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // the host's ds_tile_caches_depthwise test (cout > COLS only when cout > 32), which sized shared memory for the cache
  const bool cache_u = KSZ == 3 && p.cout > COLS && p.cin <= kDtCC;
  float* s_u = s_dw + kk * p.cin + tid * kDtCP;                    // this thread's depthwise values [<= 32] (odd pitch: no bank conflicts)

  // ---- which pixels ----
  int img, y, x, hp0;                                              // hp0: this thread's centre pixel in the staged tile
  bool valid;
  int ty0 = 0, tx0 = 0;
  long long flat0 = 0;
  if (KSZ == 3) {
    const int t = blockIdx.x % (p.tiles_x * p.tiles_y);
    img = blockIdx.x / (p.tiles_x * p.tiles_y);
    ty0 = (t / p.tiles_x) * kDtT;
    tx0 = (t % p.tiles_x) * kDtT;
    // warp = 4 rows x 8 columns: warps 0..7 tile the 16 x 16 block as 4 row-bands x 2 column-halves
    const int ly = (warp >> 1) * 4 + (lane >> 3), lx = (warp & 1) * 8 + (lane & 7);
    y = ty0 + ly;
    x = tx0 + lx;
    valid = y < p.H && x < p.W;
    hp0 = (ly + 1) * kDtS + (lx + 1);
  } else {
    flat0 = (long long)blockIdx.x * kDtThreads;
    const long long total = (long long)p.n_img * p.H * p.W;
    const long long gp = flat0 + tid;
    valid = gp < total;
    const long long g2 = valid ? gp : total - 1;
    img = (int)(g2 / ((long long)p.H * p.W));
    const int r = (int)(g2 - (long long)img * p.H * p.W);
    y = r / p.W;
    x = r - y * p.W;
    hp0 = tid;
  }

  for (int i = tid; i < kk * p.cin; i += kDtThreads) s_dw[i] = p.dw ? __ldg(p.dw + i) : 1.0f;
  const bool vec_ok = ((p.src_pitch & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.src) & 15) == 0);

  for (int cg = 0; cg < p.cout; cg += COLS) {                      // column groups (one unless cout > 32)
    __syncthreads();                                               // previous group's readers of s_pw are done
    for (int i = tid; i < p.cin * COLS; i += kDtThreads) {
      const int c = i / COLS, q = i - c * COLS;
      s_pw[i] = (cg + q < p.cout) ? __ldg(p.pw + (size_t)c * p.cout + cg + q) : 0.f;
    }
    __syncthreads();
    float acc[COLS];
#pragma unroll
    for (int q = 0; q < COLS; ++q) acc[q] = 0.f;

    for (int c0 = 0; c0 < p.cin; c0 += kDtCC) {
      const int cc = (p.cin - c0) < kDtCC ? (p.cin - c0) : kDtCC;
      // ---- stage the input chunk (skipped when a single chunk is already resident from the previous column group) ----
      if (cg == 0 || p.cin > kDtCC) {
        __syncthreads();
        if (KSZ == 3) {
          constexpr int HP = (kDtT + 2) * (kDtT + 2);
          if (vec_ok && ((c0 & 3) == 0)) {
            for (int i = tid; i < HP * (kDtCC / 4); i += kDtThreads) {
              const int px = i >> 3, q = i & 7;
              const int hy = px / (kDtT + 2), hx = px - hy * (kDtT + 2);
              const int gy = ty0 + hy - 1, gx = tx0 + hx - 1;
              float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
              if (gy >= 0 && gy < p.H && gx >= 0 && gx < p.W && 4 * q < cc)
                v = __ldg(reinterpret_cast<const float4*>(p.src + ((size_t)((size_t)img * p.H + gy) * p.W + gx) * p.src_pitch + c0 + 4 * q));
              float* d = s_in + (hy * kDtS + hx) * kDtCP + 4 * q;
              d[0] = v.x;
              d[1] = (4 * q + 1 < cc) ? v.y : 0.f;
              d[2] = (4 * q + 2 < cc) ? v.z : 0.f;
              d[3] = (4 * q + 3 < cc) ? v.w : 0.f;
            }
          } else {
            for (int i = tid; i < HP * kDtCC; i += kDtThreads) {
              const int px = i >> 5, c = i & 31;
              const int hy = px / (kDtT + 2), hx = px - hy * (kDtT + 2);
              const int gy = ty0 + hy - 1, gx = tx0 + hx - 1;
              float v = 0.f;
              if (gy >= 0 && gy < p.H && gx >= 0 && gx < p.W && c < cc)
                v = __ldg(p.src + ((size_t)((size_t)img * p.H + gy) * p.W + gx) * p.src_pitch + c0 + c);
              s_in[(hy * kDtS + hx) * kDtCP + c] = v;
            }
          }
        } else {
          const long long total = (long long)p.n_img * p.H * p.W;
          if (vec_ok && ((c0 & 3) == 0)) {
            for (int i = tid; i < kDtThreads * (kDtCC / 4); i += kDtThreads) {
              const int px = i >> 3, q = i & 7;
              float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
              if (flat0 + px < total && 4 * q < cc)
                v = __ldg(reinterpret_cast<const float4*>(p.src + (size_t)(flat0 + px) * p.src_pitch + c0 + 4 * q));
              float* d = s_in + px * kDtCP + 4 * q;
              d[0] = v.x;
              d[1] = (4 * q + 1 < cc) ? v.y : 0.f;
              d[2] = (4 * q + 2 < cc) ? v.z : 0.f;
              d[3] = (4 * q + 3 < cc) ? v.w : 0.f;
            }
          } else {
            for (int i = tid; i < kDtThreads * kDtCC; i += kDtThreads) {
              const int px = i >> 5, c = i & 31;
              float v = 0.f;
              if (flat0 + px < total && c < cc) v = __ldg(p.src + (size_t)(flat0 + px) * p.src_pitch + c0 + c);
              s_in[px * kDtCP + c] = v;
            }
          }
        }
        __syncthreads();
      }
      // ---- depthwise value of (pixel, channel) in registers, contracted at once against the pointwise row ----
      const float* sp = s_in + hp0 * kDtCP;
      for (int c = 0; c < cc; ++c) {
        float d;
        if (KSZ == 3) {
          if (cache_u && cg > 0) {
            d = s_u[c];
          } else {
            d = 0.f;
#pragma unroll
            for (int t = 0; t < 9; ++t)
              d = fmaf(sp[((t / 3 - 1) * kDtS + (t % 3 - 1)) * kDtCP + c], s_dw[t * p.cin + c0 + c], d);
            if (cache_u) s_u[c] = d;
          }
        } else {
          d = sp[c] * s_dw[c0 + c];
        }
        const float4* w4 = reinterpret_cast<const float4*>(s_pw + (c0 + c) * COLS);
#pragma unroll
        for (int g = 0; g < CG4; ++g) {
          const float4 w = w4[g];
          acc[4 * g + 0] = fmaf(d, w.x, acc[4 * g + 0]);
          acc[4 * g + 1] = fmaf(d, w.y, acc[4 * g + 1]);
          acc[4 * g + 2] = fmaf(d, w.z, acc[4 * g + 2]);
          acc[4 * g + 3] = fmaf(d, w.w, acc[4 * g + 3]);
        }
      }
    }

    // ---- epilogue: bias, PReLU, store ----
    if (valid) {
      const size_t pix = ((size_t)img * p.H + y) * p.W + x;
#pragma unroll
      for (int g = 0; g < CG4; ++g) {
        const int co0 = cg + 4 * g;
        if (co0 >= p.cout) continue;
        float v[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int co = co0 + q;
          float t = acc[4 * g + q];
          if (co < p.cout) {
            if (p.bias) t += __ldg(p.bias + co);
            if (p.alpha) t = t > 0.f ? t : __ldg(p.alpha + co) * t;
          }
          v[q] = t;
        }
        if (p.d2s_r == 0) {
          float* base;
          int col;
          if (p.split > 0 && co0 >= p.split) {
            base = p.dst2 + pix * p.dst2_pitch + p.dst2_off;
            col = co0 - p.split;
          } else {
            base = p.dst + pix * p.dst_pitch + p.dst_off;
            col = co0;
          }
          const bool whole = (co0 + 3 < p.cout) && !(p.split > 0 && co0 < p.split && co0 + 3 >= p.split);
          if (whole && ((reinterpret_cast<uintptr_t>(base + col) & 15) == 0)) {
            *reinterpret_cast<float4*>(base + col) = make_float4(v[0], v[1], v[2], v[3]);
          } else {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const int co = co0 + q;
              if (co >= p.cout) continue;
              float t = v[q];
              if (p.add) t += __ldg(p.add + pix);
              if (p.split > 0 && co >= p.split) p.dst2[pix * p.dst2_pitch + p.dst2_off + (co - p.split)] = t;
              else p.dst[pix * p.dst_pitch + p.dst_off + co] = t;
            }
          }
        } else {
          // DCR: column (i*r + j)*C + c -> (y*r + i, x*r + j, c)   (tf.depth_to_space, tf_graph.py:248)
          const int r = p.d2s_r, C = p.d2s_cout;
          const size_t HRW = (size_t)p.W * r;
          const size_t img_base = (size_t)img * p.H * r * HRW;
          if ((C & 3) == 0 && co0 + 3 < p.cout) {
            const int ij = co0 / C, c = co0 - ij * C;
            const int ii = ij / r, jj = ij - ii * r;
            float* d = p.dst + (img_base + (size_t)(y * r + ii) * HRW + (size_t)(x * r + jj)) * p.dst_pitch + c;
            if ((reinterpret_cast<uintptr_t>(d) & 15) == 0) {
              *reinterpret_cast<float4*>(d) = make_float4(v[0], v[1], v[2], v[3]);
              continue;
            }
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int co = co0 + q;
            if (co >= p.cout) continue;
            const int ij = co / C, c = co - ij * C;
            const int ii = ij / r, jj = ij - ii * r;
            p.dst[(img_base + (size_t)(y * r + ii) * HRW + (size_t)(x * r + jj)) * p.dst_pitch + c] = v[q];
          }
        }
      }
    }
  }
}

// sigmoid / tanh / selu of an activated layer's output, in place: channels [off, off + C) of a [px][pitch] buffer.
// prelu, relu and leaky_relu run inside ds_tile_kernel's epilogue through its slope vector; evaluating the other three
// there as well changed the register allocation of every ds_tile_kernel instantiation and cost the PReLU graph 1.3 %
// (bench.py `ds`), so they take this one extra pass over the layer's output instead.
__global__ void __launch_bounds__(256) ds_act_kernel(float* buf, long long npx, int pitch, int off, int C, int act) {
  const long long total = npx * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long px = i / C;
    float* q = buf + px * pitch + off + (int)(i - px * C);
    *q = act_curve(act, *q);
  }
}

// R-CNN1 of a depthwise-separable graph (cin == cout == 1, 3x3, + x2) at HR resolution: four consecutive pixels of a row
// per thread, the three input rows read as float4 + two edge scalars.
__global__ void __launch_bounds__(256) ds_single4_kernel(const float* __restrict__ src, const float* __restrict__ add,
                                                         float* __restrict__ dst, int n_img, int H, int W, const float* dw,
                                                         const float* pw, const float* bias, const float* alpha) {
  float w[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) w[t] = __ldg(dw + t) * __ldg(pw);
  const float b = bias ? __ldg(bias) : 0.f;
  const int W4 = W >> 2;
  const long long total = (long long)n_img * H * W4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int x4 = (int)(i % W4);
    const long long row = i / W4;
    const int y = (int)(row % H);
    const float* base = src + row * W + 4 * x4;
    float acc[4] = {b, b, b, b};
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
      if ((unsigned)(y + dy) >= (unsigned)H) continue;
      const float* r = base + (long long)dy * W;
      const float4 m = __ldg(reinterpret_cast<const float4*>(r));
      const float l = x4 > 0 ? __ldg(r - 1) : 0.f;
      const float rr = x4 + 1 < W4 ? __ldg(r + 4) : 0.f;
      const float v[6] = {l, m.x, m.y, m.z, m.w, rr};
#pragma unroll
      for (int q = 0; q < 4; ++q)
        acc[q] = fmaf(v[q], w[(dy + 1) * 3], fmaf(v[q + 1], w[(dy + 1) * 3 + 1], fmaf(v[q + 2], w[(dy + 1) * 3 + 2], acc[q])));
    }
    if (alpha) {
      const float a = __ldg(alpha);
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[q] = acc[q] > 0.f ? acc[q] : a * acc[q];
    }
    const float4 x2 = add ? __ldg(reinterpret_cast<const float4*>(add + row * W + 4 * x4)) : make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<float4*>(dst + row * W + 4 * x4) = make_float4(acc[0] + x2.x, acc[1] + x2.y, acc[2] + x2.z, acc[3] + x2.w);
  }
}

// Same layer (k x k) with one pixel per thread: for HR widths that are not a multiple of 4, unaligned x2 / y, or a 1x1
// R-CNN1.  Row and column come from 64-bit pixel indices, so any number of pixels is covered.
template <int KSZ>
__global__ void __launch_bounds__(256) ds_single_kernel(const float* __restrict__ src, const float* __restrict__ add,
                                                        float* __restrict__ dst, int n_img, int H, int W, const float* dw,
                                                        const float* pw, const float* bias, const float* alpha) {
  constexpr int kk = KSZ * KSZ, half = KSZ >> 1;
  float w[kk];
#pragma unroll
  for (int t = 0; t < kk; ++t) w[t] = __ldg(dw + t) * __ldg(pw);
  const float b = bias ? __ldg(bias) : 0.f;
  const long long total = (long long)n_img * H * W;
  for (long long gp = (long long)blockIdx.x * blockDim.x + threadIdx.x; gp < total; gp += (long long)gridDim.x * blockDim.x) {
    const long long row = gp / W;
    const int x = (int)(gp - row * W);
    const int y = (int)(row % H);
    float acc = b;
#pragma unroll
    for (int t = 0; t < kk; ++t) {
      const int dy = t / KSZ - half, dx = t % KSZ - half;
      if ((unsigned)(y + dy) < (unsigned)H && (unsigned)(x + dx) < (unsigned)W)
        acc = fmaf(__ldg(src + gp + (long long)dy * W + dx), w[t], acc);
    }
    if (alpha) acc = acc > 0.f ? acc : __ldg(alpha) * acc;
    if (add) acc += __ldg(add + gp);
    dst[gp] = acc;
  }
}

}  // namespace dcscn
