// CUDA-core kernels around the tensor-core convolution:
//   * conv_first_kernel : CNN1 (cin = 1, K = 9 - no GEMM shape to speak of), DCSCN.py:240-253 first iteration
//   * conv_last_kernel  : R-CNN1 (cout = 1, no bias / activation) fused with  tf.add(H[-1], x2, "output")
//                         (DCSCN.py:318-325)
//   * conv_ref_kernel   : plain fp32 FMA restatement of the tensor-core layer on the same buffers; used only by
//                         the on-GPU validation tests (option conv_impl = 1), never by default
//   * small layout helpers for the debug / parity interface
#pragma once
#include "common.h"
#include "epilogue.cuh"

namespace dcscn {

// ------------------------------------------------------------------ CNN1 -----------------------------------
struct ConvFirstParams {
  ConvGeom g;            // only n_img, H, W used
  int ksz;
  int n_pad;             // padded cout (multiple of 16)
  const float* x;        // [N, H, W] fp32 (channels == 1)
  const float* w;        // [k*k][n_pad] fp32, zero padded
  EpiParams epi;         // EPI_PLANES, out_scale 1
};

__global__ void __launch_bounds__(256) conv_first_kernel(const ConvFirstParams p) {
  // One lane = one pixel: its k*k input taps are loaded once and reused for every 16-channel group; the weights of a
  // group are warp-uniform, so the float4 shared-memory reads are broadcasts (one wavefront each).
  extern __shared__ float4 s_w4[];  // [tap][group][4]
  const int taps = p.ksz * p.ksz;
  const int groups = p.n_pad >> 4;
  for (int i = threadIdx.x; i < taps * groups * 4; i += blockDim.x) {
    const int q = i & 3, grp = (i >> 2) % groups, t = (i >> 2) / groups;
    const float* src = p.w + t * p.n_pad + grp * 16 + q * 4;
    s_w4[i] = make_float4(src[0], src[1], src[2], src[3]);
  }
  __syncthreads();
  const int half = p.ksz >> 1;
  const long long total = (long long)p.g.n_img * p.g.H * p.g.W;
  for (long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x; pix < total;
       pix += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(pix % p.g.W);
    const int y = (int)((pix / p.g.W) % p.g.H);
    const int img = (int)(pix / ((long long)p.g.W * p.g.H));
    const float* xi = p.x + (size_t)img * p.g.H * p.g.W;
    float in[25];
#pragma unroll
    for (int t = 0; t < 25; ++t) {
      if (t < taps) {
        const int yy = y + t / p.ksz - half, xx = x + t % p.ksz - half;
        in[t] = (yy >= 0 && yy < p.g.H && xx >= 0 && xx < p.g.W) ? __ldg(xi + (size_t)yy * p.g.W + xx) : 0.f;
      }
    }
    for (int grp = 0; grp < groups; ++grp) {
      float acc[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[i] = 0.f;
#pragma unroll
      for (int t = 0; t < 25; ++t) {
        if (t < taps) {
          const float v = in[t];
          const float4* w4 = s_w4 + (t * groups + grp) * 4;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 w = w4[q];
            acc[4 * q + 0] = fmaf(v, w.x, acc[4 * q + 0]);
            acc[4 * q + 1] = fmaf(v, w.y, acc[4 * q + 1]);
            acc[4 * q + 2] = fmaf(v, w.z, acc[4 * q + 2]);
            acc[4 * q + 3] = fmaf(v, w.w, acc[4 * q + 3]);
          }
        }
      }
      epilogue_store16(p.epi, p.g, p.n_pad, img, y, x, grp * 16, acc);
    }
  }
}

// 3x3 fast path: lane = 8 consecutive output channels (weights, bias, alpha live in registers for the whole kernel),
// warp = one pixel at a time, so each pixel's 2 x n_pad fp16 values leave the SM as two contiguous, fully coalesced
// rows.  HBM-write-bound by construction (CNN1 writes 2 x 208 fp16 per LR pixel and reads 4 bytes).
// ZNEG: the training forward also stores min(z, 0) (fp16) for the PReLU backward.
template <bool ZNEG>
__global__ void __launch_bounds__(256, 2) conv_first3x3_kernel(const ConvFirstParams p) {
  const int lane = threadIdx.x & 31;
  const int lanes_used = p.n_pad >> 3;
  const bool active = lane < lanes_used;
  const int c0 = lane * 8;
  float w[9][8], bias[8], alpha[8];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int i = 0; i < 8; ++i) w[t][i] = active ? __ldg(p.w + t * p.n_pad + c0 + i) : 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    bias[i] = active ? __ldg(p.epi.bias + c0 + i) : 0.f;
    alpha[i] = active ? __ldg(p.epi.alpha + c0 + i) : 1.f;
  }
  const EpiSegment seg = p.epi.seg[0];
  const float keep = p.epi.keep_prob, inv_keep = 1.0f / keep;
  const int act = p.epi.act;
  const long long total = (long long)p.g.n_img * p.g.H * p.g.W;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  constexpr int RUN = 32;                          // consecutive pixels per warp visit: a sliding 3x3 window, 3 loads / pixel
  const int W = p.g.W, H = p.g.H;
  for (long long pix0 = warp0 * RUN; pix0 < total; pix0 += nwarps * RUN) {
    const long long pix1 = pix0 + RUN < total ? pix0 + RUN : total;
    int x = (int)(pix0 % W);
    int y = (int)((pix0 / W) % H);
    float c0v[3], c1v[3], c2v[3];                  // window columns x-1, x, x+1 (rows y-1, y, y+1)
    auto load_col = [&](long long pix, int yy0, int xx, float (&col)[3]) {
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const int yy = yy0 + r - 1;
        col[r] = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? __ldg(p.x + pix + (long long)(r - 1) * W + (xx - x)) : 0.f;
      }
    };
    load_col(pix0, y, x - 1, c0v);
    load_col(pix0, y, x, c1v);
    for (long long pix = pix0; pix < pix1; ++pix) {
      load_col(pix, y, x + 1, c2v);
      float acc[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          acc[i] = fmaf(c0v[r], w[3 * r + 0][i], acc[i]);
          acc[i] = fmaf(c1v[r], w[3 * r + 1][i], acc[i]);
          acc[i] = fmaf(c2v[r], w[3 * r + 2][i], acc[i]);
        }
      }
      uint32_t ph[4], pl[4], pz[4];
#pragma unroll
      for (int i = 0; i < 8; i += 2) {
        float t0 = acc[i] + bias[i], t1 = acc[i + 1] + bias[i + 1];
        if (ZNEG) pz[i >> 1] = pack_h2(__float2half_rn(zneg_value(t0)), __float2half_rn(zneg_value(t1)));
        t0 = t0 > 0.f ? t0 : alpha[i] * t0;
        t1 = t1 > 0.f ? t1 : alpha[i + 1] * t1;
        if (!ZNEG && act >= ACT_SIGMOID) {             // slope 1 on these layers: t0, t1 are still z (their training
                                                       // forward writes no min(z, 0) plane, so ZNEG excludes them)
          t0 = act_curve_call(act, t0);
          t1 = act_curve_call(act, t1);
        }
        if (keep < 1.0f) {
          const uint64_t base = (uint64_t)pix * (uint64_t)p.n_pad + c0 + i;
          t0 = dropout_keep(p.epi.drop_seed, p.epi.drop_layer, base, keep) ? t0 * inv_keep : 0.f;
          t1 = dropout_keep(p.epi.drop_seed, p.epi.drop_layer, base + 1, keep) ? t1 * inv_keep : 0.f;
        }
        split_f16x2(t0, t1, ph[i >> 1], pl[i >> 1]);
      }
      if (active) {
        const size_t off = (size_t)pix * seg.pitch + c0;
        *reinterpret_cast<uint4*>(seg.dst_hi + off) = make_uint4(ph[0], ph[1], ph[2], ph[3]);
        if (seg.dst_lo != nullptr) *reinterpret_cast<uint4*>(seg.dst_lo + off) = make_uint4(pl[0], pl[1], pl[2], pl[3]);
        if (ZNEG) *reinterpret_cast<uint4*>(seg.dst_zneg + off) = make_uint4(pz[0], pz[1], pz[2], pz[3]);
      }
      if (++x == W) {                                // next image row (or next image): rebuild the window
        x = 0;
        if (++y == H) y = 0;
        if (pix + 1 < pix1) {
#pragma unroll
          for (int r = 0; r < 3; ++r) c0v[r] = 0.f;
          load_col(pix + 1, y, 0, c1v);
        }
      } else {
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          c0v[r] = c1v[r];
          c1v[r] = c2v[r];
        }
      }
    }
  }
}

// ---------------------------------------------------------------- R-CNN1 -----------------------------------
struct ConvLastParams {
  int n_img, H, W;       // HR resolution
  int ksz;               // 3
  int C;                 // input channels
  int pitch;             // channel pitch of src
  const float* src;      // [N, H, W, pitch] fp32
  const float* w;        // [k*k][C] fp32  (cout == 1)
  float bias;            // 0 for the reference graph
  const float* x2;       // [N, H, W] bicubic
  float* y;              // [N, H, W]
};

constexpr int kLastTW = 32, kLastTH = 8, kLastCC = 8;

__global__ void __launch_bounds__(256) conv_last_kernel(const ConvLastParams p) {
  extern __shared__ float s_mem[];
  const int half = p.ksz >> 1;
  const int PW = kLastTW + 2 * half, PH = kLastTH + 2 * half;
  float* s_w = s_mem;                                  // [taps][C]
  float* s_in = s_mem + p.ksz * p.ksz * p.C;           // [PH][PW][kLastCC]
  const int taps = p.ksz * p.ksz;
  for (int i = threadIdx.x; i < taps * p.C; i += blockDim.x) s_w[i] = p.w[i];

  const int tiles_x = (p.W + kLastTW - 1) / kLastTW, tiles_y = (p.H + kLastTH - 1) / kLastTH;
  const int tile = blockIdx.x;
  const int img = tile / (tiles_x * tiles_y);
  const int t2 = tile - img * tiles_x * tiles_y;
  const int ty = t2 / tiles_x, tx = t2 - ty * tiles_x;
  const int lx = threadIdx.x % kLastTW, ly = threadIdx.x / kLastTW;
  const int ox = tx * kLastTW + lx, oy = ty * kLastTH + ly;
  const float* src = p.src + (size_t)img * p.H * p.W * p.pitch;

  float acc = p.bias;
  for (int c0 = 0; c0 < p.C; c0 += kLastCC) {
    __syncthreads();
    for (int i = threadIdx.x; i < PH * PW * kLastCC; i += blockDim.x) {
      const int c = i % kLastCC;
      const int pp = i / kLastCC;
      const int sx = pp % PW, sy = pp / PW;
      const int gx = tx * kLastTW + sx - half, gy = ty * kLastTH + sy - half;
      float v = 0.f;
      if (gx >= 0 && gx < p.W && gy >= 0 && gy < p.H && (c0 + c) < p.C)
        v = __ldg(src + ((size_t)gy * p.W + gx) * p.pitch + c0 + c);
      s_in[i] = v;
    }
    __syncthreads();
    const int cc = (p.C - c0) < kLastCC ? (p.C - c0) : kLastCC;
    for (int t = 0; t < taps; ++t) {
      const float* si = s_in + ((ly + t / p.ksz) * PW + (lx + t % p.ksz)) * kLastCC;
      const float* wr = s_w + t * p.C + c0;
      for (int c = 0; c < cc; ++c) acc = fmaf(si[c], wr[c], acc);
    }
  }
  if (ox < p.W && oy < p.H) {
    const size_t o = ((size_t)img * p.H + oy) * p.W + ox;
    p.y[o] = acc + __ldg(p.x2 + o);
  }
}

// Same layer straight from global memory (used by the train step, where the HR feature map is materialised anyway).
// Lane = channel quad (filter taps of its 4 channels in registers), a warp walks a run of consecutive pixels of an image
// row with a sliding 3x3 window of float4 (three 16-byte loads per pixel, no index divisions in the loop) and reduces
// the lanes' partial dot products with shuffles.  Needs ksz == 3, C % 4 == 0, pitch % 4 == 0 and C <= 128.
constexpr int kLastRun = 32;
__global__ void __launch_bounds__(256) conv_last_direct_kernel(const ConvLastParams p) {
  const int lane = threadIdx.x & 31, quads = p.C >> 2;
  const bool active = lane < quads;
  float4 w[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) w[t] = active ? __ldg(reinterpret_cast<const float4*>(p.w + t * p.C) + lane) : make_float4(0.f, 0.f, 0.f, 0.f);
  const int W = p.W, H = p.H;
  const int segs = (W + kLastRun - 1) / kLastRun;       // runs never cross an image row: no wrap logic in the loop
  const long long runs = (long long)p.n_img * H * segs;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long run = warp0; run < runs; run += nwarps) {
    const long long row = run / segs;
    const int xs = (int)(run - row * segs) * kLastRun;
    const int xe = xs + kLastRun < W ? xs + kLastRun : W;
    const int y = (int)(row % H);
    const bool up = y > 0, dn = y + 1 < H;
    const float* rowp = p.src + (size_t)row * W * p.pitch + 4 * lane;   // (row, x = 0), this lane's channels
    const size_t rs = (size_t)W * p.pitch;
    auto load_col = [&](int xx, float4 (&col)[3]) {
      const bool in = active && xx >= 0 && xx < W;
      const float* c = rowp + (size_t)(xx < 0 ? 0 : xx) * p.pitch;
      col[0] = (in && up) ? __ldg(reinterpret_cast<const float4*>(c - rs)) : zero4;
      col[1] = in ? __ldg(reinterpret_cast<const float4*>(c)) : zero4;
      col[2] = (in && dn) ? __ldg(reinterpret_cast<const float4*>(c + rs)) : zero4;
    };
    float4 c0v[3], c1v[3], c2v[3];                 // window columns x-1, x, x+1 (rows y-1, y, y+1) of this lane's 4 channels
    load_col(xs - 1, c0v);
    load_col(xs, c1v);
#pragma unroll 4
    for (int x = xs; x < xe; ++x) {
      load_col(x + 1, c2v);
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const float4 w0 = w[3 * r], w1 = w[3 * r + 1], w2 = w[3 * r + 2];
        a0 = fmaf(c0v[r].x, w0.x, fmaf(c1v[r].x, w1.x, fmaf(c2v[r].x, w2.x, a0)));
        a1 = fmaf(c0v[r].y, w0.y, fmaf(c1v[r].y, w1.y, fmaf(c2v[r].y, w2.y, a1)));
        a2 = fmaf(c0v[r].z, w0.z, fmaf(c1v[r].z, w1.z, fmaf(c2v[r].z, w2.z, a2)));
        a3 = fmaf(c0v[r].w, w0.w, fmaf(c1v[r].w, w1.w, fmaf(c2v[r].w, w2.w, a3)));
      }
      float acc = (a0 + a1) + (a2 + a3);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      const long long q = row * W + x;
      if (lane == 0) p.y[q] = acc + p.bias + __ldg(p.x2 + q);
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        c0v[r] = c1v[r];
        c1v[r] = c2v[r];
      }
    }
  }
}

// Second half of the fused R-CNN1: y = sum over taps of the tap-planar partial products (written by the Up-PS
// epilogue, EPI_D2S_RDOT) at the tap-shifted pixel, + x2  (DCSCN.py:318-325).
struct ConvGatherParams {
  int n_img, H, W;   // HR resolution
  int ksz;
  const float* v;    // [parts][taps][n_img][H][W]
  int parts;         // partial plane sets to add up (EpiParams::rdot_parts)
  const float* x2;
  float* y;
};

__global__ void __launch_bounds__(256) conv_last_gather_kernel(const ConvGatherParams p) {
  const int half = p.ksz >> 1;
  const size_t plane = (size_t)p.n_img * p.H * p.W;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < plane; idx += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(idx % p.W);
    const int y = (int)((idx / p.W) % p.H);
    float acc = 0.f;
    const int taps = p.ksz * p.ksz;
    for (int t = 0; t < taps; ++t) {
      const int yy = y + t / p.ksz - half, xx = x + t % p.ksz - half;
      if (yy >= 0 && yy < p.H && xx >= 0 && xx < p.W)
        for (int q = 0; q < p.parts; ++q)
          acc += __ldg(p.v + (size_t)(q * taps + t) * plane + idx + (ptrdiff_t)(yy - y) * p.W + (xx - x));
    }
    p.y[idx] = acc + __ldg(p.x2 + idx);
  }
}

// 3x3, W % 4 == 0: four consecutive pixels of a row per thread.  Every (part, tap) plane row is read as one aligned float4
// plus one edge scalar for the dx = -1 / +1 taps (30 loads per 4 pixels with two partial plane sets instead of 72), no
// per-tap division.  Same summation order as the generic kernel above (taps outer, parts inner).
__global__ void __launch_bounds__(256) conv_last_gather4_kernel(const ConvGatherParams p) {
  const int W4 = p.W >> 2;
  const size_t plane = (size_t)p.n_img * p.H * p.W;
  const size_t total = (size_t)p.n_img * p.H * W4;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int x4 = (int)(i % W4);
    const size_t row = i / W4;                         // img * H + y
    const int y = (int)(row % p.H);
    const size_t base = row * p.W + 4 * (size_t)x4;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
      if ((unsigned)(y + dy) >= (unsigned)p.H) continue;
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx) {
        const int t = (dy + 1) * 3 + (dx + 1);
        for (int q = 0; q < p.parts; ++q) {
          const float* r = p.v + (size_t)(q * 9 + t) * plane + base + (ptrdiff_t)dy * p.W;
          const float4 m = __ldg(reinterpret_cast<const float4*>(r));
          if (dx == 0) {
            a0 += m.x; a1 += m.y; a2 += m.z; a3 += m.w;
          } else if (dx < 0) {
            const float l = x4 > 0 ? __ldg(r - 1) : 0.f;
            a0 += l; a1 += m.x; a2 += m.y; a3 += m.z;
          } else {
            const float rr = x4 + 1 < W4 ? __ldg(r + 4) : 0.f;
            a0 += m.y; a1 += m.z; a2 += m.w; a3 += rr;
          }
        }
      }
    }
    const float4 b = __ldg(reinterpret_cast<const float4*>(p.x2 + base));
    *reinterpret_cast<float4*>(p.y + base) = make_float4(a0 + b.x, a1 + b.y, a2 + b.z, a3 + b.w);
  }
}

// ---------------------------------------------------- validation conv (CUDA cores, fp32) -------------------
__global__ void __launch_bounds__(128) conv_ref_kernel(const ConvRefParams p) {
  const int groups = p.n_total_pad >> 4;
  const int half = p.ksz >> 1;
  const long long total = (long long)p.g.n_img * p.g.H * p.g.W * groups;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int grp = (int)(idx % groups);
    const long long pix = idx / groups;
    const int x = (int)(pix % p.g.W);
    const int y = (int)((pix / p.g.W) % p.g.H);
    const int img = (int)(pix / ((long long)p.g.W * p.g.H));
    float acc[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = 0.f;
    for (int t = 0; t < p.ksz * p.ksz; ++t) {
      const int yy = y + t / p.ksz - half, xx = x + t % p.ksz - half;
      if (yy < 0 || yy >= p.g.H || xx < 0 || xx >= p.g.W) continue;
      const size_t base = (((size_t)img * p.g.H + yy) * p.g.W + xx) * p.src_pitch;
      for (int c = 0; c < p.cin; ++c) {
        const int q = p.in_map[c];
        float a = __half2float(p.src_hi[base + q]);
        if (p.src_lo != nullptr) a += __half2float(p.src_lo[base + q]);
        const float* wr = p.w + ((size_t)t * p.cin + c) * p.cout;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          const int n = grp * 16 + i;
          if (n < p.cout) acc[i] = fmaf(a, __ldg(wr + n), acc[i]);
        }
      }
    }
    epilogue_store16(p.epi, p.g, p.n_total_pad, img, y, x, grp * 16, acc);
  }
}

// ------------------------------------------------- depthwise step of wide depthwise-separable graphs -----------
// The depthwise half of tf.nn.separable_conv2d (helper/tf_graph.py:155-216) for graphs too wide for ds_tile_kernel:
// u[c] = sum over the k x k taps of x[c] dw[tap][c] (SAME zero padding, no bias), read from and written to fp16 hi/lo
// planes, so that the pointwise half, bias and activation run as a 1x1 layer of conv_tc_kernel over u.  fp32 FMAs in
// tap order, one thread per pixel and 8 channel positions (16-byte loads and stores).
struct DwParams {
  int n_img, H, W;           // resolution of the layer's input (= output)
  int ksz;                   // 3 or 5; 0 = the layer has no depthwise step
  int cpad;                  // channel positions of the source region (a multiple of 16), also u's pitch
  const __half* src_hi;      // source planes, offset to the region's first position
  const __half* src_lo;      // null in f16x1
  int src_pitch;
  const float* dw;           // [k*k][cpad] fp32, zero at positions no channel maps to
  __half* u_hi;              // [px][cpad]
  __half* u_lo;              // null in f16x1
};

template <int K>
__global__ void __launch_bounds__(256) depthwise_planes_kernel(const DwParams p) {
  constexpr int half = K / 2;
  const int groups = p.cpad >> 3;
  const long long total = (long long)p.n_img * p.H * p.W * groups;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(i % groups) * 8;
    const long long pix = i / groups;
    const int x = (int)(pix % p.W);
    const int y = (int)((pix / p.W) % p.H);
    const long long img0 = pix - (long long)y * p.W - x;   // first pixel of this image
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int ty = 0; ty < K; ++ty) {
      const int yy = y + ty - half;
      if (yy < 0 || yy >= p.H) continue;
#pragma unroll
      for (int tx = 0; tx < K; ++tx) {
        const int xx = x + tx - half;
        if (xx < 0 || xx >= p.W) continue;
        const size_t off = (size_t)(img0 + (long long)yy * p.W + xx) * p.src_pitch + c0;
        const uint4 hq = __ldg(reinterpret_cast<const uint4*>(p.src_hi + off));
        const uint4 lq = p.src_lo != nullptr ? __ldg(reinterpret_cast<const uint4*>(p.src_lo + off)) : make_uint4(0, 0, 0, 0);
        const __half2* h2 = reinterpret_cast<const __half2*>(&hq);
        const __half2* l2 = reinterpret_cast<const __half2*>(&lq);
        const float4* w4 = reinterpret_cast<const float4*>(p.dw + (size_t)(ty * K + tx) * p.cpad + c0);
        const float4 wa = __ldg(w4), wb = __ldg(w4 + 1);
        const float w[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 hv = __half22float2(h2[j]), lv = __half22float2(l2[j]);
          acc[2 * j] = fmaf(hv.x + lv.x, w[2 * j], acc[2 * j]);
          acc[2 * j + 1] = fmaf(hv.y + lv.y, w[2 * j + 1], acc[2 * j + 1]);
        }
      }
    }
    uint32_t ph[4], pl[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) split_f16x2(acc[2 * j], acc[2 * j + 1], ph[j], pl[j]);
    const size_t o = (size_t)pix * p.cpad + c0;
    *reinterpret_cast<uint4*>(p.u_hi + o) = make_uint4(ph[0], ph[1], ph[2], ph[3]);
    if (p.u_lo != nullptr) *reinterpret_cast<uint4*>(p.u_lo + o) = make_uint4(pl[0], pl[1], pl[2], pl[3]);
  }
}

// ---------------------------------------------------------------- helpers ----------------------------------
__global__ void planes_to_f32_kernel(const __half* hi, const __half* lo, float* out, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float v = __half2float(hi[i]);
    if (lo != nullptr) v += __half2float(lo[i]);
    out[i] = v;
  }
}

// ------------------------------------------------------------- Pillow bicubic resize on the device ------------
// Bit-exact restatement of `Image.resize(BICUBIC)` for mode 'F' images (reference helper/utilty.py:211-239 ->
// Pillow src/libImaging/Resample.c, see helper/pil_resample.py): horizontal pass, float32 intermediate, vertical pass;
// every sample is (float) sum_x (double)pixel * w[x] accumulated in window order.  __dmul_rn / __dadd_rn keep the
// compiler from fusing the multiply-add (Pillow's x86-64 build has no FMA), which is what makes it bit-exact.
struct PilAxis {
  const double* k;     // [out][ksize] normalised weights
  const int* bounds;   // [out][2] first input index, taps
  int ksize;
};

__global__ void __launch_bounds__(256) pil_resample_h_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                             long long rows, int W, int OW, const PilAxis ax) {
  const long long total = rows * OW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / OW;
    const int xx = (int)(i - row * OW);
    const int x0 = __ldg(ax.bounds + 2 * xx), cnt = __ldg(ax.bounds + 2 * xx + 1);
    const double* k = ax.k + (size_t)xx * ax.ksize;
    const float* p = src + row * W + x0;
    double ss = 0.0;
    for (int x = 0; x < cnt; ++x) ss = __dadd_rn(ss, __dmul_rn((double)__ldg(p + x), __ldg(k + x)));
    dst[i] = (float)ss;
  }
}

__global__ void __launch_bounds__(256) pil_resample_v_kernel(const float* __restrict__ src, float* __restrict__ dst, int n,
                                                             int H, int OH, int OW, const PilAxis ax) {
  const long long per = (long long)OH * OW, total = per * n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int img = (int)(i / per);
    const int r = (int)(i - (long long)img * per);
    const int yy = r / OW, xx = r - yy * OW;
    const int y0 = __ldg(ax.bounds + 2 * yy), cnt = __ldg(ax.bounds + 2 * yy + 1);
    const double* k = ax.k + (size_t)yy * ax.ksize;
    const float* p = src + ((size_t)img * H + y0) * OW + xx;
    double ss = 0.0;
    for (int y = 0; y < cnt; ++y) ss = __dadd_rn(ss, __dmul_rn((double)__ldg(p + (size_t)y * OW), __ldg(k + y)));
    dst[i] = (float)ss;
  }
}

// ------------------------------------------------------------- training patch store ---------------------------
// What `build_input_batch` + the feed of `train_batch` did on the host (DCSCN.py:186-190, 415-420; patches of
// loader.BatchDataSets, loader.py:236-249): the uint8 patch arrays live in HBM, one launch gathers the mini-batch's
// patches by index into fp32 NHWC tensors (x scale = max_value / 255, loader.py:251-255), optionally mirrored left-right
// (bit 31 of the index; the augmentation of loader.py:318-319).
__global__ void __launch_bounds__(256) patch_gather_kernel(const uint8_t* __restrict__ store, const int* __restrict__ idx,
                                                           float* __restrict__ out, int n, int H, int W, double scale) {
  const long long per = (long long)H * W, total = per * n;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(e / per);
    const int r = (int)(e - (long long)i * per);
    const int code = __ldg(idx + i);
    const long long k = code & 0x7FFFFFFF;
    int src = r;
    if (code < 0) {                                  // mirrored patch: column W - 1 - x
      const int y = r / W, x = r - y * W;
      src = y * W + (W - 1 - x);
    }
    // numpy's `np.multiply(uint8_patch, max_value / 255.0)` is a float64 product, rounded to fp32 at the feed
    out[e] = (float)((double)__ldg(store + k * per + src) * scale);
  }
}

// ------------------------------------------------------------- random-crop training data ----------------------
// What loader.DynamicDataSets.load_batch_image does per patch on the host (reference helper/loader.py:310-355): crop an
// e x e square out of a decoded image, RGB -> Y in float64, mirror left-right, Pillow-bicubic down by 1/scale and back up.
// The decoded uint8 images live in HBM (dcscn_image_store_set); a mini-batch is a list of crop descriptors.
struct ImageEntry {
  long long offset;    // first byte of the image in the pixel store
  int height, width, channels;   // channels: 3 (RGB, interleaved) or 1 (mode 'L')
};

struct CropJob {
  int image, top, left, mirror;
  int mode8;           // 1: a mode-'L' image, resampled by Pillow's 8-bit path; 0: an RGB image, resampled as mode 'F'
  int slot;            // position of the crop inside its resampler group (mode-'F' crops, then mode-'L' crops)
};

// util._Y_ROW
#define DCSCN_Y_R (65.738 / 256.0)
#define DCSCN_Y_G (129.057 / 256.0)
#define DCSCN_Y_B (25.064 / 256.0)

// One thread per HR crop pixel (i, r, c): the source pixel is (top + r, left + (mirror ? e - 1 - c : c)).  An RGB pixel
// becomes util.convert_rgb_to_y's float64 Y, which numpy's dot (BLAS ddot) forms as fma(b, c2, fma(g, c1, r * c0)) + 16;
// the truth is fp32(Y * scale) (the float64 product of _rescaled, loader.py:323-327) and the mode-'F' resampler input is
// fp32(Y) (Image.fromarray of a float64 array).  A mode-'L' pixel is fed to the 8-bit resampler as is and its truth is
// fp32(double(u8) * scale).  scale = max_value / 255, exactly 1 at 255 (no multiply in the reference).
__global__ void __launch_bounds__(256) crop_gather_kernel(const uint8_t* __restrict__ pixels, const ImageEntry* __restrict__ table,
                                                          const CropJob* __restrict__ jobs, int n, int e, double scale,
                                                          float* __restrict__ truth, float* __restrict__ f_in,
                                                          uint8_t* __restrict__ l_in) {
  const long long per = (long long)e * e, total = per * n;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(idx / per);
    const int r = (int)(idx - (long long)i * per);
    const int y = r / e, x = r - y * e;
    const CropJob j = jobs[i];
    const ImageEntry im = table[j.image];
    const int col = j.left + (j.mirror ? e - 1 - x : x);
    const uint8_t* p = pixels + im.offset + ((long long)(j.top + y) * im.width + col) * im.channels;
    const long long dst = (long long)j.slot * per + r;
    if (im.channels == 3) {
      const double v = __dadd_rn(__fma_rn((double)__ldg(p + 2), DCSCN_Y_B,
                                          __fma_rn((double)__ldg(p + 1), DCSCN_Y_G, __dmul_rn((double)__ldg(p), DCSCN_Y_R))),
                                 16.0);
      truth[idx] = (float)__dmul_rn(v, scale);
      f_in[dst] = (float)v;
    } else {
      const uint8_t v = __ldg(p);
      truth[idx] = (float)__dmul_rn((double)v, scale);
      l_in[dst] = v;
    }
  }
}

// Pillow's ImagingResampleHorizontal_8bpc / ImagingResampleVertical_8bpc (src/libImaging/Resample.c) for mode 'L': the
// double weights of the mode-'F' tables become 22-bit fixed point, (int)(w * 2^22 + 0.5) or (int)(w * 2^22 - 0.5) for
// w < 0 (normalize_coeffs_8bpc); the int32 sum starts at 2^21 and the sample is clamp(sum >> 22, 0, 255).
__device__ __forceinline__ int pil_coeff8(double w) {
  const double s = __dmul_rn(w, 4194304.0);
  return w < 0.0 ? __double2int_rz(__dadd_rn(s, -0.5)) : __double2int_rz(__dadd_rn(s, 0.5));
}

__device__ __forceinline__ uint8_t pil_clip8(int ss) {
  const int v = ss >> 22;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

__global__ void __launch_bounds__(256) pil_resample8_h_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                              long long rows, int W, int OW, const PilAxis ax) {
  const long long total = rows * OW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / OW;
    const int xx = (int)(i - row * OW);
    const int x0 = __ldg(ax.bounds + 2 * xx), cnt = __ldg(ax.bounds + 2 * xx + 1);
    const double* k = ax.k + (size_t)xx * ax.ksize;
    const uint8_t* p = src + row * W + x0;
    int ss = 1 << 21;
    for (int x = 0; x < cnt; ++x) ss += (int)__ldg(p + x) * pil_coeff8(__ldg(k + x));
    dst[i] = pil_clip8(ss);
  }
}

__global__ void __launch_bounds__(256) pil_resample8_v_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int n,
                                                              int H, int OH, int OW, const PilAxis ax) {
  const long long per = (long long)OH * OW, total = per * n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int img = (int)(i / per);
    const int r = (int)(i - (long long)img * per);
    const int yy = r / OW, xx = r - yy * OW;
    const int y0 = __ldg(ax.bounds + 2 * yy), cnt = __ldg(ax.bounds + 2 * yy + 1);
    const double* k = ax.k + (size_t)yy * ax.ksize;
    const uint8_t* p = src + ((size_t)img * H + y0) * OW + xx;
    int ss = 1 << 21;
    for (int y = 0; y < cnt; ++y) ss += (int)__ldg(p + (size_t)y * OW) * pil_coeff8(__ldg(k + y));
    dst[i] = pil_clip8(ss);
  }
}

// out [n, H, W] (batch order) from the resampled crops of the two groups: a mode-'F' sample v becomes fp32 v * fp32(scale)
// (numpy multiplies an fp32 array by a Python float in fp32), a mode-'L' sample fp32(double(u8) * scale).
__global__ void __launch_bounds__(256) crop_place_kernel(const CropJob* __restrict__ jobs, const float* __restrict__ f_src,
                                                         const uint8_t* __restrict__ l_src, float* __restrict__ out, int n,
                                                         int H, int W, double scale) {
  const long long per = (long long)H * W, total = per * n;
  const float fscale = (float)scale;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(idx / per);
    const long long src = (long long)jobs[i].slot * per + (idx - (long long)i * per);
    out[idx] = jobs[i].mode8 ? (float)__dmul_rn((double)__ldg(l_src + src), scale) : __fmul_rn(__ldg(f_src + src), fscale);
  }
}

// ------------------------------------------------------------- self-ensemble (DCSCN.py:547-586) --------------
// The 8 transforms of helper/utilty.py:595-617 (`flip`) as index maps on an [H][W] image:
//   0 identity, 1 flipud, 2 fliplr, 3 flipud(fliplr), 4 rot90(+1), 5 rot90(-1), 6 flipud(rot90(+1)) = transpose,
//   7 flipud(rot90(-1)) = anti-transpose.  Types 4..7 swap the image's height and width.
// src_of(t, i, j) = the source pixel (p, q) of pixel (i, j) of the transformed image.
__device__ __forceinline__ void ensemble_src(int t, int i, int j, int H, int W, int* p, int* q) {
  switch (t) {
    case 0: *p = i; *q = j; break;
    case 1: *p = H - 1 - i; *q = j; break;
    case 2: *p = i; *q = W - 1 - j; break;
    case 3: *p = H - 1 - i; *q = W - 1 - j; break;
    case 4: *p = j; *q = W - 1 - i; break;
    case 5: *p = H - 1 - j; *q = i; break;
    case 6: *p = j; *q = i; break;
    default: *p = H - 1 - j; *q = W - 1 - i; break;
  }
}

// Up to four transforms of one orientation group (all < 4 or all >= 4), the batch of one forward.
struct EnsembleSel {
  int t[4];
  int count;
};

// dst[v][i][j] = src[src_of(sel.t[v], i, j)] for v in [0, count): the transformed copies that feed one batched forward.
// All `count` transforms share one output shape [OH][OW] ([H][W] for t < 4, [W][H] otherwise).
__global__ void __launch_bounds__(256) ensemble_flip_kernel(const float* __restrict__ src, float* __restrict__ dst, int H, int W,
                                                            const EnsembleSel sel) {
  const int OH = sel.t[0] < 4 ? H : W, OW = sel.t[0] < 4 ? W : H;
  const long long per = (long long)OH * OW, total = per * sel.count;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(idx / per);
    const int r = (int)(idx - (long long)v * per);
    const int i = r / OW, j = r - i * OW;
    int p, q;
    ensemble_src(sel.t[v], i, j, H, W, &p, &q);
    dst[idx] = __ldg(src + (long long)p * W + q);
  }
}

// out[p][q] = (sum over the transforms t in `mask` of y_t[inverse position]) / divisor, accumulated in fp64 in the order
// t = 0, 1, ... like the reference's `output += flip(y, i, invert=True)` on a float64 array (DCSCN.py:560-575).
// ya: the selected transforms < 4 in ascending order (shape [H][W] each), yb: the selected transforms >= 4 ([W][H] each);
// H, W = output (HR) size.  divisor = number of flips of the whole ensemble, or 1 for a rank's partial sum.
__global__ void __launch_bounds__(256) ensemble_reduce_kernel(const float* __restrict__ ya, const float* __restrict__ yb,
                                                              double* __restrict__ out, int H, int W, int mask, double divisor) {
  const long long total = (long long)H * W;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int p = (int)(idx / W), q = (int)(idx - (long long)p * W);
    double sum = 0.0;
    int sa = 0, sb = 0;                              // slot of the next selected transform inside ya / yb
    for (int t = 0; t < 8; ++t) {
      if (!((mask >> t) & 1)) continue;
      int i, j;
      switch (t) {                                  // the (i, j) of transform t whose source pixel is (p, q)
        case 0: i = p; j = q; break;
        case 1: i = H - 1 - p; j = q; break;
        case 2: i = p; j = W - 1 - q; break;
        case 3: i = H - 1 - p; j = W - 1 - q; break;
        case 4: i = W - 1 - q; j = p; break;
        case 5: i = q; j = H - 1 - p; break;
        case 6: i = q; j = p; break;
        default: i = W - 1 - q; j = H - 1 - p; break;
      }
      const float v = t < 4 ? __ldg(ya + ((long long)(sa++) * H + i) * W + j) : __ldg(yb + ((long long)(sb++) * W + i) * H + j);
      sum += (double)v;
    }
    out[idx] = sum / divisor;
  }
}

}  // namespace dcscn
