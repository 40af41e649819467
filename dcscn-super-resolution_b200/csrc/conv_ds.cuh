// Depthwise-separable DCSCN layers (reference: helper/tf_graph.py:155-216 `depthwise_separable_conv2d` /
// `build_depthwise_separable_conv`, i.e. tf.nn.separable_conv2d: depthwise k x k with channel multiplier 1 and no
// bias, then pointwise 1x1, then +bias, then PReLU; used for EVERY layer of a `--depthwise_separable` graph incl. the
// 1x1 A1/B1 (a per-channel scale) and R-CNN1).
//
// These graphs are tiny (c-DCSCN: <= 131 channels, 14,240 MAC per LR pixel at x4) and bound by HBM traffic, not
// math: one fused kernel per layer on CUDA cores, fp32 NHWC activations, no tensor cores (a 131 x 24 contraction per
// pixel does not fill a tensor-core tile).  The depthwise result never leaves registers / shared memory.
#pragma once
#include <cstdint>

namespace dcscn {

struct DsLayerParams {
  int n_img, H, W;          // resolution of this layer (input == output)
  int ksz;                  // depthwise kernel size (1 or 3)
  int cin, cout;
  const float* src;         // [N,H,W,src_pitch] fp32, already offset to the first input channel
  int src_pitch;
  const float* dw;          // [k*k][cin]   depthwise_W  [k,k,cin,1]
  const float* pw;          // [cin][cout]  pointwise_W  [1,1,cin,cout]
  const float* bias;        // [cout] or null
  const float* alpha;       // [cout] or null (no activation)
  // output: plain channel slot, or depth_to_space scatter (DCR), optionally + x2 (final layer)
  float* dst;
  int dst_pitch;            // channels per pixel of dst
  int dst_off;              // first channel written (plain mode)
  int d2s_r;                // 0 = plain; otherwise block size, dst is [N, r*H, r*W, dst_pitch] and cout = r*r*dst_cout
  int d2s_cout;
  const float* add;         // null, or [N,H,W] tensor added to channel 0 (cout must be 1): tf.add(H[-1], x2)
};

constexpr int kDsPix = 64;      // pixels per CTA (consecutive in the flattened N*H*W order; may span rows / images)
constexpr int kDsThreads = 256;

__host__ __device__ inline int ds_cin_pad(int cin) {   // multiple of 4 with an odd number of float4 per row
  int c = (cin + 3) & ~3;                              // -> consecutive pixel rows hit distinct bank groups
  if (((c >> 2) & 1) == 0) c += 4;
  return c;
}
__host__ __device__ inline int ds_cout_pad(int cout) { return (cout + 3) & ~3; }
inline size_t ds_smem_bytes(int ksz, int cin, int cout) {
  return ((size_t)kDsPix * ds_cin_pad(cin) + (size_t)ds_cin_pad(cin) * ds_cout_pad(cout) + (size_t)ksz * ksz * cin) * sizeof(float);
}

// Pointwise contraction + bias + PReLU + store for PXT pixels x 4 output channels per thread (pixels pg + j * PG).
template <int PXT>
__device__ __forceinline__ void ds_pointwise(const DsLayerParams& p, const float* s_d, const float* s_w, const int* s_x,
                                             const int* s_y, int cin_p, int cout_p, long long base, int npix) {
  const int G = cout_p >> 2;
  constexpr int PG = kDsPix / PXT;
  for (int item = threadIdx.x; item < G * PG; item += kDsThreads) {
    const int g = item % G, pg = item / G;
    float acc[PXT][4];
#pragma unroll
    for (int j = 0; j < PXT; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[j][q] = 0.f;
    const float* wcol = s_w + 4 * g;
    for (int c4 = 0; c4 < cin_p; c4 += 4) {
      const float4 w0 = *reinterpret_cast<const float4*>(wcol + (c4 + 0) * cout_p);
      const float4 w1 = *reinterpret_cast<const float4*>(wcol + (c4 + 1) * cout_p);
      const float4 w2 = *reinterpret_cast<const float4*>(wcol + (c4 + 2) * cout_p);
      const float4 w3 = *reinterpret_cast<const float4*>(wcol + (c4 + 3) * cout_p);
#pragma unroll
      for (int j = 0; j < PXT; ++j) {
        const float4 d = *reinterpret_cast<const float4*>(s_d + (pg + PG * j) * cin_p + c4);
        acc[j][0] = fmaf(d.w, w3.x, fmaf(d.z, w2.x, fmaf(d.y, w1.x, fmaf(d.x, w0.x, acc[j][0]))));
        acc[j][1] = fmaf(d.w, w3.y, fmaf(d.z, w2.y, fmaf(d.y, w1.y, fmaf(d.x, w0.y, acc[j][1]))));
        acc[j][2] = fmaf(d.w, w3.z, fmaf(d.z, w2.z, fmaf(d.y, w1.z, fmaf(d.x, w0.z, acc[j][2]))));
        acc[j][3] = fmaf(d.w, w3.w, fmaf(d.z, w2.w, fmaf(d.y, w1.w, fmaf(d.x, w0.w, acc[j][3]))));
      }
    }
#pragma unroll
    for (int j = 0; j < PXT; ++j) {
      const int px = pg + PG * j;
      if (px >= npix) continue;
      const long long gp = base + px;
      const int x = s_x[px], y = s_y[px];
      // first pixel of this image row block in the r-times larger output: (img*H*W) * r*r, then (y*r + i, x*r + j)
      const long long img_px = gp - ((long long)y * p.W + x);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int co = 4 * g + q;
        if (co >= p.cout) continue;
        float v = acc[j][q];
        if (p.bias) v += __ldg(p.bias + co);
        if (p.alpha) v = v > 0.f ? v : __ldg(p.alpha + co) * v;
        if (p.d2s_r == 0) {
          if (p.add) v += __ldg(p.add + gp);
          p.dst[(size_t)gp * p.dst_pitch + p.dst_off + co] = v;
        } else {
          // DCR: input channel (i*r + j)*C + c -> (y*r + i, x*r + j, c)   (tf.depth_to_space, tf_graph.py:248)
          const int r = p.d2s_r, ij = co / p.d2s_cout, c = co - ij * p.d2s_cout;
          const int ii = ij / r, jj = ij - ii * r;
          const size_t o = (size_t)img_px * r * r + (size_t)(y * r + ii) * (p.W * r) + (size_t)(x * r + jj);
          p.dst[o * p.dst_pitch + c] = v;
        }
      }
    }
  }
}

// One CTA: kDsPix consecutive pixels.  Phase 1: depthwise outputs [pix][cin_pad] into shared memory (a warp per
// pixel, lanes over channels: coalesced NHWC reads).  Phase 2: the pointwise contraction as a register-tiled GEMM out
// of shared memory: every thread owns 4 pixels x 4 output channels and reads float4s of the depthwise row and of the
// (staged, zero-padded) pointwise filter: 8 LDS.128 per 64 FMA.
template <int KSZ>
__global__ void __launch_bounds__(kDsThreads) ds_layer_kernel(const DsLayerParams p) {
  extern __shared__ float4 s_raw[];
  constexpr int kk = KSZ * KSZ;
  const int cin_p = ds_cin_pad(p.cin), cout_p = ds_cout_pad(p.cout);
  float* s_d = reinterpret_cast<float*>(s_raw);       // [kDsPix][cin_p]
  float* s_w = s_d + kDsPix * cin_p;                  // [cin_p][cout_p]
  float* s_dw = s_w + cin_p * cout_p;                 // [k*k][cin]
  const long long total = (long long)p.n_img * p.H * p.W;
  const long long base = (long long)blockIdx.x * kDsPix;
  const int npix = (int)((total - base) < kDsPix ? (total - base) : kDsPix);

  __shared__ int s_x[kDsPix], s_y[kDsPix];        // pixel coordinates, computed once (64-bit divisions are expensive)
  if (threadIdx.x < kDsPix) {
    const long long gp = base + threadIdx.x;
    s_x[threadIdx.x] = (int)(gp % p.W);
    s_y[threadIdx.x] = (int)((gp / p.W) % p.H);
  }
  for (int i = threadIdx.x; i < cin_p * cout_p; i += kDsThreads) {
    const int c = i / cout_p, co = i - c * cout_p;
    s_w[i] = (c < p.cin && co < p.cout) ? __ldg(p.pw + (size_t)c * p.cout + co) : 0.f;
  }
  for (int i = threadIdx.x; i < kk * p.cin; i += kDsThreads) s_dw[i] = __ldg(p.dw + i);
  __syncthreads();

  // depthwise.  3x3: a warp walks kDsPix / 8 consecutive pixels with lane = channel and a sliding 3x3 window (three
  // coalesced loads per pixel and channel, filter taps in registers, no per-element index arithmetic).
  // 1x1 (A1 / B1 of a depthwise-separable graph): a per-channel scale, one load per (pixel, channel).
  if (KSZ == 3) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int PPW = kDsPix / (kDsThreads / 32);
    const int px0 = warp * PPW;
    const int px1 = (px0 + PPW) < npix ? (px0 + PPW) : npix;
    const int W = p.W, H = p.H;
    for (int c0 = 0; c0 < p.cin && px0 < npix; c0 += 32) {
      const int c = c0 + lane;
      const bool act = c < p.cin;
      float wd[9];
#pragma unroll
      for (int t = 0; t < 9; ++t) wd[t] = act ? s_dw[t * p.cin + c] : 0.f;
      int x = s_x[px0], y = s_y[px0];
      const float* ctr = p.src + (size_t)(base + px0) * p.src_pitch + c;   // centre pixel, this lane's channel
      float l[3], m[3], r[3];
      auto load_col = [&](int xx, float (&col)[3]) {
#pragma unroll
        for (int rr = 0; rr < 3; ++rr) {
          const int yy = y + rr - 1;
          col[rr] = (act && yy >= 0 && yy < H && xx >= 0 && xx < W) ? __ldg(ctr + ((long long)(rr - 1) * W + (xx - x)) * p.src_pitch) : 0.f;
        }
      };
      load_col(x - 1, l);
      load_col(x, m);
      for (int px = px0; px < px1; ++px) {
        load_col(x + 1, r);
        float acc = 0.f;
#pragma unroll
        for (int rr = 0; rr < 3; ++rr)
          acc = fmaf(l[rr], wd[3 * rr], fmaf(m[rr], wd[3 * rr + 1], fmaf(r[rr], wd[3 * rr + 2], acc)));
        if (act) s_d[px * cin_p + c] = acc;
        ctr += p.src_pitch;
        if (++x == W) {                              // next image row (or image): rebuild the window
          x = 0;
          if (++y == H) y = 0;
          if (px + 1 < px1) {
#pragma unroll
            for (int rr = 0; rr < 3; ++rr) l[rr] = 0.f;
            load_col(0, m);
          }
        } else {
#pragma unroll
          for (int rr = 0; rr < 3; ++rr) {
            l[rr] = m[rr];
            m[rr] = r[rr];
          }
        }
      }
    }
    // zero padding: channels [cin, cin_p) of every row and the rows past the last pixel
    const int padc = cin_p - p.cin;
    for (int i = threadIdx.x; i < kDsPix * padc; i += kDsThreads) s_d[(i / padc) * cin_p + p.cin + i % padc] = 0.f;
    for (int i = threadIdx.x + npix * cin_p; i < kDsPix * cin_p; i += kDsThreads) s_d[i] = 0.f;
  } else {
    for (int i = threadIdx.x; i < kDsPix * cin_p; i += kDsThreads) {
      const int px = i / cin_p, c = i - px * cin_p;
      float v = 0.f;
      if (px < npix && c < p.cin) v = __ldg(p.src + (size_t)(base + px) * p.src_pitch + c) * s_dw[c];
      s_d[i] = v;
    }
  }
  __syncthreads();

  const int G = cout_p >> 2;               // float4 groups of output channels
  if (G * (kDsPix / 4) >= kDsThreads) ds_pointwise<4>(p, s_d, s_w, s_x, s_y, cin_p, cout_p, base, npix);
  else ds_pointwise<1>(p, s_d, s_w, s_x, s_y, cin_p, cout_p, base, npix);
}

// cin == cout == 1 (R-CNN1 of a depthwise-separable graph at HR resolution): one thread per pixel.
template <int KSZ>
__global__ void __launch_bounds__(256) ds_single_kernel(const DsLayerParams p) {
  constexpr int kk = KSZ * KSZ, half = KSZ >> 1;
  const long long total = (long long)p.n_img * p.H * p.W;
  float w[kk];
#pragma unroll
  for (int t = 0; t < kk; ++t) w[t] = __ldg(p.dw + t) * __ldg(p.pw);
  const float bias = p.bias ? __ldg(p.bias) : 0.f;
  for (long long gp = (long long)blockIdx.x * blockDim.x + threadIdx.x; gp < total; gp += (long long)gridDim.x * blockDim.x) {
    const unsigned g32 = (unsigned)gp;                     // total < 2^32 pixels (checked by the launcher)
    const unsigned row = g32 / (unsigned)p.W;
    const int x = (int)(g32 - row * (unsigned)p.W);
    const int y = (int)(row % (unsigned)p.H);
    const float* ctr = p.src + (size_t)gp * p.src_pitch;
    float acc = bias;
#pragma unroll
    for (int t = 0; t < kk; ++t) {
      const int dy = t / KSZ - half, dx = t % KSZ - half;
      if ((unsigned)(y + dy) < (unsigned)p.H && (unsigned)(x + dx) < (unsigned)p.W)
        acc = fmaf(__ldg(ctr + ((long long)dy * p.W + dx) * p.src_pitch), w[t], acc);
    }
    if (p.alpha) acc = acc > 0.f ? acc : __ldg(p.alpha) * acc;
    if (p.add) acc += __ldg(p.add + gp);
    p.dst[(size_t)gp * p.dst_pitch + p.dst_off] = acc;
  }
}

}  // namespace dcscn
