// Train-step kernels for depthwise-separable graphs (reference: helper/tf_graph.py:155-216 - every layer is
// tf.nn.separable_conv2d: depthwise k x k with multiplier 1, pointwise 1 x 1, + bias, PReLU, dropout - under the loss /
// gradient ops of DCSCN.py:334-413).  fp32 on CUDA cores: a depthwise-separable c-DCSCN has 14 kMAC per LR pixel and at
// most 131 x 32 pointwise filters; the step is bound by memory traffic and launch count, not by arithmetic.
//
// One layer, forward:   u = depthwise(x, dw);  z = u . pw + b;  h = f(z);  out = dropout(h)
//            backward:  g = d out;  dh = g * mask / keep;  dz = dh * f'(z);  d b += dz;  with PReLU f'(z) = z > 0 ? 1 : alpha
//                       and d alpha += dh * min(z, 0); the other activators take f' at z = 0 as TensorFlow's gradient ops
//                       do (act_grad_kernel, train.cuh)
//                       d pw[c][co] = sum_px u[px][c] dz[px][co];   du[px][c] = sum_co dz[px][co] pw[c][co]
//                       d dw[t][c] = sum_px x[px + t][c] du[px][c];  dx[px][c] (+)= sum_t du[px - t][c] dw[t][c]
// u is recomputed in the backward pass (one cheap kernel) instead of being kept; z (the pre-activation) is kept per layer.
#pragma once
#include "epilogue.cuh"

namespace dcscn {

// ------------------------------------------------------------------------------------- forward ----
struct DsDwParams {
  int n, H, W, C, ksz;
  const float* src;      // NHWC, element (px, c) at src[px * src_pitch + src_off + c]
  int src_pitch, src_off;
  const float* dw;       // [k*k][C]
  float* u;              // [px][C]
};

__global__ void __launch_bounds__(256) ds_dw_fwd_kernel(const DsDwParams p) {
  const long long total = (long long)p.n * p.H * p.W * p.C;
  const int half = p.ksz >> 1, taps = p.ksz * p.ksz;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % p.C);
    const long long px = i / p.C;
    const int x = (int)(px % p.W), y = (int)((px / p.W) % p.H);
    float acc = 0.f;
    for (int t = 0; t < taps; ++t) {
      const int dy = t / p.ksz - half, dx = t % p.ksz - half;
      if ((unsigned)(y + dy) < (unsigned)p.H && (unsigned)(x + dx) < (unsigned)p.W)
        acc = fmaf(__ldg(p.src + (px + (long long)dy * p.W + dx) * p.src_pitch + p.src_off + c), __ldg(p.dw + t * p.C + c), acc);
    }
    p.u[i] = acc;
  }
}

struct DsPwParams {
  long long npx;
  int H, W;              // resolution of this layer's input (for the depth_to_space scatter)
  int cin, cout;
  const float* u;        // [px][cin]
  const float* pw;       // [cin][cout]
  const float* bias;     // [cout] or null
  const float* alpha;    // [cout] PReLU slope, or null
  float* z;              // [px][cout] pre-activation, kept for the backward pass
  float* dst;            // layer output: (px, co) at dst[px * dst_pitch + dst_off + co], or depth_to_space scattered
  int dst_pitch, dst_off;
  int d2s_r, d2s_C;      // DCR: column (i*r + j)*C + c -> pixel (y*r + i, x*r + j), channel c
  const float* add;      // + x2 (cout == 1), or null
  float keep;            // dropout keep probability (only applied to activated layers, tf_graph.py:129-130)
  uint32_t seed, layer;
  int act;               // Activation; ACT_NONE = linear layer
};

__global__ void __launch_bounds__(256) ds_pw_fwd_kernel(const DsPwParams p) {
  const long long total = p.npx * p.cout;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(i % p.cout);
    const long long px = i / p.cout;
    float acc = p.bias ? __ldg(p.bias + co) : 0.f;
    const float* ur = p.u + px * p.cin;
    for (int c = 0; c < p.cin; ++c) acc = fmaf(__ldg(ur + c), __ldg(p.pw + (size_t)c * p.cout + co), acc);
    p.z[i] = acc;
    float hv = acc;
    if (p.act != ACT_NONE) {
      hv = act_apply(p.act, acc, p.alpha ? __ldg(p.alpha + co) : (p.act == ACT_LEAKY_RELU ? kLeakySlope : 0.f));
      if (p.keep < 1.0f) hv = dropout_keep(p.seed, p.layer, (uint64_t)i, p.keep) ? hv * (1.0f / p.keep) : 0.f;
    }
    if (p.d2s_r == 0) {
      if (p.add) hv += __ldg(p.add + px);
      p.dst[px * p.dst_pitch + p.dst_off + co] = hv;
    } else {
      const int r = p.d2s_r, C = p.d2s_C;
      const int x = (int)(px % p.W), y = (int)((px / p.W) % p.H);
      const long long img = px / ((long long)p.W * p.H);
      const int ij = co / C, c = co - ij * C, ii = ij / r, jj = ij - ii * r;
      const long long hp = (img * p.H * r + (long long)(y * r + ii)) * ((long long)p.W * r) + (x * r + jj);
      p.dst[hp * p.dst_pitch + p.dst_off + c] = hv;
    }
  }
}

// ------------------------------------------------------------------------------------ backward ----
struct DsActBwdParams {
  long long npx;
  int H, W, cout;
  const float* gout;     // gradient w.r.t. the layer output: same addressing as the forward store (incl. depth_to_space)
  int g_pitch, g_off;
  int d2s_r, d2s_C;
  const float* z;        // [px][cout]
  const float* alpha;    // PReLU slope, or null
  float keep;
  uint32_t seed, layer;
  float* dz;             // [px][cout]
  float* e;              // [px][cout]: dh * min(z, 0) (column sums = d alpha); only written for PReLU
  int act;               // Activation; ACT_NONE = linear layer
};

__global__ void __launch_bounds__(256) ds_act_bwd_kernel(const DsActBwdParams p) {
  const long long total = p.npx * p.cout;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(i % p.cout);
    const long long px = i / p.cout;
    float g;
    if (p.d2s_r == 0) {
      g = __ldg(p.gout + px * p.g_pitch + p.g_off + co);
    } else {
      const int r = p.d2s_r, C = p.d2s_C;
      const int x = (int)(px % p.W), y = (int)((px / p.W) % p.H);
      const long long img = px / ((long long)p.W * p.H);
      const int ij = co / C, c = co - ij * C, ii = ij / r, jj = ij - ii * r;
      const long long hp = (img * p.H * r + (long long)(y * r + ii)) * ((long long)p.W * r) + (x * r + jj);
      g = __ldg(p.gout + hp * p.g_pitch + p.g_off + c);
    }
    if (p.act != ACT_NONE) {
      if (p.keep < 1.0f) g = dropout_keep(p.seed, p.layer, (uint64_t)i, p.keep) ? g * (1.0f / p.keep) : 0.f;
      const float zz = p.z[i];
      if (p.act == ACT_PRELU) {
        p.e[i] = g * fminf(zz, 0.f);
        g = zz > 0.f ? g : __ldg(p.alpha + co) * g;
      } else if (p.act == ACT_LEAKY_RELU) {
        g = zz < 0.f ? kLeakySlope * g : g;        // Maximum's gradient: z >= 0.1 z takes the z branch, slope 1 at z = 0
      } else {
        g *= act_deriv_from_output(p.act, act_apply(p.act, zz, 0.f));
      }
    }
    p.dz[i] = g;
  }
}

// out[c] += sum over pixels of src[px][c]   (block partials, one atomicAdd per block and column).  blockIdx.y takes the
// columns [256 y, 256 y + G) with G = min(256, C - 256 y): grid.y = ceil(C / 256).
__global__ void __launch_bounds__(256) ds_colsum_kernel(const float* __restrict__ src, long long npx, int C, float* out,
                                                        int px_per_block) {
  __shared__ float s[256];
  const int c0 = blockIdx.y * 256, G = C - c0 < 256 ? C - c0 : 256;
  const int rows = 256 / G;                      // pixel rows handled in parallel by one block
  const int c = threadIdx.x % G, rg = threadIdx.x / G;
  const long long px0 = (long long)blockIdx.x * px_per_block;
  const long long px1 = px0 + px_per_block < npx ? px0 + px_per_block : npx;
  float acc = 0.f;
  if (rg < rows)
    for (long long px = px0 + rg; px < px1; px += rows) acc += src[px * C + c0 + c];
  s[threadIdx.x] = (rg < rows) ? acc : 0.f;
  __syncthreads();
  if (threadIdx.x < G) {
    float t = 0.f;
    for (int r = 0; r < rows; ++r) t += s[r * G + threadIdx.x];
    atomicAdd(out + c0 + threadIdx.x, t);
  }
}

// d pw[c][co] += sum_px u[px][c] * dz[px][co].  Each (c, co) pair is one fp32 FMA chain over the block's pixels in
// order, however the pixels are staged.  blockIdx.z takes the columns [co0, co0 + G), co0 = kDsDpwCols z, G = min(kDsDpwCols,
// cout - co0); blockIdx.y a tile of kDsDpwPairs x 256 of its cin x G pairs.  A pass stages `chunk` pixels of u and of
// those columns of dz: chunk (cin + G) floats of dynamic shared memory (ds_dpw_chunk).
struct DsDpwParams {
  long long npx;
  int cin, cout;
  const float* u;
  const float* dz;
  float* dpw;
  int px_per_block;
  int chunk;
};
constexpr int kDsDpwPairs = 17;                        // (c, co) pairs per thread: 17 x 256 = 4352 pairs per blockIdx.y
constexpr int kDsDpwChunk = 32;                        // most pixels staged per pass
constexpr int kDsDpwCols = 256;                        // most dz columns per blockIdx.z
constexpr int kDsDpwSmemFloats = 48 * 1024 / 4;        // the dynamic shared memory a launch may take without opting in

// Pixels per pass of ds_dpw_kernel for a layer: up to kDsDpwChunk, as many as fit the default 48 KB; 0 = none fits.
inline int ds_dpw_chunk(int cin, int cout) {
  const int w = cin + (cout < kDsDpwCols ? cout : kDsDpwCols);
  return kDsDpwSmemFloats / w < kDsDpwChunk ? kDsDpwSmemFloats / w : kDsDpwChunk;
}

__global__ void __launch_bounds__(256) ds_dpw_kernel(const DsDpwParams p) {
  extern __shared__ float ds_smem[];
  const int co0 = blockIdx.z * kDsDpwCols, G = p.cout - co0 < kDsDpwCols ? p.cout - co0 : kDsDpwCols;
  float* su = ds_smem;                                 // [chunk][cin]
  float* sz = ds_smem + p.chunk * p.cin;               // [chunk][G]
  const int pairs = p.cin * G;
  const int e0 = blockIdx.y * (kDsDpwPairs * 256) + threadIdx.x;
  float acc[kDsDpwPairs];
#pragma unroll
  for (int k = 0; k < kDsDpwPairs; ++k) acc[k] = 0.f;
  const long long px0 = (long long)blockIdx.x * p.px_per_block;
  const long long px1 = px0 + p.px_per_block < p.npx ? px0 + p.px_per_block : p.npx;
  for (long long base = px0; base < px1; base += p.chunk) {
    const int P = (int)((px1 - base) < p.chunk ? (px1 - base) : p.chunk);
    __syncthreads();
    for (int i = threadIdx.x; i < P * p.cin; i += 256) su[i] = p.u[base * p.cin + i];
    for (int i = threadIdx.x; i < P * G; i += 256) {
      const int q = i / G;
      sz[i] = p.dz[(base + q) * p.cout + co0 + (i - q * G)];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kDsDpwPairs; ++k) {
      const int e = e0 + k * 256;
      if (e < pairs) {
        const int c = e / G, co = e - c * G;
        float a = acc[k];
        for (int q = 0; q < P; ++q) a = fmaf(su[q * p.cin + c], sz[q * G + co], a);
        acc[k] = a;
      }
    }
  }
#pragma unroll
  for (int k = 0; k < kDsDpwPairs; ++k) {
    const int e = e0 + k * 256;
    if (e < pairs) {
      const int c = e / G;
      atomicAdd(p.dpw + (size_t)c * p.cout + co0 + (e - c * G), acc[k]);
    }
  }
}

// du[px][c] = sum_co dz[px][co] * pw[c][co]
__global__ void __launch_bounds__(256) ds_du_kernel(const float* __restrict__ dz, const float* __restrict__ pw, float* du,
                                                    long long npx, int cin, int cout) {
  const long long total = npx * cin;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cin);
    const long long px = i / cin;
    const float* zr = dz + px * cout;
    const float* wr = pw + (size_t)c * cout;
    float acc = 0.f;
    for (int co = 0; co < cout; ++co) acc = fmaf(__ldg(zr + co), __ldg(wr + co), acc);
    du[i] = acc;
  }
}

// d dw[t][c] += sum_px x[px + t][c] * du[px][c].  A block covers `cpb` channels (power of two <= 256) x 256 / cpb pixel lanes.
struct DsDdwParams {
  int n, H, W, C, ksz;
  const float* src;
  int src_pitch, src_off;
  const float* du;       // [px][C]
  float* ddw;            // [k*k][C]
  int cpb;
  int px_per_block;
};

__global__ void __launch_bounds__(256) ds_ddw_kernel(const DsDdwParams p) {
  __shared__ float s[256 * 9];
  const int cl = threadIdx.x % p.cpb, pl = threadIdx.x / p.cpb, lanes = 256 / p.cpb;
  const int c = blockIdx.y * p.cpb + cl;
  const int half = p.ksz >> 1, taps = p.ksz * p.ksz;
  const long long npx = (long long)p.n * p.H * p.W;
  const long long px0 = (long long)blockIdx.x * p.px_per_block;
  const long long px1 = px0 + p.px_per_block < npx ? px0 + p.px_per_block : npx;
  float acc[9];
#pragma unroll
  for (int t = 0; t < 9; ++t) acc[t] = 0.f;
  if (c < p.C) {
    for (long long px = px0 + pl; px < px1; px += lanes) {
      const int x = (int)(px % p.W), y = (int)((px / p.W) % p.H);
      const float g = __ldg(p.du + px * p.C + c);
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        if (t < taps) {
          const int dy = t / p.ksz - half, dx = t % p.ksz - half;
          if ((unsigned)(y + dy) < (unsigned)p.H && (unsigned)(x + dx) < (unsigned)p.W)
            acc[t] = fmaf(__ldg(p.src + (px + (long long)dy * p.W + dx) * p.src_pitch + p.src_off + c), g, acc[t]);
        }
      }
    }
  }
#pragma unroll
  for (int t = 0; t < 9; ++t) s[t * 256 + threadIdx.x] = acc[t];
  __syncthreads();
  if (pl == 0 && c < p.C) {
    for (int t = 0; t < taps; ++t) {
      float v = 0.f;
      for (int l = 0; l < lanes; ++l) v += s[t * 256 + l * p.cpb + cl];
      atomicAdd(p.ddw + t * p.C + c, v);
    }
  }
}

// dx[px][c] (+)= sum_t du[px - t][c] * dw[t][c]
struct DsDxParams {
  int n, H, W, C, ksz;
  const float* du;       // [px][C]
  const float* dw;       // [k*k][C]
  float* dst;
  int dst_pitch, dst_off;
  int accumulate;
};

__global__ void __launch_bounds__(256) ds_dx_kernel(const DsDxParams p) {
  const long long total = (long long)p.n * p.H * p.W * p.C;
  const int half = p.ksz >> 1, taps = p.ksz * p.ksz;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % p.C);
    const long long px = i / p.C;
    const int x = (int)(px % p.W), y = (int)((px / p.W) % p.H);
    float acc = 0.f;
    for (int t = 0; t < taps; ++t) {
      const int dy = t / p.ksz - half, dx = t % p.ksz - half;      // u[y - dy][x - dx] saw x[y][x] through tap t
      if ((unsigned)(y - dy) < (unsigned)p.H && (unsigned)(x - dx) < (unsigned)p.W)
        acc = fmaf(__ldg(p.du + (px - (long long)dy * p.W - dx) * p.C + c), __ldg(p.dw + t * p.C + c), acc);
    }
    float* d = p.dst + px * p.dst_pitch + p.dst_off + c;
    *d = p.accumulate ? *d + acc : acc;
  }
}

}  // namespace dcscn
