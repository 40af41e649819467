// Filter gradients on the Hopper wgmma tensor cores.
//
// Reference: the `conv2d` backward-filter op TF adds to the graph for every `tf.nn.conv2d` of DCSCN.build_graph when
// `optimizer.compute_gradients(loss)` runs (DCSCN.py:406):  dW[tap][ci][co] = sum_pixels A[p + tap][ci] * dZ[p][co].
//
// GEMM view: M = input channels, N = output channels, K = pixels.  Both operands are read straight from the NHWC
// fp16 planes by the same 4-D tiled TMA boxes the forward kernels use ({64 channels, 16 x 2 pixels}; the A box origin is
// shifted by the filter tap and TMA's out-of-bounds zero fill is TF's SAME padding), which lands them in shared memory
// as rows of 64 channels per pixel: the canonical **MN-major** 128-byte-swizzled wgmma operand (pixels = K run down
// the rows, 8-row groups 1024 bytes apart = SBO, 64-channel groups one box apart = LBO).  No transposes, no copies.
// (A K-major formulation over channel-major copies does not work: a filter tap would be a shift of the innermost TMA
// coordinate by one element, and TMA faults on innermost coordinates that are not 16-byte multiples.)
//
// Precision: the forward scheme, a = a_hi + a_lo and z = z_hi + z_lo in fp16, D += a_lo z_hi + a_hi z_lo + a_hi z_hi
// with fp32 accumulation in registers.  The pixel range is split over CTAs (each writes its partial sum;
// `wgrad_reduce_kernel` adds them in a fixed order and applies the channel-position map and the column window:
// deterministic, no atomics), which also keeps the per-accumulator product count (and with it the tensor core's
// truncation bias, DESIGN.md 4.1) small.
#pragma once
#include "conv_tc.cuh"

namespace dcscn {

constexpr int kWgTW = 16, kWgTH = 2;                 // pixel patch of one K chunk (32 pixels)
constexpr int kWgBoxBytes = kWgTW * kWgTH * 128;     // one TMA box: 32 rows of 64 fp16
constexpr int kWgTcThreads = 384;                    // warpgroup 0: TMA; warpgroups 1, 2: wgmma on input channels 0-63 / 64-127
constexpr int kWgMaxTaps = 2;                        // accumulators per consumer thread: taps x n_groups * 32 <= 128 registers
constexpr int kWgMaxN = 128;                         // column tile cap

struct WgradTcParams {
  int ksz;
  int n_img, tiles_x, tiles_y;   // chunk index -> (img, ty, tx)
  int m_tiles;            // 128-channel tiles of the input
  int n_tiles, n_pad;     // column tiles of dZ, n_pad channels each (multiple of 16, <= kWgMaxN)
  int n_groups;           // 64-channel boxes per dZ tile = ceil(n_pad / 64); the products are n_groups * 64 wide
  int tap_group;          // filter taps per CTA (<= kWgMaxTaps, 1 when n_groups == 2): they share the dZ tile of a chunk
  int ksplit;             // CTAs sharing one (tap group, m_tile, n_tile): contiguous ranges of the chunk index
  int chunks;             // n_img * tiles_y * tiles_x
  float* partial;         // [ksplit][taps][m_tiles * 128][n_tiles * n_pad]
};

__host__ __device__ inline size_t wgrad_tc_stage_bytes(int n_groups, int tap_group) {
  return (size_t)4 * tap_group * kWgBoxBytes + (size_t)2 * n_groups * kWgBoxBytes;
}

// MN-major, 128-byte swizzle: LBO (bits [16,30)) = bytes between 64-channel groups, SBO (bits [32,46)) = bytes
// between 8-pixel groups, layout type SWIZZLE_128B = 1 (bits [62,64)).
__device__ __forceinline__ uint64_t make_desc_mn(uint32_t saddr) {
  const uint32_t lo = ((saddr & 0x3FFFFu) >> 4) | ((uint32_t)(kWgBoxBytes >> 4) << 16);
  constexpr uint32_t hi = (uint32_t)(1024 >> 4) | (1u << 30);
  return ((uint64_t)hi << 32) | (uint64_t)lo;
}

__global__ void __launch_bounds__(kWgTcThreads, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                const __grid_constant__ CUtensorMap tm_z_hi, const __grid_constant__ CUtensorMap tm_z_lo,
                const WgradTcParams p, const int num_stages) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const uint32_t STAGE_BYTES = (uint32_t)wgrad_tc_stage_bytes(p.n_groups, p.tap_group);
  const uint32_t Z_OFF = 4u * (uint32_t)p.tap_group * kWgBoxBytes;
  const uint32_t ZP_BYTES = (uint32_t)p.n_groups * kWgBoxBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)num_stages * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + num_stages;

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const int taps = p.ksz * p.ksz, half = p.ksz >> 1;
  int b = blockIdx.x;
  const int ks = b % p.ksplit; b /= p.ksplit;
  const int nt = b % p.n_tiles; b /= p.n_tiles;
  const int mt = b % p.m_tiles;
  const int tap0 = (b / p.m_tiles) * p.tap_group;                    // this CTA's taps: [tap0, tap0 + ntap)
  const int ntap = (taps - tap0) < p.tap_group ? (taps - tap0) : p.tap_group;
  const int c_begin = (int)((long long)ks * p.chunks / p.ksplit);
  const int c_end = (int)((long long)(ks + 1) * p.chunks / p.ksplit);

  if (threadIdx.x == 0) {
    for (int i = 0; i < num_stages; ++i) {
      ptx::mbar_init(&full_bar[i], 1);
      ptx::mbar_init(&empty_bar[i], 2);     // one arrival per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    ptx::setmaxnreg_dec<kRegsIssue>();
    if (threadIdx.x == 0) {
      ptx::prefetch_tensormap(&tm_a_hi);
      ptx::prefetch_tensormap(&tm_a_lo);
      ptx::prefetch_tensormap(&tm_z_hi);
      ptx::prefetch_tensormap(&tm_z_lo);
      int st = 0;
      uint32_t ph = 0;
      const int per_img = p.tiles_x * p.tiles_y;
      for (int c = c_begin; c < c_end; ++c) {
        const int img = c / per_img, r = c - img * per_img;
        const int y0 = (r / p.tiles_x) * kWgTH, x0 = (r % p.tiles_x) * kWgTW;
        ptx::mbar_wait(&empty_bar[st], ph ^ 1);
        uint8_t* s = smem + (size_t)st * STAGE_BYTES;
        ptx::mbar_arrive_expect_tx(&full_bar[st], (uint32_t)(4 * ntap + 2 * p.n_groups) * kWgBoxBytes);
        for (int j = 0; j < ntap; ++j) {
          const int tap = tap0 + j;
          const int dy = tap / p.ksz - half, dx = tap % p.ksz - half;
          uint8_t* sa = s + (size_t)j * 4 * kWgBoxBytes;
          for (int g = 0; g < 2; ++g) {
            ptx::tma_load_4d(sa + g * kWgBoxBytes, &tm_a_hi, &full_bar[st], mt * 128 + g * 64, x0 + dx, y0 + dy, img);
            ptx::tma_load_4d(sa + (2 + g) * kWgBoxBytes, &tm_a_lo, &full_bar[st], mt * 128 + g * 64, x0 + dx, y0 + dy, img);
          }
        }
        for (int g = 0; g < p.n_groups; ++g) {
          ptx::tma_load_4d(s + Z_OFF + g * kWgBoxBytes, &tm_z_hi, &full_bar[st], nt * p.n_pad + g * 64, x0, y0, img);
          ptx::tma_load_4d(s + Z_OFF + ZP_BYTES + g * kWgBoxBytes, &tm_z_lo, &full_bar[st], nt * p.n_pad + g * 64, x0, y0, img);
        }
        if (++st == num_stages) { st = 0; ph ^= 1; }
      }
    }
  } else {
    ptx::setmaxnreg_inc<kRegsEpilogue>();
    const int cw = wg - 1;                           // input channels [64 cw, 64 cw + 64) of the m tile
    const int n = p.n_groups * 64;                   // product width (columns >= n_pad are computed, never stored)
    const uint32_t smem_base_u32 = ptx::smem_u32(smem);
    float acc[kWgMaxTaps][64];
#pragma unroll
    for (int j = 0; j < kWgMaxTaps; ++j)
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[j][i] = 0.f;
    int st = 0;
    uint32_t ph = 0;
    for (int c = c_begin; c < c_end; ++c) {
      ptx::mbar_wait(&full_bar[st], ph);
      const uint32_t st_addr = smem_base_u32 + (uint32_t)st * STAGE_BYTES;
      const uint32_t z_hi = st_addr + Z_OFF, z_lo = z_hi + ZP_BYTES;
      ptx::wgmma_fence();
#pragma unroll
      for (int j = 0; j < kWgMaxTaps; ++j) {
        if (j >= ntap) break;
        // 16 pixels (rows of 128 bytes) per product; the two small products first, the dominant one last
        const uint32_t a_hi = st_addr + (uint32_t)(j * 4 + cw) * kWgBoxBytes, a_lo = a_hi + 2u * kWgBoxBytes;
        ptx::wgmma_f16_n<1, 1>(n, acc[j], make_desc_mn(a_lo), make_desc_mn(z_hi), 1);
        ptx::wgmma_f16_n<1, 1>(n, acc[j], make_desc_mn(a_hi), make_desc_mn(z_lo), 1);
        ptx::wgmma_f16_n<1, 1>(n, acc[j], make_desc_mn(a_lo + 2048u), make_desc_mn(z_hi + 2048u), 1);
        ptx::wgmma_f16_n<1, 1>(n, acc[j], make_desc_mn(a_hi + 2048u), make_desc_mn(z_lo + 2048u), 1);
        ptx::wgmma_f16_n<1, 1>(n, acc[j], make_desc_mn(a_hi), make_desc_mn(z_hi), 1);
        ptx::wgmma_f16_n<1, 1>(n, acc[j], make_desc_mn(a_hi + 2048u), make_desc_mn(z_hi + 2048u), 1);
      }
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
#pragma unroll
      for (int j = 0; j < kWgMaxTaps; ++j) ptx::reg_fence(acc[j]);
      if ((threadIdx.x & 127) == 0) ptx::mbar_arrive(&empty_bar[st]);
      if (++st == num_stages) { st = 0; ph ^= 1; }
    }
    // accumulator layout: rows 16 warp + lane / 4 (+ 8), column pairs 8 i + 2 (lane % 4)
    const int wq = (threadIdx.x & 127) >> 5;
    const int m = cw * 64 + wq * 16 + (lane >> 2);
    const size_t m_total = (size_t)p.m_tiles * 128, n_total = (size_t)p.n_tiles * p.n_pad;
#pragma unroll
    for (int j = 0; j < kWgMaxTaps; ++j) {
      if (j >= ntap) break;
      float* out = p.partial + (((size_t)ks * taps + tap0 + j) * m_total + (size_t)mt * 128 + m) * n_total + (size_t)nt * p.n_pad;
#pragma unroll
      for (int i = 0; i < kWgMaxN / 8; ++i) {
        const int col = 8 * i + 2 * (lane & 3);
        if (col < p.n_pad) {
          *reinterpret_cast<float2*>(out + col) = make_float2(acc[j][4 * i], acc[j][4 * i + 1]);
          *reinterpret_cast<float2*>(out + 8 * n_total + col) = make_float2(acc[j][4 * i + 2], acc[j][4 * i + 3]);
        }
      }
    }
  }
  __syncthreads();
}

// dW[tap][ci][co] += scale * sum_s partial[s][tap][pos(ci)][col0 + co]
struct WgradReduceParams {
  const float* partial;
  int ksplit, taps, m_total, n_total;
  int cin, cout, col0;
  const int* in_map;      // [cin] row of the A matrix that holds logical input channel ci (nullptr = identity)
  float* dW;
};

__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const WgradReduceParams p) {
  const long long total = (long long)p.taps * p.cin * p.cout;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int co = (int)(i % p.cout);
    const long long r = i / p.cout;
    const int ci = (int)(r % p.cin), tap = (int)(r / p.cin);
    const int row = p.in_map ? __ldg(p.in_map + ci) : ci;
    const float* src = p.partial + ((size_t)tap * p.m_total + row) * p.n_total + p.col0 + co;
    const size_t stride = (size_t)p.taps * p.m_total * p.n_total;
    float s = 0.f;
    for (int k = 0; k < p.ksplit; ++k) s += src[(size_t)k * stride];
    p.dW[i] += s;
  }
}

}  // namespace dcscn
