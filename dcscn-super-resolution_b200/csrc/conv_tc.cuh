// Implicit-GEMM convolution on Hopper wgmma tensor cores (sm_90a).
//
// Replaces  tf.nn.conv2d(SAME, stride 1, NHWC, HWIO) + bias + PReLU  of the reference
// (helper/tf_graph.py:104-153 conv2d / build_conv; :238-249 build_pixel_shuffler_layer).
//
// GEMM view:  D[M = 128 pixels (TH x TW patch), N = cout (padded to 16, <= 112 per column tile)]
//             = sum over 64-channel input chunks, taps (kx, ky) of  A_tap[128 x 64] * W_tap[64 x N]
//   * A tiles are fetched by TMA (4-D tiled tensor map over the NHWC fp16 plane).  A k x k layer (k = 3 or 5) loads ONE
//     box of TW x (TH + k - 1) pixels per (chunk, kx), its origin shifted by (kx - k / 2, -k / 2); the k ky taps read it
//     at row offsets 0, TW, ..., (k - 1) TW.  The host only picks patches with TW a multiple of 8, so every offset is a
//     whole number of 8-row swizzle atoms and the operand descriptors stay valid.  TMA zero-fills out-of-image pixels, which IS TF's SAME padding - no halo handling in
//     the kernel.  A 1x1 layer loads one TW x TH box per chunk.
//   * fp32-equivalent precision from fp16 tensor cores:  a = a_hi + a_lo,  w*2^s = w_hi + w_lo
//     (each 11-bit significands), D += a_hi*w_hi + a_lo*w_hi + a_hi*w_lo   (3 x m64nNk16 wgmma per 16 channels,
//     fp32 accumulation in registers).  NPLANES == 1 is the single-pass fp16 "fast" mode.
//   * The tensor core's fp32 accumulator update truncates (round-toward-zero), a bias that grows linearly with the
//     number of accumulation steps.  K is therefore cut into short segments (`seg_chunks` weight tiles): each segment
//     accumulates the two correction products in `corr` and the dominant a_hi*w_hi product in `dom`, both from zero,
//     and at its end both are added into the running fp32 `sum` with round-to-nearest ("promotion").  Only `dom`
//     grows large, so only the dominant chain contributes truncation error.  `seg_chunks` == 1 (the strict setting)
//     promotes after every 16-channel K slice.  The three register sets take 3 N / 2 floats per thread, which is what
//     caps a column tile at 112 (kMaxTileN).
//   * The column-tile width N is a template parameter: the wgmma width is an immediate of the instruction, and a
//     straight-line run of same-width wgmma needs no per-instruction selection.
//   * Two shared-memory rings with their own full/empty mbarriers: activation slots (one per (chunk, kx)) and weight
//     tiles (one per (tap, chunk), read from the packed image [n_tile][tap][chunk]).  The consumers commit one wgmma
//     group per weight tile and release a slot as soon as `wgmma.wait_group 1` shows the group that last read it
//     has completed, so both rings work purely as prefetch depth.  A weight tile arrives as one bulk copy.
//   * Warp roles: warpgroup 0 = producer (warp 0 issues TMA), warpgroups 1 and 2 = consumers, one per 64-pixel half
//     of the tile: they issue the wgmma of their rows, promote, and run the epilogue (bias/PReLU/split -> global) after
//     an exchange through shared memory that gives every thread one pixel and a run of 16-column chunks.  Persistent
//     CTAs (one per SM) stride over (pixel-tile, column-tile) work items.
#pragma once
#include "common.h"
#include "epilogue.cuh"
#include "ptx.cuh"

namespace dcscn {

constexpr int kConsumerWGs = 2;                    // one per 64-pixel half of the 128-pixel tile
constexpr int kTcThreads = (1 + kConsumerWGs) * 128;
constexpr int kRegsIssue = 40, kRegsEpilogue = 232;  // setmaxnreg budgets (128*40 + 256*232 <= 64K)
constexpr int kMaxASlots = 4;                      // activation ring slots
constexpr int kMaxWSlots = 12;                     // weight ring slots
constexpr int kTcBarrierBytes = 2 * (kMaxASlots + kMaxWSlots) * 8;
constexpr int kMaxTileN = 112;                     // column tile cap: corr + dom + promoted sum = 3 N / 2 registers;
                                                   // at N = 128 (192 of them) ptxas spills inside the K loop
constexpr int kRdotSmemBytes = 9 * 128 * 4;         // fused R-CNN1 filter taps (d2s_cout <= 128) staged in shared memory
constexpr int kColSplit = 2;                       // epilogue threads per pixel, each owning a contiguous run of chunks
constexpr int kXchgStride = 36;                    // floats per pixel row of the epilogue exchange buffer (2 chunks + pad)
constexpr int kXchgBytes = kConsumerWGs * 64 * kXchgStride * 4;
constexpr int kTcKC = 64;                          // input channels per K chunk: an fp16 operand row is 128 bytes,
                                                   // one row of the SWIZZLE_128B layout

struct TcSmem {
  static constexpr int kRowBytes = kTcKC * 2;               // 128 (SWIZZLE_128B)
  static constexpr int kSbo = 8 * kRowBytes;                // 8-row core-matrix group stride
  static constexpr uint64_t kLayout = 1ull;                 // wgmma descriptor layout type: SW128 = 1
};

// wgmma shared-memory matrix descriptor of a K-major swizzled operand tile: start address >> 4 in [0,14), leading
// byte offset (unused for swizzled K-major, 1) in [16,30), stride byte offset >> 4 in [32,46), layout type in [62,64).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(TcSmem::kSbo >> 4) << 32) |
         (TcSmem::kLayout << 62);
}

// Bytes of one activation plane in a ring slot: the TMA box of TW x (TH + ksz - 1) pixels, rounded up to 1024 bytes
// so that every slot and plane starts on a swizzle-atom boundary.
__host__ __device__ inline uint32_t tc_a_plane_bytes(int TW, int TH, int ksz) {
  return ((uint32_t)TW * (uint32_t)(TH + ksz - 1) * (uint32_t)kTcKC * 2u + 1023u) & ~1023u;
}
__host__ __device__ inline uint32_t tc_w_tile_bytes(int nplanes, int n_pad) {
  return (uint32_t)nplanes * (uint32_t)n_pad * (uint32_t)kTcKC * 2u;
}

// One wgmma batch: the products of KS consecutive 16-channel K slices of a weight tile, committed as one group.
// corr += a_lo*w_hi + a_hi*w_lo, dom += a_hi*w_hi; acc_on == 0 starts both from zero.
template <int N, int NPLANES, int KS>
__device__ __forceinline__ void tile_products(float (&corr)[N / 2], float (&dom)[N / 2], uint64_t a_hi, uint64_t a_lo,
                                              uint64_t b_hi, uint64_t b_lo, uint32_t acc_on) {
  ptx::wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) {
    const uint64_t kadd = (uint64_t)ks * 2u;   // 32 bytes (16 fp16 along K) in 16-byte descriptor units
    const uint32_t on = ks == 0 ? acc_on : 1u;
    if (NPLANES == 2) {
      ptx::wgmma_f16<N, 0, 0>(corr, a_lo + kadd, b_hi + kadd, on);
      ptx::wgmma_f16<N, 0, 0>(corr, a_hi + kadd, b_lo + kadd, 1u);
    }
    ptx::wgmma_f16<N, 0, 0>(dom, a_hi + kadd, b_hi + kadd, on);
  }
  ptx::wgmma_commit();
}

template <int NPLANES, int N>
__global__ void __launch_bounds__(kTcThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo,
               const ConvTCParams p, const int a_slots, const int w_slots) {
  static_assert(N % 16 == 0 && N >= 16 && N <= kMaxTileN, "column tile width");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [a_slots x (A_hi, A_lo)] [w_slots x (W_hi, W_lo)] then barriers, R-CNN1 taps, epilogue exchange
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const ConvGeom& g = p.g;
  const int ksz = p.ksz;
  const uint32_t A_PLANE = tc_a_plane_bytes(g.TW, g.TH, ksz);
  const uint32_t A_SLOT = NPLANES * A_PLANE;
  const uint32_t A_TX = (uint32_t)NPLANES * (uint32_t)g.TW * (uint32_t)(g.TH + ksz - 1) * kTcKC * 2u;  // bytes TMA delivers
  constexpr uint32_t B_BYTES = N * kTcKC * 2;
  constexpr uint32_t W_TILE = NPLANES * B_BYTES;
  uint8_t* a_ring = smem;
  uint8_t* w_ring = smem + (size_t)a_slots * A_SLOT;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(w_ring + (size_t)w_slots * W_TILE);
  uint64_t* a_empty = a_full + kMaxASlots;
  uint64_t* w_full = a_empty + kMaxASlots;
  uint64_t* w_empty = w_full + kMaxWSlots;
  float* s_rdot = reinterpret_cast<float*>(w_empty + kMaxWSlots);   // 16-byte aligned (barriers start 1024-aligned)
  float* s_xchg = s_rdot + kRdotSmemBytes / 4;

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < a_slots; ++s) {
      ptx::mbar_init(&a_full[s], 1);
      ptx::mbar_init(&a_empty[s], kConsumerWGs);   // one arrival per consumer warpgroup
    }
    for (int s = 0; s < w_slots; ++s) {
      ptx::mbar_init(&w_full[s], 1);
      ptx::mbar_init(&w_empty[s], kConsumerWGs);
    }
    ptx::fence_barrier_init();
    ptx::fence_proxy_async();
  }
  if (p.epi.mode == EPI_D2S_RDOT)
    for (int i = threadIdx.x; i < p.epi.rdot_taps * p.epi.d2s_cout; i += blockDim.x) s_rdot[i] = p.epi.rdot_w[i];
  __syncthreads();

  const int tiles_per_img = g.tiles_x * g.tiles_y;
  const int num_items = g.n_img * tiles_per_img * p.n_tiles;
  const int half = ksz >> 1;
  const int chunks = p.chunks;

  if (wg == 0) {
    ptx::setmaxnreg_dec<kRegsIssue>();
    // ============================== TMA producer ==============================
    if (threadIdx.x == 0) {
      ptx::prefetch_tensormap(&tm_hi);
      if (NPLANES == 2) ptx::prefetch_tensormap(&tm_lo);
      int as = 0, ws = 0;
      uint32_t a_ph = 0, w_ph = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        const int n_tile = item % p.n_tiles;
        const int tile = item / p.n_tiles;
        const int img = tile / tiles_per_img;
        const int t2 = tile - img * tiles_per_img;
        const int ty = t2 / g.tiles_x, tx = t2 - ty * g.tiles_x;
        const int x0 = tx * g.TW - half, y0 = ty * g.TH - half;
        const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(p.wpack) + (size_t)n_tile * ksz * ksz * chunks * W_TILE;
        for (int ch = 0; ch < chunks; ++ch) {
          for (int dx = 0; dx < ksz; ++dx) {
            ptx::mbar_wait(&a_empty[as], a_ph ^ 1);
            uint8_t* ad = a_ring + (size_t)as * A_SLOT;
            ptx::mbar_arrive_expect_tx(&a_full[as], A_TX);
            ptx::tma_load_4d(ad, &tm_hi, &a_full[as], ch * kTcKC, x0 + dx, y0, img);
            if (NPLANES == 2) ptx::tma_load_4d(ad + A_PLANE, &tm_lo, &a_full[as], ch * kTcKC, x0 + dx, y0, img);
            if (++as == a_slots) { as = 0; a_ph ^= 1; }
            for (int dy = 0; dy < ksz; ++dy) {
              ptx::mbar_wait(&w_empty[ws], w_ph ^ 1);
              uint8_t* wd = w_ring + (size_t)ws * W_TILE;
              ptx::mbar_arrive_expect_tx(&w_full[ws], W_TILE);
              const uint8_t* wtile = wsrc + (size_t)((dy * ksz + dx) * chunks + ch) * W_TILE;
              ptx::bulk_load(wd, wtile, W_TILE, &w_full[ws]);
              if (++ws == w_slots) { ws = 0; w_ph ^= 1; }
            }
          }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<kRegsEpilogue>();
    // ============================== consumers ==================================
    const int cw = wg - 1;                   // which 64-pixel half of the tile
    const int t = threadIdx.x & 127;
    const int wq = t >> 5;                   // warp inside the warpgroup: accumulator rows 16 wq .. 16 wq + 15
    constexpr int nch = N >> 4;
    constexpr int per = (nch + kColSplit - 1) / kColSplit;
    const int n_total = p.n_tiles * N;
    const bool strict = p.seg_chunks == 1;
    const uint32_t a_ring_u32 = ptx::smem_u32(a_ring);
    const uint32_t w_ring_u32 = ptx::smem_u32(w_ring);
    const uint32_t a_off = (uint32_t)(cw * 64 * TcSmem::kRowBytes);
    const uint32_t dy_step = (uint32_t)(g.TW * TcSmem::kRowBytes);   // one image row of the box: whole 8-row atoms
    // epilogue ownership after the exchange: pixel `row`, chunks [grp * per, grp * per + my_chunks)
    const int row = cw * 64 + (t >> 1);
    const int grp = t & 1;
    const int py = row / g.TW, px = row - py * g.TW;
    const int first_chunk = grp * per;
    const int my_chunks = (nch - first_chunk) < per ? ((nch - first_chunk) > 0 ? nch - first_chunk : 0) : per;
    float* xchg = s_xchg + cw * 64 * kXchgStride;
    // a slot is released once the wgmma group that last read it has completed (one arrival per warpgroup, by thread 0)
    auto release_a = [&](int s) { ptx::mbar_arrive_if(&a_empty[s], t == 0); };
    auto release_w = [&](int s) { ptx::mbar_arrive_if(&w_empty[s], t == 0); };
    int as = 0, ws = 0;
    uint32_t a_ph = 0, w_ph = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
      const int n_tile = item % p.n_tiles;
      const int tile = item / p.n_tiles;
      const int img = tile / tiles_per_img;
      const int t2 = tile - img * tiles_per_img;
      const int ty = t2 / g.tiles_x, tx = t2 - ty * g.tiles_x;
      const int y = ty * g.TH + py, x = tx * g.TW + px;
      const bool valid = (y < g.H) && (x < g.W);

      float sum[N / 2], corr[N / 2], dom[N / 2];
#pragma unroll
      for (int i = 0; i < N / 2; ++i) sum[i] = 0.f;
      auto promote = [&]() {   // fp32 round-to-nearest: the small corrections first, then the dominant chain
        ptx::reg_fence(corr);
        ptx::reg_fence(dom);
#pragma unroll
        for (int i = 0; i < N / 2; ++i) {
          if (NPLANES == 2) sum[i] += corr[i];
          sum[i] += dom[i];
        }
      };
      uint32_t acc_on = 0;          // 0: the next products start a new segment (accumulators from zero)
      int seg_left = p.seg_chunks;  // weight tiles left in the current segment
      int pend_w = -1, pend_a = -1; // slots read by the last committed, not yet completed group
      for (int ch = 0; ch < chunks; ++ch) {
        int ksteps = p.cin_pad - ch * kTcKC;
        ksteps = (ksteps > kTcKC ? kTcKC : ksteps) >> 4;
        for (int dx = 0; dx < ksz; ++dx) {
          ptx::mbar_wait(&a_full[as], a_ph);
          const uint32_t a_addr = a_ring_u32 + (uint32_t)as * A_SLOT + a_off;
          for (int dy = 0; dy < ksz; ++dy) {
            ptx::mbar_wait(&w_full[ws], w_ph);
            const uint32_t w_addr = w_ring_u32 + (uint32_t)ws * W_TILE;
            const uint64_t a_hi = make_smem_desc(a_addr + (uint32_t)dy * dy_step);
            const uint64_t a_lo = make_smem_desc(a_addr + (uint32_t)dy * dy_step + A_PLANE);
            const uint64_t b_hi = make_smem_desc(w_addr);
            const uint64_t b_lo = make_smem_desc(w_addr + B_BYTES);
            const bool a_done = dy == ksz - 1;   // last tap that reads this activation slot
            if (strict) {
              // every 16-channel K slice (its three products) is promoted on its own
#pragma unroll 1
              for (int ks = 0; ks < ksteps; ++ks) {
                const uint64_t kadd = (uint64_t)ks * 2u;   // 32 bytes (16 fp16 along K) in 16-byte descriptor units
                // acc_on is always 0 here; a run-time 0 rather than a literal keeps ptxas from treating the products
                // as fresh definitions of corr / dom (which makes it wait for every group at every loop join)
                tile_products<N, NPLANES, 1>(corr, dom, a_hi + kadd, a_lo + kadd, b_hi + kadd, b_lo + kadd, acc_on);
                ptx::wgmma_wait<0>();
                promote();
              }
              release_w(ws);
              if (a_done) release_a(as);
            } else {
              // one straight-line batch per K-slice count: a branch inside a batch makes ptxas serialise the wgmma
              if (ksteps == 4)
                tile_products<N, NPLANES, 4>(corr, dom, a_hi, a_lo, b_hi, b_lo, acc_on);
              else if (ksteps == 1)
                tile_products<N, NPLANES, 1>(corr, dom, a_hi, a_lo, b_hi, b_lo, acc_on);
              else if (ksteps == 2)
                tile_products<N, NPLANES, 2>(corr, dom, a_hi, a_lo, b_hi, b_lo, acc_on);
              else
                tile_products<N, NPLANES, 3>(corr, dom, a_hi, a_lo, b_hi, b_lo, acc_on);
              acc_on = 1;
              const bool item_end = a_done && dx == ksz - 1 && ch == chunks - 1;
              if (--seg_left == 0 || item_end) {
                ptx::wgmma_wait<0>();
                promote();
                acc_on = 0;
                seg_left = p.seg_chunks;
                if (pend_w >= 0) release_w(pend_w);
                if (pend_a >= 0) release_a(pend_a);
                release_w(ws);
                if (a_done) release_a(as);
                pend_w = pend_a = -1;
              } else {
                ptx::wgmma_wait<1>();   // the previous weight tile's group has completed
                if (pend_w >= 0) release_w(pend_w);
                if (pend_a >= 0) release_a(pend_a);
                pend_w = ws;
                pend_a = a_done ? as : -1;
              }
            }
            if (++ws == w_slots) { ws = 0; w_ph ^= 1; }
          }
          if (++as == a_slots) { as = 0; a_ph ^= 1; }
        }
      }
      // the last weight tile ended a segment, so every group has completed; saying so here keeps ptxas from placing
      // its own wait inside the loop, ahead of the exchange that reuses the accumulator registers
      ptx::wgmma_wait<0>();

      // Exchange: the wgmma layout gives a thread rows 16 wq + lane / 4 (+ 8) and column pairs 8 j + 2 (lane % 4); the
      // epilogue wants one pixel and 16 consecutive columns per thread.  Round k moves chunks k and per + k.
      float v9[9];
#pragma unroll
      for (int i = 0; i < 9; ++i) v9[i] = 0.f;
      const int r0 = wq * 16 + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
      for (int k = 0; k < per; ++k) {
        ptx::named_bar_sync(1 + cw, 128);    // readers of the previous round are done
#pragma unroll
        for (int c = 0; c < nch; ++c) {
          if (c == k || c == per + k) {
            float* dst = xchg + (c == k ? 0 : 16);
#pragma unroll
            for (int h = 0; h < 2; ++h) {      // 8-column halves of the chunk: accumulator group j = 2 c + h
              const int j = 2 * c + h;
              dst[r0 * kXchgStride + 8 * h + cq] = sum[4 * j];
              dst[r0 * kXchgStride + 8 * h + cq + 1] = sum[4 * j + 1];
              dst[(r0 + 8) * kXchgStride + 8 * h + cq] = sum[4 * j + 2];
              dst[(r0 + 8) * kXchgStride + 8 * h + cq + 1] = sum[4 * j + 3];
            }
          }
        }
        ptx::named_bar_sync(1 + cw, 128);
        if (k < my_chunks) {
          float v[16];
          const float4* srcp = reinterpret_cast<const float4*>(xchg + (t >> 1) * kXchgStride + grp * 16);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float4 f = srcp[q];
            v[4 * q] = f.x; v[4 * q + 1] = f.y; v[4 * q + 2] = f.z; v[4 * q + 3] = f.w;
          }
          const int cg = n_tile * N + (first_chunk + k) * 16;
          if (p.epi.mode == EPI_D2S_RDOT) {
            // the host guarantees that a thread's columns are whole sub-pixels (rdot_parts == 1) or an equal share of
            // one sub-pixel (rdot_parts > 1: each share writes its own partial plane set)
            if (cg < p.epi.n_valid) {
              const int ij = cg / p.epi.d2s_cout, cc = cg - ij * p.epi.d2s_cout;
              rdot_accumulate16(p.epi, s_rdot, cg, cc, v, v9);
              const bool last = p.epi.rdot_parts > 1 ? k + 1 == my_chunks : cc + 16 == p.epi.d2s_cout;
              if (last && valid) rdot_flush(p.epi, g, img, y, x, ij, p.epi.rdot_parts > 1 ? cc / (per * 16) : 0, v9);
            }
          } else if (valid) {
            if (p.epi.mode == EPI_D2S_TAPS) taps_store16(p.epi, g, img, y, x, cg, v);
            else epilogue_store16(p.epi, g, n_total, img, y, x, cg, v);
          }
        }
      }
    }
  }

  __syncthreads();
}

}  // namespace dcscn
