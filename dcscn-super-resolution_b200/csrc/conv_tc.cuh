// Implicit-GEMM convolution on Hopper wgmma tensor cores (sm_90a).
//
// Replaces  tf.nn.conv2d(SAME, stride 1, NHWC, HWIO) + bias + PReLU  of the reference
// (helper/tf_graph.py:104-153 conv2d / build_conv; :238-249 build_pixel_shuffler_layer).
//
// GEMM view:  D[M = 128 pixels (TH x TW patch), N = cout (padded to 16, <= 128 per column tile)]
//             = sum over taps (ky,kx) and input-channel chunks of  A_tap[128 x KC] * W_tap[KC x N]
//   * A tiles are fetched by TMA (4-D tiled tensor map over the NHWC fp16 plane, box {KC, TW, TH, 1});
//     the box origin is shifted by the tap offset and TMA zero-fills out-of-image pixels, which IS
//     TF's SAME padding - no halo handling in the kernel.
//   * fp32-equivalent precision from fp16 tensor cores:  a = a_hi + a_lo,  w*2^s = w_hi + w_lo
//     (each 11-bit significands), D += a_hi*w_hi + a_lo*w_hi + a_hi*w_lo   (3 x m64nNk16 wgmma per 16 channels,
//     fp32 accumulation in registers).  NPLANES == 1 is the single-pass fp16 "fast" mode.
//   * The tensor core's fp32 accumulator update truncates (round-toward-zero), a bias that grows linearly with the
//     number of accumulation steps.  K is therefore cut into short segments (`seg_chunks` pipeline stages): each
//     segment accumulates from zero, and the sum is added into a second set of fp32 registers with round-to-nearest
//     ("promotion").  `seg_chunks` == 1 (the strict setting) promotes after every 16-channel K slice.  Accumulator + running sum take N registers per thread, which is what caps a column tile at 128.
//   * Weight tiles are the dominant L2->SM traffic (every 128-pixel tile streams the whole layer's weights).  CTAs
//     are launched in clusters of `cs` (1, 2 or 4) that walk pixel tiles in lockstep; each CTA fetches 1/cs of
//     every weight tile and multicasts it to the whole cluster (cp.async.bulk ... .multicast::cluster), and each
//     consumer warpgroup releases a pipeline stage in all cluster members (remote mbarrier arrive).
//   * Warp roles: warpgroup 0 = producer (warp 0 issues TMA), warpgroups 1 and 2 = consumers, one per 64-pixel half
//     of the tile: they issue the wgmma of their rows, promote, and run the epilogue (bias/PReLU/split -> global) after
//     an exchange through shared memory that gives every thread one pixel and a run of 16-column chunks.  Persistent
//     CTAs stride over (pixel-tile, column-tile) work items.
#pragma once
#include "common.h"
#include "epilogue.cuh"
#include "ptx.cuh"

namespace dcscn {

constexpr int kConsumerWGs = 2;                    // one per 64-pixel half of the 128-pixel tile
constexpr int kTcThreads = (1 + kConsumerWGs) * 128;
constexpr int kRegsIssue = 40, kRegsEpilogue = 232;  // setmaxnreg budgets (128*40 + 256*232 <= 64K)
constexpr int kMaxStages = 12;
constexpr int kMaxTileN = 128;                     // column tile cap: accumulator + promoted sum = n_pad registers
constexpr int kRdotSmemBytes = 9 * 128 * 4;         // fused R-CNN1 filter taps (d2s_cout <= 128) staged in shared memory
constexpr int kColSplit = 2;                       // epilogue threads per pixel, each owning a contiguous run of chunks
constexpr int kXchgStride = 36;                    // floats per pixel row of the epilogue exchange buffer (2 chunks + pad)
constexpr int kXchgBytes = kConsumerWGs * 64 * kXchgStride * 4;

template <int KC>
struct TcSmem {
  static constexpr int kRowBytes = KC * 2;                  // 128 (SWIZZLE_128B) or 64 (SWIZZLE_64B)
  static constexpr int kABytes = kTileM * kRowBytes;        // one A plane tile
  static constexpr int kSbo = 8 * kRowBytes;                // 8-row core-matrix group stride
  static constexpr uint64_t kLayout = (KC == 64) ? 1ull : 2ull;  // wgmma descriptor layout type: SW128 = 1, SW64 = 2
};

// wgmma shared-memory matrix descriptor of a K-major swizzled operand tile: start address >> 4 in [0,14), leading
// byte offset (unused for swizzled K-major, 1) in [16,30), stride byte offset >> 4 in [32,46), layout type in [62,64).
template <int KC>
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(TcSmem<KC>::kSbo >> 4) << 32) |
         (TcSmem<KC>::kLayout << 62);
}

__host__ __device__ inline size_t tc_stage_bytes(int KC, int nplanes, int n_pad) {
  return (size_t)nplanes * ((size_t)kTileM * KC * 2 + (size_t)n_pad * KC * 2);
}

template <int KC, int NPLANES>
__global__ void __launch_bounds__(kTcThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo,
               const ConvTCParams p, const int num_stages) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [stages x (A_hi, A_lo, B_hi, B_lo)] then barriers, R-CNN1 taps, epilogue exchange
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int A_BYTES = TcSmem<KC>::kABytes;
  const int B_BYTES = p.n_pad * KC * 2;
  const int STAGE_BYTES = NPLANES * (A_BYTES + B_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)num_stages * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + kMaxStages;
  float* s_rdot = reinterpret_cast<float*>(empty_bar + kMaxStages);   // 16-byte aligned (barriers start 1024-aligned)
  float* s_xchg = s_rdot + kRdotSmemBytes / 4;

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;
  const int cs = p.cluster_size;
  const uint32_t rank = cs > 1 ? ptx::cluster_ctarank() : 0u;
  const uint16_t cta_mask = (uint16_t)((1u << cs) - 1u);

  if (threadIdx.x == 0) {
    for (int s = 0; s < num_stages; ++s) {
      ptx::mbar_init(&full_bar[s], 1);
      ptx::mbar_init(&empty_bar[s], kConsumerWGs * cs);   // one arrival per consumer warpgroup of every cluster CTA
    }
    ptx::fence_barrier_init();
    ptx::fence_proxy_async();
  }
  if (p.epi.mode == EPI_D2S_RDOT)
    for (int i = threadIdx.x; i < p.epi.rdot_taps * p.epi.d2s_cout; i += blockDim.x) s_rdot[i] = p.epi.rdot_w[i];
  __syncthreads();
  if (cs > 1) ptx::cluster_sync();               // peers' barriers are initialised before anything targets them

  const ConvGeom& g = p.g;
  const int tiles_per_img = g.tiles_x * g.tiles_y;
  const int num_tiles = g.n_img * tiles_per_img;
  const int groups = (num_tiles + cs - 1) / cs;  // cs pixel tiles are processed by one cluster iteration
  const int num_items = groups * p.n_tiles;
  const int cluster_id = blockIdx.x / cs;
  const int num_clusters = gridDim.x / cs;
  const int taps = p.ksz * p.ksz;
  const int half = p.ksz >> 1;
  const int total_chunks = taps * p.chunks;

  if (wg == 0) {
    ptx::setmaxnreg_dec<kRegsIssue>();
    // ============================== TMA producer ==============================
    if (threadIdx.x == 0) {
      ptx::prefetch_tensormap(&tm_hi);
      if (NPLANES == 2) ptx::prefetch_tensormap(&tm_lo);
      const int slice_rows = p.n_pad / cs;                       // this CTA's share of every weight tile
      const uint32_t slice_bytes = (uint32_t)(slice_rows * KC * 2);
      const uint32_t slice_off = rank * slice_bytes;
      int stage = 0;
      uint32_t phase = 0;
      for (int item = cluster_id; item < num_items; item += num_clusters) {
        const int n_tile = item % p.n_tiles;
        int tile = (item / p.n_tiles) * cs + (int)rank;
        if (tile >= num_tiles) tile = num_tiles - 1;             // lockstep filler (stores are masked)
        const int img = tile / tiles_per_img;
        const int t2 = tile - img * tiles_per_img;
        const int ty = t2 / g.tiles_x, tx = t2 - ty * g.tiles_x;
        const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(p.wpack) +
                              (size_t)n_tile * total_chunks * (size_t)(NPLANES * B_BYTES);
        for (int tap = 0; tap < taps; ++tap) {
          const int dy = tap / p.ksz - half, dx = tap % p.ksz - half;
          for (int ch = 0; ch < p.chunks; ++ch) {
            ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* st = smem + (size_t)stage * STAGE_BYTES;
            ptx::mbar_arrive_expect_tx(&full_bar[stage], (uint32_t)STAGE_BYTES);
            ptx::tma_load_4d(st, &tm_hi, &full_bar[stage], ch * KC, tx * g.TW + dx, ty * g.TH + dy, img);
            if (NPLANES == 2)
              ptx::tma_load_4d(st + A_BYTES, &tm_lo, &full_bar[stage], ch * KC, tx * g.TW + dx, ty * g.TH + dy, img);
            const uint8_t* wtile = wsrc + (size_t)(tap * p.chunks + ch) * (NPLANES * B_BYTES);
            uint8_t* bdst = st + NPLANES * A_BYTES;
            if (cs == 1) {
              ptx::bulk_load(bdst, wtile, (uint32_t)(NPLANES * B_BYTES), &full_bar[stage]);
            } else {
#pragma unroll
              for (int pl = 0; pl < NPLANES; ++pl)
                ptx::bulk_load_multicast(bdst + pl * B_BYTES + slice_off, wtile + (size_t)pl * B_BYTES + slice_off,
                                         slice_bytes, &full_bar[stage], cta_mask);
            }
            if (++stage == num_stages) { stage = 0; phase ^= 1; }
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
    const int n = p.n_pad;
    const int nch = n >> 4;
    const int per = (nch + kColSplit - 1) / kColSplit;
    const int nseg = (total_chunks + p.seg_chunks - 1) / p.seg_chunks;
    const int n_total = p.n_tiles * p.n_pad;
    const uint32_t smem_base_u32 = ptx::smem_u32(smem);
    const uint32_t a_off = (uint32_t)(cw * 64 * TcSmem<KC>::kRowBytes);
    // epilogue ownership after the exchange: pixel `row`, chunks [grp * per, grp * per + my_chunks)
    const int row = cw * 64 + (t >> 1);
    const int grp = t & 1;
    const int py = row / g.TW, px = row - py * g.TW;
    const int first_chunk = grp * per;
    const int my_chunks = (nch - first_chunk) < per ? ((nch - first_chunk) > 0 ? nch - first_chunk : 0) : per;
    float* xchg = s_xchg + cw * 64 * kXchgStride;
    int stage = 0;
    uint32_t phase = 0;
    for (int item = cluster_id; item < num_items; item += num_clusters) {
      const int n_tile = item % p.n_tiles;
      const int tile = (item / p.n_tiles) * cs + (int)rank;
      const bool real = tile < num_tiles;
      const int img = tile / tiles_per_img;
      const int t2 = tile - img * tiles_per_img;
      const int ty = t2 / g.tiles_x, tx = t2 - ty * g.tiles_x;
      const int y = ty * g.TH + py, x = tx * g.TW + px;
      const bool valid = real && (y < g.H) && (x < g.W);

      float sum[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) sum[i] = 0.f;
      for (int s = 0; s < nseg; ++s) {
        const int c0 = s * p.seg_chunks;
        const int c1 = (c0 + p.seg_chunks < total_chunks) ? c0 + p.seg_chunks : total_chunks;
        float acc[64];
        if (p.seg_chunks == 1) {
          // strictest setting: the segment is one stage and every 16-channel K slice (its three products) is promoted
          // on its own, so no accumulator ever holds more than one slice
          const int ch = c0 % p.chunks;
          ptx::mbar_wait(&full_bar[stage], phase);
          const uint32_t st_addr = smem_base_u32 + (uint32_t)stage * (uint32_t)STAGE_BYTES;
          const uint64_t a_hi = make_smem_desc<KC>(st_addr + a_off);
          const uint64_t a_lo = make_smem_desc<KC>(st_addr + A_BYTES + a_off);
          const uint64_t b_hi = make_smem_desc<KC>(st_addr + NPLANES * A_BYTES);
          const uint64_t b_lo = make_smem_desc<KC>(st_addr + NPLANES * A_BYTES + B_BYTES);
          int ksteps = (p.cin_pad - ch * KC);
          ksteps = (ksteps > KC ? KC : ksteps) >> 4;
#pragma unroll 1
          for (int ks = 0; ks < ksteps; ++ks) {
            const uint64_t kadd = (uint64_t)ks * 2u;
            ptx::wgmma_fence();
            if (NPLANES == 2) {
              ptx::wgmma_f16_n<0, 0>(n, acc, a_lo + kadd, b_hi + kadd, 0);
              ptx::wgmma_f16_n<0, 0>(n, acc, a_hi + kadd, b_lo + kadd, 1);
            }
            ptx::wgmma_f16_n<0, 0>(n, acc, a_hi + kadd, b_hi + kadd, NPLANES == 2 ? 1u : 0u);
            ptx::wgmma_commit();
            ptx::wgmma_wait<0>();
            ptx::reg_fence(acc);
#pragma unroll
            for (int i = 0; i < 64; ++i) sum[i] += acc[i];
          }
          if (t == 0) {
            if (cs == 1) ptx::mbar_arrive(&empty_bar[stage]);
            else
              for (int r = 0; r < cs; ++r) ptx::mbar_arrive_cluster(&empty_bar[stage], (uint32_t)r);
          }
          if (++stage == num_stages) { stage = 0; phase ^= 1; }
          continue;
        }
        uint32_t accumulate = 0;   // every segment starts from zero
        ptx::wgmma_fence();
        // Pass A: as the stages of this segment land, issue the small correction products (a_lo*w_hi, a_hi*w_lo).
        // Pass B: the dominant a_hi*w_hi products.  The accumulator only becomes large in pass B, so only those
        // products contribute truncation error: 3x fewer "effective" steps per segment.
        int st = stage;
        uint32_t ph = phase;
        for (int c = c0; c < c1; ++c) {
          const int ch = c % p.chunks;
          ptx::mbar_wait(&full_bar[st], ph);
          if (NPLANES == 2) {
            const uint32_t st_addr = smem_base_u32 + (uint32_t)st * (uint32_t)STAGE_BYTES;
            const uint64_t a_hi = make_smem_desc<KC>(st_addr + a_off);
            const uint64_t a_lo = make_smem_desc<KC>(st_addr + A_BYTES + a_off);
            const uint64_t b_hi = make_smem_desc<KC>(st_addr + NPLANES * A_BYTES);
            const uint64_t b_lo = make_smem_desc<KC>(st_addr + NPLANES * A_BYTES + B_BYTES);
            int ksteps = (p.cin_pad - ch * KC);
            ksteps = (ksteps > KC ? KC : ksteps) >> 4;
#pragma unroll 1
            for (int ks = 0; ks < ksteps; ++ks) {
              const uint64_t kadd = (uint64_t)ks * 2u;  // 32 bytes (16 fp16 along K) in 16-byte descriptor units
              ptx::wgmma_f16_n<0, 0>(n, acc, a_lo + kadd, b_hi + kadd, accumulate);
              ptx::wgmma_f16_n<0, 0>(n, acc, a_hi + kadd, b_lo + kadd, 1);
              accumulate = 1;
            }
          }
          if (++st == num_stages) { st = 0; ph ^= 1; }
        }
        st = stage;
        for (int c = c0; c < c1; ++c) {
          const int ch = c % p.chunks;
          const uint32_t st_addr = smem_base_u32 + (uint32_t)st * (uint32_t)STAGE_BYTES;
          const uint64_t a_hi = make_smem_desc<KC>(st_addr + a_off);
          const uint64_t b_hi = make_smem_desc<KC>(st_addr + NPLANES * A_BYTES);
          int ksteps = (p.cin_pad - ch * KC);
          ksteps = (ksteps > KC ? KC : ksteps) >> 4;
#pragma unroll 1
          for (int ks = 0; ks < ksteps; ++ks) {
            const uint64_t kadd = (uint64_t)ks * 2u;
            ptx::wgmma_f16_n<0, 0>(n, acc, a_hi + kadd, b_hi + kadd, accumulate);
            accumulate = 1;
          }
          if (++st == num_stages) st = 0;
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::reg_fence(acc);
        // the segment's stages have been read: release them in every CTA of the cluster
        st = stage;
        for (int c = c0; c < c1; ++c) {
          if (t == 0) {
            if (cs == 1) ptx::mbar_arrive(&empty_bar[st]);
            else
              for (int r = 0; r < cs; ++r) ptx::mbar_arrive_cluster(&empty_bar[st], (uint32_t)r);
          }
          if (++st == num_stages) st = 0;
        }
        stage = st;
        phase = ph;
        // fp32 round-to-nearest promotion (registers past n / 2 hold no columns and are never stored)
#pragma unroll
        for (int i = 0; i < 64; ++i) sum[i] += acc[i];
      }

      // Exchange: the wgmma layout gives a thread rows 16 wq + lane / 4 (+ 8) and column pairs 8 j + 2 (lane % 4); the
      // epilogue wants one pixel and 16 consecutive columns per thread.  Round k moves chunks k and per + k.
      float v9[9];
#pragma unroll
      for (int i = 0; i < 9; ++i) v9[i] = 0.f;
      const int r0 = wq * 16 + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
      for (int k = 0; k < kMaxTileN / 16 / kColSplit; ++k) {
        if (k >= per) break;
        ptx::named_bar_sync(1 + cw, 128);    // readers of the previous round are done
#pragma unroll
        for (int c = 0; c < kMaxTileN / 16; ++c) {
          if (c < nch && (c == k || c == per + k)) {
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
          const int cg = n_tile * p.n_pad + (first_chunk + k) * 16;
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
            epilogue_store16(p.epi, g, n_total, img, y, x, cg, v);
          }
        }
      }
    }
  }

  __syncthreads();
  if (cs > 1) ptx::cluster_sync();  // nobody exits while a peer may still signal its barriers
}

}  // namespace dcscn
