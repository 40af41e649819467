// Implicit-GEMM convolution on Hopper wgmma tensor cores (sm_90a).
//
// Replaces  tf.nn.conv2d(SAME, stride 1, NHWC, HWIO) + bias + PReLU  of the reference
// (helper/tf_graph.py:104-153 conv2d / build_conv; :238-249 build_pixel_shuffler_layer).
//
// GEMM view:  D[M = 128 pixels (TH x TW patch), N = cout (padded to 16, <= 112 per column tile)]
//             = sum over 64-channel input chunks, taps (kx, ky) of  A_tap[128 x 64] * W_tap[64 x N]
//   * A tiles are fetched by TMA (4-D tiled tensor map over the NHWC fp16 plane).  A k x k layer (k = 3 or 5) on a 16 x 8
//     patch whose boxes fit (p.chunk_box) loads ONE box of W_box x (TH + k - 1) pixels per chunk, W_box = TW + k - 1,
//     at origin (-k / 2, -k / 2): each 8-pixel patch row is one 8-row operand group, W_box rows apart, and tap (kx, ky)
//     starts kx + ky W_box rows in - not a whole swizzle atom, which the address-based swizzle allows (make_smem_desc).
//     Otherwise it loads one box of TW x (TH + k - 1) pixels per (chunk, kx), its origin shifted by (kx - k / 2, -k / 2);
//     the k ky taps read it at row offsets 0, TW, ..., (k - 1) TW, with TW a multiple of 8.  TMA zero-fills out-of-image
//     pixels, which IS TF's SAME padding - no halo handling in the kernel.  A 1x1 layer loads one TW x TH box per chunk.
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
//   * Two shared-memory rings with their own full/empty mbarriers: activation slots (one per chunk or (chunk, kx)) and weight
//     tiles (one per (tap, chunk), read from the packed image [n_tile][tap][chunk]).  The consumers commit one wgmma
//     group per weight tile and release a slot as soon as `wgmma.wait_group 1` shows the group that last read it
//     has completed, so both rings work purely as prefetch depth.  A weight tile arrives as one bulk copy.
//   * Warp roles: warpgroups 1 and 2 = consumers, one per 64-pixel half of the tile: they issue the wgmma of their
//     rows and promote.  At the end of an item they store the fp32 sums into a hand-off tile in shared memory and go
//     on to the next item.  Warpgroup 0: thread 0 issues the TMA and bulk copies; warps 1-3 run the epilogue (bias /
//     activation / split -> global, or the fused R-CNN1 dot products) from the hand-off tile, one pixel and a run of
//     16-column chunks per work unit, while the consumers' wgmma of the next item run.  Two mbarriers pass the tile
//     back and forth (stage_full, stage_empty).  Persistent CTAs (one per SM) stride over (pixel-tile, column-tile)
//     work items.
#pragma once
#include "common.h"
#include "epilogue.cuh"
#include "ptx.cuh"

namespace dcscn {

constexpr int kConsumerWGs = 2;                    // one per 64-pixel half of the 128-pixel tile
constexpr int kTcThreads = (1 + kConsumerWGs) * 128;
// setmaxnreg budgets: the kernel starts at 168 registers a thread (65536 / 384, in steps of 8), a pool of 384 * 168;
// 128 * 104 + 256 * 200 fills it exactly.  200 hold the three accumulator sets of a 112-column tile (168) without a
// spill, now that the epilogue runs elsewhere; below 104 the epilogue warps spill inside their loop.
constexpr int kRegsProducer = 104, kRegsConsumer = 200;
constexpr int kRegsIssue = 40, kRegsEpilogue = 232;  // wgrad_tc_kernel's budgets (128*40 + 256*232 = 384 * 168)
constexpr int kEpiWarps = 3;                       // warps 1-3 of the producer warpgroup run the tile epilogues
constexpr int kEpiThreads = kEpiWarps * 32;
constexpr int kMaxASlots = 4;                      // activation ring slots
constexpr int kMaxWSlots = 12;                     // weight ring slots
constexpr int kTcBarrierBytes = (2 * (kMaxASlots + kMaxWSlots) + 2) * 8;   // rings + stage_full / stage_empty
constexpr int kMaxTileN = 112;                     // column tile cap: corr + dom + promoted sum = 3 N / 2 registers;
                                                   // at N = 128 (192 of them) ptxas spills inside the K loop
constexpr int kRdotSmemBytes = 9 * 128 * 4;         // fused R-CNN1 filter taps (d2s_cout <= 128) staged in shared memory
constexpr int kColSplit = 2;                       // epilogue work units per pixel, each a contiguous run of chunks

constexpr int kTcKC = 64;                          // input channels per K chunk: an fp16 operand row is 128 bytes,
                                                   // one row of the SWIZZLE_128B layout

struct TcSmem {
  static constexpr int kRowBytes = kTcKC * 2;               // 128 (SWIZZLE_128B)
  static constexpr int kSbo = 8 * kRowBytes;                // 8-row core-matrix group stride
  static constexpr uint64_t kLayout = 1ull;                 // wgmma descriptor layout type: SW128 = 1
};

// wgmma shared-memory matrix descriptor of a K-major swizzled operand tile: start address >> 4 in [0,14), leading
// byte offset (unused for swizzled K-major, 1) in [16,30), stride byte offset (between 8-row groups) >> 4 in [32,46),
// base offset 0 in [49,52), layout type in [62,64).  The 128-byte swizzle is a function of the shared-memory address
// itself, as TMA writes it (measured on H100, tests/test_gpu_wgmma_desc.py): a start any whole number of 128-byte rows
// into an atom, with any multiple of 128 bytes as the stride, reads the rows TMA stored there with base offset 0.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t sbo = TcSmem::kSbo) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(sbo >> 4) << 32) |
         (TcSmem::kLayout << 62);
}

// Width of a k x k layer's activation box: TW + k - 1 when one box per chunk serves all taps (chunk_box), else TW.
__host__ __device__ inline int tc_box_w(int TW, int ksz, int chunk_box) { return chunk_box ? TW + ksz - 1 : TW; }

// Bytes of one activation plane in a ring slot: the TMA box of box_w x (TH + ksz - 1) pixels, rounded up to 1024
// bytes so that every slot and plane starts on a swizzle-atom boundary.
__host__ __device__ inline uint32_t tc_a_plane_bytes(int box_w, int TH, int ksz) {
  return ((uint32_t)box_w * (uint32_t)(TH + ksz - 1) * (uint32_t)kTcKC * 2u + 1023u) & ~1023u;
}
__host__ __device__ inline uint32_t tc_w_tile_bytes(int nplanes, int n_pad) {
  return (uint32_t)nplanes * (uint32_t)n_pad * (uint32_t)kTcKC * 2u;
}

// The fp32 hand-off tile between the consumers and the epilogue warps: 128 pixel rows of an N-column tile.  A row holds
// the first `per` 16-column chunks (the first epilogue unit of the pixel), 4 floats of gap, then the rest; the stride
// N + 8 is 8 or 24 floats past a multiple of 32.  So the consumers' 8-byte stores (4 rows x 8 columns per half warp)
// and the epilogue's 16-byte loads (4 pixels x both units per quarter warp) each touch every bank once.
__host__ __device__ constexpr int tc_stage_stride(int n_pad) { return n_pad + 8; }
__host__ __device__ constexpr uint32_t tc_stage_bytes(int n_pad) { return 128u * (uint32_t)tc_stage_stride(n_pad) * 4u; }

#ifdef DCSCN_TC_PHASES
// Diagnostic build only (-DDCSCN_TC_PHASES, scripts/tc_phases.py): clock64() cycles summed over the consumer warpgroups
// of every CTA of a launch.  [0] K loop (item start to its last wgmma), [1] the consumers' epilogue, [2] items x
// consumer warpgroups, [3] the epilogue warps' busy cycles (summed over the kEpiWarps warps).  The host reads and
// clears them after each launch (tc_phase_report).
__device__ unsigned long long g_tc_phase[4];
#endif

// Diagnostic builds only (scripts/tc_bound.py), whose outputs are meaningless: -DDCSCN_TC_BOUND=1 (fill only) - the
// consumers wait for every slot and release it without issuing wgmma; -DDCSCN_TC_BOUND=2 (math only) - once every
// slot of a ring has been filled, the producer arrives on its full barrier without copying.  Their launch times bound
// the K loop from the fill side and the wgmma side.
#if defined(DCSCN_TC_BOUND) && DCSCN_TC_BOUND == 2
#define DCSCN_TC_COPY(filled, slots) ((filled)++ < (slots))
#else
#define DCSCN_TC_COPY(filled, slots) ((void)(filled), true)
#endif

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
  // carve: [a_slots x (A_hi, A_lo)] [w_slots x (W_hi, W_lo)] then barriers, the hand-off tile, the R-CNN1 taps
  // (EPI_D2S_RDOT only) and, when p.bias_smem, the bias and slopes of all n_tiles * N columns
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const ConvGeom& g = p.g;
  const int ksz = p.ksz;
  const bool chunk_box = p.chunk_box != 0;
  const int box_w = tc_box_w(g.TW, ksz, p.chunk_box);
  const uint32_t A_PLANE = tc_a_plane_bytes(box_w, g.TH, ksz);
  const uint32_t A_SLOT = NPLANES * A_PLANE;
  const uint32_t A_TX = (uint32_t)NPLANES * (uint32_t)box_w * (uint32_t)(g.TH + ksz - 1) * kTcKC * 2u;  // bytes TMA delivers
  constexpr uint32_t B_BYTES = N * kTcKC * 2;
  constexpr uint32_t W_TILE = NPLANES * B_BYTES;
  uint8_t* a_ring = smem;
  uint8_t* w_ring = smem + (size_t)a_slots * A_SLOT;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(w_ring + (size_t)w_slots * W_TILE);
  uint64_t* a_empty = a_full + kMaxASlots;
  uint64_t* w_full = a_empty + kMaxASlots;
  uint64_t* w_empty = w_full + kMaxWSlots;
  uint64_t* stage_full = w_empty + kMaxWSlots;    // the consumers have stored an item's sums in the hand-off tile
  uint64_t* stage_empty = stage_full + 1;          // the epilogue warps have read them
  float* s_stage = reinterpret_cast<float*>(stage_empty + 1);   // 16-byte aligned (barriers start 1024-aligned)
  float* s_rdot = s_stage + tc_stage_bytes(N) / 4;
  constexpr int kStride = tc_stage_stride(N);
  constexpr int nch = N >> 4;
  constexpr int per = (nch + kColSplit - 1) / kColSplit;   // chunks of a pixel's first epilogue unit

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
    ptx::mbar_init(stage_full, kConsumerWGs * 4);   // one arrival per consumer warp
    ptx::mbar_init(stage_empty, kEpiWarps);         // one arrival per epilogue warp
    ptx::fence_barrier_init();
    ptx::fence_proxy_async();
  }
  float* s_bias = s_rdot + (p.epi.mode == EPI_D2S_RDOT ? kRdotSmemBytes / 4 : 0);
  float* s_alpha = s_bias + p.n_tiles * N;
  if (p.epi.mode == EPI_D2S_RDOT)
    for (int i = threadIdx.x; i < p.epi.rdot_taps * p.epi.d2s_cout; i += blockDim.x) s_rdot[i] = p.epi.rdot_w[i];
  // epilogue_store16 reads them from here: an epilogue warp has few loads in flight, and an L1 miss on them is what it
  // waits for longest
  const bool bias_smem = p.bias_smem != 0;   // the host reserves them only in the EPI_PLANES / D2S plane modes
  const float* bias_src = bias_smem ? s_bias : p.epi.bias;
  const float* alpha_src = bias_smem ? s_alpha : p.epi.alpha;
  if (bias_smem)
    for (int i = threadIdx.x; i < p.n_tiles * N; i += blockDim.x) {
      s_bias[i] = p.epi.bias[i];
      s_alpha[i] = p.epi.alpha[i];
    }
  __syncthreads();

  const int tiles_per_img = g.tiles_x * g.tiles_y;
  const int num_items = g.n_img * tiles_per_img * p.n_tiles;
  const int half = ksz >> 1;
  const int chunks = p.chunks;

  if (wg == 0) {
    ptx::setmaxnreg_dec<kRegsProducer>();
    // ============================== TMA producer ==============================
    if (threadIdx.x == 0) {
      ptx::prefetch_tensormap(&tm_hi);
      if (NPLANES == 2) ptx::prefetch_tensormap(&tm_lo);
      int as = 0, ws = 0;
      uint32_t a_ph = 0, w_ph = 0;
      int a_filled = 0, w_filled = 0;   // DCSCN_TC_BOUND == 2 only
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
            if (!chunk_box || dx == 0) {   // a chunk box is loaded once, at origin (-k / 2, -k / 2)
              ptx::mbar_wait(&a_empty[as], a_ph ^ 1);
              uint8_t* ad = a_ring + (size_t)as * A_SLOT;
              if (DCSCN_TC_COPY(a_filled, a_slots)) {
                ptx::mbar_arrive_expect_tx(&a_full[as], A_TX);
                ptx::tma_load_4d(ad, &tm_hi, &a_full[as], ch * kTcKC, x0 + dx, y0, img);
                if (NPLANES == 2) ptx::tma_load_4d(ad + A_PLANE, &tm_lo, &a_full[as], ch * kTcKC, x0 + dx, y0, img);
              } else {
                ptx::mbar_arrive(&a_full[as]);
              }
              if (++as == a_slots) { as = 0; a_ph ^= 1; }
            }
            for (int dy = 0; dy < ksz; ++dy) {
              ptx::mbar_wait(&w_empty[ws], w_ph ^ 1);
              uint8_t* wd = w_ring + (size_t)ws * W_TILE;
              if (DCSCN_TC_COPY(w_filled, w_slots)) {
                ptx::mbar_arrive_expect_tx(&w_full[ws], W_TILE);
                const uint8_t* wtile = wsrc + (size_t)((dy * ksz + dx) * chunks + ch) * W_TILE;
                ptx::bulk_load(wd, wtile, W_TILE, &w_full[ws]);
              } else {
                ptx::mbar_arrive(&w_full[ws]);
              }
              if (++ws == w_slots) { ws = 0; w_ph ^= 1; }
            }
          }
        }
      }
    } else if (threadIdx.x >= 32) {
      // ============================== epilogue warps ==========================
      // Each item's sums arrive in the hand-off tile.  A work unit is one pixel and a contiguous run of 16-column chunks
      // (the first `per` chunks, or the rest); unit u = 2 pixel + run, so a warp reads 16 pixels x both runs.  A
      // thread's units all have the same run (kEpiThreads is even), so its bias and slopes stay the same.
      const int e = threadIdx.x - 32;
      const int n_total = p.n_tiles * N;
      uint32_t st_ph = 0;
#ifdef DCSCN_TC_PHASES
      long long ph_w = 0;
#endif
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        const int n_tile = item % p.n_tiles;
        const int tile = item / p.n_tiles;
        const int img = tile / tiles_per_img;
        const int t2 = tile - img * tiles_per_img;
        const int ty = t2 / g.tiles_x, tx = t2 - ty * g.tiles_x;
        ptx::mbar_wait(stage_full, st_ph);
#ifdef DCSCN_TC_PHASES
        const long long ph_t0 = clock64();
#endif
        // In the depth_to_space modes nothing is stored past n_valid: when the second runs of chunks lie wholly past it
        // (the folded Up-PS: 36 of 96 columns), the units are the pixels' first runs alone.
        const int runs = p.epi.mode != EPI_PLANES && n_tile * N + per * 16 >= p.epi.n_valid ? 1 : kColSplit;
#pragma unroll 1
        for (int u = e; u < 128 * runs; u += kEpiThreads) {
          const int row = runs == kColSplit ? u >> 1 : u, grp = runs == kColSplit ? u & 1 : 0;
          const int py = row / g.TW, px = row - py * g.TW;
          const int y = ty * g.TH + py, x = tx * g.TW + px;
          const bool valid = (y < g.H) && (x < g.W);
          const int first_chunk = grp * per;
          const int my_chunks = (nch - first_chunk) < per ? ((nch - first_chunk) > 0 ? nch - first_chunk : 0) : per;
          const float4* src = reinterpret_cast<const float4*>(s_stage + row * kStride + grp * (per * 16 + 4));
          float v9[9];
#pragma unroll
          for (int i = 0; i < 9; ++i) v9[i] = 0.f;
#pragma unroll
          for (int k = 0; k < per; ++k) {
            if (k < my_chunks) {
              float v[16];
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                const float4 f = src[4 * k + q];
                v[4 * q] = f.x; v[4 * q + 1] = f.y; v[4 * q + 2] = f.z; v[4 * q + 3] = f.w;
              }
              const int cg = n_tile * N + (first_chunk + k) * 16;
              if (p.epi.mode == EPI_D2S_RDOT) {
                // the host guarantees that a unit's columns are whole sub-pixels (rdot_parts == 1) or an equal share of
                // one sub-pixel (rdot_parts > 1: each share writes its own partial plane set)
                if (cg < p.epi.n_valid) {
                  const int ij = cg / p.epi.d2s_cout, cc = cg - ij * p.epi.d2s_cout;
                  rdot_accumulate16(p.epi, s_rdot, cg, cc, v, v9);
                  const bool last = p.epi.rdot_parts > 1 ? k + 1 == my_chunks : cc + 16 == p.epi.d2s_cout;
                  if (last && valid) rdot_flush(p.epi, g, img, y, x, ij, p.epi.rdot_parts > 1 ? cc / (per * 16) : 0, v9);
                }
              } else if (valid) {
                if (p.epi.mode == EPI_D2S_TAPS) taps_store16(p.epi, g, img, y, x, cg, v);
                else epilogue_store16<true>(p.epi, g, n_total, img, y, x, cg, v, bias_src, alpha_src);
              }
            }
          }
        }
        __syncwarp();
        ptx::mbar_arrive_if(stage_empty, lane == 0);
        st_ph ^= 1;
#ifdef DCSCN_TC_PHASES
        ph_w += clock64() - ph_t0;
#endif
      }
#ifdef DCSCN_TC_PHASES
      if (lane == 0) atomicAdd(&g_tc_phase[3], (unsigned long long)ph_w);
#endif
    }
  } else {
    ptx::setmaxnreg_inc<kRegsConsumer>();
    // ============================== consumers ==================================
    const int cw = wg - 1;                   // which 64-pixel half of the tile
    const int t = threadIdx.x & 127;
    const int wq = t >> 5;                   // warp inside the warpgroup: accumulator rows 16 wq .. 16 wq + 15
    const bool strict = p.seg_chunks == 1;
    const uint32_t a_ring_u32 = ptx::smem_u32(a_ring);
    const uint32_t w_ring_u32 = ptx::smem_u32(w_ring);
    // A chunk box holds the patch's 8-pixel rows W_box = TW + k - 1 pixels apart: each is one 8-row group of the operand
    // (stride W_box rows), tap (kx, ky) starts kx + ky W_box rows in, and this half's rows start TH / 2 box rows on.
    // A (chunk, kx) box is TW pixels wide: whole 8-row groups, 1024 bytes apart, and ky starts ky TW rows in.
    const uint32_t a_off = (uint32_t)((chunk_box ? cw * (g.TH / 2) * box_w : cw * 64) * TcSmem::kRowBytes);
    const uint32_t a_sbo = chunk_box ? (uint32_t)(box_w * TcSmem::kRowBytes) : (uint32_t)TcSmem::kSbo;
    const uint32_t dy_step = (uint32_t)(box_w * TcSmem::kRowBytes);   // one image row of the box
    // the wgmma layout gives a thread rows 16 wq + lane / 4 (+ 8) of its half and column pairs 8 j + 2 (lane % 4)
    float* stage_row = s_stage + (cw * 64 + wq * 16 + (lane >> 2)) * kStride + 2 * (lane & 3);
    uint32_t st_ph = 0;
    // a slot is released once the wgmma group that last read it has completed (one arrival per warpgroup, by thread 0)
    auto release_a = [&](int s) { ptx::mbar_arrive_if(&a_empty[s], t == 0); };
    auto release_w = [&](int s) { ptx::mbar_arrive_if(&w_empty[s], t == 0); };
    int as = 0, ws = 0;
    uint32_t a_ph = 0, w_ph = 0;
#ifdef DCSCN_TC_PHASES
    long long ph_k = 0, ph_e = 0, ph_n = 0;
#endif
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
#ifdef DCSCN_TC_PHASES
      const long long ph_t0 = clock64();
#endif
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
          if (!chunk_box || dx == 0) ptx::mbar_wait(&a_full[as], a_ph);
          const uint32_t a_addr =
              a_ring_u32 + (uint32_t)as * A_SLOT + a_off + (chunk_box ? (uint32_t)dx * TcSmem::kRowBytes : 0u);
          for (int dy = 0; dy < ksz; ++dy) {
            ptx::mbar_wait(&w_full[ws], w_ph);
            const uint32_t w_addr = w_ring_u32 + (uint32_t)ws * W_TILE;
            const uint64_t a_hi = make_smem_desc(a_addr + (uint32_t)dy * dy_step, a_sbo);
            const uint64_t a_lo = make_smem_desc(a_addr + (uint32_t)dy * dy_step + A_PLANE, a_sbo);
            const uint64_t b_hi = make_smem_desc(w_addr);
            const uint64_t b_lo = make_smem_desc(w_addr + B_BYTES);
            // last tap that reads this activation slot
            const bool a_done = dy == ksz - 1 && (!chunk_box || dx == ksz - 1);
#if defined(DCSCN_TC_BOUND) && DCSCN_TC_BOUND == 1
            release_w(ws);
            if (a_done) release_a(as);
            if (++ws == w_slots) { ws = 0; w_ph ^= 1; }
            continue;
#endif
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
          if ((!chunk_box || dx == ksz - 1) && ++as == a_slots) { as = 0; a_ph ^= 1; }
        }
      }
      // the last weight tile ended a segment, so every group has completed; saying so here keeps ptxas from placing
      // its own wait inside the loop, ahead of the stores that read the accumulator registers
      ptx::wgmma_wait<0>();
#ifdef DCSCN_TC_PHASES
      const long long ph_t1 = clock64();
#endif

      // Hand-off: once the epilogue warps have read the previous item's tile, store the sums in it (8-byte stores, the
      // second run of chunks 4 floats further on) and go on to the next item; the epilogue warps take it from here.
      ptx::mbar_wait(stage_empty, st_ph ^ 1);
#pragma unroll
      for (int j = 0; j < N / 8; ++j) {
        float* d = stage_row + 8 * j + (j / 2 >= per ? 4 : 0);
        *reinterpret_cast<float2*>(d) = make_float2(sum[4 * j], sum[4 * j + 1]);
        *reinterpret_cast<float2*>(d + 8 * kStride) = make_float2(sum[4 * j + 2], sum[4 * j + 3]);
      }
      __syncwarp();
      ptx::mbar_arrive_if(stage_full, lane == 0);
      st_ph ^= 1;
#ifdef DCSCN_TC_PHASES
      ptx::named_bar_sync(1 + cw, 128);   // the warpgroup's slowest thread ends the epilogue
      const long long ph_t2 = clock64();
      ph_k += ph_t1 - ph_t0;
      ph_e += ph_t2 - ph_t1;
      ++ph_n;
#endif
    }
#ifdef DCSCN_TC_PHASES
    if (t == 0) {
      atomicAdd(&g_tc_phase[0], (unsigned long long)ph_k);
      atomicAdd(&g_tc_phase[1], (unsigned long long)ph_e);
      atomicAdd(&g_tc_phase[2], (unsigned long long)ph_n);
    }
#endif
  }

  __syncthreads();
}

}  // namespace dcscn
