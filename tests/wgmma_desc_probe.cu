// How wgmma reads a SWIZZLE_128B K-major operand whose descriptor starts part-way into a swizzle atom
// (tests/test_gpu_wgmma_desc.py).
//
// A box of 9 rows of W_box pixels x 64 fp16 channels is TMA-loaded with the tensor-map settings of conv_tc_kernel into
// a 1024-aligned buffer.  wgmma.m64n16k16 (both operands in shared memory, K = 64 in four steps) then reads its 64 A
// rows as 8 groups of 8 consecutive pixels, group g starting at pixel r + g * W_box: the descriptor starts r rows
// (r * 128 bytes) into the box with a stride byte offset of W_box * 128.  Two descriptor forms are tried: base_offset
// = 0, and base_offset = (start address >> 7) & 7.  The reference is the same wgmma on an aligned tile that TMA loaded
// at the shifted origin (a 3-D view of the same pixels with group stride W_box), read with the ordinary descriptor.
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <vector>

#include "../dcscn-super-resolution_b200/csrc/ptx.cuh"

namespace {
using namespace dcscn;

// K-major SWIZZLE_128B descriptor: start >> 4 [0,14), LBO 1 [16,30), SBO >> 4 [32,46), base_offset [49,52), layout 1.
__device__ uint64_t desc(uint32_t saddr, uint32_t sbo, uint32_t base_offset) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(sbo >> 4) << 32) |
         ((uint64_t)(base_offset & 7) << 49) | (1ull << 62);
}

constexpr uint32_t kBox = 0, kRef = 24 * 1024, kB = 32 * 1024, kBar = 34 * 1024;

__device__ void mma64(float (&d)[8], uint32_t a, uint32_t sbo_a, uint32_t base_offset, uint32_t b) {
  ptx::wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
    ptx::wgmma_f16<16, 0, 0>(d, desc(a + 32 * ks, sbo_a, base_offset), desc(b + 32 * ks, 1024, 0), ks ? 1u : 0u);
  ptx::wgmma_commit();
  ptx::wgmma_wait<0>();
}

// out: [3][64][16] fp32 - base_offset 0, base_offset from the address, reference
__global__ void __launch_bounds__(128) probe_kernel(const __grid_constant__ CUtensorMap tm_box,
                                                    const __grid_constant__ CUtensorMap tm_ref,
                                                    const __grid_constant__ CUtensorMap tm_b, int w_box, int r,
                                                    float* out) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + kBar);
  const int t = threadIdx.x;
  if (t == 0) {
    ptx::mbar_init(bar, 1);
    ptx::fence_barrier_init();
    ptx::fence_proxy_async();
  }
  __syncthreads();
  if (t == 0) {
    ptx::mbar_arrive_expect_tx(bar, (9 * w_box + 64 + 16) * 128);
    ptx::tma_load_4d(smem + kBox, &tm_box, bar, 0, 0, 0, 0);
    ptx::tma_load_4d(smem + kRef, &tm_ref, bar, 0, 0, 0, 0);
    ptx::tma_load_4d(smem + kB, &tm_b, bar, 0, 0, 0, 0);
  }
  ptx::mbar_wait(bar, 0);
  const uint32_t base = ptx::smem_u32(smem);
  const uint32_t a_shift = base + kBox + (uint32_t)r * 128;
  const int row = (t >> 5) * 16 + ((t & 31) >> 2), col = 2 * (t & 3);
  for (int form = 0; form < 3; ++form) {
    float d[8];
    if (form == 2) mma64(d, base + kRef, 1024, 0, base + kB);
    else mma64(d, a_shift, (uint32_t)w_box * 128, form ? (a_shift >> 7) & 7 : 0, base + kB);
    float* o = out + form * 64 * 16;
    // m64n16 accumulator layout: d[4j + 2h + e] is row + 8h, column 8j + col + e
    for (int j = 0; j < 2; ++j)
      for (int h = 0; h < 2; ++h)
        for (int e = 0; e < 2; ++e) o[(row + 8 * h) * 16 + 8 * j + col + e] = d[4 * j + 2 * h + e];
  }
}

PFN_cuTensorMapEncodeTiled_v12000 encode_fn() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  return (PFN_cuTensorMapEncodeTiled_v12000)fn;
}

// conv_tc_kernel's settings: fp16, SWIZZLE_128B, 256-byte L2 promotion, zero fill
bool encode(PFN_cuTensorMapEncodeTiled_v12000 enc, CUtensorMap* tm, void* base, const cuuint64_t (&dims)[4],
            const cuuint64_t (&strides)[3], const cuuint32_t (&box)[4]) {
  cuuint32_t estr[4] = {1, 1, 1, 1};
  return enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace

// Runs the probe for one (W_box, r); out receives 3 x 64 x 16 floats.  Returns 0 on success.
extern "C" int wgmma_desc_probe(int w_box, int r, float* out) {
  PFN_cuTensorMapEncodeTiled_v12000 enc = encode_fn();
  if (!enc || w_box < 8 || w_box > 32 || r < 0 || r > 7) return 1;
  const int pixels = 9 * w_box;
  std::vector<__half> ha(pixels * 64), hb(16 * 64);
  uint32_t s = 12345u + 977u * (uint32_t)w_box;
  auto rnd = [&]() { s = s * 1664525u + 1013904223u; return (float)((s >> 9) & 0xFFFF) / 32768.0f - 1.0f; };
  for (auto& v : ha) v = __float2half(rnd());
  for (auto& v : hb) v = __float2half(rnd());
  __half *da = nullptr, *db = nullptr;
  float* dout = nullptr;
  if (cudaMalloc(&da, ha.size() * 2) || cudaMalloc(&db, hb.size() * 2) || cudaMalloc(&dout, 3 * 64 * 16 * 4)) return 2;
  cudaMemcpy(da, ha.data(), ha.size() * 2, cudaMemcpyHostToDevice);
  cudaMemcpy(db, hb.data(), hb.size() * 2, cudaMemcpyHostToDevice);
  const cuuint64_t row = 128, line = (cuuint64_t)w_box * 128;
  CUtensorMap tm_box, tm_ref, tm_b;
  bool ok = encode(enc, &tm_box, da, {64, (cuuint64_t)w_box, 9, 1}, {row, line, 9 * line},
                   {64, (cuuint32_t)w_box, 9, 1}) &&
            // pixel r + g * W_box + i as row 8 g + i of an aligned tile
            encode(enc, &tm_ref, da + r * 64, {64, 8, 8, 1}, {row, line, 8 * line}, {64, 8, 8, 1}) &&
            encode(enc, &tm_b, db, {64, 16, 1, 1}, {row, 16 * row, 16 * row}, {64, 16, 1, 1});
  int rc = ok ? 0 : 3;
  if (!rc) {
    const int smem = 35 * 1024 + 1024;
    if (cudaFuncSetAttribute(probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) rc = 4;
    if (!rc) {
      probe_kernel<<<1, 128, smem>>>(tm_box, tm_ref, tm_b, w_box, r, dout);
      if (cudaDeviceSynchronize() != cudaSuccess) rc = 5;
      else cudaMemcpy(out, dout, 3 * 64 * 16 * 4, cudaMemcpyDeviceToHost);
    }
  }
  cudaFree(da);
  cudaFree(db);
  cudaFree(dout);
  return rc;
}
