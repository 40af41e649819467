// Thin inline-PTX wrappers for the sm_90a features the DCSCN kernels use:
// mbarrier, TMA (cp.async.bulk[.tensor]), wgmma (mma_async / fence / commit_group / wait_group).
#pragma once
#include <cstdint>
#include <cuda.h>

namespace dcscn {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "elect.sync _|P1, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P1;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// Register re-balancing between warpgroups (all 4 warps of a warpgroup must execute the same one).
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}

// ---------------------------------------------------------------- mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "LAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra LAB_WAIT;\n\t"
      "DONE:\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

// --------------------------------------------------------------------- TMA ----
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}

// 4-D tiled tensor load global -> shared, completes `bytes` on the mbarrier.
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// 1-D bulk copy global -> shared (16-byte aligned, size multiple of 16).
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// Releases of a pipeline slot whose readers were wgmma (complete once wgmma.wait_group returns): executed by every
// thread and predicated on `pred` inside the instruction, so no branch breaks the warp-uniform path of a wgmma sequence
// in flight (a divergent branch there makes ptxas serialise the wgmma).  Default (.release.cta) semantics: a
// .release.cluster arrive costs a GPU-scope memory barrier per call, and the slot's next writer is the async proxy.
__device__ __forceinline__ void mbar_arrive_if(uint64_t* bar, bool pred) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %1, 0;\n\t"
      "@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"((uint32_t)pred)
      : "memory");
}

// ------------------------------------------------------------------- wgmma ----
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma sequence.
template <int R>
__device__ __forceinline__ void reg_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Named barrier over `threads` threads (a warpgroup = 128); id 0 is __syncthreads.
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// wgmma.mma_async m64nNk16, fp16 x fp16 -> fp32, both operands from shared-memory descriptors.  N is part of the
// opcode, so every width the kernels use has its own wrapper; d holds the N / 2 accumulator registers of this thread.
// TA / TB = 1: the operand is MN-major (transposed) instead of K-major.
template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_f16(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d);
#define DCSCN_WGMMA_N16(TA, TB)                                                                                      \
  template <>                                                                                                           \
  __device__ __forceinline__ void wgmma_f16<16, TA, TB>(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) { \
    asm volatile(                                                                                                       \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"                                                                   \
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, " #TA ", " #TB ";\n\t}\n"                  \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])                                                                                                            \
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));                                                                      \
  }
DCSCN_WGMMA_N16(0, 0)
DCSCN_WGMMA_N16(1, 1)
#undef DCSCN_WGMMA_N16
#define DCSCN_WGMMA_N32(TA, TB)                                                                                      \
  template <>                                                                                                           \
  __device__ __forceinline__ void wgmma_f16<32, TA, TB>(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) { \
    asm volatile(                                                                                                       \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"                                                                   \
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, " #TA ", " #TB ";\n\t}\n"                  \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])                                                                                                            \
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));                                                                      \
  }
DCSCN_WGMMA_N32(0, 0)
DCSCN_WGMMA_N32(1, 1)
#undef DCSCN_WGMMA_N32
#define DCSCN_WGMMA_N48(TA, TB)                                                                                      \
  template <>                                                                                                           \
  __device__ __forceinline__ void wgmma_f16<48, TA, TB>(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) { \
    asm volatile(                                                                                                       \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"                                                                   \
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, " #TA ", " #TB ";\n\t}\n"                  \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])                                                                                                            \
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));                                                                      \
  }
DCSCN_WGMMA_N48(0, 0)
DCSCN_WGMMA_N48(1, 1)
#undef DCSCN_WGMMA_N48
#define DCSCN_WGMMA_N64(TA, TB)                                                                                      \
  template <>                                                                                                           \
  __device__ __forceinline__ void wgmma_f16<64, TA, TB>(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) { \
    asm volatile(                                                                                                       \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"                                                                   \
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, " #TA ", " #TB ";\n\t}\n"                  \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])                                                                                                            \
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));                                                                      \
  }
DCSCN_WGMMA_N64(0, 0)
DCSCN_WGMMA_N64(1, 1)
#undef DCSCN_WGMMA_N64
#define DCSCN_WGMMA_N80(TA, TB)                                                                                      \
  template <>                                                                                                           \
  __device__ __forceinline__ void wgmma_f16<80, TA, TB>(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) { \
    asm volatile(                                                                                                       \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"                                                                   \
        "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1, " #TA ", " #TB ";\n\t}\n"                  \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])                                                                                                            \
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));                                                                      \
  }
DCSCN_WGMMA_N80(0, 0)
DCSCN_WGMMA_N80(1, 1)
#undef DCSCN_WGMMA_N80
#define DCSCN_WGMMA_N96(TA, TB)                                                                                      \
  template <>                                                                                                           \
  __device__ __forceinline__ void wgmma_f16<96, TA, TB>(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) { \
    asm volatile(                                                                                                       \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"                                                                   \
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, " #TA ", " #TB ";\n\t}\n"                  \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])                                                                                                            \
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));                                                                      \
  }
DCSCN_WGMMA_N96(0, 0)
DCSCN_WGMMA_N96(1, 1)
#undef DCSCN_WGMMA_N96
#define DCSCN_WGMMA_N112(TA, TB)                                                                                      \
  template <>                                                                                                           \
  __device__ __forceinline__ void wgmma_f16<112, TA, TB>(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) { \
    asm volatile(                                                                                                       \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %58, 0;\n\t"                                                                   \
        "wgmma.mma_async.sync.aligned.m64n112k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55}, %56, %57, p, 1, 1, " #TA ", " #TB ";\n\t}\n"                  \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])                                                                                                            \
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));                                                                      \
  }
DCSCN_WGMMA_N112(0, 0)
DCSCN_WGMMA_N112(1, 1)
#undef DCSCN_WGMMA_N112
#define DCSCN_WGMMA_N128(TA, TB)                                                                                      \
  template <>                                                                                                           \
  __device__ __forceinline__ void wgmma_f16<128, TA, TB>(float* d, uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) { \
    asm volatile(                                                                                                       \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                                                   \
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, " #TA ", " #TB ";\n\t}\n"                  \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])                                                                                                            \
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));                                                                      \
  }
DCSCN_WGMMA_N128(0, 0)
DCSCN_WGMMA_N128(1, 1)
#undef DCSCN_WGMMA_N128

// Width chosen at run time (uniform branch per instruction), for the filter-gradient kernel: one accumulator array of 64
// registers serves every product width (n <= 128, multiple of 16); registers past n / 2 are left untouched.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_n(int n, float (&d)[64], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
  switch (n) {
    case 16: wgmma_f16<16, TA, TB>(d, desc_a, desc_b, scale_d); break;
    case 32: wgmma_f16<32, TA, TB>(d, desc_a, desc_b, scale_d); break;
    case 48: wgmma_f16<48, TA, TB>(d, desc_a, desc_b, scale_d); break;
    case 64: wgmma_f16<64, TA, TB>(d, desc_a, desc_b, scale_d); break;
    case 80: wgmma_f16<80, TA, TB>(d, desc_a, desc_b, scale_d); break;
    case 96: wgmma_f16<96, TA, TB>(d, desc_a, desc_b, scale_d); break;
    case 112: wgmma_f16<112, TA, TB>(d, desc_a, desc_b, scale_d); break;
    default: wgmma_f16<128, TA, TB>(d, desc_a, desc_b, scale_d); break;
  }
}

}  // namespace ptx
}  // namespace dcscn
