// wgmma / mbarrier / bulk-copy PTX wrappers and shared-memory descriptor helpers shared by the tensor-core kernels
// (field_tc.cu: fused forward; bwd_chain.cu, bwd_wgrad.cu, bwd_dx.cu: backward).  sm_90a.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace tc {

constexpr int TM = 128;             // samples per tile (two warpgroups of 64 rows)
constexpr int ATOM_BYTES = 16384;   // 128 rows x 128 B (64 bf16 of K): one SWIZZLE_128B atom

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// try_wait is a hardware sleep that ends when the phase completes or after a time limit; the hint (20 us) stretches the
// limit so that waiting warps do not spin on the probe loop.  The wake-up on completion stays prompt.
// Bounded wait: a protocol bug must become an error, not a hung GPU.  The probe loop, the clock bound and the trap are
// one asm statement with no call and no branch visible to the compiler, so consumers can wait while wgmma groups are in
// flight (a function call or a divergent branch between wgmmas makes ptxas serialise them).  On timeout the thread
// records (1, block, barrier, parity) in `diag` (mapped host memory owned by onerf_ctx, reported by the next launch
// check on the host) and traps.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, uint32_t* diag) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .u64 t0, t1;\n\t.reg .u32 b;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
      "@p bra DONE;\n\t"
      "mov.u64 t0, %%clock64;\n"
      "WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
      "@p bra DONE;\n\t"
      "mov.u64 t1, %%clock64;\n\t"
      "sub.u64 t1, t1, t0;\n\t"
      "setp.lt.u64 p, t1, %4;\n\t"
      "@p bra WAIT;\n\t"
      "mov.u32 b, %%ctaid.x;\n\t"
      "st.volatile.u32 [%3 + 4], b;\n\t"
      "st.volatile.u32 [%3 + 8], %0;\n\t"
      "st.volatile.u32 [%3 + 12], %1;\n\t"
      "membar.sys;\n\t"
      "st.volatile.u32 [%3], 1;\n\t"
      "membar.sys;\n\t"
      "trap;\n"
      "DONE:\n\t}"
      :
      : "r"(bar), "r"(parity), "r"(20000u), "l"(diag), "n"(4000000000ll)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// make generic-proxy shared-memory writes visible to the async proxy (bulk copies / wgmma operand reads)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

// per-thread register budget of the executing warpgroup (all its warps execute it)
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// ------------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA, M = 64 rows per warpgroup, K = 16 per instruction, bf16 x bf16 -> fp32 in registers)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
template <int NR>
__device__ __forceinline__ void fence_regs(float* d) {
#pragma unroll
  for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define ONERF_WG_D32                                                                                                   \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, " \
  "%25, %26, %27, %28, %29, %30, %31}"
#define ONERF_WG_OUT32(d)                                                                                              \
  "+f"((d)[0]), "+f"((d)[1]), "+f"((d)[2]), "+f"((d)[3]), "+f"((d)[4]), "+f"((d)[5]), "+f"((d)[6]), "+f"((d)[7]),      \
      "+f"((d)[8]), "+f"((d)[9]), "+f"((d)[10]), "+f"((d)[11]), "+f"((d)[12]), "+f"((d)[13]), "+f"((d)[14]),           \
      "+f"((d)[15]), "+f"((d)[16]), "+f"((d)[17]), "+f"((d)[18]), "+f"((d)[19]), "+f"((d)[20]), "+f"((d)[21]),         \
      "+f"((d)[22]), "+f"((d)[23]), "+f"((d)[24]), "+f"((d)[25]), "+f"((d)[26]), "+f"((d)[27]), "+f"((d)[28]),         \
      "+f"((d)[29]), "+f"((d)[30]), "+f"((d)[31])
#define ONERF_WG_OUT64(d) ONERF_WG_OUT32(d), ONERF_WG_OUT32((d) + 32)
#define ONERF_WG_OUT128(d) ONERF_WG_OUT64(d), ONERF_WG_OUT64((d) + 64)
#define ONERF_WG_D64 "{" \
  "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
  "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
  "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
  "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63" "}"
#define ONERF_WG_D128 "{" \
  "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
  "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
  "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
  "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, " \
  "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, " \
  "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, " \
  "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, " \
  "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127" "}"

// D[64 x 64] += A[64 x 16] (registers: the m64k16 A fragment, bf16 pairs) . B (shared memory, K-major)
__device__ __forceinline__ void wgmma_rs_n64(float* d, const uint32_t* a, uint64_t desc_b, int scale_d = 1) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " ONERF_WG_D32 ", {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
      : ONERF_WG_OUT32(d)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d));
}
// D[64 x 64] += A (shared memory) . B (shared memory); TA / TB: operand is MN-major (transposed)
template <int TA, int TB>
__device__ __forceinline__ void wgmma_ss_n64(float* d, uint64_t desc_a, uint64_t desc_b, int scale_d = 1) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 " ONERF_WG_D32 ", %32, %33, p, 1, 1, %35, %36;\n\t}"
      : ONERF_WG_OUT32(d)
      : "l"(desc_a), "l"(desc_b), "r"(scale_d), "n"(TA), "n"(TB));
}

// Full-width shapes of the layer chain (tc_chain.cuh): D[64 x N] += A . B, N = 64, 128 or 256, both operands K-major,
// A from registers (rs) or shared memory (ss).  One instruction covers all N columns of a k16 step.  scale_d = 0 makes
// the MMA write D = A . B without reading the accumulator (the first MMA of a sum).
template <int N>
__device__ __forceinline__ void wgmma_rs(float* d, const uint32_t* a, uint64_t desc_b, int scale_d = 1) {
  if constexpr (N == 64) {
    wgmma_rs_n64(d, a, desc_b, scale_d);
  } else if constexpr (N == 128) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " ONERF_WG_D64 ", {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
        : ONERF_WG_OUT64(d)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d));
  } else {
    static_assert(N == 256, "wgmma_rs: N is 64, 128 or 256");
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %133, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 " ONERF_WG_D128 ", {%128, %129, %130, %131}, %132, p, 1, 1, 0;\n\t}"
        : ONERF_WG_OUT128(d)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d));
  }
}
template <int N>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t desc_a, uint64_t desc_b, int scale_d = 1) {
  if constexpr (N == 64) {
    wgmma_ss_n64<0, 0>(d, desc_a, desc_b, scale_d);
  } else if constexpr (N == 128) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 " ONERF_WG_D64 ", %64, %65, p, 1, 1, 0, 0;\n\t}"
        : ONERF_WG_OUT64(d)
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));
  } else {
    static_assert(N == 256, "wgmma_ss: N is 64, 128 or 256");
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 " ONERF_WG_D128 ", %128, %129, p, 1, 1, 0, 0;\n\t}"
        : ONERF_WG_OUT128(d)
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));
  }
}

// Shared-memory matrix descriptor (sm_90 GMMA):
//   [0,14) start address >> 4, [16,30) leading byte offset >> 4, [32,46) stride byte offset >> 4,
//   [62,64) layout type (1 = SWIZZLE_128B, 2 = SWIZZLE_64B)
// K-major SWIZZLE_128B (X / dZ atoms): 8-row groups 1024 B apart.  K-major SWIZZLE_64B (weight stage images): 512 B.
// MN-major SWIZZLE_128B (atoms read with K = samples): 64-wide MN blocks LBO apart, 8-row K groups 1024 B apart.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
  return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) | ((uint64_t)layout << 62);
}
__device__ __forceinline__ uint64_t desc_k_sw128(uint32_t saddr) { return make_desc(saddr, 16, 1024, 1); }
__device__ __forceinline__ uint64_t desc_k_sw64(uint32_t saddr) { return make_desc(saddr, 16, 512, 2); }
__device__ __forceinline__ uint64_t desc_mn_sw128(uint32_t saddr, uint32_t lbo_bytes) { return make_desc(saddr, lbo_bytes, 1024, 1); }

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float bf16_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }

// 16-byte chunk `chunk` (8 bf16 of K) of row `row` in a buffer made of SWIZZLE_128B atoms (64 K per atom, 128 rows)
__device__ __forceinline__ uint32_t atom_chunk_off(int row, int chunk) {
  return (uint32_t)(chunk >> 3) * ATOM_BYTES + (uint32_t)row * 128u + (uint32_t)(((chunk & 7) ^ (row & 7)) << 4);
}

// Register fragment of a warpgroup's m64nN accumulator: thread (warp w of the group, lane l) holds rows
// 16 w + l / 4 (entries 4 j, 4 j + 1) and 16 w + l / 4 + 8 (entries 4 j + 2, 4 j + 3), columns 8 j + 2 (l % 4) + {0, 1}.
// Packed to bf16 pairs as pk[2 j] (first row) / pk[2 j + 1] (second row), 16 columns (pk[4 c .. 4 c + 3]) are exactly the
// m64k16 A fragment of the next MMA: the output of one layer is the register operand of the next.

}  // namespace tc
