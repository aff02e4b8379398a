// Positional encoding of one sample row into K-major SWIZZLE_128B shared-memory atoms (the A operand "X" of the
// X-fed layers) of the fused forward kernel (field_tc.cu).
// Reference: models/embedding_helper.py:57-74 (Embedding.forward), :403-409 (channel split + PE of the voxel features).
#pragma once
#include "tc_common.cuh"

namespace tc {

// 16-byte chunk `chunk` (8 bf16 of K) of row `row` in an A buffer made of SWIZZLE_128B atoms (64 K per atom)
__device__ __forceinline__ uint32_t a_chunk_addr(uint32_t base, int row, int chunk) {
  return base + (uint32_t)(chunk >> 3) * ATOM_BYTES + (uint32_t)row * 128u + (uint32_t)(((chunk & 7) ^ (row & 7)) << 4);
}
__device__ __forceinline__ void st_chunk(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

// PE of 8 channels -> 13 chunks [f | sin 2^k f | cos 2^k f]_k at chunk0 + stride * block
__device__ __forceinline__ void pe8_to_chunks(uint32_t xbase, int row, int chunk0, int stride, const float* f) {
  float s[8], c[8];
  st_chunk(a_chunk_addr(xbase, row, chunk0), pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]),
           pack_bf16(f[6], f[7]));
#pragma unroll
  for (int j = 0; j < 8; ++j) __sincosf(f[j], &s[j], &c[j]);  // |f| = O(1), 6 octaves: error stays << bf16 ulp
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    st_chunk(a_chunk_addr(xbase, row, chunk0 + stride * (1 + 2 * k)), pack_bf16(s[0], s[1]), pack_bf16(s[2], s[3]),
             pack_bf16(s[4], s[5]), pack_bf16(s[6], s[7]));
    st_chunk(a_chunk_addr(xbase, row, chunk0 + stride * (2 + 2 * k)), pack_bf16(c[0], c[1]), pack_bf16(c[2], c[3]),
             pack_bf16(c[4], c[5]), pack_bf16(c[6], c[7]));
    if (k < 5) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {  // double-angle step to the next octave
        const float s2 = 2.0f * s[j] * c[j];
        c[j] = fmaf(-2.0f * s[j], s[j], 1.0f);
        s[j] = s2;
      }
    }
  }
}

// PE10(xyz): 63 values in reference order + one zero -> 8 chunks starting at chunk0.  Values are packed to
// bf16 pairs as they are produced and each chunk is stored once complete (the stream position is a compile-time
// constant after unrolling), so few registers stay live: the encoder warps run at the producer's register budget.
__device__ __forceinline__ void pe_xyz_to_chunks(uint32_t xbase, int row, int chunk0, float x, float y, float z) {
  uint32_t pk[4];
  float pend = 0.0f;
  int pos = 0;
  auto emit = [&](float val) {
    if ((pos & 1) == 0) pend = val;
    else pk[(pos >> 1) & 3] = pack_bf16(pend, val);
    if ((pos & 7) == 7) st_chunk(a_chunk_addr(xbase, row, chunk0 + (pos >> 3)), pk[0], pk[1], pk[2], pk[3]);
    ++pos;
  };
  emit(x); emit(y); emit(z);
  float s[3], c[3];
  sincosf(x, &s[0], &c[0]);
  sincosf(y, &s[1], &c[1]);
  sincosf(z, &s[2], &c[2]);
#pragma unroll
  for (int k = 0; k < 10; ++k) {
    emit(s[0]); emit(s[1]); emit(s[2]);
    emit(c[0]); emit(c[1]); emit(c[2]);
    if (k < 9) {
#pragma unroll
      for (int j = 0; j < 3; ++j) {  // double-angle step to the next octave
        const float s2 = 2.0f * s[j] * c[j];
        c[j] = fmaf(-2.0f * s[j], s[j], 1.0f);
        s[j] = s2;
      }
    }
  }
  emit(0.0f);
}


}  // namespace tc
