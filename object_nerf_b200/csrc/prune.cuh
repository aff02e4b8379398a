// Sample positions of the pruning pass (EmbeddingVoxel.self_pruning_empty_voxels, reference
// models/embedding_helper.py:202-245), shared by the fused tensor-core pass (field_tc.cu: prune_tc_kernel) and the fp32
// route's point generator (prune.cu).
#pragma once
#include "encode.cuh"
#include "field_common.cuh"

constexpr int kPruneSamples = 4096;          // 16^3 jittered samples per voxel
constexpr uint32_t kPruneStream = 6u;        // Philox stream id no other kernel of the library uses

struct PruneSource {
  const int64_t* cells;   // (K,3) occupied cells, torch.nonzero order
  const float* jitter;    // (K * 4096, 3) U[0,1) or null: philox_uniform(seed, kPruneStream, row * 3 + c)
  uint64_t seed;
};

// Position of sample s of voxel k (global index into cells), in the reference's fp32 operation order, every operation
// rounded on its own:  centre = float(cell) * voxel_size - voxel_offset;  p = centre + (r * voxel_size - voxel_size / 2)
__device__ __forceinline__ void prune_point(const PruneSource& src, const GridView& g, int64_t k, int s, float* p) {
  const int64_t row = k * kPruneSamples + s;
  const float half = __fdiv_rn(g.vsize, 2.0f);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float centre = __fsub_rn(__fmul_rn((float)__ldg(src.cells + k * 3 + c), g.vsize), g.off[c]);
    const float r = src.jitter ? __ldg(src.jitter + row * 3 + c) : philox_uniform(src.seed, kPruneStream, (uint64_t)row * 3 + c);
    p[c] = __fadd_rn(centre, __fsub_rn(__fmul_rn(r, g.vsize), half));
  }
}

// alpha = 1 - exp(-relu(sigma)) with IEEE expf (torch's 1 - torch.exp(-torch.relu(sigma)) for finite sigma); >= 0, so its
// bit pattern orders as an unsigned int
__device__ __forceinline__ float prune_alpha(float sigma) { return 1.0f - expf(-fmaxf(sigma, 0.0f)); }

// field_tc.cu: the fused pass over voxels [cell_begin, cell_begin + n_cells) of src.cells (fp: grid, packed, layout of the
// voxel model); atomicMax of each voxel's alpha into max_alpha[k - cell_begin], which the caller zeroes
int onerf_launch_prune_bf16(onerf_ctx* ctx, const FieldParams& fp, const PruneSource& src, int64_t cell_begin,
                            int64_t n_cells, float* max_alpha, cudaStream_t stream);
