// CLIP part similarities of the VLM part segmentation (pixie/voxel/segmentation.py:98-183); see part_segmentation.cu.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <cstdint>

namespace pixie {

constexpr int kMaxParts = 64;

// For the occupied voxels v of feat [V][C] float16 (mask[v] != 0, in index order; every voxel when mask is null), with
// f = feat[v] in fp32 and the unit query rows q [P][C] fp32:
//   sims[n][p]  = (f . q_p) / |f|                  fp32 accumulation, one pass over the features
//   probs[n][p] = softmax_p(sims[n][p] * inv_t)    (optional: probs may be null)
//   labels[n]   = argmax_p probs[n][p]              torch's rule: first index on ties, a NaN wins
//   scores[n]   = probs[n][labels[n]]
// n counts the occupied voxels; the caller gives it (n_occupied), and a mask with fewer writes only those rows.
// 1 <= P <= kMaxParts, C >= 1. Stream-ordered scratch, no host sync.
cudaError_t part_similarity(const __half* feat, const uint8_t* mask, int64_t V, int C, int n_occupied, const float* query, int P,
                            float inv_t, float* sims, int64_t* labels, float* scores, float* probs, cudaStream_t st);

}  // namespace pixie
