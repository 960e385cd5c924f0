// Exact nearest Gaussian of every filled particle (PG/particle_filling/filling.py:383-405), and the two searches of the VLM
// part segmentation (pixie/voxel/segmentation.py); see nearest.cu.
#pragma once
#include <cuda_runtime.h>

namespace pixie {

// index[j] = argmin over i of the float32 distance |query[j] - pos[i]| (one rounding per operation, sqrt correctly
// rounded), ties to the lowest i, or -1 when no Gaussian is closer than 1e10. pos [n][3], query [m][3], index [m];
// n or m may be 0. Stream-ordered scratch, no host sync.
cudaError_t nearest_gaussian(const float* pos, int n, const float* query, int m, int* index, cudaStream_t st);

// index[j] = argmin over i of the fp64 squared distance (dx*dx + dy*dy) + dz*dz between query[j] (float32, widened) and
// vert[i] (float64), one rounding per operation; ties to the lowest i; -1 for a non-finite query or without finite vertices.
// vert [n][3], query [m][3], index [m]; n or m may be 0. Stream-ordered scratch, no host sync.
cudaError_t nearest_vertex(const double* vert, int n, const float* query, int m, int* index, cudaStream_t st);

// out[q] = the mode of labels over the k nearest points of pos[q] (itself included), nearest by the fp64 squared distance
// of nearest_vertex, ties at the k-th distance to the lowest index; a tie in count goes to the smallest label.
// pos [n][3] finite, labels [n], out [n], 1 <= k <= n. Stream-ordered scratch, no host sync; deterministic.
cudaError_t knn_label_vote(const float* pos, int n, const long long* labels, int k, long long* out, cudaStream_t st);

}  // namespace pixie
