// Exact nearest Gaussian of every filled particle (PG/particle_filling/filling.py:383-405); see nearest.cu.
#pragma once
#include <cuda_runtime.h>

namespace pixie {

// index[j] = argmin over i of the float32 distance |query[j] - pos[i]| (one rounding per operation, sqrt correctly
// rounded), ties to the lowest i, or -1 when no Gaussian is closer than 1e10. pos [n][3], query [m][3], index [m];
// n or m may be 0. Stream-ordered scratch, no host sync.
int nearest_gaussian(const float* pos, int n, const float* query, int m, int* index, cudaStream_t st);

}  // namespace pixie
