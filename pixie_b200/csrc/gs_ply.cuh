// 3DGS PLY vertex records of a simulated frame (gs_simulation.py:253-322 with gaussian_model.py:177-208); see gs_ply.cu.
#pragma once
#include <cuda_runtime.h>

namespace pixie {

// records [n][14 + 3K] fp32, one PLY vertex per row: x y z, nx ny nz (0), f_dc_0..2, f_rest_0..3(K-1)-1, opacity,
// scale_0..2 (log scales), rot_0..3 (w x y z, scipy's sign). pos [n][3], cov [n][6] upper triangle, shs [n][K][3],
// opacity [n]; K in {1, 4, 9, 16}, anything else returns 2. Stream-ordered, no host sync.
int gaussian_ply_records(const float* pos, const float* cov, const float* shs, int K, const float* opacity, int n, float* records,
                         cudaStream_t st);

}  // namespace pixie
