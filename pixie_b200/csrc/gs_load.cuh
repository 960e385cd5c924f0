// Trained 3DGS checkpoint decode (gaussian_model.py load_ply + get_xyz / get_features / get_opacity / get_covariance, with
// the opacity filter of gs_simulation.py:405); see gs_load.cu.
#pragma once
#include <cuda_runtime.h>

namespace pixie {

// Word (4-byte) offsets of a checkpoint's columns within a vertex row: x y z, f_dc_0..2, f_rest_0..3(K-1)-1 in numeric
// order, opacity, scale_0..2, rot_0..3. Only the first 3(K-1) entries of `rest` are read.
struct GsColumns {
    int xyz[3], dc[3], rest[45], opacity, scale[3], rot[4];
};

constexpr int kGsLoadMaxRowWords = 448;   // 128 staged rows of at most 448 words fit the 227 KB of shared memory

// table: n rows of `row_words` 4-byte words each (the PLY's binary vertex element, little-endian, on the device). Writes
// the kept rows, in file order, to pos [.][3], shs [.][K][3], opacity [.], cov [.][6] (capacity n each) and their number
// to *m_host. With has_threshold a row is kept when sigmoid(opacity) > threshold (strict; NaN is dropped), otherwise all
// are. K is 1, 4, 9 or 16 and 1 <= row_words <= kGsLoadMaxRowWords. Host-synchronises on `st` once when filtering.
cudaError_t gaussian_checkpoint_decode(const void* table, long long n, int row_words, const GsColumns& cols, int K, int has_threshold,
                                       float threshold, float* pos, float* shs, float* opacity, float* cov, long long* m_host, cudaStream_t st);
// The same table and columns, every row, decoded as GaussianModel.load_ply then get_xyz, get_features, get_opacity,
// get_scaling and get_rotation give it: pos, shs and opacity as above, scales [n][3] = exp(scale_j), rotations [n][4] =
// rot / max(||rot||, 1e-12) (F.normalize; w x y z as stored). Stream-ordered, no host sync.
cudaError_t gaussian_checkpoint_decode_scale_rot(const void* table, long long n, int row_words, const GsColumns& cols, int K, float* pos,
                                                 float* shs, float* opacity, float* scales, float* rotations, cudaStream_t st);

}  // namespace pixie
