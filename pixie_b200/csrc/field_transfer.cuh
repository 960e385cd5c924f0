// Material-field -> particle transfer (SURVEY.md 8f-1); see field_transfer.cu.
#pragma once
#include <cuda_runtime.h>

namespace pixie {

// pred [3 + n_classes][D^3] fp32 (the packed tensor save_predictions writes), mask [D^3] fp32 (> 0 = occupied).
// ranges = {density_min, density_max, E_min, E_max, nu_min, nu_max} (log10 for density and E). Outputs hold up to D^3
// entries; *count_host receives the number of occupied voxels (the call synchronises the stream).
cudaError_t field_extract(const float* pred, int n_classes, const float* mask, int D, const double ranges[6], const double bmin[3], const double bmax[3],
                          float* pos, float* density, float* E, float* nu, int* material, float* conf, int* count_host, cudaStream_t st);

// For every query point: k nearest material points -> mean (continuous) / mode (categorical) of their properties; queries whose
// nearest point is farther than `threshold` get the defaults. defaults = {density, E, nu, conf}.
cudaError_t knn_assign(const float* query, int nq, const float* pos, const float* density, const float* E, const float* nu, const int* material,
                       const int* part, const float* conf, int m, int k, double threshold, int weighted, const float defaults[4], int def_material,
                       int def_part, float* o_density, float* o_E, float* o_nu, int* o_material, int* o_part, float* o_conf, int* n_too_far_host,
                       cudaStream_t st);

// get_particle_volume (filling.py:247-288): vol[p] = dx^3 / (particles in p's cell of the grid_n^3 grid). Stream-ordered, no host sync.
cudaError_t particle_volume(const float* pos, int n, int grid_n, float grid_dx, float* vol, cudaStream_t st);
// Per-frame export to the renderer's frame (gs_simulation.py:591-600): positions and (optionally) upper-triangular covariances.
// rotations: host array [n_rot][9] row-major, applied in reverse order like apply_inverse_rotations.
cudaError_t frame_transform(const float* pos, const float* cov, int n, float z_shift, float scale, const float mean[3], const float* rotations, int n_rot,
                            float* pos_out, float* cov_out, cudaStream_t st);

}  // namespace pixie
