// Evaluation metrics of the material networks on labelled scenes (inference_combined.py process_batch with
// compute_accuracy / masked_mean, and the ground-truth normalisation of MaterialVoxelDataset.__getitem__); see
// material_metrics.cu.
#pragma once
#include <cuda_runtime.h>

namespace pixie {

// Normalisation of the three continuous ground-truth channels, as numpy evaluates `2 * (clip(x, lo, hi) - lo) / (hi - lo) - 1`
// on float32 data: lo, hi and span = (hi - lo, computed in double) are each rounded to float32.
struct MaterialNorm {
    float lo[3], hi[3], span[3];
};

// mat [n][V][c_mat] (channels-last material_grid.npy, c_mat >= 4: density, E, nu, ..., material id last), mask [n][V] or
// null (then the mask is material id != background_id), seg [n][n_classes][V] logits, cont [n][3][V]. Writes gt [n][4][V]
// (normalised density, E, nu, then the id truncated to an integer), counts [n][2] = (total, correct) and
// sums [n][4] = (sum over voxels of (cont - gt)^2 * mask for the three channels, sum of mask), all on the device.
// Stream-ordered; returns nonzero on a CUDA error.
int material_metrics(const float* mat, int c_mat, const float* mask, const float* seg, int n_classes, const float* cont, int n, long long V,
                     const MaterialNorm& norm, int background_id, float* gt, long long* counts, double* sums, cudaStream_t st);

}  // namespace pixie
