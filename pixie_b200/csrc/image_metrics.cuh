// PSNR and SSIM of one image pair, as gaussian-splatting's metrics.py scores render/ground-truth pairs; see image_metrics.cu.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace pixie {

// a, b: [height][width][3] uint8 on the device, read as k / 255 in float32 (to_tensor). window (host): the normalised
// float32 11-tap 1D window. out [2] fp64 on the device: {psnr, ssim}. One kernel launch; the result is the same bit for
// bit on every call. Stream-ordered, no host sync.
cudaError_t image_metrics(const uint8_t* a, const uint8_t* b, int height, int width, const float window[11], double* out, cudaStream_t st);

}  // namespace pixie
