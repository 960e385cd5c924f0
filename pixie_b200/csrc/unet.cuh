// Internal C++ interface of the U-Net executor (wrapped by the C ABI in capi.cu). A failure sets the message of
// pixie_last_error().
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <string>
#include "../../include/pixie_b200.h"

namespace pixie {
using UNet = pixie_unet_s;    // the C ABI's handle is the executor itself (unet.cu)
UNet* unet_create(const pixie_unet_config& cfg);    // nullptr on failure
int unet_set_tensor(UNet* u, const char* name, const float* data, const int64_t* shape, int ndim);
int unet_finalize(UNet* u);
int unet_forward(UNet* u, const void* feat_f16, int batch, float* out, cudaStream_t st);
int unet_profile(UNet* u, const void* feat_f16, int batch, float* out, cudaStream_t st, float* ms, int* kinds, double* flops, int cap);
int unet_forward_ncdhw(UNet* u, const float* feat_f32, int batch, float* out, cudaStream_t st);
int unet_forward_host(UNet* u, const void* feat_host, int batch, float* out_host, cudaStream_t st);
int64_t unet_debug_fetch(UNet* u, const char* name, float* host_out, int64_t capacity);
std::string unet_debug_names(UNet* u);
int unet_launch_count(UNet* u);
double unet_flops(UNet* u);
int unet_check(UNet* u);
void unet_destroy(UNet* u);
}  // namespace pixie
