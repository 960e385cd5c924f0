// PSNR and SSIM of one image pair: gaussian-splatting's utils/image_utils.py psnr and utils/loss_utils.py ssim (11-tap
// Gaussian window, sigma 1.5, zero padding 5 per channel, C1 = 0.01^2, C2 = 0.03^2, mean of the map), as metrics.py applies
// them to a render and its ground truth read by to_tensor (k / 255 in float32).
//
// One launch. A 256-thread CTA owns a 32 x 16 tile of one channel: it stages the tile and its 5-pixel halo as float32 in
// shared memory, forms the five horizontal window sums (x, y, x^2, y^2, x y) of every halo row, then the vertical sums
// and the SSIM map of its pixels. Everything after the float32 inputs is fp64: sigma^2 = E[x^2] - mu^2 cancels, and in
// near-flat regions that error is divided by C2 = 9e-4. The 2D window is the outer product of the float32 1D window the
// reference normalises (the caller passes it), taken exactly in fp64; the reference rounds each product to float32 (see
// DESIGN.md). The CTA reduces its map and squared-error sums in a fixed tree, writes them to a partial slot, and the last
// CTA to finish (a fenced counter) sums the slots in index order: the result does not depend on scheduling.
#include "image_metrics.cuh"
#include "workspace.cuh"

#include <cstdint>

namespace pixie {
namespace {

constexpr int kTW = 32, kTH = 16, kR = 5, kTaps = 2 * kR + 1;
constexpr int kInW = kTW + 2 * kR, kInH = kTH + 2 * kR;
constexpr int kThreads = 256;
// the constants as the float32 tensors of the reference see them
constexpr double kC1 = (double)(float)(0.01 * 0.01);
constexpr double kC2 = (double)(float)(0.03 * 0.03);

struct Window { float g[kTaps]; };

__global__ void __launch_bounds__(kThreads) ssim_psnr_kernel(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, int H, int W,
                                                             Window win, double2* __restrict__ partials, unsigned* __restrict__ counter,
                                                             double* __restrict__ out) {
    __shared__ float sa[kInH][kInW], sb[kInH][kInW];
    __shared__ double hs[5][kInH][kTW];
    __shared__ double red[2][kThreads];
    __shared__ bool is_last;
    const int t = threadIdx.x, ch = blockIdx.z;
    const int x0 = blockIdx.x * kTW, y0 = blockIdx.y * kTH;

    for (int k = t; k < kInH * kInW; k += kThreads) {
        const int r = k / kInW, c = k % kInW, gy = y0 - kR + r, gx = x0 - kR + c;
        float va = 0.f, vb = 0.f;
        if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
            const size_t idx = ((size_t)gy * W + gx) * 3 + ch;
            va = __fdiv_rn((float)a[idx], 255.0f);
            vb = __fdiv_rn((float)b[idx], 255.0f);
        }
        sa[r][c] = va;
        sb[r][c] = vb;
    }
    __syncthreads();

    for (int k = t; k < kInH * kTW; k += kThreads) {
        const int r = k / kTW, c = k % kTW;
        double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0, s4 = 0.0;
#pragma unroll
        for (int j = 0; j < kTaps; ++j) {
            const double g = win.g[j], x = sa[r][c + j], y = sb[r][c + j];
            s0 += g * x;
            s1 += g * y;
            s2 += g * (x * x);
            s3 += g * (y * y);
            s4 += g * (x * y);
        }
        hs[0][r][c] = s0; hs[1][r][c] = s1; hs[2][r][c] = s2; hs[3][r][c] = s3; hs[4][r][c] = s4;
    }
    __syncthreads();

    double acc_ssim = 0.0, acc_se = 0.0;
    for (int k = t; k < kTH * kTW; k += kThreads) {
        const int r = k / kTW, c = k % kTW;
        if (y0 + r >= H || x0 + c >= W) continue;
        double m[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
        for (int i = 0; i < kTaps; ++i) {
            const double g = win.g[i];
#pragma unroll
            for (int q = 0; q < 5; ++q) m[q] += g * hs[q][r + i][c];
        }
        const double mu1_sq = m[0] * m[0], mu2_sq = m[1] * m[1], mu12 = m[0] * m[1];
        const double s11 = m[2] - mu1_sq, s22 = m[3] - mu2_sq, s12 = m[4] - mu12;
        acc_ssim += ((2.0 * mu12 + kC1) * (2.0 * s12 + kC2)) / ((mu1_sq + mu2_sq + kC1) * (s11 + s22 + kC2));
        const double d = (double)sa[r + kR][c + kR] - (double)sb[r + kR][c + kR];
        acc_se += d * d;
    }
    red[0][t] = acc_ssim;
    red[1][t] = acc_se;
    __syncthreads();
    for (int s = kThreads / 2; s > 0; s >>= 1) {
        if (t < s) { red[0][t] += red[0][t + s]; red[1][t] += red[1][t + s]; }
        __syncthreads();
    }
    const unsigned blocks = gridDim.x * gridDim.y * gridDim.z;
    if (t == 0) {
        partials[(blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = make_double2(red[0][0], red[1][0]);
        __threadfence();
        is_last = atomicAdd(counter, 1u) == blocks - 1;
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();

    double ps = 0.0, pe = 0.0;
    for (unsigned k = t; k < blocks; k += kThreads) {
        const double2 p = __ldcg(partials + k);
        ps += p.x;
        pe += p.y;
    }
    red[0][t] = ps;
    red[1][t] = pe;
    __syncthreads();
    for (int s = kThreads / 2; s > 0; s >>= 1) {
        if (t < s) { red[0][t] += red[0][t + s]; red[1][t] += red[1][t + s]; }
        __syncthreads();
    }
    if (t == 0) {
        const double count = 3.0 * (double)H * (double)W;
        const double mse = red[1][0] / count;
        out[0] = 20.0 * log10(1.0 / sqrt(mse));
        out[1] = red[0][0] / count;
    }
}

}  // namespace

cudaError_t image_metrics(const uint8_t* a, const uint8_t* b, int height, int width, const float window[11], double* out, cudaStream_t st) {
    Window win;
    for (int k = 0; k < kTaps; ++k) win.g[k] = window[k];
    const dim3 grid((width + kTW - 1) / kTW, (height + kTH - 1) / kTH, 3);
    const size_t blocks = (size_t)grid.x * grid.y * grid.z;
    double2* partials = nullptr;
    unsigned* counter = nullptr;
    Workspace w(st);
    PIXIE_TRY(w.carve([&] { partials = w.take<double2>(blocks); counter = w.take<unsigned>(1); }));
    PIXIE_TRY(cudaMemsetAsync(counter, 0, sizeof(unsigned), st));
    ssim_psnr_kernel<<<grid, kThreads, 0, st>>>(a, b, height, width, win, partials, counter, out);
    return cudaGetLastError();
}

}  // namespace pixie
