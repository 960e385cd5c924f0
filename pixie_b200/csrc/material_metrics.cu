// Evaluation metrics of the material networks on labelled scenes: process_batch's metric code
// (WG/trainer/inference_combined.py:108-170) with compute_accuracy and masked_mean (pixie/training_utils.py:68-87), and the
// ground-truth normalisation of MaterialVoxelDataset.__getitem__ (WG/data_utils/my_data.py:160-240), in one pass per batch.
//
// The reference loads material_grid.npy on the host, normalises it with numpy, copies it to the device NCDHW and runs a
// dozen torch reductions per batch and per sample. Here one kernel reads the raw channels-last grid, the mask, the seg
// logits and the cont prediction once (16 B loads when every array is 16 B aligned and V % 4 == 0, scalar loads
// otherwise), writes the normalised gt once (the `mat_grid` save_predictions stores) and reduces, per sample:
//   total   = #(mask != 0)                          (mask.bool(); NaN counts)
//   correct = #(argmax(seg) == trunc(id) & mask != 0) (torch.argmax: first index on ties, NaN is the maximum)
//   s_c     = sum (cont_c - gt_c)^2 * mask, c < 3   (each product a float32 op as torch does it; NaN propagates)
//   den     = sum mask
// The sums accumulate in fp64 (counts are exact integers in fp64): each thread in voxel order, then a fixed shuffle tree
// per warp, the warps in order, and the blocks of a sample in order in a second kernel. The voxel-to-thread map depends on
// V and the load path only, so a repeated call is bit-identical. The float32 replay of the scalar arithmetic
// (num / (clamp(den, 1) + 1e-8), correct / total, the batch means) is done on the host (network_files.py).
//
// Normalisation, as numpy evaluates it on float32 data: density and E go through log10(x + float32(1e-6)) (here the fp64
// log10 rounded to float32, i.e. correctly rounded in all but double-rounding cases), then each continuous channel
// through clip(x, lo, hi) (NaN passes), 2 * (x - lo), / span, - 1 with lo, hi, span = float32(hi - lo) each float32 and every
// op one __f*_rn. The id channel is float(int64(id)) = trunc(id), with -0 written as +0.
#include "material_metrics.cuh"

#include <cstdint>

namespace pixie {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxBlocks = 256;          // blocks per sample; a grid-stride loop covers the rest
constexpr int kAcc = 6;                  // s0 s1 s2 den total correct

__device__ __forceinline__ float log10_eps(float x) { return (float)log10((double)__fadd_rn(x, 1e-6f)); }

__device__ __forceinline__ float scale(float x, float lo, float hi, float span) {
    x = x < lo ? lo : (x > hi ? hi : x);
    return __fsub_rn(__fdiv_rn(__fmul_rn(2.0f, __fsub_rn(x, lo)), span), 1.0f);
}

// torch.argmax over classes, fed one class at a time
__device__ __forceinline__ void argmax_step(float x, int c, float& bv, int& best) {
    if (c == 0 || (bv == bv && (x > bv || x != x))) { bv = x; best = c; }
}

// One voxel: writes its 4 gt channels to g and adds its terms to acc.
__device__ __forceinline__ void voxel(float d, float e, float nu, float id, float mk, bool has_mask, int background_id, int best,
                                      float p0, float p1, float p2, const MaterialNorm& nm, float g[4], double acc[kAcc]) {
    const float tid = __fadd_rn(truncf(id), 0.0f);
    const float m = has_mask ? mk : (tid != (float)background_id ? 1.0f : 0.0f);
    g[0] = scale(log10_eps(d), nm.lo[0], nm.hi[0], nm.span[0]);
    g[1] = scale(log10_eps(e), nm.lo[1], nm.hi[1], nm.span[1]);
    g[2] = scale(nu, nm.lo[2], nm.hi[2], nm.span[2]);
    g[3] = tid;
    const float p[3] = {p0, p1, p2};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float df = __fsub_rn(p[c], g[c]);
        acc[c] += (double)__fmul_rn(__fmul_rn(df, df), m);
    }
    acc[3] += (double)m;
    const bool on = m != 0.0f;
    acc[4] += on ? 1.0 : 0.0;
    acc[5] += (on && (float)best == tid) ? 1.0 : 0.0;
}

// Fixed-order block reduction of kAcc doubles; thread k < kAcc returns the block total of entry k.
__device__ __forceinline__ double block_reduce(double acc[kAcc], double (*sh)[kAcc]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < kAcc; ++k) {
        double v = acc[k];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_down_sync(0xffffffffu, v, off);
        if (lane == 0) sh[warp][k] = v;
    }
    __syncthreads();
    double s = 0.0;
    if (threadIdx.x < kAcc) {
        s = sh[0][threadIdx.x];
        for (int w = 1; w < kWarps; ++w) s += sh[w][threadIdx.x];
    }
    return s;
}

struct Args {
    const float *mat, *mask, *seg, *cont;
    float* gt;
    double* partial;                     // [n][blocks][kAcc]
    long long V;
    int c_mat, n_classes, background_id;
    MaterialNorm norm;
};

// 16 B path: c_mat == 4, V % 4 == 0, all arrays 16 B aligned. One thread handles 4 consecutive voxels per step.
__global__ void __launch_bounds__(kThreads) metrics_vec_kernel(const Args a) {
    __shared__ double sh[kWarps][kAcc];
    const int s = blockIdx.y;
    const long long V = a.V, G = V / 4;
    const float4* mat = reinterpret_cast<const float4*>(a.mat + (size_t)s * V * 4);
    const float4* mask = a.mask ? reinterpret_cast<const float4*>(a.mask + (size_t)s * V) : nullptr;
    const float* seg = a.seg + (size_t)s * a.n_classes * V;
    const float* cont = a.cont + (size_t)s * 3 * V;
    float* gt = a.gt + (size_t)s * 4 * V;
    double acc[kAcc] = {0, 0, 0, 0, 0, 0};
    for (long long q = (long long)blockIdx.x * kThreads + threadIdx.x; q < G; q += (long long)gridDim.x * kThreads) {
        float4 mv[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) mv[k] = __ldcs(mat + 4 * q + k);
        const float4 mk = mask ? __ldcs(mask + q) : make_float4(0.f, 0.f, 0.f, 0.f);
        float bv[4];
        int best[4];
        for (int c = 0; c < a.n_classes; ++c) {
            const float4 l = __ldcs(reinterpret_cast<const float4*>(seg + (size_t)c * V) + q);
            argmax_step(l.x, c, bv[0], best[0]);
            argmax_step(l.y, c, bv[1], best[1]);
            argmax_step(l.z, c, bv[2], best[2]);
            argmax_step(l.w, c, bv[3], best[3]);
        }
        float4 p[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) p[c] = __ldcs(reinterpret_cast<const float4*>(cont + (size_t)c * V) + q);
        float g[4][4];
        const float mks[4] = {mk.x, mk.y, mk.z, mk.w};
        const float pv[3][4] = {{p[0].x, p[0].y, p[0].z, p[0].w}, {p[1].x, p[1].y, p[1].z, p[1].w}, {p[2].x, p[2].y, p[2].z, p[2].w}};
#pragma unroll
        for (int k = 0; k < 4; ++k)
            voxel(mv[k].x, mv[k].y, mv[k].z, mv[k].w, mks[k], mask != nullptr, a.background_id, best[k], pv[0][k], pv[1][k], pv[2][k], a.norm,
                  g[k], acc);
#pragma unroll
        for (int c = 0; c < 4; ++c) __stcs(reinterpret_cast<float4*>(gt + (size_t)c * V) + q, make_float4(g[0][c], g[1][c], g[2][c], g[3][c]));
    }
    const double r = block_reduce(acc, sh);
    if (threadIdx.x < kAcc) a.partial[((size_t)s * gridDim.x + blockIdx.x) * kAcc + threadIdx.x] = r;
}

// Scalar path: any c_mat >= 4, any V, any alignment. One thread per voxel per step.
__global__ void __launch_bounds__(kThreads) metrics_scalar_kernel(const Args a) {
    __shared__ double sh[kWarps][kAcc];
    const int s = blockIdx.y;
    const long long V = a.V;
    const int C = a.c_mat;
    const float* mat = a.mat + (size_t)s * V * C;
    const float* mask = a.mask ? a.mask + (size_t)s * V : nullptr;
    const float* seg = a.seg + (size_t)s * a.n_classes * V;
    const float* cont = a.cont + (size_t)s * 3 * V;
    float* gt = a.gt + (size_t)s * 4 * V;
    double acc[kAcc] = {0, 0, 0, 0, 0, 0};
    for (long long v = (long long)blockIdx.x * kThreads + threadIdx.x; v < V; v += (long long)gridDim.x * kThreads) {
        const float* mv = mat + (size_t)v * C;
        float bv = 0.0f;
        int best = 0;
        for (int c = 0; c < a.n_classes; ++c) argmax_step(__ldg(seg + (size_t)c * V + v), c, bv, best);
        float g[4];
        voxel(__ldg(mv), __ldg(mv + 1), __ldg(mv + 2), __ldg(mv + C - 1), mask ? __ldg(mask + v) : 0.0f, mask != nullptr, a.background_id, best,
              __ldg(cont + v), __ldg(cont + V + v), __ldg(cont + 2 * V + v), a.norm, g, acc);
#pragma unroll
        for (int c = 0; c < 4; ++c) gt[(size_t)c * V + v] = g[c];
    }
    const double r = block_reduce(acc, sh);
    if (threadIdx.x < kAcc) a.partial[((size_t)s * gridDim.x + blockIdx.x) * kAcc + threadIdx.x] = r;
}

// One block per sample: the sample's block partials in block order.
__global__ void __launch_bounds__(kThreads) metrics_final_kernel(const double* __restrict__ partial, int blocks, long long* __restrict__ counts,
                                                                 double* __restrict__ sums) {
    __shared__ double sh[kWarps][kAcc];
    const int s = blockIdx.x;
    double acc[kAcc] = {0, 0, 0, 0, 0, 0};
    for (int b = threadIdx.x; b < blocks; b += kThreads)
#pragma unroll
        for (int k = 0; k < kAcc; ++k) acc[k] += partial[((size_t)s * blocks + b) * kAcc + k];
    const double r = block_reduce(acc, sh);
    if (threadIdx.x < 4) sums[4 * s + threadIdx.x] = r;
    else if (threadIdx.x < kAcc) counts[2 * s + threadIdx.x - 4] = (long long)r;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

int material_metrics(const float* mat, int c_mat, const float* mask, const float* seg, int n_classes, const float* cont, int n, long long V,
                     const MaterialNorm& norm, int background_id, float* gt, long long* counts, double* sums, cudaStream_t st) {
    if (n <= 0) return 0;
    const bool vec = c_mat == 4 && V % 4 == 0 && aligned16(mat) && (!mask || aligned16(mask)) && aligned16(seg) && aligned16(cont) && aligned16(gt);
    const long long units = vec ? V / 4 : V;
    const int blocks = (int)(units <= 0 ? 1 : (units + kThreads - 1) / kThreads < kMaxBlocks ? (units + kThreads - 1) / kThreads : kMaxBlocks);
    double* partial = nullptr;
    if (cudaMallocAsync(&partial, (size_t)n * blocks * kAcc * sizeof(double), st) != cudaSuccess) return 1;
    const Args a{mat, mask, seg, cont, gt, partial, V, c_mat, n_classes, background_id, norm};
    const dim3 grid(blocks, n);
    if (vec) metrics_vec_kernel<<<grid, kThreads, 0, st>>>(a);
    else metrics_scalar_kernel<<<grid, kThreads, 0, st>>>(a);
    metrics_final_kernel<<<n, kThreads, 0, st>>>(partial, blocks, counts, sums);
    cudaFreeAsync(partial, st);
    return cudaGetLastError() != cudaSuccess;
}

}  // namespace pixie
