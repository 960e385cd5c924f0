// Trained 3DGS checkpoint decode: GaussianModel.load_ply (gaussian-splatting/scene/gaussian_model.py:215-260) followed by
// get_xyz / get_features / get_opacity / get_covariance (:27-31, :117-118 with utils/general_utils.py:64-110) and, when a
// threshold is given, the opacity filter of gs_simulation.py:405. The mirror image of gs_ply.cu.
//
// The reference reads each column into numpy, copies it to the device as a float32 tensor and runs the activations as
// separate torch ops. Here the vertex table goes to the device as it is in the file and one thread decodes one row. A
// block stages its contiguous span of 128 rows in shared memory with 16 B loads (the span starts at a multiple of
// 128 * 4 B, so it is aligned whenever the table is, whatever the row width), then each thread reads its row's columns
// from shared memory. Every float operation of the reference is one __f*_rn here, so nvcc cannot contract it: pos, shs and
// opacity equal torch's bit for bit; L = R diag(s) is formed as the product R @ diag(s) forms it (R_ij s_j, and NaN when
// another entry of the row of R is not finite); only the 3-term sums of L L^T, which cuBLAS does in the reference, use FMA.
//
// With a threshold, a first pass counts each block's kept rows, cub scans the counts, and the decode pass writes the kept
// rows at the block's offset plus their rank in the block (warp ballots), which keeps file order.
#include "gs_load.cuh"
#include "workspace.cuh"

#include <cub/cub.cuh>
#include <cstdint>

namespace pixie {
namespace {

constexpr int kRows = 128;                 // rows staged per block = threads per block
constexpr int kWarps = kRows / 32;

// torch's CUDA sigmoid for float: one / (one + std::exp(-a)) in float
__device__ __forceinline__ float sigmoid_rn(float a) { return __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-a))); }

__device__ __forceinline__ bool keep_row(float opacity, int has_threshold, float threshold) {
    return !has_threshold || opacity > threshold;            // NaN compares false
}

__global__ void __launch_bounds__(kRows) count_kernel(const float* __restrict__ table, long long n, int row_words, int op_col,
                                                      float threshold, long long* __restrict__ counts) {
    const long long i = (long long)blockIdx.x * kRows + threadIdx.x;
    bool keep = false;
    if (i < n) keep = keep_row(sigmoid_rn(__ldg(table + i * row_words + op_col)), 1, threshold);
    const int c = __syncthreads_count(keep);
    if (threadIdx.x == 0) counts[blockIdx.x] = c;
}

template <int K>
__global__ void __launch_bounds__(kRows) decode_kernel(const float* __restrict__ table, long long n, int row_words, const GsColumns cols,
                                                       int has_threshold, float threshold, const long long* __restrict__ offsets,
                                                       float* __restrict__ pos, float* __restrict__ shs, float* __restrict__ opacity,
                                                       float* __restrict__ cov) {
    extern __shared__ __align__(16) float rows[];
    __shared__ int warp_base[kWarps];
    const long long first = (long long)blockIdx.x * kRows;
    const int nb = (int)min((long long)kRows, n - first);
    const int count = nb * row_words;
    const float* src = table + first * row_words;
    const int t = threadIdx.x;
    if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
        const int n4 = count >> 2;
        const float4* s4 = reinterpret_cast<const float4*>(src);
        float4* d4 = reinterpret_cast<float4*>(rows);
        for (int i = t; i < n4; i += kRows) d4[i] = __ldg(s4 + i);
        for (int i = 4 * n4 + t; i < count; i += kRows) rows[i] = __ldg(src + i);
    } else {
        for (int i = t; i < count; i += kRows) rows[i] = __ldg(src + i);
    }
    __syncthreads();

    const float* row = rows + t * row_words;
    float o = 0.0f;
    bool keep = false;
    if (t < nb) {
        o = sigmoid_rn(row[cols.opacity]);
        keep = keep_row(o, has_threshold, threshold);
    }
    // rank among the block's kept rows, in row order
    const unsigned ballot = __ballot_sync(0xffffffffu, keep);
    const int lane = t & 31, warp = t >> 5;
    if (lane == 0) warp_base[warp] = __popc(ballot);
    __syncthreads();
    if (!keep) return;
    int rank = __popc(ballot & ((1u << lane) - 1u));
    for (int w = 0; w < warp; ++w) rank += warp_base[w];
    const long long m = (offsets ? offsets[blockIdx.x] : first) + rank;

#pragma unroll
    for (int c = 0; c < 3; ++c) pos[3 * m + c] = row[cols.xyz[c]];
    // get_features: shs[m][0][c] = f_dc_c, shs[m][k][c] = f_rest_{c (K-1) + k - 1} (load_ply's reshape (P, 3, K-1), transpose)
    float* sh = shs + (long long)3 * K * m;
#pragma unroll
    for (int c = 0; c < 3; ++c) sh[c] = row[cols.dc[c]];
#pragma unroll
    for (int k = 1; k < K; ++k)
#pragma unroll
        for (int c = 0; c < 3; ++c) sh[3 * k + c] = row[cols.rest[c * (K - 1) + k - 1]];
    opacity[m] = o;

    float s[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) s[j] = expf(row[cols.scale[j]]);
    // build_rotation: norm = sqrt(((r0 r0 + r1 r1) + r2 r2) + r3 r3), q = r / norm, R as general_utils.py:90-98 writes it
    const float r0 = row[cols.rot[0]], r1 = row[cols.rot[1]], r2 = row[cols.rot[2]], r3 = row[cols.rot[3]];
    const float norm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r0, r0), __fmul_rn(r1, r1)), __fmul_rn(r2, r2)), __fmul_rn(r3, r3)));
    const float w = __fdiv_rn(r0, norm), x = __fdiv_rn(r1, norm), y = __fdiv_rn(r2, norm), z = __fdiv_rn(r3, norm);
    const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
    const float xy = __fmul_rn(x, y), xz = __fmul_rn(x, z), yz = __fmul_rn(y, z);
    const float wx = __fmul_rn(w, x), wy = __fmul_rn(w, y), wz = __fmul_rn(w, z);
    float R[3][3];
    R[0][0] = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(yy, zz)));
    R[0][1] = __fmul_rn(2.0f, __fsub_rn(xy, wz));
    R[0][2] = __fmul_rn(2.0f, __fadd_rn(xz, wy));
    R[1][0] = __fmul_rn(2.0f, __fadd_rn(xy, wz));
    R[1][1] = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(xx, zz)));
    R[1][2] = __fmul_rn(2.0f, __fsub_rn(yz, wx));
    R[2][0] = __fmul_rn(2.0f, __fsub_rn(xz, wy));
    R[2][1] = __fmul_rn(2.0f, __fadd_rn(yz, wx));
    R[2][2] = __fsub_rn(1.0f, __fmul_rn(2.0f, __fadd_rn(xx, yy)));
    // L = R @ diag(s): R_ij s_j plus the other two entries of row i times 0, which only matters when one is not finite
    float L[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float zero_terms = __fadd_rn(__fmul_rn(R[i][0], 0.0f), __fadd_rn(__fmul_rn(R[i][1], 0.0f), __fmul_rn(R[i][2], 0.0f)));
#pragma unroll
        for (int j = 0; j < 3; ++j) L[i][j] = __fadd_rn(__fmul_rn(R[i][j], s[j]), zero_terms);
    }
    // strip_symmetric(L L^T): (00, 01, 02, 11, 12, 22)
    float* cv = cov + 6 * m;
    const int ii[6] = {0, 0, 0, 1, 1, 2}, jj[6] = {0, 1, 2, 1, 2, 2};
#pragma unroll
    for (int e = 0; e < 6; ++e) {
        const int a = ii[e], b = jj[e];
        cv[e] = fmaf(L[a][2], L[b][2], fmaf(L[a][1], L[b][1], __fmul_rn(L[a][0], L[b][0])));
    }
}

template <int K>
cudaError_t launch_decode(const float* table, long long n, int row_words, const GsColumns& cols, int has_threshold, float threshold,
                          const long long* offsets, float* pos, float* shs, float* opacity, float* cov, cudaStream_t st) {
    const size_t smem = (size_t)kRows * row_words * sizeof(float);
    if (smem > 48 * 1024) PIXIE_TRY(cudaFuncSetAttribute(decode_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long blocks = (n + kRows - 1) / kRows;
    decode_kernel<K><<<(unsigned)blocks, kRows, smem, st>>>(table, n, row_words, cols, has_threshold, threshold, offsets, pos, shs, opacity, cov);
    return cudaGetLastError();
}

}  // namespace

cudaError_t gaussian_checkpoint_decode(const void* table_v, long long n, int row_words, const GsColumns& cols, int K, int has_threshold,
                                       float threshold, float* pos, float* shs, float* opacity, float* cov, long long* m_host, cudaStream_t st) {
    *m_host = 0;
    if (n <= 0) return cudaSuccess;
    const float* table = static_cast<const float*>(table_v);
    const long long blocks = (n + kRows - 1) / kRows;
    long long *counts = nullptr, *offsets = nullptr;      // [blocks + 1] each, with a threshold
    Workspace w(st);
    if (has_threshold) {
        void* tmp = nullptr;
        size_t tmp_bytes = 0;
        PIXIE_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, counts, offsets, (int)(blocks + 1), st));
        PIXIE_TRY(w.carve([&] { counts = w.take<long long>(blocks + 1); offsets = w.take<long long>(blocks + 1); tmp = w.take<char>(tmp_bytes); }));
        PIXIE_TRY(cudaMemsetAsync(counts + blocks, 0, sizeof(long long), st));
        count_kernel<<<(unsigned)blocks, kRows, 0, st>>>(table, n, row_words, cols.opacity, threshold, counts);
        PIXIE_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, counts, offsets, (int)(blocks + 1), st));
        PIXIE_TRY(cudaMemcpyAsync(m_host, offsets + blocks, sizeof(long long), cudaMemcpyDeviceToHost, st));
    }
    cudaError_t e;
    switch (K) {
        case 1: e = launch_decode<1>(table, n, row_words, cols, has_threshold, threshold, offsets, pos, shs, opacity, cov, st); break;
        case 4: e = launch_decode<4>(table, n, row_words, cols, has_threshold, threshold, offsets, pos, shs, opacity, cov, st); break;
        case 9: e = launch_decode<9>(table, n, row_words, cols, has_threshold, threshold, offsets, pos, shs, opacity, cov, st); break;
        default: e = launch_decode<16>(table, n, row_words, cols, has_threshold, threshold, offsets, pos, shs, opacity, cov, st); break;
    }
    PIXIE_TRY(e);
    if (has_threshold) PIXIE_TRY(cudaStreamSynchronize(st));
    else *m_host = n;
    return cudaSuccess;
}

}  // namespace pixie
