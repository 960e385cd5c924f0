// 3DGS PLY vertex records of a simulated frame: export_gaussians_to_ply (gs_simulation.py:290-322) with
// cov3D_to_log_scales_and_quats (:253-288) and GaussianModel.save_ply / construct_list_of_attributes
// (gaussian-splatting/scene/gaussian_model.py:177-208), one thread per Gaussian.
//
// The reference runs torch.linalg.eigh and scipy's Rotation.from_matrix on the CPU. Here each covariance goes through a
// cyclic Jacobi in fp64 (eigenvalues sorted descending, sqrt(max(lambda, 1e-12)), log; the third eigenvector negated
// when det R < 0) and Markley's decision of scipy's from_matrix, so the quaternion has scipy's sign for the same R
// (w may be negative). A row is 14 + 3K floats (248 B at K = 16); a block stages its rows in shared memory, reading
// pos / shs / opacity / cov and writing the records as the block's contiguous spans with 16 B accesses where aligned.
#include "gs_ply.cuh"

#include <cstdint>

namespace pixie {
namespace {

constexpr int kThreads = 128;
constexpr int kMaxSweeps = 10;        // a 3x3 converges in 4-6 cyclic sweeps; the cap bounds the loop

// A <- J^T A J, V <- V J for the rotation J that zeroes A[P][Q] (Numerical Recipes' `jacobi` step); R is the third index
template <int P, int Q, int R>
__device__ __forceinline__ void jacobi_rotate(double (&A)[3][3], double (&V)[3][3]) {
    const double apq = A[P][Q];
    if (apq == 0.0) return;
    const double theta = (A[Q][Q] - A[P][P]) / (2.0 * apq);
    const double t = fabs(theta) > 1e150 ? 0.5 / theta : (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
    const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
    A[P][P] -= t * apq;
    A[Q][Q] += t * apq;
    A[P][Q] = A[Q][P] = 0.0;
    const double arp = A[R][P], arq = A[R][Q];
    A[R][P] = A[P][R] = c * arp - s * arq;
    A[R][Q] = A[Q][R] = s * arp + c * arq;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const double vp = V[i][P], vq = V[i][Q];
        V[i][P] = c * vp - s * vq;
        V[i][Q] = s * vp + c * vq;
    }
}

__device__ __forceinline__ void swap_pair(double (&lam)[3], double (&V)[3][3], int a, int b) {
    if (lam[a] < lam[b]) {
        const double l = lam[a]; lam[a] = lam[b]; lam[b] = l;
#pragma unroll
        for (int i = 0; i < 3; ++i) { const double v = V[i][a]; V[i][a] = V[i][b]; V[i][b] = v; }
    }
}

// cov3D_to_log_scales_and_quats for one upper-triangular covariance u = (xx, xy, xz, yy, yz, zz):
// out = (log s0, log s1, log s2, w, x, y, z); all seven NaN when any entry of u is NaN or +-Inf (the Jacobi below would
// stop on a NaN at once and fmax would turn a NaN eigenvalue into the clamp, writing a plausible Gaussian instead)
__device__ __forceinline__ void cov_to_scales_quat(const float* u, float* out) {
    bool finite = true;
#pragma unroll
    for (int i = 0; i < 6; ++i) finite &= isfinite(u[i]);
    if (!finite) {
#pragma unroll
        for (int i = 0; i < 7; ++i) out[i] = __int_as_float(0x7fc00000);
        return;
    }
    double A[3][3] = {{u[0], u[1], u[2]}, {u[1], u[3], u[4]}, {u[2], u[4], u[5]}};
    double V[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
    for (int sweep = 0; sweep < kMaxSweeps; ++sweep) {
        const double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2];
        const double diag = A[0][0] * A[0][0] + A[1][1] * A[1][1] + A[2][2] * A[2][2];
        if (!(off > 1e-36 * diag)) break;                   // also ends a zero matrix
        jacobi_rotate<0, 1, 2>(A, V);
        jacobi_rotate<0, 2, 1>(A, V);
        jacobi_rotate<1, 2, 0>(A, V);
    }
    double lam[3] = {A[0][0], A[1][1], A[2][2]};
    swap_pair(lam, V, 0, 1);                                 // descending, the eigenvectors as columns of R = V
    swap_pair(lam, V, 1, 2);
    swap_pair(lam, V, 0, 1);
#pragma unroll
    for (int i = 0; i < 3; ++i) out[i] = (float)log(sqrt(fmax(lam[i], 1e-12)));
    const double det = V[0][0] * (V[1][1] * V[2][2] - V[1][2] * V[2][1]) - V[0][1] * (V[1][0] * V[2][2] - V[1][2] * V[2][0]) +
                       V[0][2] * (V[1][0] * V[2][1] - V[1][1] * V[2][0]);
    if (det < 0.0) {                                         // right-handed: negate column 2
#pragma unroll
        for (int i = 0; i < 3; ++i) V[i][2] = -V[i][2];
    }
    // scipy Rotation.from_matrix: the largest of (R00, R11, R22, trace), first on ties, builds its component first
    const double tr = V[0][0] + V[1][1] + V[2][2];
    int choice = 0;
    double best = V[0][0];
    if (V[1][1] > best) { choice = 1; best = V[1][1]; }
    if (V[2][2] > best) { choice = 2; best = V[2][2]; }
    if (tr > best) choice = 3;
    double q[4];                                             // x y z w; choice i builds q[i], then j = i + 1, k = i + 2 (mod 3)
    if (choice == 0) {
        q[0] = 1.0 - tr + 2.0 * V[0][0]; q[1] = V[1][0] + V[0][1]; q[2] = V[2][0] + V[0][2]; q[3] = V[2][1] - V[1][2];
    } else if (choice == 1) {
        q[1] = 1.0 - tr + 2.0 * V[1][1]; q[2] = V[2][1] + V[1][2]; q[0] = V[0][1] + V[1][0]; q[3] = V[0][2] - V[2][0];
    } else if (choice == 2) {
        q[2] = 1.0 - tr + 2.0 * V[2][2]; q[0] = V[0][2] + V[2][0]; q[1] = V[1][2] + V[2][1]; q[3] = V[1][0] - V[0][1];
    } else {
        q[0] = V[2][1] - V[1][2]; q[1] = V[0][2] - V[2][0]; q[2] = V[1][0] - V[0][1]; q[3] = 1.0 + tr;
    }
    const double inv = 1.0 / sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    out[3] = (float)(q[3] * inv);
    out[4] = (float)(q[0] * inv);
    out[5] = (float)(q[1] * inv);
    out[6] = (float)(q[2] * inv);
}

// put(i, src[i]) for i < count, the block reading the span with coalesced (16 B where src is aligned) loads
template <class Put>
__device__ __forceinline__ void load_span(const float* __restrict__ src, int count, Put put) {
    if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
        const int n4 = count >> 2;
        const float4* s4 = reinterpret_cast<const float4*>(src);
        for (int i = threadIdx.x; i < n4; i += kThreads) {
            const float4 v = __ldg(s4 + i);
            put(4 * i, v.x); put(4 * i + 1, v.y); put(4 * i + 2, v.z); put(4 * i + 3, v.w);
        }
        for (int i = 4 * n4 + threadIdx.x; i < count; i += kThreads) put(i, __ldg(src + i));
    } else {
        for (int i = threadIdx.x; i < count; i += kThreads) put(i, __ldg(src + i));
    }
}

template <int K>
__global__ void __launch_bounds__(kThreads) ply_records_kernel(const float* __restrict__ pos, const float* __restrict__ cov,
                                                               const float* __restrict__ shs, const float* __restrict__ opacity, int n,
                                                               float* __restrict__ records) {
    constexpr int W = 14 + 3 * K;                            // floats per record
    constexpr int S = 3 * K;                                 // SH floats per Gaussian
    constexpr int kOpacity = 6 + S, kScale = 7 + S;
    __shared__ __align__(16) float rec[kThreads * W];
    __shared__ float cv[kThreads * 6];
    const long long first = (long long)blockIdx.x * kThreads;
    const int nb = (int)min((long long)kThreads, n - first);

    load_span(pos + 3 * first, 3 * nb, [&](int e, float v) { rec[(e / 3) * W + e % 3] = v; });
    // shs[p][k][c] -> f_dc_c (k = 0) or f_rest_{c (K-1) + k - 1}: save_ply's transpose(1, 2).flatten
    load_span(shs + (long long)S * first, S * nb, [&](int e, float v) {
        const int j = e / S, r = e % S, k = r / 3, c = r % 3;
        rec[j * W + (k == 0 ? 6 + c : 9 + c * (K - 1) + (k - 1))] = v;
    });
    load_span(opacity + first, nb, [&](int e, float v) { rec[e * W + kOpacity] = v; });
    load_span(cov + 6 * first, 6 * nb, [&](int e, float v) { cv[e] = v; });
    __syncthreads();

    const int t = threadIdx.x;
    if (t < nb) {
        float* row = rec + t * W;
        row[3] = 0.0f; row[4] = 0.0f; row[5] = 0.0f;
        cov_to_scales_quat(cv + 6 * t, row + kScale);
    }
    __syncthreads();

    float* dst = records + W * first;
    const int count = W * nb;
    if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
        const int n4 = count >> 2;
        const float4* s4 = reinterpret_cast<const float4*>(rec);
        float4* d4 = reinterpret_cast<float4*>(dst);
        for (int i = t; i < n4; i += kThreads) d4[i] = s4[i];
        for (int i = 4 * n4 + t; i < count; i += kThreads) dst[i] = rec[i];
    } else {
        for (int i = t; i < count; i += kThreads) dst[i] = rec[i];
    }
}

template <int K>
void launch(const float* pos, const float* cov, const float* shs, const float* opacity, int n, float* records, cudaStream_t st) {
    ply_records_kernel<K><<<(n + kThreads - 1) / kThreads, kThreads, 0, st>>>(pos, cov, shs, opacity, n, records);
}

}  // namespace

cudaError_t gaussian_ply_records(const float* pos, const float* cov, const float* shs, int K, const float* opacity, int n, float* records,
                                 cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    switch (K) {
        case 1: launch<1>(pos, cov, shs, opacity, n, records, st); break;
        case 4: launch<4>(pos, cov, shs, opacity, n, records, st); break;
        case 9: launch<9>(pos, cov, shs, opacity, n, records, st); break;
        default: launch<16>(pos, cov, shs, opacity, n, records, st); break;
    }
    return cudaGetLastError();
}

}  // namespace pixie
