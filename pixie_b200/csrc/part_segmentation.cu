// CLIP part similarities of the VLM part segmentation: run_clip and the label choice of clip_part_segmentation
// (pixie/voxel/segmentation.py:98-183). The reference copies the fp16 (D, D, D, C) grid to fp32, normalises it, runs a
// matmul against the unit query embeddings and a softmax. Here one pass reads each occupied voxel's C fp16 features once:
//   1. compact   cub::DeviceSelect over the mask gives the occupied voxel indices in C order (skipped without a mask)
//   2. similarity one warp per voxel (V voxels per warp for small P): lane l holds channels 8l .. 8l + 7 of each 256-channel
//                tile (one 16 B load when C % 8 == 0 and the features are 16 B aligned, else eight 2 B loads; the next
//                tile's loads are issued before the current tile is used), and
//                accumulates in fp32 the squared norm and the P dot products against the unit queries, which sit in
//                shared memory as fp32, permuted so that a warp's float4 reads are conflict-free. The P sums are reduced
//                across the warp by recursive halving, after which lane l holds part l (and l + 32): it writes the
//                similarity, and the warp forms the softmax and the argmax from the lanes' values.
// No fp32 copy of the grid exists: the features are converted in registers.
#include "part_segmentation.cuh"
#include "workspace.cuh"

#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <algorithm>
#include <cfloat>
#include <climits>

namespace pixie {
namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kTileC = 256;                          // channels per tile: 8 per lane
constexpr size_t kResidentBytes = 200 * 1024;        // all query tiles stay in shared memory up to this size

// the 8 halves at channels c0 .. c0 + 7 of a row, zero past C or for a row that is not there (ok false)
template <bool VEC>
__device__ __forceinline__ uint4 load8(const __half* __restrict__ feat, long long row, int C, int c0, bool ok) {
    const __half* src = feat + row * C + c0;
    uint4 u = make_uint4(0u, 0u, 0u, 0u);
    if constexpr (VEC) {
        if (ok && c0 < C) u = __ldg(reinterpret_cast<const uint4*>(src));
    } else {
        __half h[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) h[j] = ok && c0 + j < C ? src[j] : __float2half(0.0f);
        u = *reinterpret_cast<const uint4*>(h);
    }
    return u;
}

__device__ __forceinline__ void widen8(uint4 u, float x[8]) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float2 f = __half22float2(h[j]); x[2 * j] = f.x; x[2 * j + 1] = f.y; }
}

// the a (val, part) pair beats b under torch.argmax: a NaN beats a number, then the larger value, then the lower part
__device__ __forceinline__ bool arg_better(float a, int pa, float b, int pb) {
    const bool an = isnan(a), bn = isnan(b);
    if (an != bn) return an;
    if (!an && a != b) return a > b;
    return pa < pb;
}

// Sums a[] over the warp so that a[h * PW] ends up holding the total of part h * PW + (lane % PW). Lane groups wider than PW
// first add whole arrays (O >= PW), then each halving step O < PW keeps one half of the parts and adds the partner's.
template <int PMAX, int PW, int O>
__device__ __forceinline__ void reduce_parts(float (&a)[PMAX], int lane) {
    if constexpr (O >= 1) {
        if constexpr (O >= PW) {
#pragma unroll
            for (int i = 0; i < PMAX; ++i) a[i] += __shfl_xor_sync(0xffffffffu, a[i], O);
        } else {
            const bool upper = (lane & O) != 0;
#pragma unroll
            for (int h = 0; h < PMAX / PW; ++h)
#pragma unroll
                for (int i = 0; i < O; ++i) {
                    const float lo = a[h * PW + i], hi = a[h * PW + i + O];
                    a[h * PW + i] = (upper ? hi : lo) + __shfl_xor_sync(0xffffffffu, upper ? lo : hi, O);
                }
        }
        reduce_parts<PMAX, PW, O / 2>(a, lane);
    }
}

// PMAX: parts rounded up to 8, 16, 32 or 64; V: voxels per warp; VEC: 16 B feature loads
template <int PMAX, int V, bool VEC>
__global__ void __launch_bounds__(kThreads, 2)
similarity_kernel(const __half* __restrict__ feat, const int* __restrict__ idx, const int* __restrict__ n_found, int n, int C,
                  const float* __restrict__ query, int P, int n_tiles, bool resident, float inv_t, float* __restrict__ sims,
                  int64_t* __restrict__ labels, float* __restrict__ scores, float* __restrict__ probs) {
    extern __shared__ float4 qs[];                   // [tiles held][P][2][32]: channel 8l + 4h + j of part p at [p][h][l].j
    constexpr int PW = PMAX < 32 ? PMAX : 32;        // parts per lane group after the reduction
    constexpr int H = PMAX / PW;                     // parts per lane (1, or 2 at PMAX = 64)
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int rows = n_found ? min(n, *n_found) : n;
    const int tile_f4 = P * 64;
    auto load_tile = [&](int t, float4* dst) {
        for (int e = threadIdx.x; e < tile_f4; e += kThreads) {
            const int p = e >> 6, h = (e >> 5) & 1, l = e & 31;
            const int c0 = t * kTileC + 8 * l + 4 * h;
            const float* src = query + (size_t)p * C;
            dst[e] = make_float4(c0 < C ? src[c0] : 0.0f, c0 + 1 < C ? src[c0 + 1] : 0.0f, c0 + 2 < C ? src[c0 + 2] : 0.0f,
                                 c0 + 3 < C ? src[c0 + 3] : 0.0f);
        }
    };
    if (resident) {
        for (int t = 0; t < n_tiles; ++t) load_tile(t, qs + (size_t)t * tile_f4);
        __syncthreads();
    }
    const int group = kWarps * V;
    for (int base = blockIdx.x * group; base < rows; base += gridDim.x * group) {     // uniform over the block
        float sq[V], acc[V][PMAX];
        long long row[V];
        bool ok[V];
#pragma unroll
        for (int v = 0; v < V; ++v) {
            const int r = base + w * V + v;
            ok[v] = r < rows;
            row[v] = ok[v] ? (idx ? idx[r] : r) : 0;
            sq[v] = 0.0f;
#pragma unroll
            for (int p = 0; p < PMAX; ++p) acc[v][p] = 0.0f;
        }
        uint4 next[V];                               // the next tile's features, loaded one tile ahead
#pragma unroll
        for (int v = 0; v < V; ++v) next[v] = load8<VEC>(feat, row[v], C, 8 * lane, ok[v]);
        for (int t = 0; t < n_tiles; ++t) {
            const float4* qt = qs + (size_t)t * tile_f4;
            if (!resident) {
                __syncthreads();
                load_tile(t, qs);
                __syncthreads();
                qt = qs;
            }
            float x[V][8];
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const uint4 cur = next[v];
                if (t + 1 < n_tiles) next[v] = load8<VEC>(feat, row[v], C, (t + 1) * kTileC + 8 * lane, ok[v]);
                widen8(cur, x[v]);
#pragma unroll
                for (int j = 0; j < 8; ++j) sq[v] = fmaf(x[v][j], x[v][j], sq[v]);
            }
#pragma unroll
            for (int p = 0; p < PMAX; ++p) {
                if (p < P) {
                    const float4 a = qt[p * 64 + lane], b = qt[p * 64 + 32 + lane];
#pragma unroll
                    for (int v = 0; v < V; ++v) {
                        float s = acc[v][p];
                        s = fmaf(x[v][0], a.x, s); s = fmaf(x[v][1], a.y, s); s = fmaf(x[v][2], a.z, s); s = fmaf(x[v][3], a.w, s);
                        s = fmaf(x[v][4], b.x, s); s = fmaf(x[v][5], b.y, s); s = fmaf(x[v][6], b.z, s); s = fmaf(x[v][7], b.w, s);
                        acc[v][p] = s;
                    }
                }
            }
        }
#pragma unroll
        for (int v = 0; v < V; ++v) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) sq[v] += __shfl_xor_sync(0xffffffffu, sq[v], o);
            reduce_parts<PMAX, PW, 16>(acc[v], lane);
            const float* a = acc[v];
            if (!ok[v]) continue;                    // uniform over the warp
            const int r = base + w * V + v;
            const float nrm = sqrtf(sq[v]);
            float sim[H], z[H], e[H];
            bool own[H];
            float m = -INFINITY;
#pragma unroll
            for (int h = 0; h < H; ++h) {
                const int p = h * PW + (lane & (PW - 1));
                own[h] = lane < PW && p < P;
                sim[h] = a[h * PW] / nrm;
                z[h] = __fmul_rn(sim[h], inv_t);     // rounded on its own, as torch's sims / T, not fused into x - m
                if (own[h]) m = fmaxf(m, z[h]);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
            float sum = 0.0f;
#pragma unroll
            for (int h = 0; h < H; ++h) {
                e[h] = own[h] ? expf(__fsub_rn(z[h], m)) : 0.0f;
                sum += e[h];
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
            float best = -INFINITY;
            int bp = INT_MAX;
#pragma unroll
            for (int h = 0; h < H; ++h) {
                if (!own[h]) continue;
                const int p = h * PW + lane;
                const float pr = e[h] / sum;
                sims[(size_t)r * P + p] = sim[h];
                if (probs) probs[(size_t)r * P + p] = pr;
                if (arg_better(pr, p, best, bp)) { best = pr; bp = p; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best, o);
                const int op = __shfl_xor_sync(0xffffffffu, bp, o);
                if (arg_better(ob, op, best, bp)) { best = ob; bp = op; }
            }
            if (lane == 0) { labels[r] = bp; scores[r] = best; }
        }
    }
}

template <int PMAX, int V, bool VEC>
cudaError_t launch(const __half* feat, const int* idx, const int* n_found, int n, int C, const float* query, int P, float inv_t,
                   float* sims, int64_t* labels, float* scores, float* probs, cudaStream_t st) {
    auto kern = similarity_kernel<PMAX, V, VEC>;
    const int n_tiles = (C + kTileC - 1) / kTileC;
    const size_t tile_bytes = (size_t)P * 64 * sizeof(float4);
    const bool resident = (size_t)n_tiles * tile_bytes <= kResidentBytes;
    const size_t smem = resident ? (size_t)n_tiles * tile_bytes : tile_bytes;
    int dev = 0, sms = 0, per_sm = 0;
    PIXIE_TRY(cudaGetDevice(&dev));
    PIXIE_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    PIXIE_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PIXIE_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, smem));
    const int group = kWarps * V;
    const int blocks = std::max(1, std::min((n + group - 1) / group, sms * std::max(per_sm, 1)));
    kern<<<blocks, kThreads, smem, st>>>(feat, idx, n_found, n, C, query, P, n_tiles, resident, inv_t, sims, labels, scores, probs);
    return cudaGetLastError();
}

template <int PMAX, int V>
cudaError_t launch_vec(bool vec, const __half* feat, const int* idx, const int* n_found, int n, int C, const float* query, int P,
                       float inv_t, float* sims, int64_t* labels, float* scores, float* probs, cudaStream_t st) {
    return vec ? launch<PMAX, V, true>(feat, idx, n_found, n, C, query, P, inv_t, sims, labels, scores, probs, st)
               : launch<PMAX, V, false>(feat, idx, n_found, n, C, query, P, inv_t, sims, labels, scores, probs, st);
}

}  // namespace

cudaError_t part_similarity(const __half* feat, const uint8_t* mask, int64_t V, int C, int n_occupied, const float* query, int P,
                            float inv_t, float* sims, int64_t* labels, float* scores, float* probs, cudaStream_t st) {
    if (n_occupied <= 0 || V <= 0) return cudaSuccess;
    int* idx = nullptr;
    int* n_found = nullptr;
    Workspace w(st);
    if (mask) {
        size_t tmp_bytes = 0;
        const thrust::counting_iterator<int> iota(0);
        PIXIE_TRY(cub::DeviceSelect::Flagged(nullptr, tmp_bytes, iota, mask, (int*)nullptr, (int*)nullptr, (int)V, st));
        void* tmp;
        PIXIE_TRY(w.carve([&] { idx = w.take<int>((size_t)V); n_found = w.take<int>(1); tmp = w.take<char>(tmp_bytes); }));
        PIXIE_TRY(cub::DeviceSelect::Flagged(tmp, tmp_bytes, iota, mask, idx, n_found, (int)V, st));
    }
    const int n = mask ? n_occupied : (int)std::min<int64_t>(n_occupied, V);
    const bool vec = C % 8 == 0 && reinterpret_cast<uintptr_t>(feat) % 16 == 0;
    if (P <= 8) return launch_vec<8, 4>(vec, feat, idx, n_found, n, C, query, P, inv_t, sims, labels, scores, probs, st);
    if (P <= 16) return launch_vec<16, 2>(vec, feat, idx, n_found, n, C, query, P, inv_t, sims, labels, scores, probs, st);
    if (P <= 32) return launch_vec<32, 2>(vec, feat, idx, n_found, n, C, query, P, inv_t, sims, labels, scores, probs, st);
    return launch_vec<64, 1>(vec, feat, idx, n_found, n, C, query, P, inv_t, sims, labels, scores, probs, st);
}

}  // namespace pixie
