// DBSCAN over a particle subset on the device: the clustering step of handle_stationary_clusters
// (PG/material_field.py:365-480), which the reference runs through scikit-learn's DBSCAN on the host.
//
// Semantics are scikit-learn's (sklearn.cluster.DBSCAN, Euclidean metric): neighbours of a point are the points whose
// fp64 squared distance is <= eps^2, the point itself included; core points have >= min_samples neighbours; clusters are
// the connected components of core points, labelled 0, 1, ... in the order of each component's smallest core index; a
// non-core point within eps of a core point takes the smallest label among those core points, every other point -1.
//
// Pipeline (workspace allocated per call; two small counts come back with one stream sync):
//   1. compaction  cub::DeviceSelect::Flagged over the index sequence (stable, so the subset keeps particle order)
//   2. binning     cells of edge eps * (1 + 1e-6) from the subset's own min corner, 21 bits per axis packed into a 64-bit
//                  key (indices clamped to [0, 2^21 - 1]: clamping only merges far cells, so a within-eps pair is never two
//                  cells apart), radix sort of (key, subset index), run-length encoding into unique keys + cell starts.
//                  The 3 z-neighbours of a cell are contiguous in key order, so a point's 27 neighbour cells are 9 point
//                  ranges found by binary search over the unique keys. No dense grid, no per-cell cap.
//   3. core        one thread per point in cell order (a warp mostly shares one candidate list, so loads broadcast);
//                  counting stops at min_samples.
//   4. components  lock-free union-find over core-core pairs (each pair once): hook the larger root under the smaller with
//                  atomicCAS, path halving on find. A component's root is therefore its smallest core index; labels are
//                  the exclusive scan of the root flags.
//   5. borders     minimum label over the core neighbours.
#include "cluster.cuh"
#include "workspace.cuh"

#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <climits>
#include <cstdint>

namespace pixie {
namespace {

constexpr int kCellBits = 21;
constexpr int kMaxCell = (1 << kCellBits) - 1;
constexpr unsigned long long kPadKey = ~0ull;     // sorts after every real key (those use 63 bits)
constexpr unsigned kFull = 0xffffffffu;

// float <-> unsigned with the same order (for atomicMin / atomicMax on floats)
__device__ __forceinline__ unsigned enc_f(float f) {
    const unsigned u = __float_as_uint(f);
    return u ^ ((u >> 31) ? 0xffffffffu : 0x80000000u);
}
__device__ __forceinline__ float dec_f(unsigned k) { return __uint_as_float(k ^ ((k >> 31) ? 0x80000000u : 0xffffffffu)); }

__device__ __forceinline__ unsigned long long cell_key(int cx, int cy, int cz) {
    return ((unsigned long long)cx << (2 * kCellBits)) | ((unsigned long long)cy << kCellBits) | (unsigned long long)cz;
}

// sklearn's KD-tree rdist: ((dx^2 + dy^2) + dz^2) in fp64, rounded after every operation (no FMA contraction)
__device__ __forceinline__ bool within(const float4 a, const float4 b, double eps2) {
    const double dx = (double)a.x - (double)b.x, dy = (double)a.y - (double)b.y, dz = (double)a.z - (double)b.z;
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)) <= eps2;
}

struct Grid {
    const float4* sp;                    // [N] points in cell order: xyz, subset index (int bits) in w
    const unsigned long long* uniq;      // [R] unique cell keys (the last one is kPadKey when the subset is smaller than N)
    const int* start;                    // [R + 1] first sorted position of each cell
    const int* n_runs;                   // R (device)
    const int* m;                        // subset size M (device)
    double eps2;
};

__device__ __forceinline__ int lower_bound(const unsigned long long* a, int n, unsigned long long k) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] < k) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// calls f(j) for every sorted position j in the 27 cells around the cell of key `key`
template <class F>
__device__ __forceinline__ void for_each_candidate(const Grid& g, unsigned long long key, F&& f) {
    const int cx = (int)(key >> (2 * kCellBits)), cy = (int)((key >> kCellBits) & kMaxCell), cz = (int)(key & kMaxCell);
    const int R = *g.n_runs;
    const int z0 = max(cz - 1, 0), z1 = min(cz + 1, kMaxCell);
    for (int nx = max(cx - 1, 0); nx <= min(cx + 1, kMaxCell); ++nx)
        for (int ny = max(cy - 1, 0); ny <= min(cy + 1, kMaxCell); ++ny) {
            const int lo = lower_bound(g.uniq, R, cell_key(nx, ny, z0));
            const int hi = lower_bound(g.uniq, R, cell_key(nx, ny, z1) + 1);
            const int e = g.start[hi];
            for (int j = g.start[lo]; j < e; ++j)
                if (!f(j)) return;
        }
}

__global__ void flag_kernel(const int* __restrict__ ids, int n, int select_id, int* __restrict__ flags) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flags[i] = ids ? (ids[i] == select_id ? 1 : 0) : 1;
}

// min corner of the subset (ordered-integer atomics, one per warp and axis)
__global__ void min_corner_kernel(const float* __restrict__ pos, const int* __restrict__ index, const int* __restrict__ m_dev, int n,
                                  unsigned* __restrict__ mn) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int m = *m_dev;
    unsigned e[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu};
    if (t < m) {
        const int i = index[t];
#pragma unroll
        for (int d = 0; d < 3; ++d) e[d] = enc_f(pos[3 * (size_t)i + d]);
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const unsigned r = __reduce_min_sync(kFull, e[d]);
        if ((threadIdx.x & 31) == 0 && r != 0xffffffffu) atomicMin(mn + d, r);
    }
}

__global__ void key_kernel(const float* __restrict__ pos, const int* __restrict__ index, const int* __restrict__ m_dev, int n,
                           const unsigned* __restrict__ mn, double cell, unsigned long long* __restrict__ keys, int* __restrict__ vals) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    vals[t] = t;
    if (t >= *m_dev) { keys[t] = kPadKey; return; }
    const int i = index[t];
    int c[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const double q = floor(((double)pos[3 * (size_t)i + d] - (double)dec_f(mn[d])) / cell);
        c[d] = (int)fmin(fmax(q, 0.0), (double)kMaxCell);      // fmax also maps NaN to 0
    }
    keys[t] = cell_key(c[0], c[1], c[2]);
}

__global__ void gather_kernel(const float* __restrict__ pos, const int* __restrict__ index, const int* __restrict__ m_dev, int n,
                              const int* __restrict__ order, float4* __restrict__ sp) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n || s >= *m_dev) return;
    const int t = order[s];
    const float* p = pos + 3 * (size_t)index[t];
    sp[s] = make_float4(p[0], p[1], p[2], __int_as_float(t));
}

__global__ void __launch_bounds__(256) core_kernel(const Grid g, const unsigned long long* __restrict__ skeys, int n, int min_samples,
                                                   uint8_t* __restrict__ core_s, uint8_t* __restrict__ core_t, int* __restrict__ parent) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n || s >= *g.m) return;
    const float4 a = g.sp[s];
    int cnt = 0;
    for_each_candidate(g, skeys[s], [&](int j) {
        if (within(a, g.sp[j], g.eps2)) ++cnt;
        return cnt < min_samples;
    });
    const int t = __float_as_int(a.w);
    const uint8_t c = cnt >= min_samples ? 1 : 0;
    core_s[s] = c;
    core_t[t] = c;
    parent[t] = t;
}

// find with path halving. Only roots are ever hooked (by CAS), and a parent is never larger than its child, so the plain
// stores below can only replace a non-root's parent by one of its ancestors.
__device__ __forceinline__ int uf_find(volatile int* par, int x) {
    int next = par[x];
    while (next != x) {
        const int nn = par[next];
        if (nn != next) par[x] = nn;
        x = next;
        next = nn;
    }
    return x;
}

__device__ __forceinline__ void uf_union(int* par, int a, int b) {
    volatile int* vp = par;
    while (true) {
        a = uf_find(vp, a);
        b = uf_find(vp, b);
        if (a == b) return;
        const int lo = min(a, b), hi = max(a, b);
        if (atomicCAS(par + hi, hi, lo) == hi) return;       // hi was still a root: hooked under lo
        a = lo; b = hi;                                       // someone hooked hi meanwhile: retry from the new roots
    }
}

__global__ void __launch_bounds__(256) union_kernel(const Grid g, const unsigned long long* __restrict__ skeys, int n,
                                                    const uint8_t* __restrict__ core_s, int* parent) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n || s >= *g.m || !core_s[s]) return;
    const float4 a = g.sp[s];
    const int t = __float_as_int(a.w);
    for_each_candidate(g, skeys[s], [&](int j) {
        if (core_s[j]) {
            const float4 b = g.sp[j];
            const int u = __float_as_int(b.w);
            if (u < t && within(a, b, g.eps2)) uf_union(parent, t, u);
        }
        return true;
    });
}

__global__ void root_kernel(const int* __restrict__ m_dev, int n, const uint8_t* __restrict__ core_t, int* parent, int* __restrict__ root_flag) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n || t >= *m_dev) return;
    if (!core_t[t]) { root_flag[t] = 0; return; }
    const int r = uf_find(parent, t);
    root_flag[t] = r == t ? 1 : 0;
    parent[t] = r;                                            // flattened for label_kernel
}

__global__ void label_kernel(const int* __restrict__ m_dev, int n, const uint8_t* __restrict__ core_t, const int* __restrict__ parent,
                             const int* __restrict__ root_rank, int* __restrict__ labels) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n || t >= *m_dev) return;
    labels[t] = core_t[t] ? root_rank[parent[t]] : -1;
}

__global__ void __launch_bounds__(256) border_kernel(const Grid g, const unsigned long long* __restrict__ skeys, int n,
                                                     const uint8_t* __restrict__ core_s, int* labels) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n || s >= *g.m || core_s[s]) return;
    const float4 a = g.sp[s];
    int best = INT_MAX;
    for_each_candidate(g, skeys[s], [&](int j) {
        if (core_s[j]) {
            const float4 b = g.sp[j];
            if (within(a, b, g.eps2)) best = min(best, labels[__float_as_int(b.w)]);     // core labels only: no race
        }
        return true;
    });
    labels[__float_as_int(a.w)] = best == INT_MAX ? -1 : best;
}

// one warp-aggregated atomic per (warp, label) group
__global__ void stats_kernel(const float* __restrict__ pos, const int* __restrict__ index, const int* __restrict__ labels, int m,
                             int* __restrict__ sizes, unsigned* __restrict__ bmin, unsigned* __restrict__ bmax) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int l = t < m ? labels[t] : -1;
    unsigned e[3] = {0, 0, 0};
    if (l >= 0) {
        const int i = index[t];
#pragma unroll
        for (int d = 0; d < 3; ++d) e[d] = enc_f(pos[3 * (size_t)i + d]);
    }
    const int lane = threadIdx.x & 31;
    unsigned todo = __ballot_sync(kFull, l >= 0);
    while (todo) {
        const int L = __shfl_sync(kFull, l, __ffs(todo) - 1);
        const bool mine = l == L;
        const unsigned grp = __ballot_sync(kFull, mine);
        unsigned lo[3], hi[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            lo[d] = __reduce_min_sync(kFull, mine ? e[d] : 0xffffffffu);
            hi[d] = __reduce_max_sync(kFull, mine ? e[d] : 0u);
        }
        if (lane == __ffs(grp) - 1) {
            atomicAdd(sizes + L, __popc(grp));
#pragma unroll
            for (int d = 0; d < 3; ++d) { atomicMin(bmin + 3 * L + d, lo[d]); atomicMax(bmax + 3 * L + d, hi[d]); }
        }
        todo &= ~grp;
    }
}

__global__ void decode_kernel(unsigned* __restrict__ a, unsigned* __restrict__ b, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        a[i] = __float_as_uint(dec_f(a[i]));
        b[i] = __float_as_uint(dec_f(b[i]));
    }
}

}  // namespace

cudaError_t dbscan(const float* pos, int n, const int* ids, int select_id, double eps, int min_samples, int* index, int* labels,
                   int* n_selected_host, int* n_clusters_host, cudaStream_t st) {
    if (n <= 0) { *n_selected_host = 0; *n_clusters_host = 0; return cudaSuccess; }
    const size_t N = (size_t)n;
    // sizes of every cub call, then one allocation for everything
    size_t tb[5] = {0, 0, 0, 0, 0};
    thrust::counting_iterator<int> iota(0);
    PIXIE_TRY(cub::DeviceSelect::Flagged(nullptr, tb[0], iota, (const int*)nullptr, (int*)nullptr, (int*)nullptr, n, st));
    PIXIE_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb[1], (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                              (const int*)nullptr, (int*)nullptr, n, 0, 64, st));
    PIXIE_TRY(cub::DeviceRunLengthEncode::Encode(nullptr, tb[2], (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                                 (int*)nullptr, (int*)nullptr, n, st));
    PIXIE_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb[3], (const int*)nullptr, (int*)nullptr, n + 1, st));
    size_t tmp_bytes = 0;
    for (size_t b : tb) tmp_bytes = b > tmp_bytes ? b : tmp_bytes;
    int *counts, *n_runs, *flags, *vals_in, *order, *run_len, *start, *parent, *root_flag, *root_rank;   // counts = {M, n_clusters}
    unsigned* mn;
    void* tmp;
    unsigned long long *keys_in, *keys, *uniq;
    float4* sp;
    uint8_t *core_s, *core_t;
    Workspace w(st);
    PIXIE_TRY(w.carve([&] {
        counts = w.take<int>(2); mn = w.take<unsigned>(3); n_runs = w.take<int>(1); tmp = w.take<char>(tmp_bytes);
        flags = w.take<int>(N); keys_in = w.take<unsigned long long>(N); keys = w.take<unsigned long long>(N);
        uniq = w.take<unsigned long long>(N); vals_in = w.take<int>(N); order = w.take<int>(N); run_len = w.take<int>(N + 1);
        start = w.take<int>(N + 1); sp = w.take<float4>(N); core_s = w.take<uint8_t>(N); core_t = w.take<uint8_t>(N);
        parent = w.take<int>(N); root_flag = w.take<int>(N + 1); root_rank = w.take<int>(N + 1);
    }));

    const int B = 256, G = (int)((N + B - 1) / B);
    const double cell = eps * (1.0 + 1e-6);
    PIXIE_TRY(cudaMemsetAsync(mn, 0xff, 3 * sizeof(unsigned), st));
    PIXIE_TRY(cudaMemsetAsync(run_len, 0, (N + 1) * sizeof(int), st));
    PIXIE_TRY(cudaMemsetAsync(root_flag, 0, (N + 1) * sizeof(int), st));
    flag_kernel<<<G, B, 0, st>>>(ids, n, select_id, flags);
    PIXIE_TRY(cub::DeviceSelect::Flagged(tmp, tb[0], iota, flags, index, counts, n, st));
    min_corner_kernel<<<G, B, 0, st>>>(pos, index, counts, n, mn);
    key_kernel<<<G, B, 0, st>>>(pos, index, counts, n, mn, cell, keys_in, vals_in);
    PIXIE_TRY(cub::DeviceRadixSort::SortPairs(tmp, tb[1], keys_in, keys, vals_in, order, n, 0, 64, st));
    PIXIE_TRY(cub::DeviceRunLengthEncode::Encode(tmp, tb[2], keys, uniq, run_len, n_runs, n, st));
    PIXIE_TRY(cub::DeviceScan::ExclusiveSum(tmp, tb[3], run_len, start, n + 1, st));
    gather_kernel<<<G, B, 0, st>>>(pos, index, counts, n, order, sp);
    Grid g{sp, uniq, start, n_runs, counts, eps * eps};
    core_kernel<<<G, B, 0, st>>>(g, keys, n, min_samples, core_s, core_t, parent);
    union_kernel<<<G, B, 0, st>>>(g, keys, n, core_s, parent);
    root_kernel<<<G, B, 0, st>>>(counts, n, core_t, parent, root_flag);
    PIXIE_TRY(cub::DeviceScan::ExclusiveSum(tmp, tb[3], root_flag, root_rank, n + 1, st));
    label_kernel<<<G, B, 0, st>>>(counts, n, core_t, parent, root_rank, labels);
    border_kernel<<<G, B, 0, st>>>(g, keys, n, core_s, labels);
    PIXIE_TRY(cudaMemcpyAsync(counts + 1, root_rank + N, sizeof(int), cudaMemcpyDeviceToDevice, st));
    int host[2] = {0, 0};
    PIXIE_TRY(cudaMemcpyAsync(host, counts, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
    PIXIE_TRY(cudaStreamSynchronize(st));
    *n_selected_host = host[0];
    *n_clusters_host = host[1];
    return cudaGetLastError();
}

cudaError_t cluster_stats(const float* pos, const int* index, const int* labels, int n_selected, int n_clusters, int* sizes,
                          float* bbox_min, float* bbox_max, cudaStream_t st) {
    if (n_clusters <= 0) return cudaSuccess;
    PIXIE_TRY(cudaMemsetAsync(sizes, 0, (size_t)n_clusters * sizeof(int), st));
    PIXIE_TRY(cudaMemsetAsync(bbox_min, 0xff, (size_t)n_clusters * 3 * sizeof(float), st));     // encoded +max
    PIXIE_TRY(cudaMemsetAsync(bbox_max, 0, (size_t)n_clusters * 3 * sizeof(float), st));        // encoded -max
    unsigned* lo = reinterpret_cast<unsigned*>(bbox_min);
    unsigned* hi = reinterpret_cast<unsigned*>(bbox_max);
    if (n_selected > 0) stats_kernel<<<(n_selected + 255) / 256, 256, 0, st>>>(pos, index, labels, n_selected, sizes, lo, hi);
    decode_kernel<<<(3 * n_clusters + 255) / 256, 256, 0, st>>>(lo, hi, 3 * n_clusters);
    return cudaGetLastError();
}

}  // namespace pixie
