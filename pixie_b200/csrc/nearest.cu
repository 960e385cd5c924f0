// Exact nearest Gaussian of every filled particle: the search of get_attr_from_closest (PG/particle_filling/filling.py:
// 383-405), which the reference runs as a brute-force O(M N) Taichi loop:
//     min_dist = 1e10; min_idx = -1
//     for pj in 0..N-1: d = |q - p_j|; if d < min_dist: min_dist, min_idx = d, pj
// The answer here is the same argmin, bit for bit: d is float32 with one rounding per operation and no FMA,
// dx = q.x - p.x (likewise y, z), d = sqrt((dx*dx + dy*dy) + dz*dz) correctly rounded; ties go to the lowest index; -1
// when no Gaussian has d < 1e10 (no Gaussians, a non-finite query, or every Gaussian at least 1e10 away). A NaN or Inf
// Gaussian coordinate makes d NaN or Inf, which never wins, so such Gaussians are kept out of every bounding box.
//
// Queries are interior points and the Gaussians sit on a surface, so a query's nearest Gaussian can be half the object
// away; a uniform cell grid would walk (R / h)^3 empty cells. Instead, a bounding-volume tree over the Gaussians:
//   1. bounds    finite bounding box of the Gaussians (ordered-integer atomics)
//   2. sort      30-bit Morton codes over that box, cub radix sort of (code, index); non-finite Gaussians sort last
//   3. tree      leaves of 32 consecutive sorted Gaussians, an implicit complete binary tree (heap order, node 1 the
//                root, leaves at P .. 2P - 1) of float32 AABBs over them, built bottom up one level per launch
//   4. queries   sorted by Morton code too, so that neighbouring threads walk similar paths; each is seeded from the
//                leaf at its Morton position, then walks the tree nearest box first with a fixed-depth stack in shared
//                memory; results are scattered back to query order.
// The Morton codes decide only the order, never the answer: exactness rests on the pruning bound alone (see kSlack).
#include "nearest.cuh"

#include <cub/cub.cuh>
#include <cstdint>

namespace pixie {
namespace {

constexpr int kLeaf = 32;
constexpr int kStack = 32;                 // >= tree depth + 1: n < 2^31 gives P <= 2^26 leaves, depth <= 26
constexpr int kThreads = 128;
constexpr unsigned kNonFinite = 1u << 30;  // above every 30-bit Morton code
constexpr float kNone = 1e10f;             // the reference's initial min_dist

// Pruning. For a Gaussian at exact distance D, the float32 d above is D (1 + e) + a with |e| <= 3.5 * 2^-24 (five
// roundings under the square root: the difference twice through the square, the square, two sums; half of that after
// the root, plus the root's own rounding) and a <= 2^-74 (at most three squares that underflow, each off by <= 2^-150).
// A box is skipped only when its lower bound lb (fp64, from the float32 corners; relative error ~2^-50) exceeds both
// best_d (1 + 2^-19) and kFloor. 2^-19 is 32 units of 2^-24, so a skipped Gaussian has d > best_d: it can neither win nor
// tie. kFloor = 2^-50 >> 2^20 a covers a best_d small enough for the absolute term a to matter. A box whose bound merely
// equals best_d is visited, so an equal-d candidate with a lower index is found.
constexpr double kSlack = 1.0 + 0x1p-19;
constexpr double kFloor = 0x1p-50;

__device__ __forceinline__ unsigned enc_f(float f) {
    const unsigned u = __float_as_uint(f);
    return u ^ ((u >> 31) ? 0xffffffffu : 0x80000000u);
}
__device__ __forceinline__ float dec_f(unsigned k) { return __uint_as_float(k ^ ((k >> 31) ? 0x80000000u : 0xffffffffu)); }

__device__ __forceinline__ bool finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

// the reference's distance: float32, one rounding per operation, correctly rounded sqrt (nvcc contracts to FMA otherwise)
__device__ __forceinline__ float dist_f32(float qx, float qy, float qz, float px, float py, float pz) {
    const float dx = __fsub_rn(qx, px), dy = __fsub_rn(qy, py), dz = __fsub_rn(qz, pz);
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
}

__device__ __forceinline__ unsigned spread10(unsigned v) {      // 10 bits -> every third bit
    v &= 0x3ffu;
    v = (v | (v << 16)) & 0x030000ffu;
    v = (v | (v << 8)) & 0x0300f00fu;
    v = (v | (v << 4)) & 0x030c30c3u;
    v = (v | (v << 2)) & 0x09249249u;
    return v;
}

struct Frame {                       // the Gaussians' finite bounding box, as Morton quantisation
    float lo[3], scale[3];
};

__device__ __forceinline__ Frame load_frame(const unsigned* __restrict__ bounds) {
    Frame f;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float lo = dec_f(bounds[d]), hi = dec_f(bounds[3 + d]);
        const bool ok = hi > lo;     // false without finite Gaussians (the sentinels decode to NaN) or on a flat axis
        f.lo[d] = ok ? lo : 0.0f;
        f.scale[d] = ok ? 1023.0f / (hi - lo) : 0.0f;
    }
    return f;
}

__device__ __forceinline__ unsigned morton(const Frame& f, float x, float y, float z) {
    const float p[3] = {x, y, z};
    unsigned c[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) c[d] = (unsigned)fminf(fmaxf((p[d] - f.lo[d]) * f.scale[d], 0.0f), 1023.0f);   // NaN -> 0
    return (spread10(c[0]) << 2) | (spread10(c[1]) << 1) | spread10(c[2]);
}

__global__ void bounds_kernel(const float* __restrict__ pos, int n, unsigned* __restrict__ bounds) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float p[3] = {0.0f, 0.0f, 0.0f};
    bool ok = false;
    if (i < n) {
        p[0] = pos[3 * (size_t)i]; p[1] = pos[3 * (size_t)i + 1]; p[2] = pos[3 * (size_t)i + 2];
        ok = finite3(p[0], p[1], p[2]);
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const unsigned lo = __reduce_min_sync(0xffffffffu, ok ? enc_f(p[d]) : 0xffffffffu);
        const unsigned hi = __reduce_max_sync(0xffffffffu, ok ? enc_f(p[d]) : 0u);
        if ((threadIdx.x & 31) == 0 && lo != 0xffffffffu) { atomicMin(bounds + d, lo); atomicMax(bounds + 3 + d, hi); }
    }
}

__global__ void key_kernel(const float* __restrict__ pts, int n, const unsigned* __restrict__ bounds, bool skip_nonfinite,
                           unsigned* __restrict__ keys, int* __restrict__ vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Frame f = load_frame(bounds);
    const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
    keys[i] = skip_nonfinite && !finite3(x, y, z) ? kNonFinite : morton(f, x, y, z);
    vals[i] = i;
}

// sorted Gaussians as (x, y, z, original index)
__global__ void gather_kernel(const float* __restrict__ pos, const int* __restrict__ order, int n, float4* __restrict__ sp) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const int i = order[s];
    sp[s] = make_float4(pos[3 * (size_t)i], pos[3 * (size_t)i + 1], pos[3 * (size_t)i + 2], __int_as_float(i));
}

// leaf boxes over the finite Gaussians of each leaf; a leaf without any keeps the empty box (+Inf, -Inf), whose bound is Inf
__global__ void leaf_box_kernel(const float4* __restrict__ sp, int n, int P, float4* __restrict__ lo, float4* __restrict__ hi) {
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= P) return;
    float4 a = make_float4(INFINITY, INFINITY, INFINITY, 0.0f), b = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.0f);
    const int e = min(n, (l + 1) * kLeaf);
    for (int j = l * kLeaf; j < e; ++j) {
        const float4 p = sp[j];
        if (!finite3(p.x, p.y, p.z)) continue;
        a.x = fminf(a.x, p.x); a.y = fminf(a.y, p.y); a.z = fminf(a.z, p.z);
        b.x = fmaxf(b.x, p.x); b.y = fmaxf(b.y, p.y); b.z = fmaxf(b.z, p.z);
    }
    lo[P + l] = a;
    hi[P + l] = b;
}

// nodes [first, 2 first) from their children
__global__ void level_box_kernel(int first, float4* __restrict__ lo, float4* __restrict__ hi) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= first) return;
    const int v = first + k;
    const float4 a0 = lo[2 * v], a1 = lo[2 * v + 1], b0 = hi[2 * v], b1 = hi[2 * v + 1];
    lo[v] = make_float4(fminf(a0.x, a1.x), fminf(a0.y, a1.y), fminf(a0.z, a1.z), 0.0f);
    hi[v] = make_float4(fmaxf(b0.x, b1.x), fmaxf(b0.y, b1.y), fmaxf(b0.z, b1.z), 0.0f);
}

// squared fp64 distance from q to the box (Inf for an empty box)
__device__ __forceinline__ double box_lb2(const float4 lo, const float4 hi, double qx, double qy, double qz) {
    const double gx = fmax(fmax((double)lo.x - qx, qx - (double)hi.x), 0.0);
    const double gy = fmax(fmax((double)lo.y - qy, qy - (double)hi.y), 0.0);
    const double gz = fmax(fmax((double)lo.z - qz, qz - (double)hi.z), 0.0);
    return gx * gx + gy * gy + gz * gz;
}

__device__ __forceinline__ int lower_bound(const unsigned* __restrict__ a, int n, unsigned k) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] < k) lo = mid + 1; else hi = mid;
    }
    return lo;
}

struct Tree {
    const float4* sp;         // [n] sorted Gaussians
    const unsigned* keys;     // [n] their sorted codes
    const float4* lo;         // [2P] node boxes, heap order
    const float4* hi;
    int n, P;
};

__device__ __forceinline__ void scan_leaf(const Tree& t, int leaf, float qx, float qy, float qz, float& bd, int& bi) {
    const int e = min(t.n, (leaf + 1) * kLeaf);
    for (int j = leaf * kLeaf; j < e; ++j) {
        const float4 p = t.sp[j];
        const float d = dist_f32(qx, qy, qz, p.x, p.y, p.z);
        const int i = __float_as_int(p.w);
        if (d < bd || (d == bd && i < bi)) { bd = d; bi = i; }       // bi = -1 only while bd = 1e10: never tied
    }
}

__device__ __forceinline__ double prune_above(float bd) {
    const double r = fmax((double)bd * kSlack, kFloor);
    return r * r;
}

__global__ void __launch_bounds__(kThreads)
query_kernel(const Tree t, const float* __restrict__ query, const unsigned* __restrict__ qkeys, const int* __restrict__ qorder,
             int m, int* __restrict__ index) {
    // pending nodes and their squared bounds (rounded down to float: a smaller bound only visits more)
    __shared__ int stk_node[kStack][kThreads];
    __shared__ float stk_lb2[kStack][kThreads];
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= m) return;
    const int qi = qorder[s];
    const float qx = query[3 * (size_t)qi], qy = query[3 * (size_t)qi + 1], qz = query[3 * (size_t)qi + 2];
    if (!finite3(qx, qy, qz)) { index[qi] = -1; return; }      // every d is NaN or Inf
    float bd = kNone;
    int bi = -1;
    // seed: the leaf at the query's Morton position
    const int seed = min(lower_bound(t.keys, t.n, qkeys[s]), t.n - 1) / kLeaf;
    scan_leaf(t, seed, qx, qy, qz, bd, bi);
    double thr2 = prune_above(bd);
    const double dqx = qx, dqy = qy, dqz = qz;
    const int tid = threadIdx.x;
    int sp = 0;
    stk_node[0][tid] = 1;
    stk_lb2[0][tid] = 0.0f;
    sp = 1;
    while (sp > 0) {
        --sp;
        const int v = stk_node[sp][tid];
        if ((double)stk_lb2[sp][tid] > thr2) continue;
        if (v >= t.P) {
            const int leaf = v - t.P;
            if (leaf != seed) {
                scan_leaf(t, leaf, qx, qy, qz, bd, bi);
                thr2 = prune_above(bd);
            }
            continue;
        }
        const int c0 = 2 * v, c1 = 2 * v + 1;
        const double l0 = box_lb2(t.lo[c0], t.hi[c0], dqx, dqy, dqz);
        const double l1 = box_lb2(t.lo[c1], t.hi[c1], dqx, dqy, dqz);
        const bool first0 = l0 <= l1;                                 // the nearer child is popped first
        const int cn = first0 ? c0 : c1, cf = first0 ? c1 : c0;
        const double ln = first0 ? l0 : l1, lf = first0 ? l1 : l0;
        if (lf <= thr2) { stk_node[sp][tid] = cf; stk_lb2[sp][tid] = __double2float_rd(lf); ++sp; }
        if (ln <= thr2) { stk_node[sp][tid] = cn; stk_lb2[sp][tid] = __double2float_rd(ln); ++sp; }
    }
    index[qi] = bi;
}

struct Workspace {
    char* base = nullptr;
    size_t off = 0;
    template <class T> T* take(size_t count) {
        T* p = reinterpret_cast<T*>(base + off);
        off += (count * sizeof(T) + 255) & ~size_t(255);
        return p;
    }
};

}  // namespace

int nearest_gaussian(const float* pos, int n, const float* query, int m, int* index, cudaStream_t st) {
    if (m <= 0) return 0;
    if (n <= 0) return cudaMemsetAsync(index, 0xff, (size_t)m * sizeof(int), st) != cudaSuccess;
    const int L = (n + kLeaf - 1) / kLeaf;
    int P = 1;
    while (P < L) P <<= 1;
    size_t tb[2] = {0, 0};
    cub::DeviceRadixSort::SortPairs(nullptr, tb[0], (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr, n,
                                    0, 31, st);
    cub::DeviceRadixSort::SortPairs(nullptr, tb[1], (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr, m,
                                    0, 31, st);
    const size_t tmp_bytes = tb[0] > tb[1] ? tb[0] : tb[1];
    unsigned *bounds, *keys_in, *keys, *qkeys_in, *qkeys;
    int *vals_in, *order, *qvals_in, *qorder;
    float4 *sp, *lo, *hi;
    void* tmp;
    auto carve = [&](Workspace& w) {
        bounds = w.take<unsigned>(6); tmp = w.take<char>(tmp_bytes);
        keys_in = w.take<unsigned>(n); keys = w.take<unsigned>(n); vals_in = w.take<int>(n); order = w.take<int>(n);
        sp = w.take<float4>(n); lo = w.take<float4>(2 * (size_t)P); hi = w.take<float4>(2 * (size_t)P);
        qkeys_in = w.take<unsigned>(m); qkeys = w.take<unsigned>(m); qvals_in = w.take<int>(m); qorder = w.take<int>(m);
    };
    Workspace sizing;
    carve(sizing);
    Workspace w;
    if (cudaMallocAsync(reinterpret_cast<void**>(&w.base), sizing.off, st) != cudaSuccess) return 1;
    carve(w);

    const int B = 256;
    cudaMemsetAsync(bounds, 0xff, 3 * sizeof(unsigned), st);         // encoded +max for the minima
    cudaMemsetAsync(bounds + 3, 0, 3 * sizeof(unsigned), st);        // encoded -max for the maxima
    bounds_kernel<<<(n + B - 1) / B, B, 0, st>>>(pos, n, bounds);
    key_kernel<<<(n + B - 1) / B, B, 0, st>>>(pos, n, bounds, true, keys_in, vals_in);
    cub::DeviceRadixSort::SortPairs(tmp, tb[0], keys_in, keys, vals_in, order, n, 0, 31, st);
    gather_kernel<<<(n + B - 1) / B, B, 0, st>>>(pos, order, n, sp);
    leaf_box_kernel<<<(P + B - 1) / B, B, 0, st>>>(sp, n, P, lo, hi);
    for (int first = P / 2; first >= 1; first /= 2) level_box_kernel<<<(first + B - 1) / B, B, 0, st>>>(first, lo, hi);
    // non-finite queries get an ordinary (clamped) code here: they return -1 before using it
    key_kernel<<<(m + B - 1) / B, B, 0, st>>>(query, m, bounds, false, qkeys_in, qvals_in);
    cub::DeviceRadixSort::SortPairs(tmp, tb[1], qkeys_in, qkeys, qvals_in, qorder, m, 0, 31, st);
    const Tree t{sp, keys, lo, hi, n, P};
    query_kernel<<<(m + kThreads - 1) / kThreads, kThreads, 0, st>>>(t, query, qkeys, qorder, m, index);
    const int rc = cudaGetLastError() != cudaSuccess;
    cudaFreeAsync(w.base, st);
    return rc;
}

}  // namespace pixie
