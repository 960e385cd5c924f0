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
//
// The same tree answers two searches of the VLM part segmentation (pixie/voxel/segmentation.py), both on fp64 squared
// distances d2 = (dx*dx + dy*dy) + dz*dz, one rounding per operation, as scipy's cKDTree and scikit-learn's KDTree form them:
//   nearest_vertex  the nearest float64 occupancy vertex of every voxel (save_segmented_point_cloud's colour lookup); the
//                   tree holds the vertices rounded outward to float32 boxes and reads the fp64 coordinates to compare
//   knn_label_vote  the k nearest voxels of every voxel, self included, by (d2, index), and the mode of their labels
//                   (local_post_process_segmentation); one warp per query, one lane per leaf point, the candidates in a
//                   per-warp buffer that a radix select cuts back to the best k whenever it fills
#include "nearest.cuh"
#include "workspace.cuh"

#include <cub/cub.cuh>
#include <algorithm>
#include <cfloat>
#include <climits>
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

__device__ __forceinline__ bool finite3(double x, double y, double z) { return isfinite(x) && isfinite(y) && isfinite(z); }

// T = float (Gaussians, voxels) or double (occupancy vertices: their codes and bounds use the float32 rounding, which only
// orders them; a finite vertex past the float range is clamped to the frame's edge)
template <class T>
__global__ void bounds_kernel(const T* __restrict__ pos, int n, unsigned* __restrict__ bounds) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float p[3] = {0.0f, 0.0f, 0.0f};
    bool ok = false;
    if (i < n) {
        ok = finite3(pos[3 * (size_t)i], pos[3 * (size_t)i + 1], pos[3 * (size_t)i + 2]);
        p[0] = (float)pos[3 * (size_t)i]; p[1] = (float)pos[3 * (size_t)i + 1]; p[2] = (float)pos[3 * (size_t)i + 2];
        if (ok && !finite3(p[0], p[1], p[2])) {
#pragma unroll
            for (int d = 0; d < 3; ++d) p[d] = fminf(fmaxf(p[d], -FLT_MAX), FLT_MAX);
        }
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const unsigned lo = __reduce_min_sync(0xffffffffu, ok ? enc_f(p[d]) : 0xffffffffu);
        const unsigned hi = __reduce_max_sync(0xffffffffu, ok ? enc_f(p[d]) : 0u);
        if ((threadIdx.x & 31) == 0 && lo != 0xffffffffu) { atomicMin(bounds + d, lo); atomicMax(bounds + 3 + d, hi); }
    }
}

template <class T>
__global__ void key_kernel(const T* __restrict__ pts, int n, const unsigned* __restrict__ bounds, bool skip_nonfinite,
                           unsigned* __restrict__ keys, int* __restrict__ vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Frame f = load_frame(bounds);
    const T x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
    keys[i] = skip_nonfinite && !finite3(x, y, z) ? kNonFinite : morton(f, (float)x, (float)y, (float)z);
    vals[i] = i;
}

// sorted points as (x, y, z, original index); fp64 points also as sorted fp64 coordinates sd [n][3]
template <class T>
__global__ void gather_kernel(const T* __restrict__ pos, const int* __restrict__ order, int n, float4* __restrict__ sp,
                              double* __restrict__ sd) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const int i = order[s];
    sp[s] = make_float4((float)pos[3 * (size_t)i], (float)pos[3 * (size_t)i + 1], (float)pos[3 * (size_t)i + 2], __int_as_float(i));
    if (sd) { sd[3 * (size_t)s] = pos[3 * (size_t)i]; sd[3 * (size_t)s + 1] = pos[3 * (size_t)i + 1]; sd[3 * (size_t)s + 2] = pos[3 * (size_t)i + 2]; }
}

// leaf boxes over the finite points of each leaf; a leaf without any keeps the empty box (+Inf, -Inf), whose bound is Inf.
// fp64 points are boxed from sd, rounded outward to float32, so the box still holds them.
__global__ void leaf_box_kernel(const float4* __restrict__ sp, const double* __restrict__ sd, int n, int P, float4* __restrict__ lo,
                                float4* __restrict__ hi) {
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= P) return;
    float4 a = make_float4(INFINITY, INFINITY, INFINITY, 0.0f), b = make_float4(-INFINITY, -INFINITY, -INFINITY, 0.0f);
    const int e = min(n, (l + 1) * kLeaf);
    for (int j = l * kLeaf; j < e; ++j) {
        if (sd) {
            const double x = sd[3 * (size_t)j], y = sd[3 * (size_t)j + 1], z = sd[3 * (size_t)j + 2];
            if (!finite3(x, y, z)) continue;
            a.x = fminf(a.x, __double2float_rd(x)); a.y = fminf(a.y, __double2float_rd(y)); a.z = fminf(a.z, __double2float_rd(z));
            b.x = fmaxf(b.x, __double2float_ru(x)); b.y = fmaxf(b.y, __double2float_ru(y)); b.z = fmaxf(b.z, __double2float_ru(z));
            continue;
        }
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
    const float4* sp;         // [n] sorted points
    const double* sd;         // [n][3] their fp64 coordinates (fp64 points only, else null)
    const unsigned* keys;     // [n] their sorted codes
    const float4* lo;         // [2P] node boxes, heap order
    const float4* hi;
    int n, P;
};

// Pruning of the fp64 searches. d2 is the squared distance to a point, lb2 that to a box, both from exact float32 or
// float64 inputs with at most five roundings of relative size 2^-53, so each is within (1 +- 2^-50) of its exact value
// (a difference of two float32 that is not exact in fp64 only adds one more such rounding). A box is skipped only when lb2
// exceeds both thr * (1 + 2^-40) and 2^-900: every point in it then has d2 > thr, so it can neither beat nor tie the
// threshold. The floor covers the absolute error of squares that fall below the normal range.
constexpr double kSlack64 = 1.0 + 0x1p-40;
constexpr double kFloor64 = 0x1p-900;

__device__ __forceinline__ double d2_f64(double qx, double qy, double qz, double px, double py, double pz) {
    const double dx = __dsub_rn(qx, px), dy = __dsub_rn(qy, py), dz = __dsub_rn(qz, pz);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// Scans the sorted points of a leaf below n_scan. F64 = false: the float32 distance d of nearest_gaussian, initial best
// 1e10, which a d of exactly 1e10 does not beat. F64 = true: the fp64 squared distance to the point's fp64 coordinates,
// initial best +Inf, and n_scan the number of finite points (the non-finite ones sort after them): a finite point whose d2
// overflows to +Inf ties the initial best and takes it (unsigned bi: -1 loses every tie), so the result is -1 only
// without finite points.
template <bool F64> struct Best { using D = float; };
template <> struct Best<true> { using D = double; };

template <bool F64>
__device__ __forceinline__ void scan_leaf(const Tree& t, int leaf, int n_scan, float qx, float qy, float qz, typename Best<F64>::D& bd,
                                          int& bi) {
    const int e = min(n_scan, (leaf + 1) * kLeaf);
    for (int j = leaf * kLeaf; j < e; ++j) {
        const float4 p = t.sp[j];
        const int i = __float_as_int(p.w);
        if constexpr (F64) {
            const double d = d2_f64(qx, qy, qz, t.sd[3 * (size_t)j], t.sd[3 * (size_t)j + 1], t.sd[3 * (size_t)j + 2]);
            if (d < bd || (d == bd && (unsigned)i < (unsigned)bi)) { bd = d; bi = i; }
        } else {
            const float d = dist_f32(qx, qy, qz, p.x, p.y, p.z);
            if (d < bd || (d == bd && i < bi)) { bd = d; bi = i; }   // bi = -1 only while bd is 1e10: never tied
        }
    }
}

__device__ __forceinline__ double prune_above(float bd) {
    const double r = fmax((double)bd * kSlack, kFloor);
    return r * r;
}
__device__ __forceinline__ double prune_above(double bd2) { return fmax(bd2 * kSlack64, kFloor64); }

template <bool F64>
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
    typename Best<F64>::D bd = F64 ? (typename Best<F64>::D)INFINITY : (typename Best<F64>::D)kNone;
    int bi = -1;
    // fp64 points with a NaN or Inf coordinate (code kNonFinite, sorted last) are never scanned
    const int n_scan = F64 ? lower_bound(t.keys, t.n, kNonFinite) : t.n;
    // seed: the leaf at the query's Morton position
    const int seed = min(lower_bound(t.keys, t.n, qkeys[s]), t.n - 1) / kLeaf;
    scan_leaf<F64>(t, seed, n_scan, qx, qy, qz, bd, bi);
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
                scan_leaf<F64>(t, leaf, n_scan, qx, qy, qz, bd, bi);
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

// ------------------------------------------------------------------------------------------------ k-NN label vote
constexpr int kVoteWarps = 4;                // warps per block
constexpr int kVoteSmemCap = 1024;           // largest per-warp candidate buffer kept in shared memory

// lexicographic (d2, index) order of the candidates
__device__ __forceinline__ bool key_less(double da, int ia, double db, int ib) { return da < db || (da == db && ia < ib); }

// ascending bitonic sort of the S (a power of two) labels by one warp; each pair of a stage belongs to one lane
__device__ void warp_sort_labels(long long* l, int S, int lane) {
    for (int k = 2; k <= S; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int x = lane; x < S; x += 32) {
                const int y = x ^ j;
                if (y <= x) continue;
                const bool up = (x & k) == 0;
                const long long a = l[x], b = l[y];
                if ((b < a) == up) { l[x] = b; l[y] = a; }
            }
            __syncwarp();
        }
}

__device__ __forceinline__ int pow2_at_least(int v) { int s = 1; while (s < v) s <<= 1; return s; }

struct VoteBuf {                             // one warp's candidates: cap keys and cap labels, and a 256-bin histogram
    double* d;
    int* i;
    long long* l;
    int* hist;
};

// One 8-bit radix-select step by a warp over the n keys key(x) whose bits above shift + 8 equal prefix: finds the digit
// (bits shift .. shift + 7) of the want-th smallest of them (1-based) and appends it to prefix; want becomes the rank
// within that digit and eq the number of keys with it.
template <class Key>
__device__ __forceinline__ void radix_step(int n, Key key, int shift, unsigned long long& prefix, int& want, int& eq, int* hist, int lane) {
    for (int j = lane; j < 256; j += 32) hist[j] = 0;
    __syncwarp();
    const unsigned long long above = shift >= 56 ? 0ull : ~0ull << (shift + 8);
    for (int x = lane; x < n; x += 32) {
        const unsigned long long u = key(x);
        if ((u & above) == prefix) atomicAdd(hist + ((u >> shift) & 255u), 1);
    }
    __syncwarp();
    int c[8], tot = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) { c[j] = hist[8 * lane + j]; tot += c[j]; }
    int incl = tot;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    const int excl = incl - tot;
    const int owner = __ffs(__ballot_sync(0xffffffffu, excl < want && want <= incl)) - 1;
    int digit = 0, below = 0, count = 0, run = excl;
    bool found = false;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (!found && run + c[j] >= want) { found = true; digit = 8 * lane + j; below = run; count = c[j]; }
        run += c[j];
    }
    digit = __shfl_sync(0xffffffffu, digit, owner);
    want -= __shfl_sync(0xffffffffu, below, owner);
    eq = __shfl_sync(0xffffffffu, count, owner);
    prefix |= (unsigned long long)digit << shift;
    __syncwarp();
}

// Keeps the k best of the cnt > k candidates by (d2, index), in place and unordered, and returns the k-th key (td, ti).
// A radix select: eight digit steps over the bits of d2 (non-negative and finite, so its bits order it), then, when the
// k-th distance is shared by candidates not all kept, four over the indices of those.
__device__ void cut_to_k(const VoteBuf& b, int cnt, int k, int lane, double& td, int& ti) {
    unsigned long long pd = 0;
    int want = k, eq = 0;
    auto dkey = [&](int x) { return (unsigned long long)__double_as_longlong(b.d[x]); };
    for (int shift = 56; shift >= 0; shift -= 8) radix_step(cnt, dkey, shift, pd, want, eq, b.hist, lane);
    td = __longlong_as_double((long long)pd);
    if (want == eq) {                        // every candidate at distance td is kept: ti = the largest of their indices
        int m = -1;
        for (int x = lane; x < cnt; x += 32) if (b.d[x] == td) m = max(m, b.i[x]);
        ti = __reduce_max_sync(0xffffffffu, m);
    } else {
        unsigned long long pi = 0;
        auto ikey = [&](int x) { return b.d[x] == td ? (unsigned long long)(unsigned)b.i[x] : 1ull << 63; };
        for (int shift = 24; shift >= 0; shift -= 8) radix_step(cnt, ikey, shift, pi, want, eq, b.hist, lane);
        ti = (int)pi;
    }
    int kept = 0;                            // compaction in place: a chunk is read whole before any of it is written
    for (int base = 0; base < cnt; base += 32) {
        const int x = base + lane;
        const double d = x < cnt ? b.d[x] : 0.0;
        const int i = x < cnt ? b.i[x] : 0;
        const bool keep = x < cnt && (d < td || (d == td && i <= ti));
        const unsigned ball = __ballot_sync(0xffffffffu, keep);
        __syncwarp();
        if (keep) { const int at = kept + __popc(ball & ((1u << lane) - 1u)); b.d[at] = d; b.i[at] = i; }
        kept += __popc(ball);
        __syncwarp();
    }
}

// out[q] = the smallest of the most frequent labels among the k nearest points of point q (itself included) by (d2, index).
// A persistent grid: each warp takes queries in Morton order, sorted position s = warp, warp + warps, ...
__global__ void __launch_bounds__(kVoteWarps * 32)
knn_vote_kernel(const Tree t, const long long* __restrict__ labels, int k, int cap, double* __restrict__ gd, int* __restrict__ gi,
                long long* __restrict__ gl, long long* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char vote_smem[];
    __shared__ int hist[kVoteWarps][256];
    __shared__ int stk_node[kVoteWarps][kStack];
    __shared__ float stk_lb2[kVoteWarps][kStack];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int gw = blockIdx.x * kVoteWarps + w, warps = gridDim.x * kVoteWarps;
    VoteBuf b;
    b.hist = hist[w];
    if (gd) {
        b.d = gd + (size_t)gw * cap; b.i = gi + (size_t)gw * cap; b.l = gl + (size_t)gw * cap;
    } else {
        b.d = reinterpret_cast<double*>(vote_smem) + (size_t)w * cap;
        b.l = reinterpret_cast<long long*>(vote_smem + (size_t)kVoteWarps * cap * 8) + (size_t)w * cap;
        b.i = reinterpret_cast<int*>(vote_smem + (size_t)kVoteWarps * cap * 16) + (size_t)w * cap;
    }
    for (int s = gw; s < t.n; s += warps) {
        const float4 q = t.sp[s];
        const double qx = q.x, qy = q.y, qz = q.z;
        int cnt = 0;
        bool full = false;                   // the buffer holds the best k so far, and (thr_d, thr_i) is the k-th of them
        double thr_d = INFINITY;
        int thr_i = INT_MAX;
        const int seed = s / kLeaf;
        auto scan = [&](int leaf) {
            const int j = leaf * kLeaf + lane;
            const bool valid = j < t.n;
            double d = INFINITY;
            int i = INT_MAX;
            if (valid) {
                const float4 p = t.sp[j];
                d = d2_f64(qx, qy, qz, p.x, p.y, p.z);
                i = __float_as_int(p.w);
            }
            bool take = valid && (!full || key_less(d, i, thr_d, thr_i));
            unsigned ball = __ballot_sync(0xffffffffu, take);
            if (cnt + __popc(ball) > cap) {         // cap >= 2k + 32, so cnt > k here
                cut_to_k(b, cnt, k, lane, thr_d, thr_i);
                cnt = k;
                full = true;
                take = valid && (!full || key_less(d, i, thr_d, thr_i));
                ball = __ballot_sync(0xffffffffu, take);
            }
            if (take) {
                const int at = cnt + __popc(ball & ((1u << lane) - 1u));
                b.d[at] = d; b.i[at] = i;
            }
            cnt += __popc(ball);
            __syncwarp();
        };
        scan(seed);
        int sp = 1;
        if (lane == 0) { stk_node[w][0] = 1; stk_lb2[w][0] = 0.0f; }
        __syncwarp();
        while (sp > 0) {
            --sp;
            const int v = stk_node[w][sp];
            const double thr2 = full ? prune_above(thr_d) : INFINITY;
            if ((double)stk_lb2[w][sp] > thr2) continue;
            if (v >= t.P) {
                if (v - t.P != seed) scan(v - t.P);
                continue;
            }
            const int c0 = 2 * v, c1 = 2 * v + 1;
            const double l0 = box_lb2(t.lo[c0], t.hi[c0], qx, qy, qz);
            const double l1 = box_lb2(t.lo[c1], t.hi[c1], qx, qy, qz);
            const bool first0 = l0 <= l1;
            const int cn = first0 ? c0 : c1, cf = first0 ? c1 : c0;
            const double ln = first0 ? l0 : l1, lf = first0 ? l1 : l0;
            __syncwarp();
            if (lf <= thr2) { if (lane == 0) { stk_node[w][sp] = cf; stk_lb2[w][sp] = __double2float_rd(lf); } ++sp; }
            if (ln <= thr2) { if (lane == 0) { stk_node[w][sp] = cn; stk_lb2[w][sp] = __double2float_rd(ln); } ++sp; }
            __syncwarp();
        }
        if (cnt > k) cut_to_k(b, cnt, k, lane, thr_d, thr_i);
        cnt = k;                             // nothing is pruned before k candidates are in, so cnt >= k
        // the mode: by a histogram when every label is in [0, 256), else by sorting the k labels and counting each run
        bool small = true;
        for (int x = lane; x < k; x += 32) {
            const long long v = labels[b.i[x]];
            b.l[x] = v;
            small = small && v >= 0 && v < 256;
        }
        small = __all_sync(0xffffffffu, small);
        __syncwarp();
        int best_c = 0;
        long long best_l = LLONG_MAX;
        if (small) {
            for (int j = lane; j < 256; j += 32) b.hist[j] = 0;
            __syncwarp();
            for (int x = lane; x < k; x += 32) atomicAdd(b.hist + b.l[x], 1);
            __syncwarp();
            for (int j = lane; j < 256; j += 32)
                if (b.hist[j] > best_c) { best_c = b.hist[j]; best_l = j; }       // ascending j: the smallest label on a tie
        } else {
            const int S = pow2_at_least(k);
            for (int x = k + lane; x < S; x += 32) b.l[x] = LLONG_MAX;
            __syncwarp();
            warp_sort_labels(b.l, S, lane);
            for (int x = lane; x < cnt; x += 32) {
                const long long v = b.l[x];
                if (x + 1 < cnt && b.l[x + 1] == v) continue;
                int lo = 0, hi = x;
                while (lo < hi) { const int mid = (lo + hi) >> 1; if (b.l[mid] < v) lo = mid + 1; else hi = mid; }
                const int c = x - lo + 1;
                if (c > best_c || (c == best_c && v < best_l)) { best_c = c; best_l = v; }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const int oc = __shfl_xor_sync(0xffffffffu, best_c, o);
            const long long ol = __shfl_xor_sync(0xffffffffu, best_l, o);
            if (oc > best_c || (oc == best_c && ol < best_l)) { best_c = oc; best_l = ol; }
        }
        if (lane == 0) out[__float_as_int(q.w)] = best_l;
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------------ tree build
struct TreeBufs {
    unsigned *bounds, *keys_in, *keys;
    int *vals_in, *order;
    float4 *sp, *lo, *hi;
    double* sd;
};

int tree_leaf_count(int n) {
    const int L = (n + kLeaf - 1) / kLeaf;
    int P = 1;
    while (P < L) P <<= 1;
    return P;
}

void take_tree(Workspace& w, TreeBufs& b, int n, int P, bool f64) {
    b.bounds = w.take<unsigned>(6);
    b.keys_in = w.take<unsigned>(n); b.keys = w.take<unsigned>(n); b.vals_in = w.take<int>(n); b.order = w.take<int>(n);
    b.sp = w.take<float4>(n); b.lo = w.take<float4>(2 * (size_t)P); b.hi = w.take<float4>(2 * (size_t)P);
    b.sd = f64 ? w.take<double>(3 * (size_t)n) : nullptr;
}

long long pow2_at_least_host(long long v) { long long s = 1; while (s < v) s <<= 1; return s; }

template <class T>
cudaError_t build_tree(const T* pos, int n, int P, const TreeBufs& b, void* tmp, size_t tmp_bytes, cudaStream_t st) {
    const int B = 256;
    PIXIE_TRY(cudaMemsetAsync(b.bounds, 0xff, 3 * sizeof(unsigned), st));         // encoded +max for the minima
    PIXIE_TRY(cudaMemsetAsync(b.bounds + 3, 0, 3 * sizeof(unsigned), st));        // encoded -max for the maxima
    bounds_kernel<T><<<(n + B - 1) / B, B, 0, st>>>(pos, n, b.bounds);
    key_kernel<T><<<(n + B - 1) / B, B, 0, st>>>(pos, n, b.bounds, true, b.keys_in, b.vals_in);
    PIXIE_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, b.keys_in, b.keys, b.vals_in, b.order, n, 0, 31, st));
    gather_kernel<T><<<(n + B - 1) / B, B, 0, st>>>(pos, b.order, n, b.sp, b.sd);
    leaf_box_kernel<<<(P + B - 1) / B, B, 0, st>>>(b.sp, b.sd, n, P, b.lo, b.hi);
    for (int first = P / 2; first >= 1; first /= 2) level_box_kernel<<<(first + B - 1) / B, B, 0, st>>>(first, b.lo, b.hi);
    return cudaSuccess;
}

// the nearest point of each query, as nearest_gaussian (float32 points, float32 d) or nearest_vertex (fp64 points, fp64 d2)
template <class T>
cudaError_t nearest_search(const T* pos, int n, const float* query, int m, int* index, cudaStream_t st) {
    if (m <= 0) return cudaSuccess;
    if (n <= 0) {
        PIXIE_TRY(cudaMemsetAsync(index, 0xff, (size_t)m * sizeof(int), st));
        return cudaSuccess;
    }
    constexpr bool f64 = sizeof(T) == 8;
    const int P = tree_leaf_count(n);
    size_t tb[2] = {0, 0};
    PIXIE_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb[0], (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr,
                                              n, 0, 31, st));
    PIXIE_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb[1], (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr,
                                              m, 0, 31, st));
    const size_t tmp_bytes = tb[0] > tb[1] ? tb[0] : tb[1];
    TreeBufs b;
    unsigned *qkeys_in, *qkeys;
    int *qvals_in, *qorder;
    void* tmp;
    Workspace w(st);
    PIXIE_TRY(w.carve([&] {
        take_tree(w, b, n, P, f64); tmp = w.take<char>(tmp_bytes);
        qkeys_in = w.take<unsigned>(m); qkeys = w.take<unsigned>(m); qvals_in = w.take<int>(m); qorder = w.take<int>(m);
    }));
    PIXIE_TRY(build_tree(pos, n, P, b, tmp, tb[0], st));
    const int B = 256;
    // non-finite queries get an ordinary (clamped) code here: they return -1 before using it
    key_kernel<float><<<(m + B - 1) / B, B, 0, st>>>(query, m, b.bounds, false, qkeys_in, qvals_in);
    PIXIE_TRY(cub::DeviceRadixSort::SortPairs(tmp, tb[1], qkeys_in, qkeys, qvals_in, qorder, m, 0, 31, st));
    const Tree t{b.sp, b.sd, b.keys, b.lo, b.hi, n, P};
    query_kernel<f64><<<(m + kThreads - 1) / kThreads, kThreads, 0, st>>>(t, query, qkeys, qorder, m, index);
    return cudaGetLastError();
}

}  // namespace

cudaError_t nearest_gaussian(const float* pos, int n, const float* query, int m, int* index, cudaStream_t st) {
    return nearest_search(pos, n, query, m, index, st);
}

cudaError_t nearest_vertex(const double* vert, int n, const float* query, int m, int* index, cudaStream_t st) {
    return nearest_search(vert, n, query, m, index, st);
}

cudaError_t knn_label_vote(const float* pos, int n, const long long* labels, int k, long long* out, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    const int P = tree_leaf_count(n);
    size_t tmp_bytes = 0;
    PIXIE_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr,
                                              (int*)nullptr, n, 0, 31, st));
    // buffer: room for the best k plus at least one leaf, doubled (up to 2^30) so that a cut keeps at least as many
    // slots free as it keeps; in shared memory up to kVoteSmemCap, else one global slice per resident warp
    const int cap = (int)std::min<long long>(pow2_at_least_host(2LL * k + kLeaf), 1LL << 30);
    int dev = 0, sms = 0;
    PIXIE_TRY(cudaGetDevice(&dev));
    PIXIE_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const bool in_smem = cap <= kVoteSmemCap;
    const size_t smem = in_smem ? (size_t)kVoteWarps * cap * 20 : 0;
    int blocks = 0;
    if (in_smem) {
        PIXIE_TRY(cudaFuncSetAttribute(knn_vote_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int per_sm = 0;
        PIXIE_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, knn_vote_kernel, kVoteWarps * 32, smem));
        blocks = sms * std::max(per_sm, 1);
    } else {                                 // at most 1 GiB of global buffers
        const long long per_block = (long long)kVoteWarps * cap * 20;
        blocks = (int)std::max<long long>(1, std::min<long long>((long long)sms * 4, (1LL << 30) / per_block));
    }
    blocks = std::min(blocks, (n + kVoteWarps - 1) / kVoteWarps);
    const size_t gslots = in_smem ? 0 : (size_t)blocks * kVoteWarps * cap;
    TreeBufs b;
    void* tmp;
    double* gd;
    int* gi;
    long long* gl;
    Workspace w(st);
    PIXIE_TRY(w.carve([&] {
        take_tree(w, b, n, P, false); tmp = w.take<char>(tmp_bytes);
        gd = w.take<double>(gslots); gi = w.take<int>(gslots); gl = w.take<long long>(gslots);
    }));
    PIXIE_TRY(build_tree(pos, n, P, b, tmp, tmp_bytes, st));
    const Tree t{b.sp, nullptr, b.keys, b.lo, b.hi, n, P};
    knn_vote_kernel<<<blocks, kVoteWarps * 32, smem, st>>>(t, labels, k, cap, in_smem ? nullptr : gd, gi, gl, out);
    return cudaGetLastError();
}

}  // namespace pixie
