// Material-field -> particle transfer on the device (SURVEY.md 8f-1): the step between the U-Net and the MPM rollout.
//   field_extract : pixie/voxel/map_pred_to_coords.py:41-75 (unscale_prediction) + :198-245 (argmax id, confidence,
//                   linspace voxel centres, mask compaction in C order) -- the reference writes a PLY that
//                   PG/material_field.py reads back; here the point cloud stays on the device.
//   knn_assign    : PG/material_field.py:228-293 (perform_knn_smoothing) + :57-86 (assign_from_neighbors): exact k nearest
//                   neighbours (brute force, shared-memory tiles, distances in fp64 like sklearn's KDTree), mean / mode
//                   of the neighbours' properties, defaults for particles farther than the threshold.
#include "field_transfer.cuh"
#include "workspace.cuh"

#include <cub/cub.cuh>

namespace pixie {
namespace {

__global__ void field_flag_kernel(const float* __restrict__ mask, int n, int* __restrict__ flags) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flags[i] = mask[i] > 0.f ? 1 : 0;
}

struct ExtractArgs {
    const float* pred;     // [3 + K][D^3]
    const float* mask;
    const int* offsets;    // exclusive scan of the flags
    int D, K;
    double lo[3], hi[3];   // density_min/max (log10), E_min/max (log10), nu_min/max (Python floats in the reference)
    double bmin[3], bmax[3];
    float *pos, *density, *E, *nu, *conf;
    int* material;
};

__global__ void field_extract_kernel(const ExtractArgs a) {
    const int D = a.D, n = D * D * D;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !(a.mask[i] > 0.f)) return;
    const int o = a.offsets[i];
    const int iz = i % D, iy = (i / D) % D, ix = i / (D * D);
    // np.linspace(min, max, D): start + i * step in float64, last sample = stop exactly; stored as 'f4' in the PLY
    const int idx[3] = {ix, iy, iz};
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const double step = (a.bmax[d] - a.bmin[d]) / (double)(D - 1);
        // i * step and + start are two separately rounded float64 operations in numpy: no FMA contraction here
        const double c = idx[d] == D - 1 ? a.bmax[d] : __dadd_rn(__dmul_rn((double)idx[d], step), a.bmin[d]);
        a.pos[3 * o + d] = (float)c;
    }
    // unscale_prediction: clip to [-1, 1]; density and E are log10-scaled, nu linear; float32 arithmetic like numpy's
    float c3[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) c3[c] = fminf(fmaxf(a.pred[(size_t)c * n + i], -1.f), 1.f);
    const float dl = (c3[0] + 1.0f) * (float)((a.hi[0] - a.lo[0]) / 2.0) + (float)a.lo[0];
    const float el = (c3[1] + 1.0f) * (float)((a.hi[1] - a.lo[1]) / 2.0) + (float)a.lo[1];
    a.density[o] = powf(10.f, dl);
    a.E[o] = powf(10.f, el);
    a.nu[o] = (c3[2] + 1.0f) * (float)((a.hi[2] - a.lo[2]) / 2.0) + (float)a.lo[2];
    // get_mat_id: a (1, 64, 64, 64) class block holds class indices, stored as 'i4' in the PLY (float -> int truncates);
    // otherwise argmax over the class channels (first maximum), so a single channel of another size gives 0.
    // conf = the maximum for K > 1, else 1
    float bv = a.pred[(size_t)3 * n + i];
    if (a.K == 1 && D == 64) {
        a.material[o] = (int)bv;
    } else {
        int best = 0;
        for (int k = 1; k < a.K; ++k) {
            const float v = a.pred[(size_t)(3 + k) * n + i];
            if (v > bv) { bv = v; best = k; }
        }
        a.material[o] = best;
    }
    a.conf[o] = a.K > 1 ? bv : 1.0f;
}

constexpr int kKnnMaxK = 16;
constexpr int kKnnTile = 256;

// numpy's pairwise float32 summation for n <= 128 (the order np.mean uses for the k neighbour values)
__device__ __forceinline__ float numpy_sum_f32(const float* a, int n) {
    if (n < 8) {
        float r = 0.f;
        for (int i = 0; i < n; ++i) r += a[i];
        return r;
    }
    float r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    int i = 8;
    for (; i < n - (n % 8); i += 8)
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] += a[i + j];
    float res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res += a[i];
    return res;
}

struct KnnArgs {
    const float* query; int nq;
    const float *pos, *density, *E, *nu, *conf; const int *material, *part; int m;
    int k; double threshold; int weighted;
    float def_density, def_E, def_nu, def_conf; int def_material, def_part;
    float *o_density, *o_E, *o_nu, *o_conf; int *o_material, *o_part;
    int* n_too_far;
};

__device__ __forceinline__ int mode_unweighted(const int* v, int k) {
    // Counter(v).most_common(1): highest count, ties -> first encountered
    int best = v[0], bc = 0;
    for (int i = 0; i < k; ++i) {
        bool seen = false;
        for (int j = 0; j < i; ++j) seen |= (v[j] == v[i]);
        if (seen) continue;
        int c = 0;
        for (int j = i; j < k; ++j) c += (v[j] == v[i]);
        if (c > bc) { bc = c; best = v[i]; }
    }
    return best;
}
__device__ __forceinline__ int mode_weighted(const int* v, const double* w, int k) {
    // np.unique + np.bincount(weights) + argmax: highest vote, ties -> smallest value
    int best = 0; double bw = -1.0; bool have = false;
    for (int i = 0; i < k; ++i) {
        bool seen = false;
        for (int j = 0; j < i; ++j) seen |= (v[j] == v[i]);
        if (seen) continue;
        double s = 0;
        for (int j = 0; j < k; ++j) if (v[j] == v[i]) s += w[j];      // bincount adds in index order
        if (!have || s > bw || (s == bw && v[i] < best)) { bw = s; best = v[i]; have = true; }
    }
    return best;
}

__global__ void __launch_bounds__(128)
knn_assign_kernel(const KnnArgs a) {
    __shared__ float sp[kKnnTile * 3];
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = q < a.nq;
    double qx = 0, qy = 0, qz = 0;
    if (live) { qx = a.query[3 * q]; qy = a.query[3 * q + 1]; qz = a.query[3 * q + 2]; }
    double bd[kKnnMaxK];
    int bi[kKnnMaxK];
    const int k = a.k;
    for (int j = 0; j < kKnnMaxK; ++j) { bd[j] = 1e300; bi[j] = -1; }
    for (int t0 = 0; t0 < a.m; t0 += kKnnTile) {
        const int cnt = min(kKnnTile, a.m - t0);
        __syncthreads();
        for (int j = threadIdx.x; j < cnt * 3; j += blockDim.x) sp[j] = a.pos[(size_t)t0 * 3 + j];
        __syncthreads();
        if (!live) continue;
        for (int j = 0; j < cnt; ++j) {
            const double dx = qx - (double)sp[3 * j], dy = qy - (double)sp[3 * j + 1], dz = qz - (double)sp[3 * j + 2];
            const double d2 = dx * dx + dy * dy + dz * dz;
            if (d2 < bd[k - 1]) {
                // insertion into the ascending list; equal distances keep the lower index first
                int pos = k - 1;
                while (pos > 0 && bd[pos - 1] > d2) { bd[pos] = bd[pos - 1]; bi[pos] = bi[pos - 1]; --pos; }
                bd[pos] = d2; bi[pos] = t0 + j;
            }
        }
    }
    if (!live) return;
    const int kk = min(k, a.m);
    const double d0 = sqrt(bd[0]);
    if (!(kk > 0) || d0 > a.threshold) {
        a.o_density[q] = a.def_density; a.o_E[q] = a.def_E; a.o_nu[q] = a.def_nu; a.o_conf[q] = a.def_conf;
        a.o_material[q] = a.def_material; a.o_part[q] = a.def_part;
        atomicAdd(a.n_too_far, 1);
        return;
    }
    float vd[kKnnMaxK], ve[kKnnMaxK], vn[kKnnMaxK], vc[kKnnMaxK];
    int vm[kKnnMaxK], vp[kKnnMaxK];
    double w[kKnnMaxK];
    double wsum = 0;
    for (int j = 0; j < kk; ++j) {
        const int i = bi[j];
        vd[j] = a.density[i]; ve[j] = a.E[i]; vn[j] = a.nu[i]; vc[j] = a.conf[i];
        vm[j] = a.material[i]; vp[j] = a.part[i];
        w[j] = 1.0 / (sqrt(bd[j]) + 1e-8);
        wsum += w[j];
    }
    if (a.weighted) {
        for (int j = 0; j < kk; ++j) w[j] /= wsum;
        double sd = 0, se = 0, sn = 0, sc = 0;
        for (int j = 0; j < kk; ++j) { sd += w[j] * (double)vd[j]; se += w[j] * (double)ve[j]; sn += w[j] * (double)vn[j]; sc += w[j] * (double)vc[j]; }
        a.o_density[q] = (float)sd; a.o_E[q] = (float)se; a.o_nu[q] = (float)sn; a.o_conf[q] = (float)sc;
        a.o_material[q] = mode_weighted(vm, w, kk); a.o_part[q] = mode_weighted(vp, w, kk);
    } else {
        const float fk = (float)kk;
        a.o_density[q] = numpy_sum_f32(vd, kk) / fk; a.o_E[q] = numpy_sum_f32(ve, kk) / fk;
        a.o_nu[q] = numpy_sum_f32(vn, kk) / fk; a.o_conf[q] = numpy_sum_f32(vc, kk) / fk;
        a.o_material[q] = mode_unweighted(vm, kk); a.o_part[q] = mode_unweighted(vp, kk);
    }
}


// ---- per-frame export (SURVEY.md 8f-2)
// get_particle_volume (PG/particle_filling/filling.py:247-288): particles per cell of a grid_n^3 grid, vol = dx^3 / count.
__device__ __forceinline__ int cell_of(float p, float dx, int n) {
    const int i = (int)floorf(p / dx);            // ti.floor(p / grid_dx, dtype=int) in f32
    return min(max(i, 0), n - 1);                 // the Taichi kernel indexes out of range here; we clamp
}
__global__ void volume_count_kernel(const float* __restrict__ pos, int n, float dx, int gn, int* __restrict__ grid) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const int i = cell_of(pos[3 * p], dx, gn), j = cell_of(pos[3 * p + 1], dx, gn), k = cell_of(pos[3 * p + 2], dx, gn);
    atomicAdd(grid + ((size_t)i * gn + j) * gn + k, 1);
}
__global__ void volume_assign_kernel(const float* __restrict__ pos, int n, float dx, int gn, const int* __restrict__ grid, float* __restrict__ vol) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const int i = cell_of(pos[3 * p], dx, gn), j = cell_of(pos[3 * p + 1], dx, gn), k = cell_of(pos[3 * p + 2], dx, gn);
    vol[p] = (dx * dx * dx) / (float)grid[((size_t)i * gn + j) * gn + k];
}

// gs_simulation.py:591-600: pos_render = apply_inverse_rotations(undotransform2origin(undoshift2center111(pos, z_shift), scale, mean), Rs),
// cov3D_render = apply_inverse_cov_rotations(cov / scale^2, Rs)   (utils/transformation_utils.py:19-20, 57-87, 101-126)
struct FrameArgs {
    const float *pos, *cov; int n;
    float z_shift, scale, mean[3];
    float R[8][9]; int n_rot;
    float *pos_out, *cov_out;
};
__global__ void frame_transform_kernel(const FrameArgs a) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= a.n) return;
    float v[3] = {a.pos[3 * p] - 1.0f - 0.0f, a.pos[3 * p + 1] - 1.0f - 0.0f, a.pos[3 * p + 2] - 1.0f - a.z_shift};
#pragma unroll
    for (int d = 0; d < 3; ++d) v[d] = a.mean[d] + v[d] / a.scale;
    for (int r = a.n_rot - 1; r >= 0; --r) {               // torch.mm(position, R): row vector times R
        const float* R = a.R[r];
        const float x = v[0] * R[0] + v[1] * R[3] + v[2] * R[6];
        const float y = v[0] * R[1] + v[1] * R[4] + v[2] * R[7];
        const float z = v[0] * R[2] + v[1] * R[5] + v[2] * R[8];
        v[0] = x; v[1] = y; v[2] = z;
    }
    a.pos_out[3 * p] = v[0]; a.pos_out[3 * p + 1] = v[1]; a.pos_out[3 * p + 2] = v[2];
    if (!a.cov) return;
    const float s2 = a.scale * a.scale;
    float u[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) u[i] = a.cov[6 * p + i] / s2;
    float M[9] = {u[0], u[1], u[2], u[1], u[3], u[4], u[2], u[4], u[5]};      // get_mat_from_upper
    for (int r = a.n_rot - 1; r >= 0; --r) {               // apply_cov_rotation(cov, R.T): R^T (cov R)
        const float* R = a.R[r];
        float T[9], O[9];
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) T[3 * i + j] = M[3 * i] * R[j] + M[3 * i + 1] * R[3 + j] + M[3 * i + 2] * R[6 + j];
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) O[3 * i + j] = R[i] * T[j] + R[3 + i] * T[3 + j] + R[6 + i] * T[6 + j];
#pragma unroll
        for (int i = 0; i < 9; ++i) M[i] = O[i];
    }
    float* o = a.cov_out + 6 * (size_t)p;                   // get_uppder_from_mat
    o[0] = M[0]; o[1] = M[1]; o[2] = M[2]; o[3] = M[4]; o[4] = M[5]; o[5] = M[8];
}

}  // namespace

cudaError_t field_extract(const float* pred, int n_classes, const float* mask, int D, const double ranges[6], const double bmin[3], const double bmax[3],
                          float* pos, float* density, float* E, float* nu, int* material, float* conf, int* count_host, cudaStream_t st) {
    const int n = D * D * D;
    int *flags = nullptr, *offsets = nullptr;
    void* tmp = nullptr;
    size_t tmp_bytes = 0;
    PIXIE_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, flags, offsets, n + 1, st));
    Workspace w(st);
    PIXIE_TRY(w.carve([&] { flags = w.take<int>(n + 1); offsets = w.take<int>(n + 1); tmp = w.take<char>(tmp_bytes); }));
    PIXIE_TRY(cudaMemsetAsync(flags, 0, (size_t)(n + 1) * sizeof(int), st));
    field_flag_kernel<<<(n + 255) / 256, 256, 0, st>>>(mask, n, flags);
    PIXIE_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, flags, offsets, n + 1, st));
    ExtractArgs a{};
    a.pred = pred; a.mask = mask; a.offsets = offsets; a.D = D; a.K = n_classes;
    for (int c = 0; c < 3; ++c) { a.lo[c] = ranges[2 * c]; a.hi[c] = ranges[2 * c + 1]; a.bmin[c] = bmin[c]; a.bmax[c] = bmax[c]; }
    a.pos = pos; a.density = density; a.E = E; a.nu = nu; a.conf = conf; a.material = material;
    field_extract_kernel<<<(n + 255) / 256, 256, 0, st>>>(a);
    PIXIE_TRY(cudaMemcpyAsync(count_host, offsets + n, sizeof(int), cudaMemcpyDeviceToHost, st));
    PIXIE_TRY(cudaStreamSynchronize(st));
    return cudaGetLastError();
}

cudaError_t knn_assign(const float* query, int nq, const float* pos, const float* density, const float* E, const float* nu, const int* material,
                       const int* part, const float* conf, int m, int k, double threshold, int weighted, const float defaults[4], int def_material,
                       int def_part, float* o_density, float* o_E, float* o_nu, int* o_material, int* o_part, float* o_conf, int* n_too_far_host,
                       cudaStream_t st) {
    Workspace w(st);
    int* d_cnt = nullptr;
    PIXIE_TRY(w.carve([&] { d_cnt = w.take<int>(1); }));
    PIXIE_TRY(cudaMemsetAsync(d_cnt, 0, sizeof(int), st));
    KnnArgs a{};
    a.query = query; a.nq = nq; a.pos = pos; a.density = density; a.E = E; a.nu = nu; a.conf = conf; a.material = material; a.part = part; a.m = m;
    a.k = k; a.threshold = threshold; a.weighted = weighted;
    a.def_density = defaults[0]; a.def_E = defaults[1]; a.def_nu = defaults[2]; a.def_conf = defaults[3]; a.def_material = def_material; a.def_part = def_part;
    a.o_density = o_density; a.o_E = o_E; a.o_nu = o_nu; a.o_conf = o_conf; a.o_material = o_material; a.o_part = o_part; a.n_too_far = d_cnt;
    if (nq > 0) knn_assign_kernel<<<(nq + 127) / 128, 128, 0, st>>>(a);
    PIXIE_TRY(cudaMemcpyAsync(n_too_far_host, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, st));
    PIXIE_TRY(cudaStreamSynchronize(st));
    return cudaGetLastError();
}

cudaError_t particle_volume(const float* pos, int n, int grid_n, float grid_dx, float* vol, cudaStream_t st) {
    const size_t cells = (size_t)grid_n * grid_n * grid_n;
    Workspace w(st);
    int* grid = nullptr;
    PIXIE_TRY(w.carve([&] { grid = w.take<int>(cells); }));
    PIXIE_TRY(cudaMemsetAsync(grid, 0, cells * sizeof(int), st));
    if (n > 0) {
        volume_count_kernel<<<(n + 255) / 256, 256, 0, st>>>(pos, n, grid_dx, grid_n, grid);
        volume_assign_kernel<<<(n + 255) / 256, 256, 0, st>>>(pos, n, grid_dx, grid_n, grid, vol);
    }
    return cudaGetLastError();
}

cudaError_t frame_transform(const float* pos, const float* cov, int n, float z_shift, float scale, const float mean[3], const float* rotations, int n_rot,
                            float* pos_out, float* cov_out, cudaStream_t st) {
    FrameArgs a{};
    a.pos = pos; a.cov = cov; a.n = n; a.z_shift = z_shift; a.scale = scale;
    for (int d = 0; d < 3; ++d) a.mean[d] = mean[d];
    for (int r = 0; r < n_rot; ++r)
        for (int i = 0; i < 9; ++i) a.R[r][i] = rotations[9 * r + i];
    a.n_rot = n_rot; a.pos_out = pos_out; a.cov_out = cov_out;
    if (n > 0) frame_transform_kernel<<<(n + 255) / 256, 256, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace pixie
