// Particle filling of hollow Gaussian objects (PG/particle_filling/filling.py:291-380, Taichi f32 / i32 in the reference).
// A trained Gaussian scene only covers the object's surface; filling adds particles to the cells the Gaussians make dense
// and to the cells they enclose, so that MPM simulates a solid rather than a shell.
//   fill_density : densify_grids (:26-87), one thread per Gaussian.
//   fill_grids   : fill_dense_grids (:90-114) + internal_filling (:117-234): per-cell new counts, cub scans in C order of
//                  cells, one host sync for the totals, then emission with counter-based random offsets.
#include "particle_fill.cuh"
#include "workspace.cuh"

#include <cub/cub.cuh>
#include <curand_kernel.h>

namespace pixie {
namespace {

// Cyclic Jacobi on a symmetric 3x3 matrix in fp64: eigenvalues keep their sign (ti.sym_eig semantics; an SVD would return
// |lambda| and change the 1e-8 clamp for slightly indefinite covariances). Sorted ascending like numpy's eigh; columns of V
// are the eigenvectors.
__device__ void sym_eig3(const float c[6], double w[3], double V[3][3]) {
    double a[3][3] = {{c[0], c[1], c[2]}, {c[1], c[3], c[4]}, {c[2], c[4], c[5]}};
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int q = 0; q < 3; ++q) V[r][q] = r == q ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 32; ++sweep) {
        const double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2];
        const double diag = a[0][0] * a[0][0] + a[1][1] * a[1][1] + a[2][2] * a[2][2];
        if (!(off > 1e-34 * diag) && !(diag == 0.0 && off > 0.0)) break;
#pragma unroll
        for (int pq = 0; pq < 3; ++pq) {
            const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
            if (a[p][q] == 0.0) continue;
            const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
            const double t = fabs(theta) > 1e150 ? 0.5 / theta : (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
            const double cs = 1.0 / sqrt(t * t + 1.0), sn = t * cs;
#pragma unroll
            for (int k = 0; k < 3; ++k) {            // A J
                const double akp = a[k][p], akq = a[k][q];
                a[k][p] = cs * akp - sn * akq;
                a[k][q] = sn * akp + cs * akq;
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) {            // J^T A
                const double apk = a[p][k], aqk = a[q][k];
                a[p][k] = cs * apk - sn * aqk;
                a[q][k] = sn * apk + cs * aqk;
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) {            // V J
                const double vkp = V[k][p], vkq = V[k][q];
                V[k][p] = cs * vkp - sn * vkq;
                V[k][q] = sn * vkp + cs * vkq;
            }
        }
    }
    w[0] = a[0][0]; w[1] = a[1][1]; w[2] = a[2][2];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2 - i; ++j)
            if (w[j] > w[j + 1]) {
                const double tw = w[j]; w[j] = w[j + 1]; w[j + 1] = tw;
#pragma unroll
                for (int k = 0; k < 3; ++k) { const double tv = V[k][j]; V[k][j] = V[k][j + 1]; V[k][j + 1] = tv; }
            }
}

// Cells are held in 64 bits, and |cell| and the window radius are capped at 2^40 cells (far wider than any grid), so that
// a Gaussian at |p / dx| ~ 1e30 gets an empty window instead of wrapping around.
__device__ __forceinline__ long long cap_cells(float x) { return (long long)fminf(fmaxf(x, -0x1p40f), 0x1p40f); }

// Gaussians per cell with the clamp of get_particle_volume (the reference indexes out of range for a Gaussian outside the
// grid); the splat window below is the reference's window around the unclamped cell, clipped to the grid.
__device__ __forceinline__ int clamp_cell(long long i, int n) { return (int)min(max(i, 0ll), (long long)n - 1); }

__global__ void __launch_bounds__(128)
fill_density_kernel(const float* __restrict__ pos, const float* __restrict__ opacity, const float* __restrict__ cov, int n,
                    int gn, float dx, int* __restrict__ count, float* __restrict__ density) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n) return;
    const float p[3] = {pos[3 * g], pos[3 * g + 1], pos[3 * g + 2]};
    long long c0[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) c0[d] = cap_cells(floorf(__fdiv_rn(p[d], dx)));   // ti.floor(x / grid_dx, dtype=int), IEEE f32
    atomicAdd(count + ((size_t)clamp_cell(c0[0], gn) * gn + clamp_cell(c0[1], gn)) * gn + clamp_cell(c0[2], gn), 1);

    float cv[6];
#pragma unroll
    for (int e = 0; e < 6; ++e) cv[e] = cov[6 * g + e];
    double wd[3], Vd[3][3];
    sym_eig3(cv, wd, Vd);
    // f32 from here on, in the reference's operation order: sig clamped to 1e-8, M = Q diag(1/sig), P = M Q^T, no FMA
    float sig[3], Q[3][3], M[3][3], P[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        sig[k] = fmaxf((float)wd[k], 1e-8f);
#pragma unroll
        for (int r = 0; r < 3; ++r) Q[r][k] = (float)Vd[r][k];
    }
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int k = 0; k < 3; ++k) M[r][k] = __fmul_rn(Q[r][k], __fdiv_rn(1.0f, sig[k]));
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int q = 0; q < 3; ++q)
            P[r][q] = __fadd_rn(__fadd_rn(__fmul_rn(M[r][0], Q[q][0]), __fmul_rn(M[r][1], Q[q][1])), __fmul_rn(M[r][2], Q[q][2]));
    float rr = 0.0f;
#pragma unroll
    for (int k = 0; k < 3; ++k) rr = fmaxf(rr, sqrtf(sig[k]));
    // r = ceil(max sqrt(sig) / dx). The window [c0 - r, c0 + r] is clipped to the grid, not r: a Gaussian whose cell lies
    // outside the grid can still reach across all of it. An empty window becomes lo = gn or hi = -1, both safe as int.
    const long long r = cap_cells(ceilf(__fdiv_rn(rr, dx)));
    const float op = opacity[g];
    int lo[3], hi[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        lo[d] = (int)min(max(c0[d] - r, 0ll), (long long)gn);
        hi[d] = (int)max(min(c0[d] + r, (long long)gn - 1), -1ll);
    }
    for (int ci = lo[0]; ci <= hi[0]; ++ci)
        for (int cj = lo[1]; cj <= hi[1]; ++cj)
            for (int ck = lo[2]; ck <= hi[2]; ++ck) {
                float gw = 0.0f;                      // compute_density (:13-23): 8 corners in i, j, k order
#pragma unroll
                for (int u = 0; u < 2; ++u)
#pragma unroll
                    for (int v = 0; v < 2; ++v)
#pragma unroll
                        for (int w = 0; w < 2; ++w) {
                            const float d0 = __fsub_rn(p[0], __fmul_rn((float)(ci + u), dx));
                            const float d1 = __fsub_rn(p[1], __fmul_rn((float)(cj + v), dx));
                            const float d2 = __fsub_rn(p[2], __fmul_rn((float)(ck + w), dx));
                            float y[3];
#pragma unroll
                            for (int q = 0; q < 3; ++q)
                                y[q] = __fadd_rn(__fadd_rn(__fmul_rn(P[q][0], d0), __fmul_rn(P[q][1], d1)), __fmul_rn(P[q][2], d2));
                            const float e = __fadd_rn(__fadd_rn(__fmul_rn(d0, y[0]), __fmul_rn(d1, y[1])), __fmul_rn(d2, y[2]));
                            gw = __fadd_rn(gw, expf(__fmul_rn(-0.5f, e)));
                        }
                atomicAdd(density + ((size_t)ci * gn + cj) * gn + ck, __fdiv_rn(__fmul_rn(op, gw), 8.0f));
            }
}

// fill_dense_grids: a cell denser than the threshold and holding fewer than max_ppc Gaussians is topped up to max_ppc.
__global__ void dense_count_kernel(int* __restrict__ count, const float* __restrict__ density, int cells, float thres, int ppc,
                                   int* __restrict__ add) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cells) return;
    int k = 0;
    if (density[c] > thres && count[c] < ppc) {
        k = ppc - count[c];
        count[c] = ppc;
    }
    add[c] = k;
}

// internal_filling tests every empty cell with one ray march per direction (O(n^4) over the grid). The same answers come
// from one pass per axis line (O(n^3)):
//   collision_search(c, d) = "some cell strictly beyond c along d has density > thres" = a suffix OR of the dense flags
//     along the line, read from the far end;
//   collision_times(c, ray_dir) starts from state = (count[c] > 0), which is false for every cell internal_filling tests
//     (count == 0), and counts false -> true transitions over the cells strictly beyond c = the number of runs of dense
//     cells beyond c. Prepending cell t to the cells beyond it adds a run exactly when t is dense and t's successor is not,
//     so a suffix count over the line gives it for every cell.
// Bits of flags[c]: 1 << d = collision_search hit along direction d (0: +x, 1: -x, 2: +y, 3: -y, 4: +z, 5: -z);
// 64 = odd number of runs along ray_dir. One launch per axis (`axis` 0..2); the first one writes, the others OR in.
__global__ void classify_kernel(const float* __restrict__ density, int gn, float thres, int axis, int ray_dir,
                                unsigned char* __restrict__ flags) {
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= gn * gn) return;
    const int u = l / gn, v = l % gn;                 // v fastest: coalesced along k for axes 0 and 1
    const size_t n2 = (size_t)gn * gn;
    size_t base, stride;
    if (axis == 0) { base = (size_t)u * gn + v; stride = n2; }
    else if (axis == 1) { base = (size_t)u * n2 + v; stride = gn; }
    else { base = (size_t)u * n2 + (size_t)v * gn; stride = 1; }
    const unsigned char plus = 1u << (2 * axis), minus = 1u << (2 * axis + 1);
    // +direction: cells t+1 .. n-1 are beyond t; walk from the far end
    bool any = false, next = false;
    int runs = 0;
    for (int t = gn - 1; t >= 0; --t) {
        const size_t c = base + (size_t)t * stride;
        unsigned char f = axis == 0 ? 0 : flags[c];
        f = (unsigned char)(f | (any ? plus : 0) | (ray_dir == 2 * axis && (runs & 1) ? 64 : 0));
        flags[c] = f;
        const bool b = density[c] > thres;
        runs += b && !next;
        any |= b;
        next = b;
    }
    // -direction: cells 0 .. t-1 are beyond t
    any = false; next = false; runs = 0;
    for (int t = 0; t < gn; ++t) {
        const size_t c = base + (size_t)t * stride;
        flags[c] = (unsigned char)(flags[c] | (any ? minus : 0) | (ray_dir == 2 * axis + 1 && (runs & 1) ? 64 : 0));
        const bool b = density[c] > thres;
        runs += b && !next;
        any |= b;
        next = b;
    }
}

__global__ void interior_count_kernel(int* __restrict__ count, const unsigned char* __restrict__ flags, int cells, int exclude_dir,
                                      int ppc, int* __restrict__ add) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= cells) return;
    const unsigned need = 0x3Fu & ~(1u << exclude_dir);
    const unsigned f = flags[c];
    int k = 0;
    if (count[c] == 0 && (f & need) == need && (f & 64u)) {
        k = ppc;                                      // max_particles_per_cell - grid[i, j, k] with grid == 0
        count[c] = ppc;
    }
    add[c] = k;
}

// (cell + U[0,1)^3) * dx + origin. U = 24 random bits * 2^-24 from Philox keyed on (seed, output index), so the output
// depends on the seed only; cell + U is kept below cell + 1 where the f32 add would round up onto the next cell's face.
__device__ __forceinline__ void emit(float* out, int idx, int i, int j, int k, float dx, float o0, float o1, float o2,
                                     unsigned long long seed) {
    curandStatePhilox4_32_10_t st;
    curand_init(seed, (unsigned long long)idx, 0ull, &st);
    const uint4 r = curand4(&st);
    const unsigned bits[3] = {r.x, r.y, r.z};
    const int cell[3] = {i, j, k};
    const float org[3] = {o0, o1, o2};
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float lo = (float)cell[d], hi = (float)(cell[d] + 1);
        float t = __fadd_rn(lo, (float)(bits[d] >> 8) * 0x1p-24f);
        if (t >= hi) t = nextafterf(hi, lo);
        out[3 * (size_t)idx + d] = __fadd_rn(__fmul_rn(t, dx), org[d]);
    }
}

__global__ void emit_kernel(const int* __restrict__ add_d, const int* __restrict__ off_d, const int* __restrict__ add_i,
                            const int* __restrict__ off_i, int n_dense, int gn, float dx, float o0, float o1, float o2,
                            unsigned long long seed, float* __restrict__ out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= gn * gn * gn) return;
    const int nd = add_d[c], ni = add_i[c];
    if (nd == 0 && ni == 0) return;
    const int k = c % gn, j = (c / gn) % gn, i = c / (gn * gn);
    for (int t = 0; t < nd; ++t) emit(out, off_d[c] + t, i, j, k, dx, o0, o1, o2, seed);
    for (int t = 0; t < ni; ++t) emit(out, n_dense + off_i[c] + t, i, j, k, dx, o0, o1, o2, seed);
}

}  // namespace

cudaError_t fill_density(const float* pos, const float* opacity, const float* cov, int n, int grid_n, float grid_dx, int* count,
                         float* density, cudaStream_t st) {
    const size_t cells = (size_t)grid_n * grid_n * grid_n;
    PIXIE_TRY(cudaMemsetAsync(count, 0, cells * sizeof(int), st));
    PIXIE_TRY(cudaMemsetAsync(density, 0, cells * sizeof(float), st));
    if (n > 0) fill_density_kernel<<<(n + 127) / 128, 128, 0, st>>>(pos, opacity, cov, n, grid_n, grid_dx, count, density);
    return cudaGetLastError();
}

cudaError_t fill_grids(int* count, const float* density, int grid_n, float grid_dx, const float origin[3], float density_thres,
                       float search_thres, int max_ppc, int exclude_dir, int ray_dir, unsigned long long seed, float* out, int max_samples,
                       int* n_dense_host, int* n_total_host, cudaStream_t st) {
    const int cells = grid_n * grid_n * grid_n;
    const int blocks = (cells + 255) / 256;
    int *add_d = nullptr, *off_d = nullptr, *add_i = nullptr, *off_i = nullptr;
    unsigned char* flags = nullptr;
    void* tmp = nullptr;
    size_t tmp_bytes = 0;
    PIXIE_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, add_d, off_d, cells + 1, st));
    // stream-ordered workspace: the only host sync is the one that brings back the totals
    Workspace w(st);
    PIXIE_TRY(w.carve([&] {
        add_d = w.take<int>(cells + 1); off_d = w.take<int>(cells + 1); add_i = w.take<int>(cells + 1); off_i = w.take<int>(cells + 1);
        flags = w.take<unsigned char>(cells); tmp = w.take<char>(tmp_bytes);
    }));
    // the extra last entry stays 0, so off[cells] is the total
    PIXIE_TRY(cudaMemsetAsync(add_d + cells, 0, sizeof(int), st));
    PIXIE_TRY(cudaMemsetAsync(add_i + cells, 0, sizeof(int), st));
    dense_count_kernel<<<blocks, 256, 0, st>>>(count, density, cells, density_thres, max_ppc, add_d);
    for (int axis = 0; axis < 3; ++axis)
        classify_kernel<<<(grid_n * grid_n + 127) / 128, 128, 0, st>>>(density, grid_n, search_thres, axis, ray_dir, flags);
    interior_count_kernel<<<blocks, 256, 0, st>>>(count, flags, cells, exclude_dir, max_ppc, add_i);
    PIXIE_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, add_d, off_d, cells + 1, st));
    PIXIE_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, add_i, off_i, cells + 1, st));
    int n_int = 0;
    PIXIE_TRY(cudaMemcpyAsync(n_dense_host, off_d + cells, sizeof(int), cudaMemcpyDeviceToHost, st));
    PIXIE_TRY(cudaMemcpyAsync(&n_int, off_i + cells, sizeof(int), cudaMemcpyDeviceToHost, st));
    PIXIE_TRY(cudaStreamSynchronize(st));
    *n_total_host = *n_dense_host + n_int;
    if (*n_total_host > 0 && *n_total_host <= max_samples)
        emit_kernel<<<blocks, 256, 0, st>>>(add_d, off_d, add_i, off_i, *n_dense_host, grid_n, grid_dx, origin[0], origin[1], origin[2],
                                            seed, out);
    return cudaGetLastError();
}

}  // namespace pixie
