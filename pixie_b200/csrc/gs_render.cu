// Forward Gaussian-splatting rasterizer for sm_90a: the frames gs_simulation.py:573-631 renders with `--render_img`
// (Inria's diff-gaussian-rasterization, scale_modifier 1, prefiltered false, precomputed 3D covariances), and the dataset
// views gaussian-splatting's render.py renders (the same rasterizer fed scales and rotations instead of covariances).
//
//   preprocess  one thread per Gaussian: near cull (view z <= 0.2), EWA projection of the covariance (x/z, y/z clamped to
//               1.3 tan(fov)), +0.3 on the 2D diagonal (the covariance given, or built from scale and rotation as
//               forward.cu's computeCov3D builds it), conic, radius ceil(3 sqrt(lambda_max)), 16x16-tile rectangle, and
//               the colour: spherical harmonics toward the camera as utils/render_utils.py:113-130 evaluates them (+0.5,
//               clamped at 0), or the caller's colours. Writes one 48-byte record per Gaussian for the blend.
//   binning     inclusive scan of the tile counts; one host sync for the total; one (tile << 32 | depth bits) key per
//               (Gaussian, tile) in Gaussian order; stable radix sort over 32 + bit width(tile count) bits, so equal depths
//               keep index order; per-tile [begin, end) ranges.
//   blend       one 256-thread CTA per tile, front to back. Batches of 256 records are gathered into double-buffered
//               shared memory with cp.async: batch b+1 is in flight while batch b blends. The CTA leaves at the first
//               batch boundary where every pixel has saturated.
//
// A renderer's buffers serve every frame it draws, and a frame returns once its blend is enqueued. So each frame's stream
// first waits for the event the previous frame recorded after its blend: frames drawn on different streams run one after
// another, in call order, and a frame on the same stream pays nothing for it.
//
// The per-Gaussian arithmetic follows the reference's operation order (glm's column-major products, the double-precision
// pixel mapping) so radii and composited sets agree with it; see DESIGN.md §7.
#include "gs_render.cuh"
#include "ptx.cuh"
#include "workspace.cuh"

#include <cub/cub.cuh>

#include <cstdint>
#include <string>

namespace pixie {

namespace {

constexpr int kTile = 16;
constexpr int kBlock = kTile * kTile;

// {mean2D.x, mean2D.y, conic.x, conic.y}, {conic.z, opacity, r, g}, {b, 0, 0, 0}: three 16-byte cp.async pieces
struct __align__(16) GsRecord { float4 a, b, c; };

struct Cam {
    float view[16], proj[16], campos[3];
    float tan_fovx, tan_fovy, focal_x, focal_y;
    int W, H, grid_x, grid_y;
};

__device__ __forceinline__ float ndc2pix(float v, int S) { return ((v + 1.0) * S - 1.0) * 0.5; }

__device__ __forceinline__ void tile_rect(float px, float py, int r, int gx, int gy, int& x0, int& y0, int& x1, int& y1) {
    x0 = min(gx, max(0, (int)((px - r) / kTile)));
    y0 = min(gy, max(0, (int)((py - r) / kTile)));
    x1 = min(gx, max(0, (int)((px + r + kTile - 1) / kTile)));
    y1 = min(gy, max(0, (int)((py + r + kTile - 1) / kTile)));
}

// 3x3 product in glm's column-major form: m[c][r]
__device__ __forceinline__ void mat3_mul(const float (&A)[3][3], const float (&B)[3][3], float (&R)[3][3]) {
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int r = 0; r < 3; ++r) R[c][r] = A[0][r] * B[c][0] + A[1][r] * B[c][1] + A[2][r] * B[c][2];
}

constexpr float SH_C0 = 0.28209479177387814f;
constexpr float SH_C1 = 0.4886025119029199f;
constexpr float SH_C2_0 = 1.0925484305920792f, SH_C2_1 = -1.0925484305920792f, SH_C2_2 = 0.31539156525252005f,
                SH_C2_3 = -1.0925484305920792f, SH_C2_4 = 0.5462742152960396f;
constexpr float SH_C3_0 = -0.5900435899266435f, SH_C3_1 = 2.890611442640554f, SH_C3_2 = -0.4570457994644658f,
                SH_C3_3 = 0.3731763325901154f, SH_C3_4 = -0.4570457994644658f, SH_C3_5 = 1.445305721320277f,
                SH_C3_6 = -0.5900435899266435f;

// Real spherical harmonics up to degree 3 at unit direction (x, y, z), one channel; sh points at coefficient 0 of it
// with a stride of 3 floats between coefficients.
__device__ __forceinline__ float eval_sh(int deg, const float* sh, float x, float y, float z) {
    float r = SH_C0 * sh[0];
    if (deg > 0) {
        r = r - SH_C1 * y * sh[3] + SH_C1 * z * sh[6] - SH_C1 * x * sh[9];
        if (deg > 1) {
            const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            r = r + SH_C2_0 * xy * sh[12] + SH_C2_1 * yz * sh[15] + SH_C2_2 * (2.0f * zz - xx - yy) * sh[18] +
                SH_C2_3 * xz * sh[21] + SH_C2_4 * (xx - yy) * sh[24];
            if (deg > 2) {
                r = r + SH_C3_0 * y * (3.0f * xx - yy) * sh[27] + SH_C3_1 * xy * z * sh[30] +
                    SH_C3_2 * y * (4.0f * zz - xx - yy) * sh[33] + SH_C3_3 * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * sh[36] +
                    SH_C3_4 * x * (4.0f * zz - xx - yy) * sh[39] + SH_C3_5 * z * (xx - yy) * sh[42] +
                    SH_C3_6 * x * (xx - 3.0f * yy) * sh[45];
            }
        }
    }
    return r;
}

// forward.cu's computeCov3D at scale_modifier 1: S = diag(scale), R from the quaternion (r = rot.x) written as glm's
// column-major constructor lists it (so R here is the transpose of the usual rotation matrix), M = S R, Sigma = M^T M; the
// upper triangle in forward.cu's order (Sigma[0][0], [0][1], [0][2], [1][1], [1][2], [2][2]).
__device__ __forceinline__ void cov3d_from_scale_rot(const float* __restrict__ scale, const float* __restrict__ rot, float (&cov)[6]) {
    const float S[3][3] = {{scale[0], 0.0f, 0.0f}, {0.0f, scale[1], 0.0f}, {0.0f, 0.0f, scale[2]}};
    const float r = rot[0], x = rot[1], y = rot[2], z = rot[3];
    const float R[3][3] = {{1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y)},
                           {2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x)},
                           {2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y)}};
    float M[3][3], Mt[3][3], Sig[3][3];
    mat3_mul(S, R, M);
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) Mt[a][b] = M[b][a];
    mat3_mul(Mt, M, Sig);
    cov[0] = Sig[0][0]; cov[1] = Sig[0][1]; cov[2] = Sig[0][2];
    cov[3] = Sig[1][1]; cov[4] = Sig[1][2]; cov[5] = Sig[2][2];
}

// kScaleRot: the covariance comes from scales [n][3] and rotations [n][4] (computeCov3D) instead of cov3d [n][6]
template <bool kScaleRot>
__global__ void __launch_bounds__(256) gs_preprocess_kernel(const float* __restrict__ means, const float* __restrict__ cov3d,
                                                            const float* __restrict__ scales, const float* __restrict__ rotations,
                                                            const float* __restrict__ opacity, const float* __restrict__ shs,
                                                            const float* __restrict__ colors, int n, int sh_coeffs, int deg,
                                                            Cam c, int* __restrict__ radii, float* __restrict__ depths,
                                                            GsRecord* __restrict__ rec, unsigned long long* __restrict__ touched) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    radii[i] = 0;
    touched[i] = 0;
    const float* v = c.view;
    const float px = means[3 * i], py = means[3 * i + 1], pz = means[3 * i + 2];
    // view space (transformPoint4x3 of the row-vector matrix)
    float tx = v[0] * px + v[4] * py + v[8] * pz + v[12];
    float ty = v[1] * px + v[5] * py + v[9] * pz + v[13];
    const float tz = v[2] * px + v[6] * py + v[10] * pz + v[14];
    if (tz <= 0.2f) return;
    const float* m = c.proj;
    const float hx = m[0] * px + m[4] * py + m[8] * pz + m[12];
    const float hy = m[1] * px + m[5] * py + m[9] * pz + m[13];
    const float hw = m[3] * px + m[7] * py + m[11] * pz + m[15];
    const float pw = 1.0f / (hw + 0.0000001f);
    const float ndc_x = hx * pw, ndc_y = hy * pw;

    // EWA: cov2D = (J W) V (J W)^T with the mean's x/z, y/z clamped to 1.3 tan(fov)
    const float limx = 1.3f * c.tan_fovx, limy = 1.3f * c.tan_fovy;
    const float txtz = tx / tz, tytz = ty / tz;
    tx = fminf(limx, fmaxf(-limx, txtz)) * tz;
    ty = fminf(limy, fmaxf(-limy, tytz)) * tz;
    const float J[3][3] = {{c.focal_x / tz, 0.0f, -(c.focal_x * tx) / (tz * tz)},
                           {0.0f, c.focal_y / tz, -(c.focal_y * ty) / (tz * tz)},
                           {0.0f, 0.0f, 0.0f}};
    const float Wm[3][3] = {{v[0], v[4], v[8]}, {v[1], v[5], v[9]}, {v[2], v[6], v[10]}};
    float built[6];
    if constexpr (kScaleRot) cov3d_from_scale_rot(scales + 3 * i, rotations + 4 * i, built);
    const float* s = kScaleRot ? built : cov3d + 6 * i;
    const float V[3][3] = {{s[0], s[1], s[2]}, {s[1], s[3], s[4]}, {s[2], s[4], s[5]}};
    float T[3][3], Tt[3][3], A[3][3], S[3][3];
    mat3_mul(Wm, J, T);
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) Tt[a][b] = T[b][a];
    mat3_mul(Tt, V, A);
    mat3_mul(A, T, S);
    const float cxx = S[0][0] + 0.3f, cxy = S[0][1], cyy = S[1][1] + 0.3f;

    const float det = cxx * cyy - cxy * cxy;
    if (det == 0.0f) return;
    const float det_inv = 1.f / det;
    const float mid = 0.5f * (cxx + cyy);
    const float l1 = mid + sqrtf(fmaxf(0.1f, mid * mid - det));
    const float l2 = mid - sqrtf(fmaxf(0.1f, mid * mid - det));
    const float radius = ceilf(3.f * sqrtf(fmaxf(l1, l2)));
    const float2 xy = {ndc2pix(ndc_x, c.W), ndc2pix(ndc_y, c.H)};
    int x0, y0, x1, y1;
    tile_rect(xy.x, xy.y, (int)radius, c.grid_x, c.grid_y, x0, y0, x1, y1);
    if ((x1 - x0) * (y1 - y0) == 0) return;

    float rgb[3];
    if (shs != nullptr) {
        // utils/render_utils.py:121-128: direction from the camera centre, normalised; +0.5, clamped at 0. forward.cu's
        // computeColorFromSH evaluates the same expressions in the same order, so both entry points share this code.
        const float dx = px - c.campos[0], dy = py - c.campos[1], dz = pz - c.campos[2];
        const float len = sqrtf(dx * dx + dy * dy + dz * dz);
        const float ux = dx / len, uy = dy / len, uz = dz / len;
        const float* sh = shs + (size_t)i * sh_coeffs * 3;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) rgb[ch] = fmaxf(eval_sh(deg, sh + ch, ux, uy, uz) + 0.5f, 0.0f);
    } else {
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) rgb[ch] = colors[3 * i + ch];
    }
    depths[i] = tz;
    radii[i] = (int)radius;
    rec[i] = GsRecord{make_float4(xy.x, xy.y, cyy * det_inv, -cxy * det_inv),
                      make_float4(cxx * det_inv, opacity[i], rgb[0], rgb[1]), make_float4(rgb[2], 0.f, 0.f, 0.f)};
    touched[i] = (unsigned long long)((y1 - y0) * (x1 - x0));
}

__global__ void __launch_bounds__(256) gs_keys_kernel(int n, const GsRecord* __restrict__ rec, const float* __restrict__ depths,
                                                      const int* __restrict__ radii, const unsigned long long* __restrict__ offsets,
                                                      int gx, int gy, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || radii[i] <= 0) return;
    uint32_t off = (uint32_t)(i == 0 ? 0ull : offsets[i - 1]);
    const float4 a = rec[i].a;
    int x0, y0, x1, y1;
    tile_rect(a.x, a.y, radii[i], gx, gy, x0, y0, x1, y1);
    const uint64_t dbits = __float_as_uint(depths[i]);
    for (int y = y0; y < y1; ++y)
        for (int x = x0; x < x1; ++x) {
            keys[off] = ((uint64_t)(uint32_t)(y * gx + x) << 32) | dbits;
            vals[off] = (uint32_t)i;
            ++off;
        }
}

__global__ void __launch_bounds__(256) gs_ranges_kernel(int L, const uint64_t* __restrict__ keys, uint2* __restrict__ ranges) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L) return;
    const uint32_t tile = (uint32_t)(keys[i] >> 32);
    if (i == 0) ranges[tile].x = 0;
    else {
        const uint32_t prev = (uint32_t)(keys[i - 1] >> 32);
        if (tile != prev) { ranges[prev].y = i; ranges[tile].x = i; }
    }
    if (i == L - 1) ranges[tile].y = L;
}

__device__ __forceinline__ void stage_batch(GsRecord* dst, const GsRecord* __restrict__ rec, const uint32_t* __restrict__ list,
                                            uint2 range, int batch, int t) {
    const uint32_t k = range.x + (uint32_t)batch * kBlock + t;
    if (k < range.y) {
        const GsRecord* src = rec + list[k];
        ptx::cp_async_16(&dst[t].a, &src->a);
        ptx::cp_async_16(&dst[t].b, &src->b);
        ptx::cp_async_16(&dst[t].c, &src->c);
    }
    ptx::cp_async_commit();   // one group per batch, empty or not, so wait_group counts stay uniform
}

__global__ void __launch_bounds__(kBlock) gs_blend_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ list,
                                                          const GsRecord* __restrict__ rec, int W, int H, float3 bg,
                                                          float* __restrict__ out) {
    __shared__ GsRecord buf[2][kBlock];
    const int t = threadIdx.y * kTile + threadIdx.x;
    const int px = blockIdx.x * kTile + threadIdx.x, py = blockIdx.y * kTile + threadIdx.y;
    const bool inside = px < W && py < H;
    bool done = !inside;
    const uint2 range = ranges[blockIdx.y * gridDim.x + blockIdx.x];
    const int rounds = (int)((range.y - range.x + kBlock - 1) / kBlock);
    int todo = (int)(range.y - range.x);
    const float pxf = (float)px, pyf = (float)py;
    float T = 1.0f, C0 = 0.f, C1 = 0.f, C2 = 0.f;

    if (rounds > 0) stage_batch(buf[0], rec, list, range, 0, t);
    for (int b = 0; b < rounds; ++b, todo -= kBlock) {
        // every thread is past batch b-1, so its buffer may be refilled; leave once all pixels have saturated
        if (__syncthreads_count(done) == kBlock) break;
        if (b + 1 < rounds) stage_batch(buf[(b + 1) & 1], rec, list, range, b + 1, t);
        else ptx::cp_async_commit();
        ptx::cp_async_wait<1>();
        __syncthreads();
        const GsRecord* cur = buf[b & 1];
        const int cnt = min(kBlock, todo);
        for (int j = 0; !done && j < cnt; ++j) {
            const float4 a = cur[j].a;
            const float4 q = cur[j].b;
            const float dx = a.x - pxf, dy = a.y - pyf;
            const float power = -0.5f * (a.z * dx * dx + q.x * dy * dy) - a.w * dx * dy;
            if (power > 0.0f) continue;
            const float alpha = fminf(0.99f, q.y * expf(power));
            if (alpha < 1.0f / 255.0f) continue;
            const float test_T = T * (1 - alpha);
            if (test_T < 0.0001f) { done = true; continue; }
            C0 += q.z * alpha * T;
            C1 += q.w * alpha * T;
            C2 += cur[j].c.x * alpha * T;
            T = test_T;
        }
    }
    ptx::cp_async_wait<0>();   // no copy may land in shared memory after the CTA has left
    if (inside) {
        const size_t pix = (size_t)py * W + px, plane = (size_t)H * W;
        out[pix] = C0 + T * bg.x;
        out[plane + pix] = C1 + T * bg.y;
        out[2 * plane + pix] = C2 + T * bg.z;
    }
}

int bit_width(uint32_t v) {
    int b = 0;
    while (v >> b) ++b;
    return b;
}

}  // namespace

}  // namespace pixie

// The C ABI's handle, pixie::GsRenderer.
struct pixie_gs_renderer_s {
    // per Gaussian
    size_t cap_n = 0;
    float* depths = nullptr;
    pixie::GsRecord* rec = nullptr;
    unsigned long long* touched = nullptr;
    unsigned long long* offsets = nullptr;
    // per (Gaussian, tile) pair
    size_t cap_pairs = 0;
    uint64_t *keys_in = nullptr, *keys_out = nullptr;
    uint32_t *vals_in = nullptr, *vals_out = nullptr;
    // per tile, and cub's scratch
    size_t cap_tiles = 0, cap_tmp = 0;
    uint2* ranges = nullptr;
    void* tmp = nullptr;
    unsigned long long* total_host = nullptr;   // pinned
    cudaEvent_t ev[6] = {};
    cudaEvent_t last = nullptr;                  // recorded after each frame's last kernel; the next frame waits for it
};

namespace pixie {

namespace {

template <typename T>
cudaError_t grow(T*& p, size_t& cap, size_t need, size_t elem = sizeof(T)) {
    if (need <= cap) return cudaSuccess;
    const cudaError_t e = cudaFree(p);
    p = nullptr;
    cap = 0;
    PIXIE_TRY(e);
    PIXIE_TRY(cudaMalloc(reinterpret_cast<void**>(&p), need * elem));
    cap = need;
    return cudaSuccess;
}

cudaError_t create_members(GsRenderer* r) {
    PIXIE_TRY(cudaMallocHost(&r->total_host, sizeof(unsigned long long)));
    for (auto& e : r->ev) PIXIE_TRY(cudaEventCreate(&e));
    return cudaEventCreateWithFlags(&r->last, cudaEventDisableTiming);
}

}  // namespace

GsRenderer* gs_renderer_create() {
    GsRenderer* r = new GsRenderer();
    if (const cudaError_t e = create_members(r)) {
        gs_renderer_destroy(r);
        fail("gs_renderer_create", e);
        return nullptr;
    }
    return r;
}

void gs_renderer_destroy(GsRenderer* r) {
    if (!r) return;
    cudaFree(r->depths); cudaFree(r->rec); cudaFree(r->touched); cudaFree(r->offsets);
    cudaFree(r->keys_in); cudaFree(r->keys_out); cudaFree(r->vals_in); cudaFree(r->vals_out);
    cudaFree(r->ranges); cudaFree(r->tmp);
    if (r->total_host) cudaFreeHost(r->total_host);
    for (auto& e : r->ev)
        if (e) cudaEventDestroy(e);
    if (r->last) cudaEventDestroy(r->last);
    delete r;
}

namespace {

int render_frame(GsRenderer* r, const GsRenderArgs& a, int* n_rendered, float* phase_ms, cudaStream_t st) {
    const int n = a.n;
    Cam c;
    for (int k = 0; k < 16; ++k) { c.view[k] = a.view[k]; c.proj[k] = a.proj[k]; }
    for (int k = 0; k < 3; ++k) c.campos[k] = a.campos[k];
    c.tan_fovx = a.tan_fovx; c.tan_fovy = a.tan_fovy;
    c.focal_x = a.width / (2.0f * a.tan_fovx);
    c.focal_y = a.height / (2.0f * a.tan_fovy);
    c.W = a.width; c.H = a.height;
    c.grid_x = (a.width + kTile - 1) / kTile;
    c.grid_y = (a.height + kTile - 1) / kTile;
    const int tiles = c.grid_x * c.grid_y;
    const int bits = bit_width((uint32_t)tiles);
    // arrays that share one capacity are each re-allocated from zero
    auto regrow = [](auto*& p, size_t want) { size_t cap = 0; return grow(p, cap, want); };
    cudaError_t e;

    if (n > r->cap_n) {
        const size_t want = (size_t)n + n / 4;
        e = regrow(r->depths, want);
        if (e == cudaSuccess) e = regrow(r->rec, want);
        if (e == cudaSuccess) e = regrow(r->touched, want);
        if (e == cudaSuccess) e = regrow(r->offsets, want);
        if (e != cudaSuccess) { r->cap_n = 0; return fail("gs_render: device allocation (per Gaussian)", e); }
        r->cap_n = want;
    }
    if ((e = grow(r->ranges, r->cap_tiles, (size_t)tiles)) != cudaSuccess) return fail("gs_render: device allocation (tile ranges)", e);

    const bool timed = phase_ms != nullptr;
    auto mark = [&](int k) { return timed ? cudaEventRecord(r->ev[k], st) : cudaSuccess; };
    if ((e = mark(0)) != cudaSuccess) return fail("gs_render: phase event", e);
    if (n > 0 && a.cov)
        gs_preprocess_kernel<false><<<(n + 255) / 256, 256, 0, st>>>(a.means, a.cov, nullptr, nullptr, a.opacity, a.shs, a.colors, n,
                                                                    a.sh_coeffs, a.sh_degree, c, a.radii, r->depths, r->rec, r->touched);
    else if (n > 0)
        gs_preprocess_kernel<true><<<(n + 255) / 256, 256, 0, st>>>(a.means, nullptr, a.scales, a.rotations, a.opacity, a.shs, a.colors, n,
                                                                   a.sh_coeffs, a.sh_degree, c, a.radii, r->depths, r->rec, r->touched);
    if ((e = mark(1)) != cudaSuccess) return fail("gs_render: phase event", e);

    unsigned long long total = 0;
    if (n > 0) {
        size_t need = 0;
        if ((e = cub::DeviceScan::InclusiveSum(nullptr, need, r->touched, r->offsets, n, st)) != cudaSuccess) return fail("gs_render: scan", e);
        if ((e = grow(reinterpret_cast<char*&>(r->tmp), r->cap_tmp, need, 1)) != cudaSuccess) return fail("gs_render: device allocation (scan)", e);
        if ((e = cub::DeviceScan::InclusiveSum(r->tmp, need, r->touched, r->offsets, n, st)) != cudaSuccess) return fail("gs_render: scan", e);
        e = cudaMemcpyAsync(r->total_host, r->offsets + (n - 1), sizeof(unsigned long long), cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) return fail("gs_render: reading the pair count", e);
        total = *r->total_host;
    }
    if (total > 0x7fffffffull)
        return fail("gs_render: " + std::to_string(total) + " (Gaussian, tile) pairs exceed 2^31 - 1");
    const int L = (int)total;
    if (L > 0) {
        if ((size_t)L > r->cap_pairs) {
            const size_t want = (size_t)L + L / 4;
            e = regrow(r->keys_in, want);
            if (e == cudaSuccess) e = regrow(r->keys_out, want);
            if (e == cudaSuccess) e = regrow(r->vals_in, want);
            if (e == cudaSuccess) e = regrow(r->vals_out, want);
            if (e != cudaSuccess) { r->cap_pairs = 0; return fail("gs_render: device allocation (pairs)", e); }
            r->cap_pairs = want;
        }
        gs_keys_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, r->rec, r->depths, a.radii, r->offsets, c.grid_x, c.grid_y, r->keys_in,
                                                       r->vals_in);
    }
    if ((e = mark(2)) != cudaSuccess) return fail("gs_render: phase event", e);
    if (L > 0) {
        size_t need = 0;
        if ((e = cub::DeviceRadixSort::SortPairs(nullptr, need, r->keys_in, r->keys_out, r->vals_in, r->vals_out, L, 0, 32 + bits, st)) != cudaSuccess)
            return fail("gs_render: sort", e);
        if ((e = grow(reinterpret_cast<char*&>(r->tmp), r->cap_tmp, need, 1)) != cudaSuccess) return fail("gs_render: device allocation (sort)", e);
        if ((e = cub::DeviceRadixSort::SortPairs(r->tmp, need, r->keys_in, r->keys_out, r->vals_in, r->vals_out, L, 0, 32 + bits, st)) !=
            cudaSuccess)
            return fail("gs_render: sort", e);
    }
    if ((e = mark(3)) != cudaSuccess) return fail("gs_render: phase event", e);
    if ((e = cudaMemsetAsync(r->ranges, 0, (size_t)tiles * sizeof(uint2), st)) != cudaSuccess) return fail("gs_render: clearing the tile ranges", e);
    if (L > 0) gs_ranges_kernel<<<(L + 255) / 256, 256, 0, st>>>(L, r->keys_out, r->ranges);
    if ((e = mark(4)) != cudaSuccess) return fail("gs_render: phase event", e);
    gs_blend_kernel<<<dim3(c.grid_x, c.grid_y), dim3(kTile, kTile), 0, st>>>(r->ranges, r->vals_out, r->rec, c.W, c.H,
                                                                          make_float3(a.bg[0], a.bg[1], a.bg[2]), a.image);
    if ((e = mark(5)) != cudaSuccess) return fail("gs_render: phase event", e);
    if ((e = cudaGetLastError()) != cudaSuccess) return fail("gs_render: kernel launch", e);
    if (timed) {
        if ((e = cudaEventSynchronize(r->ev[5])) != cudaSuccess) return fail("gs_render: phase timing", e);
        for (int k = 0; k < 5; ++k)
            if ((e = cudaEventElapsedTime(&phase_ms[k], r->ev[k], r->ev[k + 1])) != cudaSuccess) return fail("gs_render: phase timing", e);
    }
    if (n_rendered) *n_rendered = L;
    return 0;
}

}  // namespace

int gs_render(GsRenderer* r, const GsRenderArgs& a, int* n_rendered, float* phase_ms, cudaStream_t st) {
    if (const cudaError_t e = cudaStreamWaitEvent(st, r->last, 0)) return fail("gs_render: waiting for the previous frame", e);
    const int rc = render_frame(r, a, n_rendered, phase_ms, st);
    // recorded on failure too: whatever the frame enqueued before failing still reads and writes the shared buffers
    const cudaError_t e = cudaEventRecord(r->last, st);
    if (e != cudaSuccess && rc == 0) return fail("gs_render: recording the frame's end", e);
    return rc;
}

}  // namespace pixie
