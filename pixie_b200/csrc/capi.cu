// extern "C" boundary of libpixie_b200.so (include/pixie_b200.h). No torch types cross it.
#include "../../include/pixie_b200.h"
#include "mpm.cuh"
#include "unet.cuh"
#include "unet_kernels.cuh"
#include "field_transfer.cuh"
#include "cluster.cuh"
#include "particle_fill.cuh"
#include "nearest.cuh"
#include "gs_render.cuh"
#include "gs_ply.cuh"
#include "gs_load.cuh"
#include "image_metrics.cuh"
#include "material_metrics.cuh"
#include "part_segmentation.cuh"
#include "workspace.cuh"

#include <algorithm>
#include <cstring>
#include <string>

namespace {
thread_local std::string g_err;
}  // namespace

namespace pixie {
int fail(const std::string& message) { g_err = message; return 1; }
int fail(const std::string& what, cudaError_t e) {
    cudaGetLastError();
    return fail(what + ": " + cudaGetErrorString(e));
}
}  // namespace pixie

using pixie::fail;

namespace {
// 0 on success, otherwise fail(op, e)
int check(const char* op, cudaError_t e) { return e == cudaSuccess ? 0 : fail(op, e); }
}  // namespace

extern "C" {

const char* pixie_last_error(void) { return g_err.c_str(); }
int pixie_abi_version(void) { return 2; }

int pixie_device_ok(void) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return 0; }
    int major = 0;
    if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) { cudaGetLastError(); return 0; }
    return major == 9 ? 1 : 0;
}

static int require_device() {
    if (!pixie_device_ok()) return fail("pixie_b200 requires an sm_90 (H100) CUDA device; there is no CPU fallback");
    return 0;
}

// ------------------------------------------------------------------------------------- U-Net
int pixie_unet_create(const pixie_unet_config* cfg, pixie_unet_t* out) {
    if (!cfg || !out) return fail("null argument");
    if (require_device()) return 1;
    *out = pixie::unet_create(*cfg);
    return *out ? 0 : 1;
}
int pixie_unet_set_tensor(pixie_unet_t h, const char* name, const float* host_data, const int64_t* shape, int ndim) {
    if (!h || !name || !host_data) return fail("null argument");
    return pixie::unet_set_tensor(h, name, host_data, shape, ndim);
}
int pixie_unet_finalize(pixie_unet_t h) {
    if (!h) return fail("null handle");
    return pixie::unet_finalize(h);
}
int pixie_unet_forward(pixie_unet_t h, const void* feat, int batch, float* out, void* stream) {
    if (!h || !feat || !out) return fail("null argument");
    return pixie::unet_forward(h, feat, batch, out, (cudaStream_t)stream);
}
int pixie_unet_forward_ncdhw(pixie_unet_t h, const float* feat, int batch, float* out, void* stream) {
    if (!h || !feat || !out) return fail("null argument");
    return pixie::unet_forward_ncdhw(h, feat, batch, out, (cudaStream_t)stream);
}
int pixie_unet_forward_host(pixie_unet_t h, const void* feat, int batch, float* out, void* stream) {
    if (!h || !feat || !out) return fail("null argument");
    return pixie::unet_forward_host(h, feat, batch, out, (cudaStream_t)stream);
}
int pixie_unet_profile(pixie_unet_t h, const void* feat, int batch, float* out, void* stream, float* ms, int* kinds, double* flops, int cap) {
    if (!h || !feat || !out || !ms || !kinds || !flops) { fail("null argument"); return -1; }
    return pixie::unet_profile(h, feat, batch, out, (cudaStream_t)stream, ms, kinds, flops, cap);
}
int pixie_field_extract(const float* pred, int n_classes, const float* mask, int D, const double ranges[6], const double bmin[3], const double bmax[3],
                        float* pos, float* density, float* E, float* nu, int* material, float* conf, int* count_host, void* stream) {
    if (!pred || !mask || !ranges || !bmin || !bmax || !pos || !density || !E || !nu || !material || !conf || !count_host) return fail("null argument");
    if (D < 2 || D > 1290 || n_classes < 1)
        return fail("field_extract: need 2 <= D <= 1290 (D^3 voxels are indexed in int32) and at least one class channel");
    if (require_device()) return 1;
    return check("field_extract", pixie::field_extract(pred, n_classes, mask, D, ranges, bmin, bmax, pos, density, E, nu, material, conf,
                                                       count_host, (cudaStream_t)stream));
}
int pixie_knn_assign(const float* query, int nq, const float* pos, const float* density, const float* E, const float* nu, const int* material,
                     const int* part, const float* conf, int m, int k, double threshold, int weighted, const float defaults[4], int def_material,
                     int def_part, float* o_density, float* o_E, float* o_nu, int* o_material, int* o_part, float* o_conf, int* n_too_far_host,
                     void* stream) {
    if (!query || !pos || !density || !E || !nu || !material || !part || !conf || !defaults || !o_density || !o_E || !o_nu || !o_material ||
        !o_part || !o_conf || !n_too_far_host) return fail("null argument");
    if (k < 1 || k > 16) return fail("knn_assign: k must be in [1, 16]");
    if (m < 1) return fail("knn_assign: empty material point cloud");
    if (k > m) return fail("knn_assign: k exceeds the number of material points");
    if (require_device()) return 1;
    return check("knn_assign", pixie::knn_assign(query, nq, pos, density, E, nu, material, part, conf, m, k, threshold, weighted, defaults,
                                                 def_material, def_part, o_density, o_E, o_nu, o_material, o_part, o_conf, n_too_far_host,
                                                 (cudaStream_t)stream));
}
int pixie_dbscan(const float* pos, int n, const int* ids, int select_id, double eps, int min_samples, int* index, int* labels,
                 int* n_selected_host, int* n_clusters_host, void* stream) {
    if (!n_selected_host || !n_clusters_host || (n > 0 && (!pos || !index || !labels))) return fail("null argument");
    if (n < 0) return fail("dbscan: negative point count");
    if (!(eps > 0.0) || min_samples < 1) return fail("dbscan: need eps > 0 and min_samples >= 1");
    if (require_device()) return 1;
    return check("dbscan", pixie::dbscan(pos, n, ids, select_id, eps, min_samples, index, labels, n_selected_host, n_clusters_host,
                                         (cudaStream_t)stream));
}
int pixie_cluster_stats(const float* pos, const int* index, const int* labels, int n_selected, int n_clusters, int* sizes,
                        float* bbox_min, float* bbox_max, void* stream) {
    if (n_selected < 0 || n_clusters < 0) return fail("cluster_stats: negative count");
    if ((n_selected > 0 && (!pos || !index || !labels)) || (n_clusters > 0 && (!sizes || !bbox_min || !bbox_max))) return fail("null argument");
    if (require_device()) return 1;
    return check("cluster_stats", pixie::cluster_stats(pos, index, labels, n_selected, n_clusters, sizes, bbox_min, bbox_max, (cudaStream_t)stream));
}
int pixie_particle_volume(const float* pos, int n, int grid_n, float grid_dx, float* vol, void* stream) {
    if (n < 0) return fail("particle_volume: negative point count");
    if (n > 0 && (!pos || !vol)) return fail("null argument");
    if (grid_n < 1 || !(grid_dx > 0.f)) return fail("particle_volume: bad grid");
    if (require_device()) return 1;
    return check("particle_volume", pixie::particle_volume(pos, n, grid_n, grid_dx, vol, (cudaStream_t)stream));
}
int pixie_frame_transform(const float* pos, const float* cov, int n, float z_shift, float scale, const float mean[3], const float* rotations,
                          int n_rot, float* pos_out, float* cov_out, void* stream) {
    if (n < 0) return fail("frame_transform: negative point count");
    if (!mean || (n > 0 && (!pos || !pos_out || (cov && !cov_out))) || (n_rot > 0 && !rotations)) return fail("null argument");
    if (n_rot < 0 || n_rot > 8) return fail("frame_transform: at most 8 rotations");
    if (require_device()) return 1;
    return check("frame_transform", pixie::frame_transform(pos, cov, n, z_shift, scale, mean, rotations, n_rot, pos_out, cov_out, (cudaStream_t)stream));
}
int pixie_gaussian_ply_records(const float* pos, const float* cov, const float* shs, int K, const float* opacity, int n, float* records,
                               void* stream) {
    if (n < 0) return fail("gaussian_ply_records: negative point count");
    if (K != 1 && K != 4 && K != 9 && K != 16) return fail("gaussian_ply_records: K must be 1, 4, 9 or 16 SH coefficients");
    if (n > 0 && (!pos || !cov || !shs || !opacity || !records)) return fail("null argument");
    if (require_device()) return 1;
    return check("gaussian_ply_records", pixie::gaussian_ply_records(pos, cov, shs, K, opacity, n, records, (cudaStream_t)stream));
}
// The checks both checkpoint decodes share: K, the row stride and the column offsets (cols [11 + 3K] bytes) into c.
static int checkpoint_columns(const char* op, int row_bytes, const int* cols, int K, pixie::GsColumns& c) {
    const std::string who(op);
    if (K != 1 && K != 4 && K != 9 && K != 16) return fail(who + ": K must be 1, 4, 9 or 16 SH coefficients");
    if (row_bytes < 4 || row_bytes % 4 != 0 || row_bytes / 4 > pixie::kGsLoadMaxRowWords)
        return fail(who + ": the row stride must be a multiple of 4 bytes, at most " + std::to_string(4 * pixie::kGsLoadMaxRowWords));
    const int row_words = row_bytes / 4, n_cols = 11 + 3 * K;
    c = pixie::GsColumns{};
    int* dst[59];
    int k = 0;
    for (int i = 0; i < 3; ++i) dst[k++] = &c.xyz[i];
    for (int i = 0; i < 3; ++i) dst[k++] = &c.dc[i];
    for (int i = 0; i < 3 * (K - 1); ++i) dst[k++] = &c.rest[i];
    dst[k++] = &c.opacity;
    for (int i = 0; i < 3; ++i) dst[k++] = &c.scale[i];
    for (int i = 0; i < 4; ++i) dst[k++] = &c.rot[i];
    for (int i = 0; i < n_cols; ++i) {
        if (cols[i] < 0 || cols[i] % 4 != 0 || cols[i] / 4 >= row_words)
            return fail(who + ": column " + std::to_string(i) + " is not a 4-byte aligned offset inside the row");
        *dst[i] = cols[i] / 4;
    }
    return 0;
}
int pixie_gaussian_checkpoint_decode(const void* table, long long n, int row_bytes, const int* cols, int K, int has_threshold, float threshold,
                                     float* pos, float* shs, float* opacity, float* cov, long long* m_host, void* stream) {
    if (!cols || !m_host || (n > 0 && (!table || !pos || !shs || !opacity || !cov))) return fail("null argument");
    if (n < 0) return fail("gaussian_checkpoint_decode: negative row count");
    pixie::GsColumns c;
    if (checkpoint_columns("gaussian_checkpoint_decode", row_bytes, cols, K, c)) return 1;
    if (require_device()) return 1;
    return check("gaussian_checkpoint_decode", pixie::gaussian_checkpoint_decode(table, n, row_bytes / 4, c, K, has_threshold, threshold, pos, shs,
                                                                                 opacity, cov, m_host, (cudaStream_t)stream));
}
int pixie_gaussian_checkpoint_decode_scale_rot(const void* table, long long n, int row_bytes, const int* cols, int K, float* pos, float* shs,
                                               float* opacity, float* scales, float* rotations, void* stream) {
    if (!cols || (n > 0 && (!table || !pos || !shs || !opacity || !scales || !rotations))) return fail("null argument");
    if (n < 0) return fail("gaussian_checkpoint_decode_scale_rot: negative row count");
    pixie::GsColumns c;
    if (checkpoint_columns("gaussian_checkpoint_decode_scale_rot", row_bytes, cols, K, c)) return 1;
    if (require_device()) return 1;
    return check("gaussian_checkpoint_decode_scale_rot", pixie::gaussian_checkpoint_decode_scale_rot(table, n, row_bytes / 4, c, K, pos, shs, opacity,
                                                                                                     scales, rotations, (cudaStream_t)stream));
}
int pixie_image_metrics(const uint8_t* a, const uint8_t* b, int height, int width, const float window[11], double* out, void* stream) {
    if (!a || !b || !window || !out) return fail("null argument");
    if (height < 1 || width < 1 || (long long)height * width > 2147483647LL / 3) return fail("image_metrics: bad image size");
    if (require_device()) return 1;
    return check("image_metrics", pixie::image_metrics(a, b, height, width, window, out, (cudaStream_t)stream));
}
int pixie_material_metrics(const float* mat, int c_mat, const float* mask, const float* seg, int n_classes, const float* cont, int n,
                           int64_t voxels, const double* ranges, int background_id, float* gt, long long* counts, double* sums, void* stream) {
    if (!ranges || (n > 0 && (!mat || !seg || !cont || !gt || !counts || !sums))) return fail("null argument");
    if (n < 0 || voxels < 1) return fail("material_metrics: need n >= 0 samples of at least one voxel");
    if (c_mat < 4) return fail("material_metrics: the material grid needs at least 4 channels (density, E, nu, ..., material id)");
    if (n_classes < 1) return fail("material_metrics: need at least one class");
    pixie::MaterialNorm nm;
    for (int c = 0; c < 3; ++c) {
        const double lo = ranges[2 * c], hi = ranges[2 * c + 1];
        nm.lo[c] = (float)lo;
        nm.hi[c] = (float)hi;
        nm.span[c] = (float)(hi - lo);
    }
    if (require_device()) return 1;
    return check("material_metrics", pixie::material_metrics(mat, c_mat, mask, seg, n_classes, cont, n, voxels, nm, background_id, gt, counts, sums,
                                                             (cudaStream_t)stream));
}
// n^3 cells and their offsets are int32 on the device
static bool fill_grid_ok(int grid_n) { return grid_n >= 1 && grid_n <= 1290; }
int pixie_fill_density(const float* pos, const float* opacity, const float* cov, int n, int grid_n, float grid_dx, int* count, float* density,
                       void* stream) {
    if (!count || !density || (n > 0 && (!pos || !opacity || !cov))) return fail("null argument");
    if (n < 0 || !fill_grid_ok(grid_n) || !(grid_dx > 0.f)) return fail("fill_density: need n >= 0, 1 <= grid_n <= 1290 and grid_dx > 0");
    if (require_device()) return 1;
    return check("fill_density", pixie::fill_density(pos, opacity, cov, n, grid_n, grid_dx, count, density, (cudaStream_t)stream));
}
int pixie_fill_grids(int* count, const float* density, int grid_n, float grid_dx, const float origin[3], float density_thres, float search_thres,
                     int max_particles_per_cell, int exclude_dir, int ray_cast_dir, unsigned long long seed, float* out, int max_samples,
                     int* n_dense_host, int* n_total_host, void* stream) {
    if (!count || !density || !origin || !n_dense_host || !n_total_host || (max_samples > 0 && !out)) return fail("null argument");
    if (!fill_grid_ok(grid_n) || !(grid_dx > 0.f)) return fail("fill_grids: need 1 <= grid_n <= 1290 and grid_dx > 0");
    if (max_particles_per_cell < 1 || (long long)grid_n * grid_n * grid_n * max_particles_per_cell > 2147483647LL)
        return fail("fill_grids: need 1 <= max_particles_per_cell and grid_n^3 * max_particles_per_cell < 2^31");
    if (exclude_dir < 0 || exclude_dir > 5 || ray_cast_dir < 0 || ray_cast_dir > 5) return fail("fill_grids: directions must be in 0..5");
    if (max_samples < 0) return fail("fill_grids: negative max_samples");
    if (require_device()) return 1;
    if (check("fill_grids", pixie::fill_grids(count, density, grid_n, grid_dx, origin, density_thres, search_thres, max_particles_per_cell,
                                              exclude_dir, ray_cast_dir, seed, out, max_samples, n_dense_host, n_total_host, (cudaStream_t)stream)))
        return 1;
    if (*n_total_host > max_samples)
        return fail("fill_grids: filling adds " + std::to_string(*n_total_host) + " particles (" + std::to_string(*n_dense_host) +
                       " in dense cells) but max_samples is " + std::to_string(max_samples));
    return 0;
}
int pixie_nearest_gaussian(const float* pos, int n, const float* query, int m, int* index, void* stream) {
    if (n < 0 || m < 0) return fail("nearest_gaussian: negative count");
    if ((n > 0 && m > 0 && !pos) || (m > 0 && (!query || !index))) return fail("null argument");
    if (require_device()) return 1;
    return check("nearest_gaussian", pixie::nearest_gaussian(pos, n, query, m, index, (cudaStream_t)stream));
}
int pixie_nearest_vertex(const double* vert, int n, const float* query, int m, int* index, void* stream) {
    if (n < 0 || m < 0) return fail("nearest_vertex: negative count");
    if ((n > 0 && m > 0 && !vert) || (m > 0 && (!query || !index))) return fail("null argument");
    if (require_device()) return 1;
    return check("nearest_vertex", pixie::nearest_vertex(vert, n, query, m, index, (cudaStream_t)stream));
}
int pixie_knn_label_vote(const float* pos, int n, const int64_t* labels, int k, int64_t* out, void* stream) {
    if (n < 0) return fail("knn_label_vote: negative count");
    if (n > 0 && (k < 1 || k > n)) return fail("knn_label_vote: k must be in [1, n]");
    if (n > 0 && (!pos || !labels || !out)) return fail("null argument");
    if (require_device()) return 1;
    return check("knn_label_vote", pixie::knn_label_vote(pos, n, (const long long*)labels, k, (long long*)out, (cudaStream_t)stream));
}
// ------------------------------------------------------------------------------------- VLM part segmentation
int pixie_part_similarity(const void* feat, const uint8_t* mask, int64_t n_voxels, int C, int n_occupied, const float* query, int P,
                          float inv_temperature, float* sims, int64_t* labels, float* scores, float* probs, void* stream) {
    if (n_voxels < 0 || n_occupied < 0) return fail("part_similarity: negative count");
    if (n_voxels > INT32_MAX) return fail("part_similarity: more than 2^31 - 1 voxels");
    if (C < 1) return fail("part_similarity: C must be >= 1");
    if (P < 1 || P > pixie::kMaxParts) return fail("part_similarity: P must be in [1, " + std::to_string(pixie::kMaxParts) + "]");
    if (n_occupied > n_voxels) return fail("part_similarity: more occupied voxels than voxels");
    if (n_occupied > 0 && (!feat || !query || !sims || !labels || !scores)) return fail("null argument");
    if (require_device()) return 1;
    return check("part_similarity", pixie::part_similarity((const __half*)feat, mask, n_voxels, C, n_occupied, query, P, inv_temperature,
                                                           sims, labels, scores, probs, (cudaStream_t)stream));
}
// ------------------------------------------------------------------------------------- Gaussian rasteriser
int pixie_gs_renderer_create(pixie_gs_renderer_t* out) {
    if (!out) return fail("null argument");
    if (require_device()) return 1;
    *out = pixie::gs_renderer_create();
    return *out ? 0 : 1;
}
// The checks and argument block both rasterizer entry points share; the caller sets the covariance source.
static int gs_render_args(pixie_gs_renderer_t h, const float* means, const float* opacity, const float* shs, int sh_coeffs, int sh_degree,
                          int n, const float view[16], const float proj[16], const float campos[3], float tan_fovx, float tan_fovy,
                          int width, int height, const float bg[3], float* image, int* radii, pixie::GsRenderArgs& a) {
    if (!h) return fail("null handle");
    if (!view || !proj || !campos || !bg || !image || (n > 0 && (!means || !opacity || !radii))) return fail("null argument");
    if (n < 0) return fail("gs_render: negative Gaussian count");
    if (width < 1 || height < 1 || (long long)width * height > 2147483647LL) return fail("gs_render: bad image size");
    if (!(tan_fovx > 0.f) || !(tan_fovy > 0.f)) return fail("gs_render: tan(fov) must be positive");
    if (shs && (sh_degree < 0 || sh_degree > 3 || (sh_degree + 1) * (sh_degree + 1) > sh_coeffs))
        return fail("gs_render: need 0 <= sh_degree <= 3 and (sh_degree + 1)^2 <= sh_coeffs");
    a = pixie::GsRenderArgs{};
    a.means = means; a.opacity = opacity; a.shs = shs;
    a.n = n; a.sh_coeffs = sh_coeffs; a.sh_degree = sh_degree;
    std::memcpy(a.view, view, sizeof(a.view));
    std::memcpy(a.proj, proj, sizeof(a.proj));
    std::memcpy(a.campos, campos, sizeof(a.campos));
    std::memcpy(a.bg, bg, sizeof(a.bg));
    a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy; a.width = width; a.height = height; a.image = image; a.radii = radii;
    return 0;
}
int pixie_gs_render(pixie_gs_renderer_t h, const float* means, const float* cov, const float* opacity, const float* shs, int sh_coeffs,
                    int sh_degree, const float* colors, int n, const float view[16], const float proj[16], const float campos[3],
                    float tan_fovx, float tan_fovy, int width, int height, const float bg[3], float* image, int* radii, int* n_rendered,
                    float* phase_ms, void* stream) {
    if (h && n > 0 && (!cov || (!shs && !colors))) return fail("null argument");
    pixie::GsRenderArgs a;
    if (gs_render_args(h, means, opacity, shs, sh_coeffs, sh_degree, n, view, proj, campos, tan_fovx, tan_fovy, width, height, bg, image,
                       radii, a))
        return 1;
    a.cov = cov; a.colors = shs ? nullptr : colors;
    return pixie::gs_render(h, a, n_rendered, phase_ms, (cudaStream_t)stream);
}
int pixie_gs_render_scale_rot(pixie_gs_renderer_t h, const float* means, const float* scales, const float* rotations, const float* opacity,
                              const float* shs, int sh_coeffs, int sh_degree, int n, const float view[16], const float proj[16],
                              const float campos[3], float tan_fovx, float tan_fovy, int width, int height, const float bg[3], float* image,
                              int* radii, int* n_rendered, float* phase_ms, void* stream) {
    if (h && n > 0 && (!scales || !rotations || !shs)) return fail("null argument");
    pixie::GsRenderArgs a;
    if (gs_render_args(h, means, opacity, shs, sh_coeffs, sh_degree, n, view, proj, campos, tan_fovx, tan_fovy, width, height, bg, image,
                       radii, a))
        return 1;
    a.scales = scales; a.rotations = rotations;
    return pixie::gs_render(h, a, n_rendered, phase_ms, (cudaStream_t)stream);
}
void pixie_gs_renderer_destroy(pixie_gs_renderer_t h) { pixie::gs_renderer_destroy(h); }
int pixie_pack_predictions(const float* seg_logits_dev, const float* cont_dev, float* out_dev, int batch, int64_t voxels, int n_classes, void* stream) {
    if (!seg_logits_dev || !cont_dev || !out_dev) return fail("null argument");
    if (require_device()) return 1;
    return check("pack_predictions",
                 (cudaError_t)pixie::launch_pack_predictions(seg_logits_dev, cont_dev, out_dev, batch, voxels, n_classes, (cudaStream_t)stream));
}
int pixie_unet_launch_count(pixie_unet_t h) { return h ? pixie::unet_launch_count(h) : 0; }
double pixie_unet_flops(pixie_unet_t h) { return h ? pixie::unet_flops(h) : 0.0; }
int pixie_unet_check(pixie_unet_t h) {
    if (!h) return fail("null handle");
    return pixie::unet_check(h);
}
int64_t pixie_unet_debug_fetch(pixie_unet_t h, const char* name, float* host_out, int64_t capacity) {
    if (!h || !name) { fail("null argument"); return -1; }
    return pixie::unet_debug_fetch(h, name, host_out, capacity);
}
int64_t pixie_unet_debug_names(pixie_unet_t h, char* buf, int64_t capacity) {
    if (!h || (!buf && capacity > 0)) { fail("null argument"); return -1; }
    const std::string s = pixie::unet_debug_names(h);
    if (capacity > 0) {
        const size_t n = std::min(s.size(), (size_t)capacity - 1);
        memcpy(buf, s.data(), n);
        buf[n] = '\0';
    }
    return (int64_t)s.size();
}
void pixie_unet_destroy(pixie_unet_t h) { pixie::unet_destroy(h); }

// ------------------------------------------------------------------------------------- MPM
int pixie_mpm_create(int n_particles, int n_grid, float grid_lim, pixie_mpm_t* out) {
    if (!out) return fail("null argument");
    if (require_device()) return 1;
    *out = pixie::mpm_create(n_particles, n_grid, grid_lim);
    return *out ? 0 : 1;
}
int pixie_mpm_bind(pixie_mpm_t h, int field, void* dev_ptr) { return h ? pixie::mpm_bind(h, field, dev_ptr) : fail("null handle"); }
int pixie_mpm_set_params(pixie_mpm_t h, const pixie_mpm_params* p) { return !p ? fail("null params") : h ? pixie::mpm_set_params(h, *p) : fail("null handle"); }
int pixie_mpm_add_bc(pixie_mpm_t h, const pixie_mpm_bc* bc) { return !bc ? fail("null bc") : h ? pixie::mpm_add_bc(h, *bc) : fail("null handle"); }
int pixie_mpm_clear_bcs(pixie_mpm_t h) { return h ? pixie::mpm_clear_bcs(h) : fail("null handle"); }
int pixie_mpm_set_time(pixie_mpm_t h, double t) { return h ? pixie::mpm_set_time(h, t) : fail("null handle"); }
int pixie_mpm_get_time(pixie_mpm_t h, double* t) { return h ? pixie::mpm_get_time(h, t) : fail("null handle"); }
int pixie_mpm_step(pixie_mpm_t h, int n, double dt, void* stream) { return h ? pixie::mpm_step(h, n, dt, (cudaStream_t)stream) : fail("null handle"); }
int pixie_mpm_compute_mu_lam(pixie_mpm_t h, void* s) { return h ? pixie::mpm_compute_mu_lam(h, (cudaStream_t)s) : fail("null handle"); }
int pixie_mpm_compute_bulk(pixie_mpm_t h, void* s) { return h ? pixie::mpm_compute_bulk(h, (cudaStream_t)s) : fail("null handle"); }
int pixie_mpm_compute_mass(pixie_mpm_t h, void* s) { return h ? pixie::mpm_compute_mass(h, (cudaStream_t)s) : fail("null handle"); }
int pixie_mpm_compute_cov_from_F(pixie_mpm_t h, void* s) { return h ? pixie::mpm_compute_cov_from_F(h, (cudaStream_t)s) : fail("null handle"); }
int pixie_mpm_compute_R_from_F(pixie_mpm_t h, void* s) { return h ? pixie::mpm_compute_R_from_F(h, (cudaStream_t)s) : fail("null handle"); }
int pixie_mpm_apply_additional_params(pixie_mpm_t h, const float* boxes, int n_boxes, void* s) {
    return h ? pixie::mpm_apply_additional_params(h, boxes, n_boxes, (cudaStream_t)s) : fail("null handle");
}
int pixie_mpm_select_box(pixie_mpm_t h, const float point[3], const float size[3], int* mask, void* s) {
    return h ? pixie::mpm_select_box(h, point, size, mask, (cudaStream_t)s) : fail("null handle");
}
int pixie_mpm_select_cylinder(pixie_mpm_t h, const float point[3], const float normal[3], float hh, float radius, int* mask, void* s) {
    return h ? pixie::mpm_select_cylinder(h, point, normal, hh, radius, mask, (cudaStream_t)s) : fail("null handle");
}
int pixie_mpm_sync(pixie_mpm_t h, void* s) { return h ? pixie::mpm_sync(h, (cudaStream_t)s) : fail("null handle"); }
int pixie_mpm_set_active_count(pixie_mpm_t h, int n_active) { return h ? pixie::mpm_set_active_count(h, n_active) : fail("null handle"); }
int pixie_mpm_grid_ptrs(pixie_mpm_t h, float** mv4, float** v4) { return h ? pixie::mpm_grid_ptrs(h, mv4, v4) : fail("null handle"); }
int pixie_mpm_exchange_buffer(pixie_mpm_t h, void** base, size_t* bytes) { return h ? pixie::mpm_exchange_buffer(h, base, bytes) : fail("null handle"); }
int pixie_mpm_slab_attach(pixie_mpm_t h, int x0, int x1, int slack, const void* left, const void* right) {
    return h ? pixie::mpm_slab_attach(h, x0, x1, slack, left, right) : fail("null handle");
}
int pixie_mpm_slab_phase(pixie_mpm_t h, int phase, double dt, void* s) { return h ? pixie::mpm_slab_phase(h, phase, dt, (cudaStream_t)s) : fail("null handle"); }
int pixie_mpm_slab_error(pixie_mpm_t h, int* flag) { return h ? pixie::mpm_slab_error(h, flag) : fail("null handle"); }
int pixie_mpm_slab_excursion(pixie_mpm_t h, int* d_out, void* s) { return h ? pixie::mpm_slab_excursion(h, d_out, (cudaStream_t)s) : fail("null handle"); }
int pixie_ipc_export(const void* dev_ptr, unsigned char handle[64]) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t size");
    cudaIpcMemHandle_t hd;
    if (check("cudaIpcGetMemHandle", cudaIpcGetMemHandle(&hd, const_cast<void*>(dev_ptr)))) return 1;
    memcpy(handle, &hd, 64);
    return 0;
}
int pixie_ipc_open(const unsigned char handle[64], void** dev_ptr) {
    cudaIpcMemHandle_t hd;
    memcpy(&hd, handle, 64);
    return check("cudaIpcOpenMemHandle", cudaIpcOpenMemHandle(dev_ptr, hd, cudaIpcMemLazyEnablePeerAccess));
}
int pixie_ipc_close(void* dev_ptr) { return check("cudaIpcCloseMemHandle", cudaIpcCloseMemHandle(dev_ptr)); }
long long pixie_mpm_launch_count(pixie_mpm_t h) { return h ? pixie::mpm_launch_count(h) : 0; }
void pixie_mpm_destroy(pixie_mpm_t h) { pixie::mpm_destroy(h); }

}  // extern "C"
