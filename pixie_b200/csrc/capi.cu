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
#include "material_metrics.cuh"

#include <algorithm>
#include <cstring>
#include <string>

namespace {
thread_local std::string g_err;
int set_err(const std::string& e) { g_err = e; return 1; }
// 0 on success, otherwise 1 with "<op>: <CUDA's description of e>" as the last error
int check(const char* op, cudaError_t e) { return e == cudaSuccess ? 0 : set_err(std::string(op) + ": " + cudaGetErrorString(e)); }
}  // namespace

struct pixie_unet_s { pixie::UNet* u; };
struct pixie_mpm_s { pixie::Mpm* m; };
struct pixie_gs_renderer_s { pixie::GsRenderer* r; };

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
    if (!pixie_device_ok()) return set_err("pixie_b200 requires an sm_90 (H100) CUDA device; there is no CPU fallback");
    return 0;
}

// ------------------------------------------------------------------------------------- U-Net
int pixie_unet_create(const pixie_unet_config* cfg, pixie_unet_t* out) {
    if (!cfg || !out) return set_err("null argument");
    if (require_device()) return 1;
    std::string e;
    pixie::UNet* u = pixie::unet_create(*cfg, e);
    if (!u) return set_err(e);
    *out = new pixie_unet_s{u};
    return 0;
}
int pixie_unet_set_tensor(pixie_unet_t h, const char* name, const float* host_data, const int64_t* shape, int ndim) {
    if (!h || !name || !host_data) return set_err("null argument");
    if (pixie::unet_set_tensor(h->u, name, host_data, shape, ndim)) return set_err(pixie::unet_error(h->u));
    return 0;
}
int pixie_unet_finalize(pixie_unet_t h) {
    if (!h) return set_err("null handle");
    if (pixie::unet_finalize(h->u)) return set_err(pixie::unet_error(h->u));
    return 0;
}
int pixie_unet_forward(pixie_unet_t h, const void* feat, int batch, float* out, void* stream) {
    if (!h || !feat || !out) return set_err("null argument");
    if (pixie::unet_forward(h->u, feat, batch, out, (cudaStream_t)stream)) return set_err(pixie::unet_error(h->u));
    return 0;
}
int pixie_unet_forward_ncdhw(pixie_unet_t h, const float* feat, int batch, float* out, void* stream) {
    if (!h || !feat || !out) return set_err("null argument");
    if (pixie::unet_forward_ncdhw(h->u, feat, batch, out, (cudaStream_t)stream)) return set_err(pixie::unet_error(h->u));
    return 0;
}
int pixie_unet_forward_host(pixie_unet_t h, const void* feat, int batch, float* out, void* stream) {
    if (!h || !feat || !out) return set_err("null argument");
    if (pixie::unet_forward_host(h->u, feat, batch, out, (cudaStream_t)stream)) return set_err(pixie::unet_error(h->u));
    return 0;
}
int pixie_unet_profile(pixie_unet_t h, const void* feat, int batch, float* out, void* stream, float* ms, int* kinds, double* flops, int cap) {
    if (!h || !feat || !out || !ms || !kinds || !flops) { set_err("null argument"); return -1; }
    const int n = pixie::unet_profile(h->u, feat, batch, out, (cudaStream_t)stream, ms, kinds, flops, cap);
    if (n < 0) set_err(pixie::unet_error(h->u));
    return n;
}
int pixie_field_extract(const float* pred, int n_classes, const float* mask, int D, const double ranges[6], const double bmin[3], const double bmax[3],
                        float* pos, float* density, float* E, float* nu, int* material, float* conf, int* count_host, void* stream) {
    if (!pred || !mask || !ranges || !bmin || !bmax || !pos || !density || !E || !nu || !material || !conf || !count_host) return set_err("null argument");
    if (D < 2 || D > 1290 || n_classes < 1)
        return set_err("field_extract: need 2 <= D <= 1290 (D^3 voxels are indexed in int32) and at least one class channel");
    if (require_device()) return 1;
    return check("field_extract", pixie::field_extract(pred, n_classes, mask, D, ranges, bmin, bmax, pos, density, E, nu, material, conf,
                                                       count_host, (cudaStream_t)stream));
}
int pixie_knn_assign(const float* query, int nq, const float* pos, const float* density, const float* E, const float* nu, const int* material,
                     const int* part, const float* conf, int m, int k, double threshold, int weighted, const float defaults[4], int def_material,
                     int def_part, float* o_density, float* o_E, float* o_nu, int* o_material, int* o_part, float* o_conf, int* n_too_far_host,
                     void* stream) {
    if (!query || !pos || !density || !E || !nu || !material || !part || !conf || !defaults || !o_density || !o_E || !o_nu || !o_material ||
        !o_part || !o_conf || !n_too_far_host) return set_err("null argument");
    if (k < 1 || k > 16) return set_err("knn_assign: k must be in [1, 16]");
    if (m < 1) return set_err("knn_assign: empty material point cloud");
    if (k > m) return set_err("knn_assign: k exceeds the number of material points");
    if (require_device()) return 1;
    return check("knn_assign", pixie::knn_assign(query, nq, pos, density, E, nu, material, part, conf, m, k, threshold, weighted, defaults,
                                                 def_material, def_part, o_density, o_E, o_nu, o_material, o_part, o_conf, n_too_far_host,
                                                 (cudaStream_t)stream));
}
int pixie_dbscan(const float* pos, int n, const int* ids, int select_id, double eps, int min_samples, int* index, int* labels,
                 int* n_selected_host, int* n_clusters_host, void* stream) {
    if (!n_selected_host || !n_clusters_host || (n > 0 && (!pos || !index || !labels))) return set_err("null argument");
    if (n < 0) return set_err("dbscan: negative point count");
    if (!(eps > 0.0) || min_samples < 1) return set_err("dbscan: need eps > 0 and min_samples >= 1");
    if (require_device()) return 1;
    return check("dbscan", pixie::dbscan(pos, n, ids, select_id, eps, min_samples, index, labels, n_selected_host, n_clusters_host,
                                         (cudaStream_t)stream));
}
int pixie_cluster_stats(const float* pos, const int* index, const int* labels, int n_selected, int n_clusters, int* sizes,
                        float* bbox_min, float* bbox_max, void* stream) {
    if (n_selected < 0 || n_clusters < 0) return set_err("cluster_stats: negative count");
    if ((n_selected > 0 && (!pos || !index || !labels)) || (n_clusters > 0 && (!sizes || !bbox_min || !bbox_max))) return set_err("null argument");
    if (require_device()) return 1;
    return check("cluster_stats", pixie::cluster_stats(pos, index, labels, n_selected, n_clusters, sizes, bbox_min, bbox_max, (cudaStream_t)stream));
}
int pixie_particle_volume(const float* pos, int n, int grid_n, float grid_dx, float* vol, void* stream) {
    if (n < 0) return set_err("particle_volume: negative point count");
    if (n > 0 && (!pos || !vol)) return set_err("null argument");
    if (grid_n < 1 || !(grid_dx > 0.f)) return set_err("particle_volume: bad grid");
    if (require_device()) return 1;
    return check("particle_volume", pixie::particle_volume(pos, n, grid_n, grid_dx, vol, (cudaStream_t)stream));
}
int pixie_frame_transform(const float* pos, const float* cov, int n, float z_shift, float scale, const float mean[3], const float* rotations,
                          int n_rot, float* pos_out, float* cov_out, void* stream) {
    if (n < 0) return set_err("frame_transform: negative point count");
    if (!mean || (n > 0 && (!pos || !pos_out || (cov && !cov_out))) || (n_rot > 0 && !rotations)) return set_err("null argument");
    if (n_rot < 0 || n_rot > 8) return set_err("frame_transform: at most 8 rotations");
    if (require_device()) return 1;
    return check("frame_transform", pixie::frame_transform(pos, cov, n, z_shift, scale, mean, rotations, n_rot, pos_out, cov_out, (cudaStream_t)stream));
}
int pixie_gaussian_ply_records(const float* pos, const float* cov, const float* shs, int K, const float* opacity, int n, float* records,
                               void* stream) {
    if (n < 0) return set_err("gaussian_ply_records: negative point count");
    if (K != 1 && K != 4 && K != 9 && K != 16) return set_err("gaussian_ply_records: K must be 1, 4, 9 or 16 SH coefficients");
    if (n > 0 && (!pos || !cov || !shs || !opacity || !records)) return set_err("null argument");
    if (require_device()) return 1;
    return check("gaussian_ply_records", pixie::gaussian_ply_records(pos, cov, shs, K, opacity, n, records, (cudaStream_t)stream));
}
int pixie_gaussian_checkpoint_decode(const void* table, long long n, int row_bytes, const int* cols, int K, int has_threshold, float threshold,
                                     float* pos, float* shs, float* opacity, float* cov, long long* m_host, void* stream) {
    if (!cols || !m_host || (n > 0 && (!table || !pos || !shs || !opacity || !cov))) return set_err("null argument");
    if (n < 0) return set_err("gaussian_checkpoint_decode: negative row count");
    if (K != 1 && K != 4 && K != 9 && K != 16) return set_err("gaussian_checkpoint_decode: K must be 1, 4, 9 or 16 SH coefficients");
    if (row_bytes < 4 || row_bytes % 4 != 0 || row_bytes / 4 > pixie::kGsLoadMaxRowWords)
        return set_err("gaussian_checkpoint_decode: the row stride must be a multiple of 4 bytes, at most " +
                       std::to_string(4 * pixie::kGsLoadMaxRowWords));
    const int row_words = row_bytes / 4, n_cols = 11 + 3 * K;
    pixie::GsColumns c{};
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
            return set_err("gaussian_checkpoint_decode: column " + std::to_string(i) + " is not a 4-byte aligned offset inside the row");
        *dst[i] = cols[i] / 4;
    }
    if (require_device()) return 1;
    return check("gaussian_checkpoint_decode", pixie::gaussian_checkpoint_decode(table, n, row_words, c, K, has_threshold, threshold, pos, shs, opacity,
                                                                                 cov, m_host, (cudaStream_t)stream));
}
int pixie_material_metrics(const float* mat, int c_mat, const float* mask, const float* seg, int n_classes, const float* cont, int n,
                           int64_t voxels, const double* ranges, int background_id, float* gt, long long* counts, double* sums, void* stream) {
    if (!ranges || (n > 0 && (!mat || !seg || !cont || !gt || !counts || !sums))) return set_err("null argument");
    if (n < 0 || voxels < 1) return set_err("material_metrics: need n >= 0 samples of at least one voxel");
    if (c_mat < 4) return set_err("material_metrics: the material grid needs at least 4 channels (density, E, nu, ..., material id)");
    if (n_classes < 1) return set_err("material_metrics: need at least one class");
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
    if (!count || !density || (n > 0 && (!pos || !opacity || !cov))) return set_err("null argument");
    if (n < 0 || !fill_grid_ok(grid_n) || !(grid_dx > 0.f)) return set_err("fill_density: need n >= 0, 1 <= grid_n <= 1290 and grid_dx > 0");
    if (require_device()) return 1;
    return check("fill_density", pixie::fill_density(pos, opacity, cov, n, grid_n, grid_dx, count, density, (cudaStream_t)stream));
}
int pixie_fill_grids(int* count, const float* density, int grid_n, float grid_dx, const float origin[3], float density_thres, float search_thres,
                     int max_particles_per_cell, int exclude_dir, int ray_cast_dir, unsigned long long seed, float* out, int max_samples,
                     int* n_dense_host, int* n_total_host, void* stream) {
    if (!count || !density || !origin || !n_dense_host || !n_total_host || (max_samples > 0 && !out)) return set_err("null argument");
    if (!fill_grid_ok(grid_n) || !(grid_dx > 0.f)) return set_err("fill_grids: need 1 <= grid_n <= 1290 and grid_dx > 0");
    if (max_particles_per_cell < 1 || (long long)grid_n * grid_n * grid_n * max_particles_per_cell > 2147483647LL)
        return set_err("fill_grids: need 1 <= max_particles_per_cell and grid_n^3 * max_particles_per_cell < 2^31");
    if (exclude_dir < 0 || exclude_dir > 5 || ray_cast_dir < 0 || ray_cast_dir > 5) return set_err("fill_grids: directions must be in 0..5");
    if (max_samples < 0) return set_err("fill_grids: negative max_samples");
    if (require_device()) return 1;
    if (check("fill_grids", pixie::fill_grids(count, density, grid_n, grid_dx, origin, density_thres, search_thres, max_particles_per_cell,
                                              exclude_dir, ray_cast_dir, seed, out, max_samples, n_dense_host, n_total_host, (cudaStream_t)stream)))
        return 1;
    if (*n_total_host > max_samples)
        return set_err("fill_grids: filling adds " + std::to_string(*n_total_host) + " particles (" + std::to_string(*n_dense_host) +
                       " in dense cells) but max_samples is " + std::to_string(max_samples));
    return 0;
}
int pixie_nearest_gaussian(const float* pos, int n, const float* query, int m, int* index, void* stream) {
    if (n < 0 || m < 0) return set_err("nearest_gaussian: negative count");
    if ((n > 0 && m > 0 && !pos) || (m > 0 && (!query || !index))) return set_err("null argument");
    if (require_device()) return 1;
    return check("nearest_gaussian", pixie::nearest_gaussian(pos, n, query, m, index, (cudaStream_t)stream));
}
// ------------------------------------------------------------------------------------- Gaussian rasteriser
int pixie_gs_renderer_create(pixie_gs_renderer_t* out) {
    if (!out) return set_err("null argument");
    if (require_device()) return 1;
    pixie::GsRenderer* r = pixie::gs_renderer_create();
    if (!r) return set_err("gs_renderer_create: out of memory");
    *out = new pixie_gs_renderer_s{r};
    return 0;
}
int pixie_gs_render(pixie_gs_renderer_t h, const float* means, const float* cov, const float* opacity, const float* shs, int sh_coeffs,
                    int sh_degree, const float* colors, int n, const float view[16], const float proj[16], const float campos[3],
                    float tan_fovx, float tan_fovy, int width, int height, const float bg[3], float* image, int* radii, int* n_rendered,
                    float* phase_ms, void* stream) {
    if (!h) return set_err("null handle");
    if (!view || !proj || !campos || !bg || !image || (n > 0 && (!means || !cov || !opacity || !radii || (!shs && !colors))))
        return set_err("null argument");
    if (n < 0) return set_err("gs_render: negative Gaussian count");
    if (width < 1 || height < 1 || (long long)width * height > 2147483647LL) return set_err("gs_render: bad image size");
    if (!(tan_fovx > 0.f) || !(tan_fovy > 0.f)) return set_err("gs_render: tan(fov) must be positive");
    if (shs && (sh_degree < 0 || sh_degree > 3 || (sh_degree + 1) * (sh_degree + 1) > sh_coeffs))
        return set_err("gs_render: need 0 <= sh_degree <= 3 and (sh_degree + 1)^2 <= sh_coeffs");
    pixie::GsRenderArgs a{};
    a.means = means; a.cov = cov; a.opacity = opacity; a.shs = shs; a.colors = shs ? nullptr : colors;
    a.n = n; a.sh_coeffs = sh_coeffs; a.sh_degree = sh_degree;
    std::memcpy(a.view, view, sizeof(a.view));
    std::memcpy(a.proj, proj, sizeof(a.proj));
    std::memcpy(a.campos, campos, sizeof(a.campos));
    std::memcpy(a.bg, bg, sizeof(a.bg));
    a.tan_fovx = tan_fovx; a.tan_fovy = tan_fovy; a.width = width; a.height = height; a.image = image; a.radii = radii;
    if (pixie::gs_render(h->r, a, n_rendered, phase_ms, (cudaStream_t)stream)) return set_err(pixie::gs_error(h->r));
    return 0;
}
void pixie_gs_renderer_destroy(pixie_gs_renderer_t h) {
    if (!h) return;
    pixie::gs_renderer_destroy(h->r);
    delete h;
}
int pixie_pack_predictions(const float* seg_logits_dev, const float* cont_dev, float* out_dev, int batch, int64_t voxels, int n_classes, void* stream) {
    if (!seg_logits_dev || !cont_dev || !out_dev) return set_err("null argument");
    if (require_device()) return 1;
    return check("pack_predictions",
                 (cudaError_t)pixie::launch_pack_predictions(seg_logits_dev, cont_dev, out_dev, batch, voxels, n_classes, (cudaStream_t)stream));
}
int pixie_unet_launch_count(pixie_unet_t h) { return h ? pixie::unet_launch_count(h->u) : 0; }
double pixie_unet_flops(pixie_unet_t h) { return h ? pixie::unet_flops(h->u) : 0.0; }
int pixie_unet_check(pixie_unet_t h) {
    if (!h) return set_err("null handle");
    if (pixie::unet_check(h->u)) return set_err(pixie::unet_error(h->u));
    return 0;
}
int64_t pixie_unet_debug_fetch(pixie_unet_t h, const char* name, float* host_out, int64_t capacity) {
    if (!h || !name) { set_err("null argument"); return -1; }
    const int64_t n = pixie::unet_debug_fetch(h->u, name, host_out, capacity);
    if (n < 0) set_err(pixie::unet_error(h->u));
    return n;
}
int64_t pixie_unet_debug_names(pixie_unet_t h, char* buf, int64_t capacity) {
    if (!h || (!buf && capacity > 0)) { set_err("null argument"); return -1; }
    const std::string s = pixie::unet_debug_names(h->u);
    if (capacity > 0) {
        const size_t n = std::min(s.size(), (size_t)capacity - 1);
        memcpy(buf, s.data(), n);
        buf[n] = '\0';
    }
    return (int64_t)s.size();
}
void pixie_unet_destroy(pixie_unet_t h) {
    if (!h) return;
    pixie::unet_destroy(h->u);
    delete h;
}

// ------------------------------------------------------------------------------------- MPM
int pixie_mpm_create(int n_particles, int n_grid, float grid_lim, pixie_mpm_t* out) {
    if (!out) return set_err("null argument");
    if (require_device()) return 1;
    std::string e;
    pixie::Mpm* m = pixie::mpm_create(n_particles, n_grid, grid_lim, e);
    if (!m) return set_err(e);
    *out = new pixie_mpm_s{m};
    return 0;
}
#define MPM_CALL(expr) do { if (!h) return set_err("null handle"); if (expr) return set_err(pixie::mpm_error(h->m)); return 0; } while (0)
int pixie_mpm_bind(pixie_mpm_t h, int field, void* dev_ptr) { MPM_CALL(pixie::mpm_bind(h->m, field, dev_ptr)); }
int pixie_mpm_set_params(pixie_mpm_t h, const pixie_mpm_params* p) { if (!p) return set_err("null params"); MPM_CALL(pixie::mpm_set_params(h->m, *p)); }
int pixie_mpm_add_bc(pixie_mpm_t h, const pixie_mpm_bc* bc) { if (!bc) return set_err("null bc"); MPM_CALL(pixie::mpm_add_bc(h->m, *bc)); }
int pixie_mpm_clear_bcs(pixie_mpm_t h) { MPM_CALL(pixie::mpm_clear_bcs(h->m)); }
int pixie_mpm_set_time(pixie_mpm_t h, double t) { MPM_CALL(pixie::mpm_set_time(h->m, t)); }
int pixie_mpm_get_time(pixie_mpm_t h, double* t) { MPM_CALL(pixie::mpm_get_time(h->m, t)); }
int pixie_mpm_step(pixie_mpm_t h, int n, double dt, void* stream) { MPM_CALL(pixie::mpm_step(h->m, n, dt, (cudaStream_t)stream)); }
int pixie_mpm_compute_mu_lam(pixie_mpm_t h, void* s) { MPM_CALL(pixie::mpm_compute_mu_lam(h->m, (cudaStream_t)s)); }
int pixie_mpm_compute_bulk(pixie_mpm_t h, void* s) { MPM_CALL(pixie::mpm_compute_bulk(h->m, (cudaStream_t)s)); }
int pixie_mpm_compute_mass(pixie_mpm_t h, void* s) { MPM_CALL(pixie::mpm_compute_mass(h->m, (cudaStream_t)s)); }
int pixie_mpm_compute_cov_from_F(pixie_mpm_t h, void* s) { MPM_CALL(pixie::mpm_compute_cov_from_F(h->m, (cudaStream_t)s)); }
int pixie_mpm_compute_R_from_F(pixie_mpm_t h, void* s) { MPM_CALL(pixie::mpm_compute_R_from_F(h->m, (cudaStream_t)s)); }
int pixie_mpm_apply_additional_params(pixie_mpm_t h, const float* boxes, int n_boxes, void* s) {
    MPM_CALL(pixie::mpm_apply_additional_params(h->m, boxes, n_boxes, (cudaStream_t)s));
}
int pixie_mpm_select_box(pixie_mpm_t h, const float point[3], const float size[3], int* mask, void* s) {
    MPM_CALL(pixie::mpm_select_box(h->m, point, size, mask, (cudaStream_t)s));
}
int pixie_mpm_select_cylinder(pixie_mpm_t h, const float point[3], const float normal[3], float hh, float radius, int* mask, void* s) {
    MPM_CALL(pixie::mpm_select_cylinder(h->m, point, normal, hh, radius, mask, (cudaStream_t)s));
}
int pixie_mpm_sync(pixie_mpm_t h, void* s) { MPM_CALL(pixie::mpm_sync(h->m, (cudaStream_t)s)); }
int pixie_mpm_set_active_count(pixie_mpm_t h, int n_active) { MPM_CALL(pixie::mpm_set_active_count(h->m, n_active)); }
int pixie_mpm_grid_ptrs(pixie_mpm_t h, float** mv4, float** v4) { MPM_CALL(pixie::mpm_grid_ptrs(h->m, mv4, v4)); }
int pixie_mpm_exchange_buffer(pixie_mpm_t h, void** base, size_t* bytes) { MPM_CALL(pixie::mpm_exchange_buffer(h->m, base, bytes)); }
int pixie_mpm_slab_attach(pixie_mpm_t h, int x0, int x1, int slack, const void* left, const void* right) {
    MPM_CALL(pixie::mpm_slab_attach(h->m, x0, x1, slack, left, right));
}
int pixie_mpm_slab_phase(pixie_mpm_t h, int phase, double dt, void* s) { MPM_CALL(pixie::mpm_slab_phase(h->m, phase, dt, (cudaStream_t)s)); }
int pixie_mpm_slab_error(pixie_mpm_t h, int* flag) { MPM_CALL(pixie::mpm_slab_error(h->m, flag)); }
int pixie_mpm_slab_excursion(pixie_mpm_t h, int* d_out, void* s) { MPM_CALL(pixie::mpm_slab_excursion(h->m, d_out, (cudaStream_t)s)); }
int pixie_ipc_export(const void* dev_ptr, unsigned char handle[64]) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t size");
    cudaIpcMemHandle_t hd;
    if (cudaIpcGetMemHandle(&hd, const_cast<void*>(dev_ptr)) != cudaSuccess) return set_err(std::string("cudaIpcGetMemHandle: ") + cudaGetErrorString(cudaGetLastError()));
    memcpy(handle, &hd, 64);
    return 0;
}
int pixie_ipc_open(const unsigned char handle[64], void** dev_ptr) {
    cudaIpcMemHandle_t hd;
    memcpy(&hd, handle, 64);
    if (cudaIpcOpenMemHandle(dev_ptr, hd, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess)
        return set_err(std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(cudaGetLastError()));
    return 0;
}
int pixie_ipc_close(void* dev_ptr) {
    if (cudaIpcCloseMemHandle(dev_ptr) != cudaSuccess) return set_err(std::string("cudaIpcCloseMemHandle: ") + cudaGetErrorString(cudaGetLastError()));
    return 0;
}
long long pixie_mpm_launch_count(pixie_mpm_t h) { return h ? pixie::mpm_launch_count(h->m) : 0; }
void pixie_mpm_destroy(pixie_mpm_t h) {
    if (!h) return;
    pixie::mpm_destroy(h->m);
    delete h;
}

}  // extern "C"
