/* pixie_b200 — C ABI of the H100-native hot path of vlongle/pixie.
 *
 * The reference has no FFI registry: its "boundary" for this path is three Python surfaces
 * (SURVEY.md §8b).  This header is what a binding of those surfaces calls; the reference-side stub a
 * maintainer would add (ctypes) is shown in INTEGRATION.md and shipped as pixie_b200/_lib.py.
 *
 * Conventions: plain pointers and sizes only (no torch types); every function returns 0 on success
 * and a non-zero code on failure. A failure always leaves a message for pixie_last_error() (one per host
 * thread, replaced by the next failure); when a CUDA call failed it reads "<operation>: <CUDA's
 * description>", and the thread's CUDA error is left clear, so the next call does not fail on it;
 * device pointers are BORROWED (the caller — torch in the Python shims — owns all tensors, as Warp
 * arrays alias torch memory in warp_utils.py:244-324); `stream` is a cudaStream_t passed as void*.
 * There is no CPU fallback: every entry point that computes requires an sm_90 (H100) device.
 */
#ifndef PIXIE_B200_H_
#define PIXIE_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* pixie_last_error(void);
/* ABI version of this header (checked by the Python loader). */
int pixie_abi_version(void);
/* 1 if the current CUDA device is sm_90 (H100), 0 otherwise / no device. */
int pixie_device_ok(void);

/* ===================================================================== U-Net (material field) ====
 * Replaces SegmentationUNet / RegressionUNet.__call__ under torch.no_grad()
 *   (third_party/Wavelet-Generation/trainer/training_discrete.py:50-88,
 *    training_continuous_mse.py:48-89, called at inference_combined.py:124-126),
 * i.e. FeatureProjector.forward (models/module/diffusion_network.py:588) followed by
 * MyUNetModel.forward (diffusion_network.py:899-935).
 */
typedef struct pixie_unet_s* pixie_unet_t;

typedef struct {
    int feature_channels;     /* channels of the input voxel grid (config: training.feature_channels) */
    int cond_dim;             /* projector output / U-Net input channels (32)                          */
    int model_channels;       /* 64                                                                   */
    int num_res_blocks;       /* 3                                                                    */
    int n_levels;             /* len(channel_mult)                                                    */
    int channel_mult[8];      /* (1,1,2,4)                                                            */
    int grid_size;            /* D = H = W of the voxel grid (64)                                     */
    int out_channels;         /* 8 (num_classes, segmentation) or 3 (regression)                      */
    int max_batch;            /* largest batch forward() will be called with                          */
    int precision;            /* 0: fp16 operands, fp32 accumulate (1 tensor-core pass; max-abs ~5e-3 vs fp32)
                               * 1: "fp16x3": operands split in fp16 hi + lo, three fp16 passes (max-abs ~6e-5)
                               * 2: "fp16e5": one fp16 pass + one E5M2 pass (kind::f8f6f4, twice the MMA rate) that adds
                               *    a_lo*w + a*w_lo = 2 pass-equivalents (max-abs ~3e-4, inside the 1e-3 tolerance) */
} pixie_unet_config;

/* Constructor arguments of SegmentationUNet / RegressionUNet (attention_resolutions must be ()). */
int pixie_unet_create(const pixie_unet_config* cfg, pixie_unet_t* out);
/* load_state_dict: one call per state-dict entry, reference key names, host fp32, torch layout
 * (training_utils.py:191-225 load_checkpoint -> model.load_state_dict). */
int pixie_unet_set_tensor(pixie_unet_t h, const char* name, const float* host_data,
                          const int64_t* shape, int ndim);
/* Packs weights (fp16, phase order), allocates workspaces, encodes TMA descriptors.
 * Fails if any state-dict entry of the architecture is missing. */
int pixie_unet_finalize(pixie_unet_t h);
/* forward(feat_grid): input fp16 channels-last (N, D, H, W, C) on the device — the on-disk layout of
 * clip_features_features.npy (pixie/voxel/voxelize.py:86,111); output fp32 (N, out_channels, D, H, W). */
int pixie_unet_forward(pixie_unet_t h, const void* feat_ndhwc_f16_dev, int batch,
                       float* out_ncdhw_f32_dev, void* stream);
/* Same, for callers holding the reference's fp32 (N, C, D, H, W) tensor (my_data.py:221): converts on
 * the device, then runs forward. */
int pixie_unet_forward_ncdhw(pixie_unet_t h, const float* feat_ncdhw_f32_dev, int batch,
                             float* out_ncdhw_f32_dev, void* stream);
/* End-to-end call for one batch with HOST buffers: pinned fp16 NDHWC in, fp32 NCDHW out (host);
 * host->device and device->host copies are issued on `stream` inside the call; returns after sync. */
int pixie_unet_forward_host(pixie_unet_t h, const void* feat_ndhwc_f16_host, int batch,
                            float* out_ncdhw_f32_host, void* stream);
/* Per-launch device times of one forward (CUDA events on `stream`, after one warm-up forward):
 * fills ms[i], kinds[i] (PIXIE_OP_*), flops[i] (algorithmic FLOPs, convolutions only) for each of the
 * n launches and returns n (<0 on error). Used by bench.py for the live roofline numbers. */
enum pixie_op_kind { PIXIE_OP_CONV = 0, PIXIE_OP_MOMENTS = 1, PIXIE_OP_NORM = 2, PIXIE_OP_UPSAMPLE = 3, PIXIE_OP_ATTENTION = 4 };
int pixie_unet_profile(pixie_unet_t h, const void* feat_ndhwc_f16_dev, int batch, float* out_ncdhw_f32_dev,
                       void* stream, float* ms, int* kinds, double* flops, int cap);
/* save_predictions packing (inference_combined.py:173-199, argmax :125): (3 + n_classes, D, H, W) fp32 =
 * continuous channels followed by the one-hot of argmax(seg_logits). All pointers device, planar NCDHW. */
int pixie_pack_predictions(const float* seg_logits_dev, const float* cont_dev, float* out_dev, int batch,
                           int64_t voxels, int n_classes, void* stream);
/* ---- material field -> particles (SURVEY.md 8f-1). All array pointers are DEVICE pointers unless marked host.
 * pixie_field_extract: pixie/voxel/map_pred_to_coords.py:41-75 (unscale_prediction: clip to [-1,1], 10**log for density
 * and E, linear nu) + :122-126, 198-245 (material id = argmax of the class channels, or the truncated class index when
 * n_classes == 1 and D == 64; confidence = max class value, 1 for one channel; np.linspace voxel centres, mask > 0
 * compaction in C order). pred = packed (3 + n_classes, D, D, D) fp32, mask = (D, D, D) fp32. ranges (host) =
 * {density_min, density_max, E_min, E_max, nu_min, nu_max} of normalization_ranges.yaml. Outputs need room for D^3
 * entries; *count_host = number of occupied voxels. Synchronises `stream`. */
int pixie_field_extract(const float* pred_dev, int n_classes, const float* mask_dev, int D, const double ranges_host[6],
                        const double min_bounds_host[3], const double max_bounds_host[3], float* pos_dev, float* density_dev,
                        float* E_dev, float* nu_dev, int* material_dev, float* conf_dev, int* count_host, void* stream);
/* pixie_knn_assign: PG/material_field.py:228-293 (perform_knn_smoothing) with assign_from_neighbors (:57-86): exact k nearest
 * material points per query (k <= 16), continuous properties = mean (np.mean order) or inverse-distance weighted mean,
 * categorical = mode (Counter.most_common / weighted bincount); queries farther than nn_distance_threshold from their nearest
 * point (compared in fp64, like scikit-learn's distances) receive the defaults {density, E, nu, conf}, default_material,
 * default_part. *n_too_far_host counts them. k must not exceed n_points (scikit-learn raises there too). */
int pixie_knn_assign(const float* query_dev, int n_query, const float* pos_dev, const float* density_dev, const float* E_dev,
                     const float* nu_dev, const int* material_dev, const int* part_dev, const float* conf_dev, int n_points, int k,
                     double nn_distance_threshold, int weighted, const float defaults_host[4], int default_material, int default_part,
                     float* out_density_dev, float* out_E_dev, float* out_nu_dev, int* out_material_dev, int* out_part_dev,
                     float* out_conf_dev, int* n_too_far_host, void* stream);
/* pixie_dbscan: the clustering of PG/material_field.py:365-480 (handle_stationary_clusters), scikit-learn DBSCAN semantics:
 * over the points i of pos [n][3] with ids_dev[i] == select_id (every point when ids_dev is NULL), in index order, neighbours
 * = fp64 squared distance <= eps^2 (self included), core = >= min_samples neighbours, clusters = connected core points labelled
 * in the order of their smallest core index, border points take the smallest adjacent label, the rest -1.
 * index_dev[t] = original index of the t-th selected point, labels_dev[t] = its label (both need room for n entries).
 * *n_selected_host / *n_clusters_host receive the counts. Synchronises `stream`. */
int pixie_dbscan(const float* pos_dev, int n, const int* ids_dev, int select_id, double eps, int min_samples, int* index_dev,
                 int* labels_dev, int* n_selected_host, int* n_clusters_host, void* stream);
/* pixie_cluster_stats: for the output of pixie_dbscan, per cluster the number of points (core + border) and the float32
 * bounding box of pos over them: sizes_dev [n_clusters], bbox_min_dev / bbox_max_dev [n_clusters][3]. */
int pixie_cluster_stats(const float* pos_dev, const int* index_dev, const int* labels_dev, int n_selected, int n_clusters,
                        int* sizes_dev, float* bbox_min_dev, float* bbox_max_dev, void* stream);
/* ---- either side of the substep loop (SURVEY.md 8f-2).
 * pixie_particle_volume: get_particle_volume, PG/particle_filling/filling.py:247-288 (Taichi in the reference): particles per cell
 * of a grid_n^3 grid of spacing grid_dx, vol = grid_dx^3 / count. Positions outside the grid are clamped to the border cells
 * (the reference indexes out of range). Stream-ordered, no host sync. */
int pixie_particle_volume(const float* pos_dev, int n, int grid_n, float grid_dx, float* vol_dev, void* stream);
/* pixie_frame_transform: per-frame hand-over to the rasteriser, gs_simulation.py:591-600 with utils/transformation_utils.py:19-20,
 * 57-87, 101-126: pos_render = apply_inverse_rotations(mean + (pos - (1,1,1+z_shift)) / scale, Rs); cov_render =
 * apply_inverse_cov_rotations(cov / scale^2, Rs) on the 6 upper-triangular entries (cov_dev may be NULL). rotations_host:
 * [n_rot][9] row-major in the order they were applied forward (n_rot <= 8). */
int pixie_frame_transform(const float* pos_dev, const float* cov_dev, int n, float z_shift_value, float scale_origin,
                          const float original_mean_pos_host[3], const float* rotations_host, int n_rot, float* pos_out_dev,
                          float* cov_out_dev, void* stream);
/* pixie_gaussian_ply_records: one 3DGS PLY vertex per Gaussian, as export_gaussians_to_ply (gs_simulation.py:290-322) with
 * cov3D_to_log_scales_and_quats (:253-288) and GaussianModel.save_ply / construct_list_of_attributes
 * (gaussian-splatting/scene/gaussian_model.py:177-208) write it. records_dev [n][14 + 3K] fp32: x y z, nx ny nz (0),
 * f_dc_0..2 = shs[p][0][0..2], f_rest_{c (K-1) + k - 1} = shs[p][k][c] (k >= 1), opacity, scale_0..2, rot_0..3. The scales
 * are log sqrt(max(lambda, 1e-12)) of the covariance's eigenvalues in descending order; rot is the quaternion (w, x, y, z)
 * of R = the eigenvectors as columns, the third negated when det R < 0, by scipy's Rotation.from_matrix (Markley's
 * decision, so w may be negative). pos_dev [n][3], cov_dev [n][6] upper triangle (xx xy xz yy yz zz), shs_dev [n][K][3]
 * with K in {1, 4, 9, 16}, opacity_dev [n]. Stream-ordered, no host sync. */
int pixie_gaussian_ply_records(const float* pos_dev, const float* cov_dev, const float* shs_dev, int K, const float* opacity_dev, int n,
                               float* records_dev, void* stream);
/* pixie_gaussian_checkpoint_decode: a trained 3DGS checkpoint, as GaussianModel.load_ply
 * (gaussian-splatting/scene/gaussian_model.py:215-260) then get_xyz, get_features, get_opacity and get_covariance() give it,
 * optionally filtered by gs_simulation.py:405. table_dev: the PLY's binary little-endian vertex element as it is in the file,
 * n rows of row_bytes bytes (a multiple of 4). cols [11 + 3K] host: the byte offsets within a row of the float32 columns
 * x y z, f_dc_0..2, f_rest_0..3(K-1)-1 (in numeric order), opacity, scale_0..2, rot_0..3; each a multiple of 4. K in
 * {1, 4, 9, 16}. Outputs, capacity n rows each: pos_dev [.][3], shs_dev [.][K][3] (shs[p][0][c] = f_dc_c,
 * shs[p][k][c] = f_rest_{c (K-1) + k - 1}), opacity_dev [.] = sigmoid(opacity), cov_dev [.][6] = the upper triangle
 * (xx xy xz yy yz zz) of L L^T, L = build_rotation(rot) diag(exp(scale)). With has_threshold only the rows with
 * opacity > threshold (float32, strict, NaN dropped) are written, compacted in file order; *m_host receives their number
 * (n without a threshold). Host-synchronises on the stream once when filtering. */
int pixie_gaussian_checkpoint_decode(const void* table_dev, long long n, int row_bytes, const int* cols, int K, int has_threshold,
                                     float threshold, float* pos_dev, float* shs_dev, float* opacity_dev, float* cov_dev,
                                     long long* m_host, void* stream);
/* pixie_gaussian_checkpoint_decode_scale_rot: the same table and columns, every row, as GaussianModel.load_ply then get_xyz,
 * get_features, get_opacity, get_scaling and get_rotation give it (what gaussian-splatting's render.py hands the rasterizer):
 * pos_dev [n][3], shs_dev [n][K][3] and opacity_dev [n] as pixie_gaussian_checkpoint_decode writes them, scales_dev [n][3] =
 * exp(scale_j), rotations_dev [n][4] = rot / max(||rot||, 1e-12) (F.normalize; w x y z as stored). Stream-ordered, no host
 * sync. */
int pixie_gaussian_checkpoint_decode_scale_rot(const void* table_dev, long long n, int row_bytes, const int* cols, int K, float* pos_dev,
                                               float* shs_dev, float* opacity_dev, float* scales_dev, float* rotations_dev, void* stream);
/* pixie_image_metrics: PSNR and SSIM of one image pair as gaussian-splatting's metrics.py scores it (utils/image_utils.py psnr,
 * utils/loss_utils.py ssim with its 11-tap sigma-1.5 window, zero padding 5, C1 = 0.01^2, C2 = 0.03^2). a_dev, b_dev:
 * [height][width][3] uint8, read as k / 255 in float32. window_host: the normalised float32 1D window; the 2D window is its
 * outer product, exact in fp64. out_dev [2] fp64 = {psnr (inf for identical images), ssim}, computed in fp64 and reduced in
 * a fixed order (bit-identical on a repeat). One kernel launch, stream-ordered, no host sync. */
int pixie_image_metrics(const uint8_t* a_dev, const uint8_t* b_dev, int height, int width, const float window_host[11], double* out_dev,
                        void* stream);
/* pixie_material_metrics: the evaluation of the material networks on labelled scenes, process_batch's metric code
 * (WG/trainer/inference_combined.py:108-170, compute_accuracy / masked_mean of pixie/training_utils.py:68-87) together with
 * the ground-truth normalisation of MaterialVoxelDataset.__getitem__ (WG/data_utils/my_data.py:160-240).
 * mat_dev [n][voxels][c_mat] fp32: material_grid.npy as it is on disk (channels-last; density, E, nu, ..., id last).
 * mask_dev [n][voxels] fp32 (clip_features_mask.npy) or NULL, in which case the mask is (trunc(id) != background_id).
 * seg_dev [n][n_classes][voxels] logits, cont_dev [n][3][voxels]. ranges (host) = {density_min, density_max, E_min, E_max,
 * nu_min, nu_max} (log10 space for density and E). Outputs, device: gt_dev [n][4][voxels] = save_predictions' mat_grid
 * (density, E: 2 (clip(log10(x + 1e-6), lo, hi) - lo) / (hi - lo) - 1; nu the same without the log; id as float(int64(id)));
 * counts_dev [n][2] = (#(mask != 0), #(argmax == id & mask != 0)), torch.argmax rules (first index, NaN is the maximum);
 * sums_dev [n][4] = (sum (cont_c - gt_c)^2 * mask for c = 0..2, sum mask), fp64 in a fixed order (bit-identical on a
 * repeat). Stream-ordered, no host sync. */
int pixie_material_metrics(const float* mat_dev, int c_mat, const float* mask_dev, const float* seg_dev, int n_classes, const float* cont_dev,
                           int n, int64_t voxels, const double ranges[6], int background_id, float* gt_dev, long long* counts_dev,
                           double* sums_dev, void* stream);
/* ---- particle filling of hollow Gaussian objects (PG/particle_filling/filling.py:26-380, Taichi in the reference).
 * pixie_fill_density: densify_grids (:26-87). count_dev [grid_n^3] int32 = Gaussians per cell (a Gaussian outside the grid
 * counts in the nearest border cell; the reference indexes out of range), density_dev [grid_n^3] fp32 = sum over the
 * Gaussians of opacity * the mean over the cell's 8 corner nodes of exp(-1/2 d^T P d), P = Q diag(1/max(sig, 1e-8)) Q^T from
 * the signed eigen-decomposition of the covariance, over the (2r+1)^3 cells around the Gaussian's cell that lie in the grid,
 * r = ceil(max sqrt(sig) / grid_dx). pos [n][3] in the grid's frame, opacity [n], cov [n][6] upper triangle. Both grids are
 * overwritten; C order (x slowest). */
int pixie_fill_density(const float* pos_dev, const float* opacity_dev, const float* cov_dev, int n, int grid_n, float grid_dx,
                       int* count_dev, float* density_dev, void* stream);
/* pixie_fill_grids: fill_dense_grids (:90-114) then internal_filling (:117-234) on the grids of pixie_fill_density. A cell
 * with density > density_thres and count < max_particles_per_cell gets the difference; then every cell whose count is still
 * 0, that sees a cell with density > search_thres in each axis direction other than exclude_dir (0 +x, 1 -x, 2 +y, 3 -y,
 * 4 +z, 5 -z) and an odd number of such runs along ray_cast_dir, gets max_particles_per_cell. count_dev is updated in place
 * like the reference's grid. New particles (cell + U[0,1)^3) * grid_dx + origin go to out_dev [max_samples][3]: dense-cell
 * ones first, each group in C order of cells, offsets from Philox keyed on (seed, output index). *n_dense_host /
 * *n_total_host receive the counts (the call synchronises `stream` once); a total above max_samples fails and writes nothing
 * to out_dev. */
int pixie_fill_grids(int* count_dev, const float* density_dev, int grid_n, float grid_dx, const float origin_host[3],
                     float density_thres, float search_thres, int max_particles_per_cell, int exclude_dir, int ray_cast_dir,
                     unsigned long long seed, float* out_dev, int max_samples, int* n_dense_host, int* n_total_host, void* stream);
/* pixie_nearest_gaussian: the search of get_attr_from_closest (filling.py:383-405). index_dev[j] = the i minimising the
 * float32 distance d = sqrt((dx*dx + dy*dy) + dz*dz), dx = query[j].x - pos[i].x (one rounding per operation), ties to the
 * lowest i; -1 when no Gaussian has d < 1e10 (n = 0, a non-finite query, or all Gaussians that far). Exact, through a
 * bounding-volume tree (not O(m n)). pos_dev [n][3], query_dev [m][3], index_dev [m] int32; n or m may be 0. Stream-ordered,
 * no host sync; repeat calls give identical results. */
int pixie_nearest_gaussian(const float* pos_dev, int n, const float* query_dev, int m, int* index_dev, void* stream);
/* ---- VLM part segmentation (pixie/voxel/segmentation.py). All three are stream-ordered, with no host sync.
 * pixie_part_similarity: run_clip and the labels of clip_part_segmentation (:98-183) in one pass over the features. For the
 * occupied voxels v (mask_dev[v] != 0, in index order; every voxel when mask_dev is NULL) of feat_dev [n_voxels][C] float16,
 * f = feat[v] widened to fp32 and query_dev [P][C] fp32 unit rows: sims_dev [n][P] = (f . q_p) / |f| accumulated in fp32,
 * probs_dev [n][P] = softmax over p of sims * inv_temperature (probs_dev may be NULL), labels_dev [n] int64 = the argmax of
 * the probabilities (first index on ties, a NaN wins, as torch.argmax), scores_dev [n] = the probability at the label.
 * n = n_occupied, the number of nonzero mask entries (n_voxels without a mask). A zero or NaN feature row gives NaN
 * similarities, label 0 and a NaN score. 1 <= P <= 64, C >= 1; no fp32 copy of the features is made. */
int pixie_part_similarity(const void* feat_dev, const uint8_t* mask_dev, int64_t n_voxels, int C, int n_occupied, const float* query_dev,
                          int P, float inv_temperature, float* sims_dev, int64_t* labels_dev, float* scores_dev, float* probs_dev,
                          void* stream);
/* pixie_knn_label_vote: local_post_process_segmentation (:190-226). out_dev[q] = the mode of labels_dev over the k nearest
 * points of pos_dev[q] (itself included) by the fp64 squared distance (dx*dx + dy*dy) + dz*dz of the float32 coordinates,
 * ties at the k-th distance to the lowest index; a tie in count goes to the smallest label. pos_dev [n][3] finite,
 * labels_dev / out_dev [n] int64, 1 <= k <= n. Exact, through the tree of pixie_nearest_gaussian; deterministic. */
int pixie_knn_label_vote(const float* pos_dev, int n, const int64_t* labels_dev, int k, int64_t* out_dev, void* stream);
/* pixie_nearest_vertex: the colour lookup of save_segmented_point_cloud (:283-301). index_dev[j] = the i minimising the fp64
 * squared distance (dx*dx + dy*dy) + dz*dz between query_dev[j] (float32) and vert_dev[i] (float64), ties to the lowest i;
 * a vertex with a NaN or Inf coordinate is never chosen, a finite one is even where d2 overflows to Inf;
 * -1 for a non-finite query or when no vertex is finite. vert_dev [n][3], query_dev [m][3], index_dev [m] int32. */
int pixie_nearest_vertex(const double* vert_dev, int n, const float* query_dev, int m, int* index_dev, void* stream);
/* ---- Gaussian-splatting rasteriser, forward only (gs_simulation.py:573-631 with `--render_img`: Inria's
 * diff-gaussian-rasterization at scale_modifier 1, prefiltered false, precomputed 3D covariances).
 * A renderer keeps its device buffers between frames and grows them when a frame needs more; once warm, a frame allocates
 * nothing. pixie_gs_render draws one frame on `stream`: means_dev [n][3], cov_dev [n][6] (upper triangle xx xy xz yy yz zz,
 * the solver's export order), opacity_dev [n]; colours from shs_dev [n][sh_coeffs][3] evaluated at degree sh_degree (<= 3,
 * (sh_degree + 1)^2 <= sh_coeffs) toward campos as utils/render_utils.py:113-130 does (+0.5, clamped at 0), or, when
 * shs_dev is NULL, colors_dev [n][3] as given. view / proj: world_view_transform and full_proj_transform as the reference
 * stores them (16 floats each, row-vector convention). image_dev [3][height][width] receives the unclamped RGB image over
 * bg, radii_dev [n] the screen radius (0 = culled). The call synchronises `stream` once, for the number of (Gaussian, tile)
 * pairs, which goes to *n_rendered_host (may be NULL). phase_ms_host, when not NULL, receives the times in ms of preprocess,
 * scan + keys, sort, ranges and blend (CUDA events; the call then synchronises a second time). The frame returns with its
 * sort and blend still running on `stream`; the next frame of the same renderer, on any stream, first waits for them, so
 * frames run in call order whatever streams they are drawn on. A renderer is not safe to call from two host threads at
 * once: callers serialise its calls. */
typedef struct pixie_gs_renderer_s* pixie_gs_renderer_t;
int pixie_gs_renderer_create(pixie_gs_renderer_t* out);
int pixie_gs_render(pixie_gs_renderer_t h, const float* means_dev, const float* cov_dev, const float* opacity_dev,
                    const float* shs_dev, int sh_coeffs, int sh_degree, const float* colors_dev, int n, const float view_host[16],
                    const float proj_host[16], const float campos_host[3], float tan_fovx, float tan_fovy, int width, int height,
                    const float bg_host[3], float* image_dev, int* radii_dev, int* n_rendered_host, float* phase_ms_host,
                    void* stream);
/* pixie_gs_render_scale_rot: one frame as pixie_gs_render draws it, with the covariances built in the preprocess from
 * scales_dev [n][3] and rotations_dev [n][4] (unit quaternions w x y z) as forward.cu's computeCov3D builds them at
 * scale_modifier 1, and the colours from shs_dev (required) as its computeColorFromSH evaluates them: what
 * gaussian_renderer.render passes with PipelineParams' defaults (gaussian-splatting's render.py). */
int pixie_gs_render_scale_rot(pixie_gs_renderer_t h, const float* means_dev, const float* scales_dev, const float* rotations_dev,
                              const float* opacity_dev, const float* shs_dev, int sh_coeffs, int sh_degree, int n, const float view_host[16],
                              const float proj_host[16], const float campos_host[3], float tan_fovx, float tan_fovy, int width, int height,
                              const float bg_host[3], float* image_dev, int* radii_dev, int* n_rendered_host, float* phase_ms_host,
                              void* stream);
void pixie_gs_renderer_destroy(pixie_gs_renderer_t h);
/* Number of kernel launches one forward() issues (for gpu_launches accounting) and algorithmic
 * FLOPs of one forward at batch 1 (2 * MACs of every Conv3d/Conv1d of the reference graph). */
int pixie_unet_launch_count(pixie_unet_t h);
/* Reads the device-side pipeline watchdog flag (non-zero return = a convolution timed out). */
int pixie_unet_check(pixie_unet_t h);
double pixie_unet_flops(pixie_unet_t h);
/* Test hook: copy a named intermediate fp32 activation (channels-last) to host. Names are module
 * paths of the reference ("unet.input_blocks.3.0", "projector", ...). Returns element count or <0. */
int64_t pixie_unet_debug_fetch(pixie_unet_t h, const char* name, float* host_out, int64_t capacity);
/* Test hook: the activations debug_fetch can copy, one "name channels side" line each, written NUL-terminated into buf.
 * Returns the length of the full list (excluding the NUL; larger than capacity - 1 means truncated) or <0. */
int64_t pixie_unet_debug_names(pixie_unet_t h, char* buf, int64_t capacity);
void pixie_unet_destroy(pixie_unet_t h);

/* ===================================================================== MPM (PhysGaussian rollout) =
 * Replaces MPM_Simulator_WARP (third_party/PhysGaussian/mpm_solver_warp/mpm_solver_warp.py:47-1210)
 * and the Warp kernels of mpm_utils.py:282-663 it launches.
 */
typedef struct pixie_mpm_s* pixie_mpm_t;

/* Particle / model arrays, bound as borrowed device pointers (fp32 unless noted). Layouts follow
 * MPMStateStruct / MPMModelStruct (warp_utils.py:6-74): vec3 = 3 floats, mat33 = 9 floats row-major. */
enum pixie_mpm_field {
    PIXIE_MPM_X = 0,          /* particle_x        [n][3]  */
    PIXIE_MPM_V = 1,          /* particle_v        [n][3]  */
    PIXIE_MPM_F = 2,          /* particle_F        [n][9]  */
    PIXIE_MPM_F_TRIAL = 3,    /* particle_F_trial  [n][9]  */
    PIXIE_MPM_C = 4,          /* particle_C        [n][9]  */
    PIXIE_MPM_STRESS = 5,     /* particle_stress   [n][9]  */
    PIXIE_MPM_R = 6,          /* particle_R        [n][9]  */
    PIXIE_MPM_COV = 7,        /* particle_cov      [n*6]   */
    PIXIE_MPM_INIT_COV = 8,   /* particle_init_cov [n*6]   */
    PIXIE_MPM_VOL = 9,        /* particle_vol      [n]     */
    PIXIE_MPM_MASS = 10,      /* particle_mass     [n]     */
    PIXIE_MPM_DENSITY = 11,   /* particle_density  [n]     */
    PIXIE_MPM_E = 12,         /* model.E           [n]     */
    PIXIE_MPM_NU = 13,        /* model.nu          [n]     */
    PIXIE_MPM_MU = 14,        /* model.mu          [n]     */
    PIXIE_MPM_LAM = 15,       /* model.lam         [n]     */
    PIXIE_MPM_BULK = 16,      /* model.bulk        [n]     */
    PIXIE_MPM_YIELD = 17,     /* model.yield_stress[n]     */
    PIXIE_MPM_MATERIAL = 18,  /* particle_material [n] int32 */
    PIXIE_MPM_SELECTION = 19, /* particle_selection[n] int32 */
    PIXIE_MPM_FIELD_COUNT = 20
};

/* Scalar members of MPMModelStruct set by set_parameters_dict (mpm_solver_warp.py:287-463). */
typedef struct {
    int n_grid;
    float grid_lim;
    float gravity[3];
    float rpic_damping;
    float grid_v_damping_scale;
    float alpha;               /* Drucker-Prager, from friction_angle (mpm_solver_warp.py:84-86) */
    float hardening;
    float xi;
    float plastic_viscosity;
    float softening;
    int update_cov_with_F;
} pixie_mpm_params;

/* Boundary conditions (closures of mpm_solver_warp.py:749-1210), evaluated in registration order. */
enum pixie_mpm_bc_kind {
    PIXIE_BC_SURFACE_COLLIDER = 0,   /* add_surface_collider   :749-843  (grid)      */
    PIXIE_BC_CUBOID = 1,             /* set_velocity_on_cuboid :852-908  (grid, moving box) */
    PIXIE_BC_BOUNDING_BOX = 2,       /* add_bounding_box       :910-977  (grid)      */
    PIXIE_BC_IMPULSE = 3,            /* add_impulse_on_particles :982-1029 (particles, needs mask) */
    PIXIE_BC_VELOCITY_TRANSLATION = 4, /* enforce_particle_velocity_translation :1031-1075 (mask) */
    PIXIE_BC_VELOCITY_ROTATION = 5   /* enforce_particle_velocity_rotation :1080-1179 (mask)     */
};

typedef struct {
    int kind;
    float point[3];
    float normal[3];
    float size[3];
    float velocity[3];          /* cuboid velocity / translation velocity / impulse force          */
    float start_time, end_time;
    float friction;
    int surface_type;           /* 0 sticky, 1 slip, 2 separate, 11 cut                            */
    int reset;
    float horizontal_axis_1[3], horizontal_axis_2[3];
    float half_height_and_radius[2];
    float rotation_scale, translation_scale;
    const int* mask_dev;        /* particle BCs: int32 [n] selection mask (borrowed), else NULL    */
} pixie_mpm_bc;

int pixie_mpm_create(int n_particles, int n_grid, float grid_lim, pixie_mpm_t* out);
/* bind, set_params, add_bc, clear_bcs, set_time / get_time, set_active_count and the slab set-up write pending results
 * back and copy on the legacy default stream, which does not wait for non-blocking streams: a caller that steps on such a
 * stream calls pixie_mpm_sync(h, stream) and synchronises that stream first (pixie_b200.mpm_solver_warp does). */
int pixie_mpm_bind(pixie_mpm_t h, int field, void* dev_ptr);
int pixie_mpm_set_params(pixie_mpm_t h, const pixie_mpm_params* p);
int pixie_mpm_add_bc(pixie_mpm_t h, const pixie_mpm_bc* bc);
int pixie_mpm_clear_bcs(pixie_mpm_t h);
/* Simulation clock (self.time, mpm_solver_warp.py:637). */
int pixie_mpm_set_time(pixie_mpm_t h, double t);
int pixie_mpm_get_time(pixie_mpm_t h, double* t);
/* n_substeps x p2g2p(step, dt) (mpm_solver_warp.py:514-637) without host round trips. dt is the
 * Python float the reference accumulates into self.time; kernels receive it rounded to fp32. */
int pixie_mpm_step(pixie_mpm_t h, int n_substeps, double dt, void* stream);
/* Small setup / export kernels (same arithmetic as the Warp ones they replace). */
int pixie_mpm_compute_mu_lam(pixie_mpm_t h, void* stream);                 /* mpm_utils.py:282-288 */
int pixie_mpm_compute_bulk(pixie_mpm_t h, void* stream);                   /* mpm_utils.py:290-293 */
int pixie_mpm_compute_mass(pixie_mpm_t h, void* stream);                   /* warp_utils.py:233-241 */
int pixie_mpm_compute_cov_from_F(pixie_mpm_t h, void* stream);             /* mpm_utils.py:529-553 */
int pixie_mpm_compute_R_from_F(pixie_mpm_t h, void* stream);               /* mpm_utils.py:556-580 */
/* apply_additional_params for a LIST of boxes in one launch (mpm_utils.py:591-610; the reference
 * launches it once per box, material_field.py:343-363). boxes: [n_boxes][10] =
 * point xyz, size xyz, E, nu, density, material(as float); the array may live on the host or on the device. */
int pixie_mpm_apply_additional_params(pixie_mpm_t h, const float* boxes, int n_boxes, void* stream);
/* selection_* mask kernels (mpm_utils.py:613-663): writes int32 mask_dev[n]. */
int pixie_mpm_select_box(pixie_mpm_t h, const float point[3], const float size[3], int* mask_dev, void* stream);
int pixie_mpm_select_cylinder(pixie_mpm_t h, const float point[3], const float normal[3],
                              float half_height, float radius, int* mask_dev, void* stream);
/* The default path keeps a cell-sorted struct-of-arrays private copy of the particle state between steps (the bound
 * arrays stay in the caller's order and are what every other entry point reads): pixie_mpm_sync writes the results back
 * into the bound arrays and must precede any read of them; every other entry point that touches the bound arrays calls it
 * internally. After a sync the caller may modify its arrays: the next step re-reads them. It is a no-op when nothing was
 * stepped since the last sync. */
int pixie_mpm_sync(pixie_mpm_t h, void* stream);
/* Live particles = the prefix [0, n_active) of the bound arrays (slab runs migrate particles between ranks). */
int pixie_mpm_set_active_count(pixie_mpm_t h, int n_active);
/* Borrowed pointers to the grid arrays owned by the handle (for tests): the {mv.xyz, m} float4[n^3] scatter grid (cleared by
 * the sweep that consumed it; in slab mode this is grid 0 of the two) and the {v.xyz, 0} float4[n^3] velocities the last
 * substep's sweep wrote. */
int pixie_mpm_grid_ptrs(pixie_mpm_t h, float** grid_mv4, float** grid_v_out);
/* ---- Slab mode of the default path (BASELINE config 5, no reference counterpart). Every handle owns an exchange buffer
 * [256-byte flag block][{mv.xyz, m} grid 0][grid 1] (float4[n_grid^3] each, x slowest; the two grids alternate by substep
 * parity); pixie_mpm_slab_attach gives it the x-neighbours' buffers (pointers valid in this process: from pixie_ipc_open for
 * a neighbour in another process, or the neighbour's own pointer inside one process). A substep is then two launches with
 * ONE flag handshake between neighbours and no host round trip: scatter (particle kernel; stencils may reach `slack` + 2
 * planes into the neighbours' ranges) and the grid sweep, which raises this rank's scatter_done, waits for the neighbours'
 * and adds their partial sums on the shared planes straight from their memory (NVLink) while it updates owned + shared
 * planes; a rank's own partial sums on shared planes are cleared one substep later (the other grid is in use meanwhile).
 * pixie_mpm_step runs whole substeps (CUDA graph); pixie_mpm_slab_phase runs ONE phase (0 scatter, 1 nothing, 2 sweep) so
 * that a single-process driver can sequence the phases of several slabs on one stream. Particles whose stencil base
 * leaves [x0 - slack, x1 + slack) raise error 2 (migrate more often); a neighbour that never shows up raises error 1.
 * pixie_mpm_set_active_count must be called after every particle migration (it also clears the shared planes). */
int pixie_mpm_exchange_buffer(pixie_mpm_t h, void** base, size_t* bytes);
int pixie_mpm_slab_attach(pixie_mpm_t h, int x0, int x1, int slack, const void* left_xbuf, const void* right_xbuf);
int pixie_mpm_slab_phase(pixie_mpm_t h, int phase, double dt, void* stream);
int pixie_mpm_slab_error(pixie_mpm_t h, int* flag);
/* Migration check without a write-back: the number of planes by which the farthest live particle's stencil base lies
 * outside [x0, x1) (towards a side that has a neighbour) is max-ed into the DEVICE int *d_out, which the caller zeroes. */
int pixie_mpm_slab_excursion(pixie_mpm_t h, int* d_out, void* stream);
/* cudaIpc plumbing for the exchange buffers (64-byte opaque handles, exchanged by the caller, e.g. over torch.distributed). */
int pixie_ipc_export(const void* dev_ptr, unsigned char handle[64]);
int pixie_ipc_open(const unsigned char handle[64], void** dev_ptr);
int pixie_ipc_close(void* dev_ptr);
/* Kernels of this library launched for the handle so far (CUDA-graph replays count their nodes; cub's sort passes do not count). */
long long pixie_mpm_launch_count(pixie_mpm_t h);
void pixie_mpm_destroy(pixie_mpm_t h);

#ifdef __cplusplus
}
#endif
#endif /* PIXIE_B200_H_ */
