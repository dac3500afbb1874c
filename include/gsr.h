/* gsr.h -- C ABI of the H100-native differentiable 3DGS tile rasterizer (libgsr_b200.so).
 *
 * This is the drop-in seam for the torch-free core of the reference rasterizer,
 *   CudaRasterizer::Rasterizer::{forward, backward, markVisible}
 *   ($RAST/cuda_rasterizer/rasterizer.h:24-91, $RAST = submodules/gaustudio-diff-gaussian-rasterization),
 * which the reference's pybind layer ($RAST/rasterize_points.cu:35-231, $RAST/ext.cpp:15-19) binds.
 * Plain pointers and sizes only: no torch / glm / std:: types.  All float* are DEVICE pointers to
 * contiguous float32 (the reference's convention, rasterize_points.cu:97-117); optional inputs are NULL
 * when absent (the reference passes the data pointer of an empty tensor, i.e. nullptr).
 * Every entry point enqueues its work on `stream` (a cudaStream_t passed as void*); the reference uses
 * the legacy default stream everywhere (forward.cu:416,459; rasterizer_impl.cu:148,280,292,306,317).
 *
 * Return convention: >= 0 success, < 0 error (text via gsr_last_error()).  With `debug` != 0 each stage is
 * followed by a stream synchronize + error check, mirroring CHECK_CUDA (auxiliary.h:166-173).
 */
#ifndef GSR_H_INCLUDED
#define GSR_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSR_ABI_VERSION 1

/* Scratch allocator callback.  Replaces the three `std::function<char*(size_t)>` resize closures the
 * reference takes (rasterizer.h:35-37, built by resizeFunctional at rasterize_points.cu:27-33).
 * Must return a device pointer to at least `bytes` bytes (any alignment >= 16), valid until the matching
 * backward call has completed.  The buffers are opaque to the caller, exactly like the reference's
 * geomBuffer / binningBuffer / imgBuffer (gaustudio_diff_gaussian_rasterization/__init__.py:97,106). */
typedef char* (*gsr_alloc_fn)(void* user, size_t bytes);

int gsr_abi_version(void);
const char* gsr_last_error(void);

/* Sizes of the three opaque buffers (what the allocator callbacks will be asked for). */
size_t gsr_geometry_bytes(int P);
size_t gsr_image_bytes(int width, int height);
size_t gsr_binning_bytes(int64_t num_rendered);

/* Replaces Rasterizer::forward (rasterizer.h:34-60, impl rasterizer_impl.cu:198-343).
 * Same arguments in the same order, plus:
 *   r_capacity : 0  -> exact mode: one blocking 8-byte device->host read of num_rendered sizes the binning
 *                      buffer (the reference does the same at rasterizer_impl.cu:284);
 *                >0 -> pipelined mode: no host sync; the binning buffer is sized for r_capacity tile
 *                      instances; if the view needs more, nothing is rendered for the overflowing tiles and
 *                      *r_host (if given) receives the true count so the caller can detect it
 *                      (num_rendered > r_capacity) and re-run.
 *   r_host     : optional PINNED host int64 that asynchronously receives num_rendered (either mode).
 * Returns num_rendered (exact mode), r_capacity (pipelined mode), or < 0 on error.
 * Exact mode speculates (gsr_set_speculation): from the second view of a (device, P, width, height) on, the binning
 * buffer is sized for 1.25 x the previous view's count and the rest of the forward is enqueued BEFORE the host blocks
 * on the count, so the GPU does not idle across the read; a view that needs more is re-binned with its exact count
 * before the call returns.  Same results and the same returned value either way; `binning_alloc` may then be called
 * twice in one forward (the last pointer is the one to keep, as with the reference's resize closure). */
int64_t gsr_forward(gsr_alloc_fn geometry_alloc, void* geometry_user, gsr_alloc_fn binning_alloc,
                    void* binning_user, gsr_alloc_fn image_alloc, void* image_user, int P, int D, int M,
                    const float* background, int width, int height, const float* means3D, const float* shs,
                    const float* colors_precomp, const float* opacities, const float* scales,
                    float scale_modifier, const float* rotations, const float* cov3D_precomp,
                    const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx,
                    float tan_fovy, int prefiltered, float* out_color, float* out_depth,
                    float* out_median_depth, float* out_opacity, int* radii, int debug, int64_t r_capacity,
                    int64_t* r_host, void* stream);

/* Replaces Rasterizer::backward (rasterizer.h:62-91, impl rasterizer_impl.cu:347-452).  Same arguments in
 * the same order (+ stream).  All ten outputs are fully written (no pre-zeroing needed, unlike the
 * reference which accumulates into torch::zeros tensors, rasterize_points.cu:160-169); dL_dconic and
 * dL_ddepth are internal in the reference's Python API and may be NULL here.
 * Shapes: dL_dmean2D[P,3] dL_dconic[P,2,2] dL_dopacity[P] dL_dcolor[P,3] dL_ddepth[P] dL_dmean3D[P,3]
 *         dL_dcov3D[P,6] dL_dsh[P,M,3] dL_dscale[P,3] dL_drot[P,4]. */
int gsr_backward(int P, int D, int M, int64_t R, const float* background, int width, int height,
                 const float* means3D, const float* shs, const float* colors_precomp, const float* scales,
                 float scale_modifier, const float* rotations, const float* cov3D_precomp,
                 const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                 float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer,
                 const float* dL_dpix, const float* dL_dpix_depth, const float* dL_dpix_median_depth,
                 const float* dL_dpix_final_opacity, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity,
                 float* dL_dcolor, float* dL_ddepth, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                 float* dL_dscale, float* dL_drot, int debug, void* stream);

/* Fused-activation variants -- the step immediately before the path in every caller (SURVEY.md §8f rank 1):
 * gaustudio's VanillaRenderer.get_gaussians_properties (gaustudio/renderers/vanilla_renderer.py:28-52) runs
 * exp(_scale), sigmoid(_opacity), normalize(_rot) and cat(_f_dc, _f_rest) as separate elementwise kernels on
 * every view (gaustudio/models/vanilla_sg.py:58-63,102-106; models/utils.py:6-32).  These entry points take the
 * model's RAW attributes instead -- log_scales[P,3], raw_rotations[P,4], opacity_logits[P], f_dc[P,1,3],
 * f_rest[P,M-1,3] -- and apply the activations inside the projection kernel; the backward returns gradients
 * w.r.t. the raw attributes (dL_dlog_scale, dL_draw_rot, dL_dopacity_logit, dL_df_dc, dL_df_rest).  Everything
 * else is identical to gsr_forward / gsr_backward; the opaque buffers are interchangeable.
 * gsr_backward_fused: dL_dcolor[P,3] and dL_dcov3D[P,6] (the gradients w.r.t. the intermediate colours and 3D
 * covariances) may be NULL; they are not written then. */
int64_t gsr_forward_fused(gsr_alloc_fn geometry_alloc, void* geometry_user, gsr_alloc_fn binning_alloc,
                          void* binning_user, gsr_alloc_fn image_alloc, void* image_user, int P, int D, int M,
                          const float* background, int width, int height, const float* means3D, const float* f_dc,
                          const float* f_rest, const float* opacity_logits, const float* log_scales,
                          float scale_modifier, const float* raw_rotations, const float* viewmatrix,
                          const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy,
                          int prefiltered, float* out_color, float* out_depth, float* out_median_depth,
                          float* out_opacity, int* radii, int debug, int64_t r_capacity, int64_t* r_host,
                          void* stream);
int gsr_backward_fused(int P, int D, int M, int64_t R, const float* background, int width, int height,
                       const float* means3D, const float* f_dc, const float* f_rest, const float* opacity_logits,
                       const float* log_scales, float scale_modifier, const float* raw_rotations,
                       const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                       float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer,
                       const float* dL_dpix, const float* dL_dpix_depth, const float* dL_dpix_median_depth,
                       const float* dL_dpix_final_opacity, float* dL_dmean2D, float* dL_dopacity_logit,
                       float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_df_dc, float* dL_df_rest,
                       float* dL_dlog_scale, float* dL_draw_rot, int debug, void* stream);

/* Replaces Rasterizer::markVisible (rasterizer.h:27-32, impl rasterizer_impl.cu:54-66,141-153).
 * present: device bool[P] (1 byte each). */
int gsr_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                     unsigned char* present, void* stream);

/* Depth -> normal map (the "rendered normal" of gaustudio's vanilla path:
 * gaustudio/datasets/__init__.py:106-112,307-380, Camera.depth2point + Camera.depth2normal with k=3).
 * depth: device float[H*W]; out: device float[H*W*3]; rot: optional device float[9] (row-major 3x3, the
 * `inverse(extrinsics[:3,:3]).t()` of coordinate='world') or NULL for camera coordinates. */
int gsr_depth2normal(const float* depth, int width, int height, float fx, float fy, float cx, float cy,
                     float d_min, float d_max, const float* rot, float* out, void* stream);

/* Depth -> 3-D points (Camera.depth2point, gaustudio/datasets/__init__.py:307-339; the step after the path in
 * gaustudio/scripts/extract_mesh.py:95-115).  out: device float[H*W*3]; cam_to_world: optional device float[16]
 * (row-major inverse(extrinsics)) for coordinate='world', NULL for camera coordinates. */
int gsr_depth2point(const float* depth, int width, int height, float fx, float fy, float cx, float cy,
                    const float* cam_to_world, float* out, void* stream);

/* ---- extraction post-pass: what gaustudio/scripts/extract_pcd.py runs on every rendered view (SURVEY 8f row 2) ----
 *
 * masked_bilateral_filter (extract_pcd.py:185-238), which the reference executes on the CPU through OpenCV:
 *   out_mask  = !dilate(!mask, d x d box)                              (cv2.dilate, default border)
 *   out_depth = bilateralFilter((depth - min)/(max - min), d, sigma_color, sigma_space) * (max - min) + min
 *               on out_mask pixels (min/max over them, masked-out pixels entering the filter as 0, disc support of
 *               radius d/2, centre weight 1, REFLECT_101 border), the input depth elsewhere.
 * depth/out_depth: device float[H*W]; mask/out_mask: device uint8[H*W] (torch.bool layout); d odd, 1..15;
 * scratch: 2 device words owned by the caller (the depth range never visits the host).
 * Reference quirk kept: max == min (constant depth, one surviving pixel) divides 0 by 0 and yields NaN there too. */
int gsr_masked_bilateral(const float* depth, const unsigned char* mask, int width, int height, int d,
                         float sigma_color, float sigma_space, float* out_depth, unsigned char* out_mask,
                         unsigned int* scratch, void* stream);

/* Per-view normal extraction (extract_pcd.py:325-335): cam = depth2normal(filtered_depth, 'camera') with -1 where
 * !fg_mask; world = cam @ rot (rot = inverse(extrinsics[:3,:3]).t(), device float[9], applied to the -1 fill too,
 * as normal2worldnormal does); valid = sum(world) > -3 && median_depth < depth_limit && opacity > opacity_min.
 * Outputs: cam_normals float[H*W*3] (optional), neg_world_normals float[H*W*3] (= -world, what the fusion
 * consumes), valid uint8[H*W]. */
int gsr_extract_normals(const float* filtered_depth, const unsigned char* fg_mask, const float* opacity,
                        const float* median_depth, int width, int height, float fx, float fy, float cx, float cy,
                        const float* rot, float depth_limit, float opacity_min, float* cam_normals,
                        float* neg_world_normals, unsigned char* valid, void* stream);

/* One view of one accumulation pass of normal_fusion (extract_pcd.py:117-136 first pass, :143-165 second pass):
 * for entry i with Gaussian id = ids[i]:  v = cam - xyz[id];  w = confidences[i] * |dot(v/|v|, n_i)| / (|v| + 1e-6);
 * with mean_normals != NULL the entry is dropped unless |n_i - mean_normals[id]| < threshold;
 * sum_normals[id] += n_i * w; sum_weights[id] += w; touched[id] = 1 (optional).  Accumulators are dense over the
 * P Gaussians (the reference's torch.unique / inverse indices are `nonzero(touched)`), zeroed by the caller.
 * (cam_x, cam_y, cam_z) is what the reference uses as the camera position: extrinsics[:3, 3]. */
int gsr_normal_fusion_pass(int64_t n, const int64_t* ids, const float* normals, const float* confidences, int P,
                           const float* xyz, float cam_x, float cam_y, float cam_z, const float* mean_normals,
                           float threshold, float* sum_normals, float* sum_weights, unsigned char* touched,
                           void* stream);

/* mean_normals[i] = normalize(sum_normals[i] / sum_weights[i]) (extract_pcd.py:139-140,167-168; 0/0 stays NaN). */
int gsr_normal_fusion_mean(int P, const float* sum_normals, const float* sum_weights, float* mean_normals,
                           void* stream);

/* k nearest neighbours among n points (the neighbour search of the fusion's final smoothing, extract_pcd.py:170-181,
 * done there on the host with scipy's cKDTree: a D2H + H2D round trip per extraction).  Uniform-grid search on the device.
 *   points      float[n*3], SORTED by cell id of the grid below (cell = (z*dims.y + y)*dims.x + x)
 *   cell_start  int32[num_cells + 1]: index of the first point of every cell (exclusive prefix of the cell counts)
 *   grid        DEVICE float[8]: origin.xyz, 1/cell_size, dims.xyz (as floats), unused -- kept on the device so the
 *               caller never has to read the bounding box back
 *   out_index   int32[n*k]: neighbours of point i (indices into `points`), ascending distance, the point itself first;
 *   out_dist    float[n*k]: their Euclidean distances.  k <= 16.  Entries are -1 / +inf if fewer than k points exist. */
int gsr_knn_grid(int n, int k, const float* points, const int* cell_start, const float* grid, int* out_index,
                 float* out_dist, void* stream);

/* ---- optimizer step after the path (SURVEY 8f row 3) ----
 * Fused multi-tensor Adam / AdamW: replaces `torch.optim.<optimizer_name>(param_groups, **args).step()` of
 * gaustudio/pipelines/optimizers/base.py:19-30 (+ zero_grad, :32-34) for optimizer_name in {Adam, AdamW}
 * (configs/vanilla.yaml:30-46: AdamW, eps 1e-15, one learning rate per Gaussian attribute) with ONE launch over
 * all groups.  Per element: grad' = grad * grad_scale (1/world after a summing all-reduce);
 *   decoupled != 0 (AdamW): p *= 1 - lr*weight_decay     else (Adam): grad' += weight_decay * p
 *   m += (grad' - m)(1 - beta1);  v = v*beta2 + (1 - beta2) grad'^2;
 *   p -= lr/(1 - beta1^step) * m / (sqrt(v)/sqrt(1 - beta2^step) + eps);   grad = 0 if zero_grad.
 * beta1 / beta2 / eps are doubles like torch's Python scalars (1 - beta2 must not be formed in float: 1.3e-5 off).
 * `groups` is a HOST array of n_groups (<= GSR_ADAM_MAX_GROUPS) descriptors of DEVICE float tensors; step >= 1. */
#define GSR_ADAM_MAX_GROUPS 16
typedef struct gsr_adam_group {
  float* param;
  float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  int64_t numel;
  float lr;
  float weight_decay;
  float* grad2; /* optional second gradient tensor (NULL: none): the step uses grad + grad2 -- two all-reduce buckets of
                   one data-parallel step -- and zero_grad clears both */
} gsr_adam_group;
int gsr_adam_step(int n_groups, const gsr_adam_group* groups, double beta1, double beta2, double eps, int64_t step,
                  int decoupled, float grad_scale, int zero_grad, void* stream);

/* Introspection for parity tests: copies internal state of the last forward out of the opaque buffers into
 * caller-provided DEVICE arrays (any may be NULL):
 *   point_list  uint32[R]   Gaussian index per sorted tile instance (== BinningState::point_list)
 *   ranges      uint32[T*2] per-tile [start,end) (== ImageState::ranges; empty tiles are (0,0))
 *   n_contrib   uint32[H*W] final_T float[H*W]     (== ImageState::n_contrib / accum_alpha)
 *   means2D float[P*2] conic_opacity float[P*4] depths float[P] rgb float[P*3] cov3D float[P*6]
 *   tiles_touched uint32[P] clamped uint8[P*3]     (== GeometryState members, rasterizer_impl.h:33-47) */
int gsr_debug_export(int P, int width, int height, int64_t R, const char* geom_buffer,
                     const char* binning_buffer, const char* image_buffer, uint32_t* point_list,
                     uint32_t* ranges, uint32_t* n_contrib, float* final_T, float* means2D, float* conic_opacity,
                     float* depths, float* rgb, float* cov3D, uint32_t* tiles_touched, unsigned char* clamped,
                     void* stream);

/* CTA -> tile order of the one-CTA-per-tile kernels (per-tile sort, compositing forward / backward): 1 = longest tile
 * first (default: shortest makespan when ONE view is in flight: -9 % / -6 % on the two compositing kernels at cfg 3),
 * 0 = raster order (about 1.5 % more throughput when several views are pipelined on different streams: each kernel's
 * long tail of crowded tiles overlaps the next kernel), 2 = shortest first.  Process-wide; returns the previous mode;
 * mode < 0 restores the default (or the GSR_TILE_ORDER environment variable).  Results never depend on it. */
int gsr_set_tile_order(int mode);

/* Exact-mode speculation of gsr_forward (see there): 1 = on (default; GSR_SPECULATE=0 in the environment turns the
 * default off), 0 = always the plain blocking read (what `debug` uses), < 0 = back to the default.  Process-wide;
 * returns the previous setting (-1 = default).  gsr_speculation_stats: forwards whose guess held / that had to re-bin. */
int gsr_set_speculation(int on);
int gsr_speculation_stats(int64_t* hits, int64_t* redos);

/* Optional per-stage device timing (CUDA events recorded on the caller's stream around each kernel).
 * Stages: 0 preprocess_fwd, 1 tile_scan, 2 scatter, 3 tile_sort, 4 render_fwd, 5 render_bwd,
 *         6 preprocess_bwd, 7 depth2normal.  gsr_profile_read synchronises the recorded events, adds their
 * elapsed times (ms) into ms[GSR_NUM_STAGES] / launch counts into counts[GSR_NUM_STAGES] and clears them. */
#define GSR_NUM_STAGES 8
int gsr_profile_enable(int on);
int gsr_profile_read(float* ms, int* counts);

#ifdef __cplusplus
}
#endif
#endif /* GSR_H_INCLUDED */
