/* gsr.h -- C ABI of the H100-native differentiable 3DGS tile rasterizer (libgsr_b200.so).
 *
 * This is the drop-in seam for the torch-free core of the reference rasterizer,
 *   CudaRasterizer::Rasterizer::{forward, backward, markVisible}
 *   ($RAST/cuda_rasterizer/rasterizer.h:24-91, $RAST = submodules/gaustudio-diff-gaussian-rasterization),
 * which the reference's pybind layer ($RAST/rasterize_points.cu:35-231, $RAST/ext.cpp:15-19) binds.
 * Plain pointers and sizes only: no torch / glm / std:: types.  All float* are DEVICE pointers to
 * contiguous float32 (the reference's convention, rasterize_points.cu:97-117); optional inputs are NULL
 * when absent (the reference passes the data pointer of an empty tensor, i.e. nullptr).
 * Alignment: the per-Gaussian quaternions are moved as one 16-byte vector, so `rotations` / `raw_rotations`
 * and the backward's `dL_drot` / `dL_draw_rot` and `dL_dconic` must be 16-byte aligned (a contiguous tensor
 * viewed at an element offset that is not a multiple of 4 is not); the entry points return -1 otherwise.
 * Every other pointer needs only float alignment.
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

/* Contribution statistics of one rendered view (DESIGN.md §7l): the forward's per-pixel walk replayed on the buffers
 * of a gsr_forward, gsr_forward_fused or gsr_forward_mip (exact or pipelined mode; R is the forward's return value,
 * as for gsr_backward), with the forward's own blend and termination decisions.  For every Gaussian i it ADDS
 *   weight[i]     += sum of w = alpha T over the pixels where i blended (per view in 32.32 fixed point, exact integer
 *                    sums, then folded into the double in stream order);
 *   count[i]      += the pixels whose walk reached the transmittance test at i: the pixels it blended plus the one
 *                    pair per pixel that ended the pixel (T (1 - alpha) < 1e-4, no weight);
 *   max_weight[i]  = max(max_weight[i], largest w), max_weight >= 0 on entry.
 * Results do not depend on scheduling, tile order or speculation.  geom_buffer's backward scratch is used (a later
 * gsr_backward of the same forward re-initialises it).  Shapes: weight double[P], count int64[P], max_weight
 * float[P]. */
int gsr_contribution(int P, int64_t R, int width, int height, char* geom_buffer, const char* binning_buffer,
                     const char* image_buffer, double* weight, int64_t* count, float* max_weight, void* stream);

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

/* ---- mesh extraction: what gaustudio/scripts/extract_mesh.py:86-186 runs after the render ----
 * A TSDF volume of 8^3-voxel bricks in a hash table on the device, unbounded in space like vdbfusion's VDB grid, in ONE
 * caller-owned state buffer of gsr_tsdf_bytes(capacity_bricks) bytes; capacity_bricks is 1..262144 and every call on
 * the volume passes the value it was initialised with.  Voxel i covers [i, i+1) * voxel_size on each axis.
 *
 * Replaces vdbfusion.VDBVolume(voxel_size, sdf_trunc, space_carving=False) (extract_mesh.py:86).  Enqueues the
 * clearing of `state`; no host synchronisation. */
size_t gsr_tsdf_bytes(int64_t capacity_bricks); /* 0 when capacity_bricks is out of range */
int gsr_tsdf_init(void* state, int64_t capacity_bricks, double voxel_size, double sdf_trunc, void* stream);

/* Replaces VDBVolume.integrate(points, extrinsic=origin) (extract_mesh.py:115) with its default constant weight.
 * points: device float[n*3]; valid: optional device uint8[n] (torch.bool), points with valid == 0 are skipped.
 * Per point p, d = p - origin: the voxels a DDA visits on the ray segment t in [max(0, |d| - trunc), |d| + trunc]
 * get sdf = s*|p - c| (c the voxel centre, s = +1 iff dot(c - origin, p - c) >= 0); sdf > -trunc adds the sample
 * min(trunc, sdf), as the integer rint(sample * 2^20 / trunc), with weight 1.  The stored value is the mean sample.
 * Float64 per-ray arithmetic and integer sums: the result does not depend on thread or call order.  Two launches,
 * no host synchronisation.  Running out of bricks is reported by the next gsr_tsdf_extract / gsr_tsdf_export. */
int gsr_tsdf_integrate(void* state, int64_t capacity_bricks, int64_t n, const float* points,
                       const unsigned char* valid, double origin_x, double origin_y, double origin_z, void* stream);

/* Replaces VDBVolume.extract_triangle_mesh(min_weight) (extract_mesh.py:145).  Marching cubes over the cubes whose
 * corners are the voxel centres v + {0,1}^3 and all have weight > min_weight (>= 0); a corner with tsdf >= 0 is
 * outside; one vertex per crossing edge (linear zero crossing, computed in double); faces point towards positive tsdf.
 * Order: bricks by key, then voxel.  Reads the counts back to the host once (blocking), then asks vertex_alloc for
 * float[V*3] and face_alloc for int64[F*3] (not called for an empty mesh); scratch_alloc is asked once for temporary
 * device memory.  Returns V and writes F to *n_faces, or -1 -- also when the volume ran out of bricks, with the
 * capacity it needs in the error text. */
int64_t gsr_tsdf_extract(void* state, int64_t capacity_bricks, double min_weight, gsr_alloc_fn scratch_alloc,
                         void* scratch_user, gsr_alloc_fn vertex_alloc, void* vertex_user, gsr_alloc_fn face_alloc,
                         void* face_user, int64_t* n_faces, void* stream);

/* Introspection for tests (vdbfusion exposes its grid through VDBVolume.tsdf / weights): returns the number of
 * bricks n (blocking) and, for the non-NULL outputs, writes the bricks in key order: brick_keys int64[n]
 * (((bz + 2^20) << 42) | ((by + 2^20) << 21) | (bx + 2^20)), sums int64[n*512] and weights int32[n*512], voxel
 * (x, y, z) of a brick at local index (z*8 + y)*8 + x. */
int64_t gsr_tsdf_export(void* state, int64_t capacity_bricks, gsr_alloc_fn scratch_alloc, void* scratch_user,
                        int64_t* brick_keys, int64_t* sums, int* weights, void* stream);

/* Replaces open3d's TriangleMesh.cluster_connected_triangles (extract_mesh.py:160-166): triangles are connected when
 * they share an edge.  faces: device int64[n_faces*3] with indices in [0, n_vertices); labels: device int64[n_faces],
 * the smallest face index of each face's component.  No host synchronisation. */
int gsr_mesh_face_components(int64_t n_faces, const int64_t* faces, int64_t n_vertices, gsr_alloc_fn scratch_alloc,
                             void* scratch_user, int64_t* labels, void* stream);

/* ---- mesh rendering and texturing: what gaustudio/scripts/render_mesh.py and texture_mesh.py run through pytorch3d's
 * MeshRasterizer (faces_per_pixel=1, blur_radius=0, no back-face culling) ----
 * vertices: device float[n_vertices*3]; faces: device int64[n_faces*3]; counts are 0..2^31-1, width / height 1..32768.
 * camera: HOST double[12], the world->camera rotation R (row-major, 9 values) then t (3 values), i.e. the top 3x4 of
 * Camera.extrinsics; fx, fy, cx, cy the pinhole intrinsics.  Pixel (column i, row j) samples the image point (i, j).
 *
 * Scratch of gsr_mesh_raster_bytes(n_vertices, n_faces, width, height) device bytes (0 for out-of-range sizes).  Its
 * first width*height*8 bytes are the z-buffer and must be all 0xff bytes before the first call; every call leaves
 * them so, so one scratch serves any number of views of the same (or a smaller) mesh at the same image size. */
size_t gsr_mesh_raster_bytes(int64_t n_vertices, int64_t n_faces, int width, int height);

/* Hard z-buffer.  Per vertex, in float64 without contraction: p = R x + t, u = fx px/pz + cx, v = fy py/pz + cy,
 * snapped to rint(256 u), rint(256 v) (ties to even); usable iff pz > znear and |u|, |v| < 2^20.  A face is drawn iff
 * its indices are in [0, n_vertices), its vertices usable and its exact int64 doubled area non-zero.  A sample is
 * covered when every edge function (oriented by the area's sign) is > 0, or == 0 on a top-left edge (y down).  Depth
 * is the perspective-correct view z 1/sum(l_i/z_i), l_i = E_i/A in double, rounded to float; the smallest depth wins,
 * then the smallest face index.  face_id: device int32[H*W] (-1: no face); depth: device float[H*W] (-1: no face).
 * No host synchronisation. */
int gsr_mesh_rasterize(int64_t n_vertices, const float* vertices, int64_t n_faces, const int64_t* faces,
                       const double* camera, double fx, double fy, double cx, double cy, double znear, int width,
                       int height, void* scratch, size_t scratch_bytes, int* face_id, float* depth, void* stream);

/* Per pixel of face_id (from gsr_mesh_rasterize with the same mesh and camera); both outputs optional (NULL):
 *   normal float[H*W*3]: R normalize(n_a + n_b + n_c) of the hit face's vertex_normals (float[V*3]), 0 without a face;
 *   color  float[H*W*3]: perspective-correct barycentric interpolation of vertex_colors (float[V*3]) with the
 *          barycentrics of the rasterizer's edge functions; 1 on a hit when vertex_colors is NULL; 0 without a face.
 * No host synchronisation. */
int gsr_mesh_shade(int64_t n_vertices, const float* vertices, int64_t n_faces, const int64_t* faces,
                   const double* camera, double fx, double fy, double cx, double cy, int width, int height,
                   const int* face_id, const float* vertex_normals, const float* vertex_colors, float* normal,
                   float* color, void* stream);

/* One view of texture_mesh.py:76-146, views numbered from 0 in the order they are applied.  face_stamp int32[F] and
 * vertex_stamp int32[V] are zeroed by the caller once before the first view.  Every face owning a pixel of face_id gets
 * face_stamp = view + 1; such a face with unit normal n = cross(v1 - v0, v2 - v0)/|.| (float64) adds rint(dot(n, d) *
 * 2^40) to stats[0] and 1 to stats[1] (device int64[2], zeroed by the caller; d = the third row of R, the optical
 * axis), and with dot(n, d) < -0.05 stamps its vertices.  A stamped vertex whose unsnapped projection lies in
 * [0, W-1] x [0, H-1] gets clamp(bilinear(image, u, v), 0, 1) in vertex_colors (float[V*3]); image: device float[H*W*3].
 * No host synchronisation. */
int gsr_mesh_texture_view(int64_t n_vertices, const float* vertices, int64_t n_faces, const int64_t* faces,
                          const double* camera, double fx, double fy, double cx, double cy, int width, int height,
                          const int* face_id, const float* image, int view, int* face_stamp, int* vertex_stamp,
                          int64_t* stats, float* vertex_colors, void* stream);

/* ---- Shape-as-Points meshing: the `--meshing sap` step of gaustudio/scripts/extract_pcd.py (models/sap.py and the
 * DPSR of utils/graphics_utils.py, res = 256, sig = 2, scale = shift = True, weighted = False) ----
 * n is 1..2^31-1 and res 2..512.  Grids are float[res^3] indexed (x*res + y)*res + z, grid node k at k/res.  The FFTs
 * between the stages are the caller's (torch.fft.rfftn / irfftn over the three grid axes).  Every sum has a fixed
 * order: the same inputs give the same bits.  Only gsr_sap_marching_cubes synchronises with the host.
 *
 * xyz: device float[n*3].  Writes transform (device float[4]) = (c, s) with c = mean(xyz) and s = 1.2 max|xyz - c|
 * over all coordinates (both reduced in double, stored as float32), and points01 (device float[n*3]) =
 * ((xyz - c)/s + 1)/2 in float32.  scratch_alloc is asked once. */
int gsr_sap_normalize(int64_t n, const float* xyz, gsr_alloc_fn scratch_alloc, void* scratch_user, float* points01,
                      float* transform, void* stream);

/* point_rasterize(weighted=False): grid (device float[3*res^3], one grid per normal component) = sum over points of
 * normal * trilinear weight towards the 8 nodes around the point, cell i0 = floor(p / cs), cs = float32(1/res), node
 * i0 + 1 wrapped to 0 at res.  points01: device float[n*3] in [0, 1) (cell indices are clamped into the grid);
 * normals: device float[n*3].  Deterministic: points are bucketed by cell (stable in point index) and every node
 * gathers from its 8 cells in a fixed order, summing in double.  scratch_alloc is asked once. */
int gsr_sap_splat(int64_t n, const float* points01, const float* normals, int res, gsr_alloc_fn scratch_alloc,
                  void* scratch_user, float* grid, void* stream);

/* The spectral solve of DPSR.forward: spectrum is rfftn of the three grids, complex64 [3][res][res][res/2+1]; writes
 * phi_hat (complex64 [res][res][res/2+1]) = -i sum_d 2 pi w_d G N_d / (-sum_d (2 pi w_d)^2 + 1e-6), 0 at w = 0, with
 * w numpy's integer fftfreq on the first two axes and rfftfreq on the last, G = exp(-0.5 (sig 2 |w| / res)^2) formed
 * in double and rounded to float.  sig is positive and finite. */
int gsr_sap_spectral(int res, double sig, const float* spectrum, float* phi_hat, void* stream);

/* Shift and scale: offset = mean over the points of the trilinear interpolation of phi (device float[res^3]) at
 * points01 (the splat's weights; summed in double in a fixed order), fv0 = phi[0] - offset, and psi (device
 * float[res^3]) = tanh(-(phi - offset) / |fv0| * 0.5).  scratch_alloc is asked once. */
int gsr_sap_shift_scale(int64_t n, const float* points01, int res, const float* phi, gsr_alloc_fn scratch_alloc,
                        void* scratch_user, float* psi, void* stream);

/* Marching cubes of psi at 0 over the (res-1)^3 cubes of the grid, with the tables of the TSDF extraction: one vertex
 * per crossing edge (linear zero crossing in double), faces facing psi > 0 (outside: psi is
 * positive on the side the normals point, as in the reference).  A vertex at index coordinates q lands at
 * (q/res * 2 - 1) * s + c with (c, s) from transform (device float[4], gsr_sap_normalize's).  Order: vertices by node
 * then axis, faces by cube then table entry.  Reads the counts back once (blocking), then asks vertex_alloc for
 * float[V*3] and face_alloc for int64[F*3] (not called for an empty mesh); scratch_alloc is asked once.  Returns V
 * and writes F to *n_faces, or -1. */
int64_t gsr_sap_marching_cubes(int res, const float* psi, const float* transform, gsr_alloc_fn scratch_alloc,
                               void* scratch_user, gsr_alloc_fn vertex_alloc, void* vertex_user,
                               gsr_alloc_fn face_alloc, void* face_user, int64_t* n_faces, void* stream);

/* ---- point-cloud cleaning: clean_point_cloud of gaustudio/scripts/extract_pcd.py:30-51 (Open3D's
 * remove_statistical_outlier, then remove_normal_outliers) ----
 * n is 1..2^31-1 and k 1..64; xyz and normals are device float[n*3].  Neighbours are exact: squared distances are
 * (dx dx + dy dy) + dz dz in double from the float32 coordinates, ties to the lower index.  Every sum has a fixed
 * order: the same inputs give the same bits.  No host synchronisation; scratch_alloc is asked once per call.
 *
 * Test entry: the K = min(k, n) nearest points of every point, itself included, ascending; index int32[n*k] and
 * sq_dist double[n*k] (row i, columns >= K untouched). */
int gsr_clean_knn(int64_t n, const float* xyz, int k, gsr_alloc_fn scratch_alloc, void* scratch_user, int* index,
                  double* sq_dist, void* stream);

/* PointCloud::RemoveStatisticalOutliers(k, std_ratio): avg_dist (device double[n]) = the mean distance to the
 * K = min(k, n) nearest points, the point itself included; stats (device double[3]) = (mean, std, threshold) with
 * mean = sum avg / n, std = sqrt(sum_{avg > 0} (avg - mean)^2 / (n - 1)) and threshold = mean + std_ratio std;
 * keep (device uint8[n]) = avg > 0 && avg < threshold.  std_ratio is positive and finite. */
int gsr_clean_statistical(int64_t n, const float* xyz, int k, double std_ratio, gsr_alloc_fn scratch_alloc,
                          void* scratch_user, double* avg_dist, double* stats, unsigned char* keep, void* stream);

/* remove_normal_outliers(k, angle_threshold): mean_angle (device double[n]) = the mean over the min(k, n) - 1 nearest
 * points other than the point itself of acos(min(|n_i . n_j|, 1)), the dot product in double (NaN when there are
 * none, or a normal is NaN); keep (device uint8[n]) = mean_angle < angle_threshold.  angle_threshold is finite. */
int gsr_clean_normal(int64_t n, const float* xyz, const float* normals, int k, double angle_threshold,
                     gsr_alloc_fn scratch_alloc, void* scratch_user, double* mean_angle, unsigned char* keep,
                     void* stream);

/* distCUDA2 of simple_knn (graphdeco's and gaustudio's initial scales): dist2 (device float[n]) = float of the mean of
 * the squared distances to the 3 nearest points other than the point itself, the exact search and rounding of
 * gsr_clean_knn, summed (d1 + d2) + d3 in double; a missing neighbour (n <= 3) counts as +inf. */
int gsr_dist2(int64_t n, const float* xyz, gsr_alloc_fn scratch_alloc, void* scratch_user, float* dist2, void* stream);

/* ---- Gaussian initialization: gaustudio/pipelines/initializers/{pcd,mesh}.py (csrc/gsr_init.cu) ----
 * normal2rotation of pcd.py:12-37 in float32, the reference's op order: normals device float[n*3] -> rot device
 * float[n*4] (16-byte aligned), the raw quaternion (w, x, y, z) of [R0 | R1 | normalize(n)]. */
int gsr_normal2rotation(int64_t n, const float* normals, float* rot, void* stream);

/* open3d's compute_vertex_normals: each vertex sums the face normals (v1 - v0) x (v2 - v0) of its faces in ascending
 * face order, in double, then divides by the norm (a zero sum stays zero); normals device float[nv*3].  verts device
 * float[nv*3], faces device int64[nf*3] with indices in [0, nv), nf < 2^31 / 3.  scratch_alloc is asked once. */
int gsr_mesh_vertex_normals(int64_t nv, const float* verts, int64_t nf, const int64_t* faces,
                            gsr_alloc_fn scratch_alloc, void* scratch_user, float* normals, void* stream);

/* SuGaR placement of the mesh initializer (mesh.py:95-250) with n in {1, 3, 4, 6} Gaussians per face, row f n + s for
 * slot s of face f: xyz float[3] the barycentric combination, rot float[4] (16-byte aligned) normal2rotation of the
 * normalised interpolated vertex normal, f_dc float[3] RGB2SH of the interpolated colour (of ones when colors is NULL),
 * scale float[3] log(2 min_edge radius_n + 1e-7) twice and log(1e-7), opacity float[1] +inf.  float32 torch ops. */
int gsr_mesh_gaussians(int64_t nf, int n, const float* verts, const int64_t* faces, const float* vertex_normals,
                       const float* colors, float* xyz, float* rot, float* f_dc, float* scale, float* opacity,
                       void* stream);

/* open3d's VoxelGrid::CreateFromTriangleMeshWithinBounds on [-0.5, 0.5]^3 with res (1..1024) cells per axis: cell
 * (i, j, k), box centre (-0.5 + idx voxel_size) + voxel_size / 2 per axis and half-size voxel_size / 2, is occupied iff
 * tribox3 (in double, its op order, a touch overlaps) passes for some triangle.  verts device double[nv*3], faces
 * device int64[nf*3].  Reads counts back three times (blocking); asks alloc once with each of column_user, hit_user
 * and sort_user for scratch, then with out_user for int32[2U + 1 + H]: the occupied cells' linear indices
 * (i res + j) res + k ascending (uint32[U]), the CSR offsets (int32[U + 1]) and each cell's triangles ascending
 * (int32[H]).  Returns U (0: nothing allocated) and writes H to *n_pairs, or -1. */
int64_t gsr_voxelize(int64_t nv, const double* verts, int64_t nf, const int64_t* faces, int res, double voxel_size,
                     gsr_alloc_fn alloc, void* column_user, void* hit_user, void* sort_user, void* out_user,
                     int64_t* n_pairs, void* stream);

/* Voxel colours: for each of gsr_voxelize's cells, the closest point of the mesh to its centre (squared distance in
 * double, ties to the lower triangle), searched over the triangles of the occupied cells within +-1, and rgb
 * (device float[ncell*3]) the barycentric interpolation there of colors (device float[nv*3]), in double. */
int gsr_voxel_colors(int64_t ncell, const unsigned* cells, const int* offsets, const int* tris, int res,
                     double voxel_size, const double* verts, const int64_t* faces, const float* colors, float* rgb,
                     void* stream);

/* ---- VisualHull: space carving of gaustudio/pipelines/initializers/mask.py (csrc/gsr_hull.cu) ----
 * res is 2..512, radius r > 0 and (tx, ty, tz) the reference's `translate`, all finite.  The grid has res^3 nodes,
 * node g = (i res + j) res + k at float32(lin[j] - tx, lin[i] - ty, lin[k] - tz) with lin = np.linspace(-r, r, res)
 * (i step + start in double, no contraction, the last node exactly r): the reference's meshgrid order.
 *
 * Carve: occ (device uint8[res^3]) = 1 iff the node passes the reference's Camera.insideView for every camera, in
 * order, evaluated in double from the float32 node and the float32 full_proj_transform P (device float[n_cams*16],
 * row-major as stored): clip = [x y z 1] P summed in row order, clip_z > 0, ndc = clip_xy / clip_w in [-1, 1]^2 (inf
 * and NaN fail), px = min(trunc((ndc_x + 1) 0.5 W), W - 1), py likewise with H, and mask[py][px] != 0.  views (device
 * int64[n_cams*3]) = (W, H, offset of the camera's [H][W] mask in masks, or -1: no mask, every pixel inside); masks
 * is device uint8.  n_cams = 0 fills every node.  No atomics. */
int gsr_hull_carve(int res, double radius, double tx, double ty, double tz, int n_cams, const float* proj,
                   const int64_t* views, const unsigned char* masks, unsigned char* occ, void* stream);

/* Marching cubes of occ (gsr_hull_carve's) at threshold in (0, 1): mcubes.marching_cubes(volume, threshold) with the
 * reference's fliplr and axis swap.  One vertex per grid edge whose ends differ, at index coordinate q = c + threshold
 * from an empty node c, c + (1 - threshold) from a filled one (double), mapped to the world per axis as
 * ((q / (res - 1)) (2 r) - r) - t in double and rounded once; world x comes from the grid's j axis and y from its i
 * axis.  Faces face the empty side.  Order: vertices by node then axis (i, j, k), faces by cube then table entry.  Reads
 * the counts back once (blocking), then asks vertex_alloc for float[V*3] and face_alloc for int64[F*3] (not called for
 * an empty mesh); scratch_alloc is asked once.  Returns V and writes F to *n_faces, or -1. */
int64_t gsr_hull_marching_cubes(int res, const unsigned char* occ, double threshold, double radius, double tx,
                                double ty, double tz, gsr_alloc_fn scratch_alloc, void* scratch_user,
                                gsr_alloc_fn vertex_alloc, void* vertex_user, gsr_alloc_fn face_alloc, void* face_user,
                                int64_t* n_faces, void* stream);

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

/* Introspection for tests: copies the per-Gaussian accumulator of the last gsr_backward / gsr_backward_fused on
 * geom_buffer into the caller's DEVICE float[P][12], ordered on `stream`.  It holds what the compositing backward added
 * up and the projection backward read: {dL/dcolor r, g, b, dL/ddepth, dL/dopacity, Sx, Sy, Sxx, Sxy, Syy, -, -}, the
 * layout of `accum` at gsr_debug_projection_backward (the last two slots are 0).  Returns -1 on a NULL buffer. */
int gsr_debug_accumulator(int P, const char* geom_buffer, float* accum, void* stream);

/* Test hook: the projection backward alone, on per-Gaussian screen-space sums chosen by the caller.
 * gsr_backward / gsr_backward_fused zero an accumulator, let the compositing backward add ten sums per Gaussian to it
 * and then run the projection backward on it; this entry point copies `accum` (DEVICE float[P][12]) into that
 * accumulator instead and runs only the projection backward, with the same argument checks and kernel-path choice.
 * Accumulator layout per Gaussian: {dL/dcolor r, g, b, dL/ddepth, dL/dopacity, Sx, Sy, Sxx, Sxy, Syy, -, -} with
 * S.. = sum over pixels of dL/dG * G * (dx, dy, dx^2, dx dy, dy^2), d = mean2D - pixel.
 * fused = 0: the arguments of gsr_backward (opacities, f_dc, f_rest, dL_df_dc, dL_df_rest unused);
 * fused = 1: those of gsr_backward_fused, with scales / rotations / opacities / dL_dsh... naming the raw attributes and
 * their gradients, shs / colors_precomp / cov3D_precomp / dL_dsh unused, and dL_dconic / dL_ddepth written when given.
 * geom_buffer must hold a forward of the same Gaussians and camera (radii, colour-clamp bits). */
int gsr_debug_projection_backward(int fused, int P, int D, int M, int width, int height, const float* means3D,
                                  const float* shs, const float* colors_precomp, const float* f_dc, const float* f_rest,
                                  const float* opacities, const float* scales, float scale_modifier,
                                  const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                                  const float* projmatrix, const float* campos, float tan_fovx, float tan_fovy,
                                  const int* radii, char* geom_buffer, const float* accum, float* dL_dmean2D,
                                  float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_ddepth,
                                  float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_df_dc,
                                  float* dL_df_rest, float* dL_dscale, float* dL_drot, int debug, void* stream);

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

/* ---- Surfel (2D Gaussian) rasterizer: the contract of the 2DGS renderer, DESIGN.md §3, surfel rasterizer ----
 * Per Gaussian: means3D[P,3], scales[P,2] (two activated tangent scales), rotations[P,4] (normalised quaternion
 * w,x,y,z; 16-byte aligned), opacities[P], exactly one of shs[P,M,3] / colors_precomp[P,3].  viewmatrix / projmatrix
 * are the 3DGS path's (row-vector layout: p_view = [p,1] @ viewmatrix, clip = [p,1] @ projmatrix).
 * Projection: culled when p_view.z <= 0.2.  Tangent axes t_u = R[:,0] s_u mod, t_v = R[:,1] s_v mod, normal R[:,2].
 * The splat point (u,v) has pixel-homogeneous coordinates h = (u,v,1).(Tu, Tv, Tw), with
 * h = (W/2 c.x + (W-1)/2 c.w, H/2 c.y + (H-1)/2 c.w, c.w) for c = [p + u t_u + v t_v, 1] @ projmatrix.  The view
 * normal is flipped to face the camera (culled when perpendicular to the centre ray).  Screen box with
 * Q = diag(9,9,-1): d = Tw'Q Tw (culled when 0), mean2D = (Tu'Q Tw, Tv'Q Tw)/d, half extents
 * sqrt(max(1e-4, mean2D^2 - (Tu'Q Tu, Tv'Q Tv)/d)), radius = ceil(max(half, 3*0.707106)); the tile rect is getRect's
 * (every tile binned; an empty rect culls).  Colour: the 3DGS path's SH (clamped at 0) or colors_precomp.
 * Per pixel (x,y), front to back in (depth, index) order: k = x Tw - Tu, l = y Tw - Tv, p = k x l (skip if p.z == 0),
 * s = p.xy/p.z, rho3 = |s|^2, rho2 = 2|mean2D - (x,y)|^2; z = rho3 <= rho2 ? s.Tw.xy + Tw.z : Tw.z (skip if z < 0.2);
 * alpha = min(0.99, o exp(-min(rho3,rho2)/2)) (skip if < 1/255; the pixel ends where T(1-alpha) < 1e-4);
 * w = alpha T blends colour, z, n_view; distortion with m = 100/99.8 (1 - 0.2/z); the median is the last splat
 * blended while T > 0.5.
 * Outputs: out_color[3,H,W] = C + T bg;  out_allmap[9,H,W] = {expected depth sum D, 1-T, normal (3), median depth,
 * distortion, median weight, median Gaussian index (float)}; median channels are 0 where no splat blends at T > 0.5.
 * radii[P] (optional) as the 3DGS path.  Allocators, `debug`, `stream` and the return value (num_rendered = sum of
 * the rect areas, after the one blocking count read) as gsr_forward; `prefiltered` is accepted and has no effect.
 * Returns -1 with an error text, before any work, on NULL required pointers, P < 0, non-positive sizes, D outside
 * 0..3 or M < (D+1)^2 with shs, not exactly one of shs / colors_precomp, or misaligned rotations. */
size_t gsr_surfel_geometry_bytes(int P);
size_t gsr_surfel_image_bytes(int width, int height);
int64_t gsr_surfel_forward(gsr_alloc_fn geometry_alloc, void* geometry_user, gsr_alloc_fn binning_alloc,
                           void* binning_user, gsr_alloc_fn image_alloc, void* image_user, int P, int D, int M,
                           const float* background, int width, int height, const float* means3D, const float* shs,
                           const float* colors_precomp, const float* opacities, const float* scales,
                           float scale_modifier, const float* rotations, const float* viewmatrix,
                           const float* projmatrix, const float* cam_pos, int prefiltered, float* out_color,
                           float* out_allmap, int* radii, int debug, void* stream);

/* Backward of gsr_surfel_forward (same Gaussians, camera and buffers; R = its return value; shs NULL when colours
 * were precomputed).  Upstream: dL_dpix[3,H,W] and dL_dallmap[9,H,W]; channels 7 and 8 (median weight and index)
 * carry no gradient and are not read.  Every branch is differentiated (ray-splat and low-pass branches, median depth
 * through the median splat's z, distortion, normal with its flip held constant); the 0.99 alpha clamp passes none.
 * Outputs, fully written (no pre-zeroing): dL_dmean2D[P,3] = gradient w.r.t. a screen-space translation of the
 * splat (Tu += dx Tw, Tv += dy Tw, mean2D += d) in NDC units (x W/2, y H/2; third component 0), dL_dopacity[P],
 * dL_dcolor[P,3], dL_dmean3D[P,3], dL_dsh[P,M,3] (required with shs), dL_dscale[P,2], dL_drot[P,4] (16-byte
 * aligned).  Culled Gaussians get zeros. */
int gsr_surfel_backward(int P, int D, int M, int64_t R, const float* background, int width, int height,
                        const float* means3D, const float* shs, const float* scales, float scale_modifier,
                        const float* rotations, const float* viewmatrix, const float* projmatrix, const float* campos,
                        char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
                        const float* dL_dallmap, float* dL_dmean2D, float* dL_dopacity, float* dL_dcolor,
                        float* dL_dmean3D, float* dL_dsh, float* dL_dscale, float* dL_drot, int debug, void* stream);

/* ---- Mip-Splatting: the mip_renderer (DESIGN.md, Mip-Splatting) ----
 * gsr_forward_mip: gsr_forward with the 2D Mip filter of width kernel_size (finite, >= 0) in the projection.  Per
 * Gaussian, with (a, b, c) = J W Sigma W^T J^T (the 2D covariance before gsr_forward's 0.3 dilation):
 *   det0 = max(1e-6, ac - b^2), det1 = max(1e-6, (a+k)(c+k) - b^2), coef = sqrt(det0 / (det1 + 1e-6) + 1e-6), or 0
 *   when either clamp fired;  cov' = (a+k, b, c+k) gives the conic, radius and tiles;  opacity' = opacity * coef.
 * Everything else -- colours, depth, means2D, radii, allocators, modes, the buffers and the return value -- is
 * gsr_forward's; gsr_debug_export reads opacity' in conic_opacity.  Only the un-fused inputs are taken.
 * gsr_backward_mip: gsr_backward for such a forward, plus the forward's input `opacities` and the same kernel_size;
 * dL_dopacity is w.r.t. the input opacity.  gsr_debug_projection_backward_mip: gsr_debug_projection_backward (fused = 0)
 * for such a forward.  All three return -1 with an error text, before any work, on a bad kernel_size or NULL
 * opacities (backward), then run the checks of the entry point they extend. */
int64_t gsr_forward_mip(gsr_alloc_fn geometry_alloc, void* geometry_user, gsr_alloc_fn binning_alloc,
                        void* binning_user, gsr_alloc_fn image_alloc, void* image_user, int P, int D, int M,
                        const float* background, int width, int height, const float* means3D, const float* shs,
                        const float* colors_precomp, const float* opacities, const float* scales,
                        float scale_modifier, const float* rotations, const float* cov3D_precomp,
                        const float* viewmatrix, const float* projmatrix, const float* cam_pos, float tan_fovx,
                        float tan_fovy, int prefiltered, float* out_color, float* out_depth,
                        float* out_median_depth, float* out_opacity, int* radii, int debug, int64_t r_capacity,
                        int64_t* r_host, float kernel_size, void* stream);
int gsr_backward_mip(int P, int D, int M, int64_t R, const float* background, int width, int height,
                     const float* means3D, const float* shs, const float* colors_precomp, const float* scales,
                     float scale_modifier, const float* rotations, const float* cov3D_precomp,
                     const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                     float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer,
                     const float* dL_dpix, const float* dL_dpix_depth, const float* dL_dpix_median_depth,
                     const float* dL_dpix_final_opacity, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity,
                     float* dL_dcolor, float* dL_ddepth, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                     float* dL_dscale, float* dL_drot, int debug, const float* opacities, float kernel_size,
                     void* stream);
int gsr_debug_projection_backward_mip(int P, int D, int M, int width, int height, const float* means3D,
                                      const float* shs, const float* colors_precomp, const float* opacities,
                                      const float* scales, float scale_modifier, const float* rotations,
                                      const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                                      const float* campos, float tan_fovx, float tan_fovy, const int* radii,
                                      char* geom_buffer, const float* accum, float* dL_dmean2D, float* dL_dconic,
                                      float* dL_dopacity, float* dL_dcolor, float* dL_ddepth, float* dL_dmean3D,
                                      float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
                                      float kernel_size, int debug, void* stream);

/* Mip-Splatting's 3D smoothing filter (MipPointCloud.compute_3D_filter) over all cameras in one pass.
 * cameras: DEVICE float[n_cameras*16], per camera R (9, row-major, Camera.R: p = x @ R + T), T (3), fx, fy (> 0),
 * width, height.  Per Gaussian x: camera c sees it iff p.z > 0.2 and u = p.x/z' fx + W/2, v = p.y/z' fy + H/2
 * (z' = max(p.z, 0.001)) lie in [-0.15 W, 1.15 W] x [-0.15 H, 1.15 H]; d = min(100000, min of p.z over those cameras);
 * a Gaussian no camera sees gets the largest d of the seen ones; filter_3D[P] = d / max_c fx * sqrt(0.2).
 * scratch: DEVICE uint32[3] owned by the caller; afterwards scratch[2] holds the number of seen Gaussians (when it is
 * 0 the filter is meaningless).  No host synchronisation; the result does not depend on thread order. */
int gsr_mip_filter3d(int P, const float* means3D, int n_cameras, const float* cameras, float* filter_3D,
                     unsigned int* scratch, void* stream);

/* ---- Scaffold-GS: the scaffold_renderer (DESIGN.md §7d) ----
 * gsr_scaffold_visible: radii[N] (int32) of N Gaussians at the anchors, with activated scales[N,3] (times
 * scale_modifier) and rotations[N,4] (16-byte aligned), or cov3D_precomp[N,6], under the Mip projection of width
 * kernel_size (finite, >= 0).  Bit-identical to the radii gsr_forward_mip writes for the same means, scales,
 * rotations and camera (the radius does not depend on the opacity).  No host synchronisation. */
int gsr_scaffold_visible(int N, const float* means3D, const float* scales, const float* rotations,
                         const float* cov3D_precomp, float scale_modifier, const float* viewmatrix,
                         const float* projmatrix, int width, int height, float tan_fovx, float tan_fovy,
                         float kernel_size, int* radii, void* stream);

/* Neural-Gaussian decoding of Nv visible anchors with k = 1..32 offsets each.  opacity[Nv,k] (the opacity MLP's
 * output); offset j of visible anchor i is kept iff opacity[i,j] > 0.
 * gsr_scaffold_count: base[Nv+1] (int32) = exclusive prefix of the kept counts, base[Nv] = M; scratch: DEVICE
 * int32[(Nv + 1023) / 1024].  No host synchronisation.
 * gsr_scaffold_decode: kept rows in anchor-major, offset-minor order (row base[i] + rank of j among i's kept offsets).
 * vis[Nv] (int64): anchor index of visible anchor i; anchor[N,3], offset[N,k,3], scaling[N,6] (activated) are
 * full-size; color[Nv,3k] and cov[Nv,7k] are the colour and covariance MLPs' outputs.  For v = vis[i],
 * S = scaling[v], c = color[i,3j..], s = cov[i,7j..]:
 *   xyz[M,3] = anchor[v] + offset[v,j] * S[0:3]   rgb[M,3] = c   out_opacity[M] = opacity[i,j]
 *   scales[M,3] = S[3:6] * sigmoid(s[0:3])        rotations[M,4] = s[3:7] / max(|s[3:7]|, 1e-12) (16-byte aligned)
 * each product and sum rounded on its own.
 * gsr_scaffold_decode_backward: with the upstream gradients of the five outputs ([M,...], read only where M > 0),
 * writes dL_dopacity_mlp[Nv,k], dL_dcolor[Nv,3k], dL_dcov[Nv,7k] (zero for dropped offsets) and the full-size
 * dL_danchor[N,3], dL_doffset[N,k,3], dL_dscaling[N,6] (zero for anchors that are not visible and for dropped offsets).
 * One thread per visible anchor sums its offsets in order: no atomics, the same bits on every run.
 * All three return -1 with an error text, before any work, on k outside 1..32, Nv < 0 (or Nv > N), a product of
 * the sizes beyond int32, NULL required pointers or misaligned rotations. */
int gsr_scaffold_count(int Nv, int k, const float* opacity, int* base, int* scratch, void* stream);
int gsr_scaffold_decode(int Nv, int k, const int64_t* vis, const int* base, const float* anchor, const float* offset,
                        const float* scaling, const float* opacity, const float* color, const float* cov, float* xyz,
                        float* rgb, float* out_opacity, float* scales, float* rotations, void* stream);
int gsr_scaffold_decode_backward(int N, int Nv, int k, const int64_t* vis, const int* base, const float* offset,
                                 const float* scaling, const float* opacity, const float* cov, const float* dL_dxyz,
                                 const float* dL_drgb, const float* dL_dopacity, const float* dL_dscales,
                                 const float* dL_drotations, float* dL_dopacity_mlp, float* dL_dcolor, float* dL_dcov,
                                 float* dL_danchor, float* dL_doffset, float* dL_dscaling, void* stream);

/* ---- adaptive density control of 3DGS / 2DGS training (DESIGN.md §7e) ----
 * gsr_densify_stats: the statistics of one view after its backward (graphdeco's add_densification_stats).  For every
 * i with radii[i] > 0: accum[i] += sqrt(g[i,0]^2 + g[i,1]^2), denom[i] += 1, max_radii2D[i] = max(max_radii2D[i],
 * radii[i]), where g = viewspace_grad [P,3].  accum, denom, max_radii2D: float32[P].  One launch, no host
 * synchronisation: it can be captured in a CUDA graph.
 * gsr_densify_count: the decisions of densify_and_prune over P Gaussians with raw log-scales scale[P,scale_dim]
 * (scale_dim 2 or 3) and opacity logits opacity[P]: grad = accum / denom (NaN -> 0), smax = max_c exp(scale);
 * clone iff grad >= max_grad and smax <= clone_max_scale; split iff grad >= max_grad and smax > clone_max_scale; a row
 * (original, clone, or child with scale log(exp(scale) * (1 / 1.6f))) is pruned iff sigmoid(opacity) < min_opacity or,
 * when prune_big != 0, its smax > big_scale.  scratch: DEVICE int32[GSR_DENSIFY_SCRATCH_INTS(P)]; afterwards its first
 * four entries hold the totals (originals kept, clones kept, child pairs kept, splits).  No host synchronisation.
 * gsr_densify_apply: writes every output tensor of the step in one launch, from the scratch of gsr_densify_count, its
 * four totals (read back by the caller) and noise z [2 n_split, 3].  Each entry maps src [P, width] to dst [P_new,
 * width], P_new = n_orig + n_clone + 2 n_pair: surviving originals in index order, then surviving clones in source order,
 * then the first children (z rows 0..n_split-1 by split rank), then the second children (z rows n_split..).  Roles:
 *   COPY, ROT: raw copies (ROT, 16-byte aligned, is also the rotation of the children's xyz)
 *   XYZ: children get R(rot) (z (.) exp(scale)) + xyz, with a zero third scale when scale_dim is 2
 *   SCALE: children get log(exp(scale) * (1 / 1.6f))
 *   MOMENT: optimizer state shaped like its parameter: survivors keep their bits, clones and children get zeros.
 * Exactly one XYZ (width 3), SCALE (width scale_dim) and ROT (width 4) entry, other entries of width 1..4096 (every
 * float of every row is written); at most GSR_DENSIFY_MAX_ENTRIES.
 * Every value except the children's xyz is rounded op by op as torch's CUDA kernels round it.
 * All three return -1 with an error text, before any work, on bad sizes or counts (P_new must fit in int32), a scale
 * width other than 2 or 3, NULL required pointers, bad entries or non-finite thresholds. */
#define GSR_DENSIFY_MAX_ENTRIES 24
#define GSR_DENSIFY_COPY 0
#define GSR_DENSIFY_XYZ 1
#define GSR_DENSIFY_SCALE 2
#define GSR_DENSIFY_ROT 3
#define GSR_DENSIFY_MOMENT 4
#define GSR_DENSIFY_SCRATCH_INTS(P) (4 + 5 * (int64_t)(P) + 4 * (((int64_t)(P) + 1023) / 1024))
typedef struct gsr_densify_entry {
  const float* src;
  float* dst;
  int width; /* floats per row */
  int role;  /* GSR_DENSIFY_* */
} gsr_densify_entry;
int gsr_densify_stats(int P, const float* viewspace_grad, const int* radii, float* accum, float* denom,
                      float* max_radii2D, void* stream);
int gsr_densify_count(int P, int scale_dim, const float* accum, const float* denom, const float* scale,
                      const float* opacity, float max_grad, float min_opacity, float clone_max_scale, int prune_big,
                      float big_scale, int* scratch, void* stream);
int gsr_densify_apply(int P, int scale_dim, const int* scratch, int n_orig, int n_clone, int n_pair, int n_split,
                      const float* noise, int n_entries, const gsr_densify_entry* entries, void* stream);

/* ---- photometric training loss: L1 + D-SSIM of graphdeco's train.py (DESIGN.md §7f) ----
 * img1 (the render) and img2 (the target): `planes` (image, channel) planes of H x W float32 each, contiguous.  The
 * window is graphdeco's create_window(11, C) (taps of gaussian(11, 1.5), zero padding of 5), applied per plane.
 * gsr_ssim_scratch_bytes: size of the device scratch of gsr_ssim_forward (0 on bad sizes).
 * gsr_ssim_forward: sums[0] = sum |img1 - img2|, sums[1] = sum of the SSIM map, over every element (float32[2],
 * summed in double in a fixed order: the same bits on every run).  partials: NULL, or float32[3, planes, H, W] that
 * receives the maps D0, D1, D2 of the backward.
 * gsr_ssim_backward: d_img1[planes, H, W] = d_sums[0] sign(img1 - img2) + d_sums[1] d(sum S)/d img1 from the maps of
 * the forward; d_sums is a DEVICE float32[2].  Every element of d_img1 is written.
 * Neither synchronises with the host.  All three refuse, before any work, planes, H or W < 1 and element counts beyond
 * int64; the two entries also NULL pointers (partials only in the backward) and grids beyond 2^31 - 1 tiles. */
size_t gsr_ssim_scratch_bytes(int64_t planes, int H, int W);
int gsr_ssim_forward(int64_t planes, int H, int W, const float* img1, const float* img2, float* partials,
                     void* scratch, float* sums, void* stream);
int gsr_ssim_backward(int64_t planes, int H, int W, const float* img1, const float* img2, const float* partials,
                      const float* d_sums, float* d_img1, void* stream);

/* ---- 2DGS normal-consistency loss (DESIGN.md §7g) ----
 * rend_normal: float32[3, H, W], world space; surf_depth: float32[H, W], view-space depth; alpha: float32[H, W];
 * world_view: the camera's world_view_transform as stored (float32[16], row-vector convention); fx, fy, cx, cy: the
 * pinhole intrinsics.  Pixel (x, y) back-projects to P = z ((x + 0.5 - cx) / fx, (y + 0.5 - cy) / fy, 1).  The surface
 * normal s of an interior pixel is normalize(u x v), u = P(x, y+1) - P(x, y-1), v = P(x+1, y) - P(x-1, y), eps 1e-12;
 * s = 0 on the border and when H < 3 or W < 3.
 * gsr_normal_consistency_scratch_bytes: size of the device scratch of the forward (0 on bad sizes).
 * gsr_normal_consistency_forward: loss[0] = mean over the H W pixels of 1 - alpha <rend_normal, s M3^T> (M3 the
 * rotation block of world_view), summed in double in a fixed order: the same bits on every run.
 * gsr_normal_consistency_backward: d_rend_normal[3, H, W] and d_surf_depth[H, W] of the loss times d_loss, a DEVICE
 * float32[1]; alpha gets no gradient.  Every element of both is written; nothing is stored between the two calls.
 * Neither synchronises with the host.  All three refuse, before any work, H or W < 1 and grids beyond 2^31 - 1 tiles;
 * the two entries also non-finite or zero fx / fy and NULL pointers. */
size_t gsr_normal_consistency_scratch_bytes(int H, int W);
int gsr_normal_consistency_forward(int H, int W, const float* rend_normal, const float* surf_depth, const float* alpha,
                                   const float* world_view, float fx, float fy, float cx, float cy, void* scratch,
                                   float* loss, void* stream);
int gsr_normal_consistency_backward(int H, int W, const float* rend_normal, const float* surf_depth,
                                    const float* alpha, const float* world_view, float fx, float fy, float cx,
                                    float cy, const float* d_loss, float* d_rend_normal, float* d_surf_depth,
                                    void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GSR_H_INCLUDED */
