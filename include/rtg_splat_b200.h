/*
 * rtg_splat_b200.h -- C ABI of librtg_splat_b200.so (sm_90a).
 *
 * Drop-in boundary for RTG-SLAM's data-parallel hot path. Every entry point names the
 * reference interface it replaces ("RAST/" = submodules/diff-gaussian-rasterizer-depth/ of
 * MisEty/RTG-SLAM). Plain pointers and sizes only; no torch types. All device pointers are
 * CUDA device memory on the current device, fp32 / int32, contiguous. Every call is
 * asynchronous on `stream` (a cudaStream_t passed as void*; NULL = legacy default stream) and
 * performs no host<->device synchronisation.
 *
 * Return value: 0 on success, negative RtgStatus on error; rtg_last_error() holds the message
 * (thread-local).
 */
#ifndef RTG_SPLAT_B200_H
#define RTG_SPLAT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum RtgStatus {
    RTG_OK = 0,
    RTG_ERR_INVALID_ARGUMENT = -1,
    RTG_ERR_CUDA = -2,
    RTG_ERR_UNSUPPORTED = -3,
};

const char *rtg_last_error(void);
int rtg_version(void);

/* Per-view constants: replaces GaussianRasterizationSettings
 * (RAST/diff_gaussian_rasterization_depth/__init__.py:284-303) as marshalled by
 * RasterizeGaussiansCUDA (RAST/rasterize_points.cu:37-64). Matrices stay on the device, exactly as
 * the reference passes them (viewmatrix = W2C transposed, projmatrix = full projection,
 * scene/cameras.py:96-110). */
typedef struct RtgSplatView {
    int32_t image_height, image_width;
    float tanfovx, tanfovy;
    float cx, cy;
    float scale_modifier;
    float color_sigma;
    float opaque_threshold;
    float depth_threshold;
    float normal_threshold; /* cosine */
    float T_threshold;
    int32_t sh_degree;
    int32_t prefiltered; /* flags word: RTG_VIEW_* below; any other bit is rejected (RTG_ERR_INVALID_ARGUMENT) */
    const float *viewmatrix; /* device, 16 floats */
    const float *projmatrix; /* device, 16 floats */
    const float *campos;     /* device, 3 floats  */
    const float *bg;         /* device, 3 floats  */
} RtgSplatView;

/* Bits of RtgSplatView.prefiltered. Every entry point that takes a view honours them.
 *   RTG_VIEW_PREFILTERED  the reference's `prefiltered`: a Gaussian outside the frustum traps (the caller promised there
 *                         is none).
 *   RTG_VIEW_ANTIALIASED  antialiased rendering (the 2-D Mip filter of Mip-Splatting): each splat keeps its 0.3 px^2
 *                         dilation and its opacity o becomes o' = o * comp, comp = sqrt(max(det0 / det, 2.5e-5)), with
 *                         det0 = a0 c0 - b^2 the determinant of the undilated 2-D covariance and det that of the dilated
 *                         one, so that a splat integrates to what it did before the dilation. o' is used everywhere o is
 *                         (alpha, the 1/255 cut-off, opaque depth hits, hit weights, T_map); the conic, radius and tiles are
 *                         the dilated covariance's. The backward returns dL/do = dL/do' comp and takes
 *                         dL/do' o dcomp/dcov2D through the covariance chain (means, scales, rotations, cov3D_precomp,
 *                         camera); the clamp is not differentiated. A backward, tangent or Gauss-Newton call must be given
 *                         the flags of the forward whose state it reads. */
enum { RTG_VIEW_PREFILTERED = 1, RTG_VIEW_ANTIALIASED = 2, RTG_VIEW_FLAGS = 3 };

/* Device counters written by rtg_splat_forward (int32 each). */
enum { RTG_CNT_NUM_RENDERED = 0, RTG_CNT_NUM_TILES = 1, RTG_CNT_OVERFLOW = 2, RTG_CNT_MAX_TILE_LEN = 3,
       RTG_CNT_ENTRIES_NEEDED = 4, /* instances with every tile's bucket padded to 4 entries: what R_cap must hold */
       RTG_CNT_WORDS = 8 };

/* Sizes of the three state buffers kept between forward and backward. Replaces the
 * geomBuffer / imgBuffer / binningBuffer resize callbacks (RAST/rasterize_points.cu:27-35,
 * required<T>() in RAST/cuda_rasterizer/rasterizer_impl.h). `R_cap` is the capacity, in
 * (Gaussian,tile) instances, of the binning buffer: the reference sizes it after a blocking
 * read-back of num_rendered (rasterizer_impl.cu:304); here the caller provides a capacity and
 * the forward raises counters[RTG_CNT_OVERFLOW] (and renders nothing) if it was too small. */
int rtg_splat_workspace_bytes(int32_t P, int32_t H, int32_t W, int64_t R_cap, size_t *geom_bytes, size_t *img_bytes,
                              size_t *bin_bytes);

/* Replaces CudaRasterizer::Rasterizer::forward (RAST/cuda_rasterizer/rasterizer.h:28-66,
 * rasterizer_impl.cu:205-437) together with the output initialisation of
 * RasterizeGaussiansCUDA (rasterize_points.cu:79-87): every element of every output is written.
 * Exactly one of (shs | colors_precomp) and one of (scales+rotations | cov3D_precomp) must be
 * non-NULL, as in GaussianRasterizer.forward (__init__.py:335-347). `M` = SH coefficients per
 * Gaussian. `counters`: device, RTG_CNT_WORDS int32. `counters_host` (may be NULL): pinned, device-mapped
 * host memory that receives a copy of the counters straight from the scan kernel; `scan_done_event` (may be
 * NULL): a cudaEvent_t recorded right after that kernel, so a caller can learn num_rendered / overflow
 * while the rest of the forward is still executing (the reference blocks the whole device instead,
 * rasterizer_impl.cu:304,346). */
int rtg_splat_forward(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                      const float *colors_precomp, const float *opacities, const float *scales, const float *rotations,
                      const float *cov3D_precomp, const int32_t *tile_mask, void *geom_ws, void *img_ws, void *bin_ws,
                      int64_t R_cap, float *out_color, float *out_depth, int32_t *out_hit_color, int32_t *out_hit_depth,
                      float *out_hit_color_weight, float *out_hit_depth_weight, float *out_T, int32_t *radii,
                      int32_t *counters, int32_t *counters_host, void *scan_done_event, void *stream);

/* Replaces CudaRasterizer::Rasterizer::backward (rasterizer.h:68-105, rasterizer_impl.cu:441-560)
 * and the zero-initialisation of RasterizeGaussiansBackwardCUDA (rasterize_points.cu:195-203):
 * every element of every non-NULL gradient output is written. The three state buffers, `R_cap` and
 * `counters` are those of the matching forward call; `final_T` is the forward's out_T,
 * `hit_image` its out_hit_depth (__init__.py:172-235). `grad2d_scratch`: P*16 floats that must be
 * all-zero on entry and are left all-zero on exit. Optional outputs (may be NULL):
 * dL_dcolors_precomp, dL_dcov3D, dL_dmeans2D. Internally the zero-fill of the culled rows runs on a library-owned
 * side stream that forks from and joins back into `stream` within this call (event fork/join, graph-capturable);
 * to the caller all work is ordered on `stream`. */
int rtg_splat_backward(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                       const float *colors_precomp, const float *scales, const float *rotations,
                       const float *cov3D_precomp, const int32_t *radii, const void *geom_ws, const void *img_ws,
                       const void *bin_ws, int64_t R_cap, const int32_t *counters, const float *final_T, const int32_t *hit_image, const float *dL_dcolor,
                       const float *dL_ddepth, float *grad2d_scratch, float *dL_dmeans3D, float *dL_dsh,
                       float *dL_dcolors_precomp, float *dL_dopacity, float *dL_dscales, float *dL_drotations,
                       float *dL_dcov3D, float *dL_dmeans2D, void *stream);

/* rtg_splat_backward without the zero fill: only the gradient rows of Gaussians with radii > 0 are written, the
 * others keep whatever the buffers held. For consumers that take `radii` themselves (rtg_map_adam_step): saves the
 * 105 MB of zero stores per 1 M Gaussians that a dense consumer needs. Same arguments. */
int rtg_splat_backward_visible(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                               const float *colors_precomp, const float *scales, const float *rotations,
                               const float *cov3D_precomp, const int32_t *radii, const void *geom_ws, const void *img_ws,
                               const void *bin_ws, int64_t R_cap, const int32_t *counters, const float *final_T,
                               const int32_t *hit_image, const float *dL_dcolor, const float *dL_ddepth, float *grad2d_scratch,
                               float *dL_dmeans3D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                               float *dL_dscales, float *dL_drotations, float *dL_dcov3D, float *dL_dmeans2D, void *stream);

/* rtg_splat_backward (visible_rows_only == 0) or rtg_splat_backward_visible (!= 0) that also differentiates the camera:
 * the per-Gaussian gradients are those of the extended call, and `dL_dcamera` (device, 35 floats, all written) receives
 * dL/dviewmatrix (16, the storage order of `view->viewmatrix`), dL/dprojmatrix (16) and dL/dcampos (3) -- the plain
 * elementwise derivative of the same loss with respect to the arrays the forward read, for any matrices it accepts.
 * Entries the forward never reads (viewmatrix 3, 7, 11, 15) get 0; intrinsics and the discrete decisions (culling,
 * tile cut-off, alpha < 1/255, opaque hit, plane test) are not differentiated. `camera_scratch`: caller-owned device
 * memory of rtg_splat_camera_scratch_bytes(P) bytes, 8-byte aligned, for the per-block partial sums; the reduction has a
 * fixed order, so identical gradient records give a bit-identical dL_dcamera. Whole-map calls only (no tile-sharded
 * exchange step). */
size_t rtg_splat_camera_scratch_bytes(int32_t P);
int rtg_splat_backward_camera(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                              const float *colors_precomp, const float *scales, const float *rotations,
                              const float *cov3D_precomp, const int32_t *radii, const void *geom_ws, const void *img_ws,
                              const void *bin_ws, int64_t R_cap, const int32_t *counters, const float *final_T,
                              const int32_t *hit_image, const float *dL_dcolor, const float *dL_ddepth, float *grad2d_scratch,
                              float *dL_dmeans3D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                              float *dL_dscales, float *dL_drotations, float *dL_dcov3D, float *dL_dmeans2D,
                              int32_t visible_rows_only, float *dL_dcamera, void *camera_scratch, void *stream);

/* The same backward in two calls with the same argument list, for callers that put an exchange step between the
 * compositing backward and the per-Gaussian backward (tile-sharded multi-GPU rendering, SURVEY.md section 8(e)):
 *   rtg_splat_backward_render : zero-fill of the culled rows + backward of renderCUDA (backward.cu:808-1066); on return
 *                               `grad2d_scratch` holds, per Gaussian, the 16-float record of partial sums
 *                               {colour 3, six moments of opacity*G*dL/dalpha (the 2-D gradients are linear in them),
 *                               depth-path dL/dmean 3, depth-path dL/d(surfel normal) 3, unused 1}
 *                               over the tiles this forward rendered -- sum it across ranks (e.g. ncclAllReduce);
 *   rtg_splat_backward_finish : computeCov2DCUDA + preprocessCUDA backward (backward.cu:273-548) from the records,
 *                               which it clears again. Visibility (radii) does not depend on tile_mask, so ranks
 *                               that render different tiles of one frame agree on which records exist.
 * rtg_splat_backward == rtg_splat_backward_render followed by rtg_splat_backward_finish. */
int rtg_splat_backward_render(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                              const float *colors_precomp, const float *scales, const float *rotations,
                              const float *cov3D_precomp, const int32_t *radii, const void *geom_ws, const void *img_ws,
                              const void *bin_ws, int64_t R_cap, const int32_t *counters, const float *final_T,
                              const int32_t *hit_image, const float *dL_dcolor, const float *dL_ddepth, float *grad2d_scratch,
                              float *dL_dmeans3D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                              float *dL_dscales, float *dL_drotations, float *dL_dcov3D, float *dL_dmeans2D, void *stream);
int rtg_splat_backward_finish(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                              const float *colors_precomp, const float *scales, const float *rotations,
                              const float *cov3D_precomp, const int32_t *radii, const void *geom_ws, const void *img_ws,
                              const void *bin_ws, int64_t R_cap, const int32_t *counters, const float *final_T,
                              const int32_t *hit_image, const float *dL_dcolor, const float *dL_ddepth, float *grad2d_scratch,
                              float *dL_dmeans3D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity,
                              float *dL_dscales, float *dL_drotations, float *dL_dcov3D, float *dL_dmeans2D, void *stream);

/* ---- Gaussian-sharded rendering (SURVEY.md section 8(e); BASELINE configs[4]) ----------------------------------
 * Rank r owns the Gaussians [p_begin, p_end) of the P-Gaussian map (parameters, gradients, optimizer state: arrays of
 * p_end - p_begin rows) and a subset of the 16x16 tiles. The forward of rtg_splat_forward is split around the exchange
 * of the per-Gaussian records, the backward around the exchange of the gradient records:
 *   rtg_splat_forward_preprocess  clears the binning counters and runs preprocessCUDA (forward.cu:238-354) on the owned
 *                                 Gaussians: writes rows [p_begin, p_end) of the geometry workspace (sized for P) and of
 *                                 `radii` (P entries) -- then all-gather those rows across ranks (their byte offsets inside
 *                                 the workspace: rtg_splat_geom_layout; splat 32 B, colour 16 B, surfel 32 B per Gaussian);
 *   rtg_splat_forward_render      tile histogram of ALL P records over the tiles of `tile_mask` (this rank's tiles), scan,
 *                                 scatter, per-tile sort, compositing: outputs as rtg_splat_forward, valid on those tiles.
 *                                 [tile_row_begin, tile_row_end): tile rows outside which tile_mask is all zero (a rank that
 *                                 owns a band of rows passes it so that the binning passes clip every rectangle to the band
 *                                 before expanding it: per-rank work / N instead of constant); 0, 0 = no clipping;
 *   rtg_splat_backward_render_shard   compositing backward over this rank's tiles into `grad2d_scratch` (P records, zero on
 *                                 entry) + zero-fill of the owned gradient rows -- then reduce-scatter the records so that
 *                                 the owner of [p_begin, p_end) holds their sums;
 *   rtg_splat_backward_finish_shard   per-Gaussian backward of the owned Gaussians; here `grad2d_scratch` must be indexable
 *                                 at records [p_begin, p_end) (pass the reduce-scatter output minus p_begin records).
 * In the *_shard calls means3D / shs / ... / dL_d* point to the OWNED rows (row 0 = Gaussian p_begin); radii, the
 * workspaces and the image-sized arrays are global. */
int rtg_splat_geom_layout(int32_t P, size_t *splat_offset, size_t *rgb_offset, size_t *hit_offset, size_t *vis_list_offset);
int rtg_splat_forward_preprocess(const RtgSplatView *view, int32_t P, int32_t p_begin, int32_t p_end, int32_t M, const float *means3D,
                                 const float *shs, const float *colors_precomp, const float *opacities, const float *scales,
                                 const float *rotations, const float *cov3D_precomp, void *geom_ws, void *bin_ws, int64_t R_cap,
                                 int32_t *radii, void *stream);
int rtg_splat_forward_render(const RtgSplatView *view, int32_t P, const int32_t *tile_mask, void *geom_ws, void *img_ws, void *bin_ws,
                             int64_t R_cap, float *out_color, float *out_depth, int32_t *out_hit_color, int32_t *out_hit_depth,
                             float *out_hit_color_weight, float *out_hit_depth_weight, float *out_T, const int32_t *radii,
                             int32_t *counters, int32_t *counters_host, void *scan_done_event, int32_t tile_row_begin,
                             int32_t tile_row_end, void *stream);
int rtg_splat_backward_render_shard(int32_t p_begin, int32_t p_end, const RtgSplatView *view, int32_t P, int32_t M,
                                    const float *means3D, const float *shs, const float *colors_precomp, const float *scales,
                                    const float *rotations, const float *cov3D_precomp, const int32_t *radii, const void *geom_ws,
                                    const void *img_ws, const void *bin_ws, int64_t R_cap, const int32_t *counters,
                                    const float *final_T, const int32_t *hit_image, const float *dL_dcolor, const float *dL_ddepth,
                                    float *grad2d_scratch, float *dL_dmeans3D, float *dL_dsh, float *dL_dcolors_precomp,
                                    float *dL_dopacity, float *dL_dscales, float *dL_drotations, float *dL_dcov3D,
                                    float *dL_dmeans2D, void *stream);
int rtg_splat_backward_finish_shard(int32_t p_begin, int32_t p_end, const RtgSplatView *view, int32_t P, int32_t M,
                                    const float *means3D, const float *shs, const float *colors_precomp, const float *scales,
                                    const float *rotations, const float *cov3D_precomp, const int32_t *radii, const void *geom_ws,
                                    const void *img_ws, const void *bin_ws, int64_t R_cap, const int32_t *counters,
                                    const float *final_T, const int32_t *hit_image, const float *dL_dcolor, const float *dL_ddepth,
                                    float *grad2d_scratch, float *dL_dmeans3D, float *dL_dsh, float *dL_dcolors_precomp,
                                    float *dL_dopacity, float *dL_dscales, float *dL_drotations, float *dL_dcov3D,
                                    float *dL_dmeans2D, void *stream);

/* ---- gradient of the transmittance map ------------------------------------------------------------------------
 * `dL_dT`: device, (H, W) fp32 laid out like dL_ddepth, 4-byte aligned: dL/dT_map of the forward's out_T. T_map is the
 * product of (1 - alpha) over the (pixel, Gaussian) pairs that added colour, and it is differentiated through every one
 * of them (dT_map/dalpha = -T_map / (1 - alpha)), exactly as the background term. Not differentiated, as for colour: the
 * min(0.99, .) clamp of alpha and the discrete decisions (alpha < 1/255, T_threshold termination, opaque hit, tile
 * cut-off, culling). hit_color_weight / hit_depth_weight stay non-differentiable: their gradient is dropped. dL_dT NULL
 * runs exactly the call without it.
 *   rtg_splat_backward_dt         rtg_splat_backward_camera's arguments with dL_dT after dL_ddepth; dL_dcamera may be NULL
 *                                 (no camera gradient; camera_scratch is then ignored). visible_rows_only as there.
 *   rtg_splat_backward_render_dt  the compositing half (rtg_splat_backward_render for 0, P; rtg_splat_backward_render_shard
 *                                 for an owned range) with dL_dT; the records carry the term, so the finish calls are
 *                                 the existing ones.
 * Both validate their arguments on the host before any CUDA work. */
int rtg_splat_backward_dt(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                          const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                          const int32_t *radii, const void *geom_ws, const void *img_ws, const void *bin_ws, int64_t R_cap,
                          const int32_t *counters, const float *final_T, const int32_t *hit_image, const float *dL_dcolor,
                          const float *dL_ddepth, const float *dL_dT, float *grad2d_scratch, float *dL_dmeans3D, float *dL_dsh,
                          float *dL_dcolors_precomp, float *dL_dopacity, float *dL_dscales, float *dL_drotations,
                          float *dL_dcov3D, float *dL_dmeans2D, int32_t visible_rows_only, float *dL_dcamera,
                          void *camera_scratch, void *stream);
int rtg_splat_backward_render_dt(int32_t p_begin, int32_t p_end, const RtgSplatView *view, int32_t P, int32_t M,
                                 const float *means3D, const float *shs, const float *colors_precomp, const float *scales,
                                 const float *rotations, const float *cov3D_precomp, const int32_t *radii, const void *geom_ws,
                                 const void *img_ws, const void *bin_ws, int64_t R_cap, const int32_t *counters,
                                 const float *final_T, const int32_t *hit_image, const float *dL_dcolor, const float *dL_ddepth,
                                 const float *dL_dT, float *grad2d_scratch, float *dL_dmeans3D, float *dL_dsh,
                                 float *dL_dcolors_precomp, float *dL_dopacity, float *dL_dscales, float *dL_drotations,
                                 float *dL_dcov3D, float *dL_dmeans2D, void *stream);

/* ---- pose refinement against a frozen map (no reference counterpart) -----------------------------------------------
 * rtg_splat_backward_pose: rtg_splat_backward_dt's camera gradient without any per-Gaussian gradient, for a loss in which
 * only the camera is optimised. Same arguments minus the eight per-Gaussian outputs and visible_rows_only; dL_dT may be
 * NULL; dL_dcamera (35 floats, all written) and camera_scratch as in rtg_splat_backward_camera, both required. The
 * compositing backward is the same; the per-Gaussian pass computes only the camera terms, stores nothing per Gaussian
 * and needs no zero fill. `grad2d_scratch` is all-zero on entry and left all-zero, as in every backward. Identical
 * gradient records give a bit-identical dL_dcamera (fixed-order reduction). Validates on the host before any CUDA work. */
int rtg_splat_backward_pose(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                            const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                            const int32_t *radii, const void *geom_ws, const void *img_ws, const void *bin_ws, int64_t R_cap,
                            const int32_t *counters, const float *final_T, const int32_t *hit_image, const float *dL_dcolor,
                            const float *dL_ddepth, const float *dL_dT, float *grad2d_scratch, float *dL_dcamera,
                            void *camera_scratch, void *stream);

/* rtg_pose_adam_step: one Adam step of a camera pose on the device, from the camera gradients of the last backward. The
 * pose is W2C (world to camera, row-major 4x4, double, kept on the device so that hundreds of steps do not drift it off
 * SE(3)); the rasterizer reads viewmatrix = W2C^T, projmatrix = viewmatrix @ projection (`projection`: the camera's
 * projection_matrix as stored, 16 floats) and campos = -R^T t. The step
 *   1. collects G = dL/dW2C through those three arrays and the gradient of the left twist xi = (rho, phi) at zero,
 *      W2C(xi) = exp(xi^) W2C: with A = G W2C^T, dL/drho_k = A[k][3], dL/dphi = (A21 - A12, A02 - A20, A10 - A01);
 *   2. takes one bias-corrected Adam step on that 6-vector from xi = 0 (torch.optim.Adam's update: lr_trans for rho,
 *      lr_rot for phi, `step` >= 1 counted by the caller as in rtg_adam_step), moments exp_avg / exp_avg_sq (6 floats
 *      each, rho then phi) carried across calls;
 *   3. applies W2C <- exp(xi^) W2C with the closed-form SE(3) exponential, resets xi to zero, and rewrites viewmatrix,
 *      projmatrix and campos in place from the double pose.
 * A NULL gradient pointer counts as zero. One single-block launch; validates on the host before any CUDA work. */
typedef struct RtgPoseAdam {
    double *pose;                                                  /* 16, W2C row-major, updated in place */
    float *exp_avg, *exp_avg_sq;                                   /* 6 each */
    const float *dL_dviewmatrix, *dL_dprojmatrix, *dL_dcampos;     /* 16, 16, 3 (rtg_splat_backward_camera's layout) */
    const float *projection;                                       /* 16 */
    float *viewmatrix, *projmatrix, *campos;                       /* 16, 16, 3: written */
    float lr_trans, lr_rot;
    float beta1, beta2, eps;
    int32_t step;
} RtgPoseAdam;
int rtg_pose_adam_step(const RtgPoseAdam *s, void *stream);

/* ---- Gauss-Newton pose step (forward-mode tangents of the render) ---------------------------------------------------
 * Pose and twist as in rtg_pose_adam_step: W2C(xi) = exp(xi^) W2C with xi = (rho, phi); under it a view-space point moves
 * as rho + phi x p_c, a view-space direction as phi x n, the view rotation as [phi]x W and campos as -W^T rho. The
 * tangents are those of the render the forward (the workspaces and counters of one rtg_splat_forward) produced; the
 * discrete decisions (cull, tile and patch cut-offs, 1/255, opaque hit, plane test, T_threshold), the 1.3*tanfov clamp
 * of the EWA Jacobian, clamped SH channels and the intrinsics are not differentiated, as in the reverse-mode gradients.
 *
 * rtg_splat_pose_gn_scratch_bytes: device scratch of both entry points (per-Gaussian tangent rows, per-tile partial sums;
 * 16-byte aligned). */
size_t rtg_splat_pose_gn_scratch_bytes(int32_t P, int32_t H, int32_t W);

/* rtg_splat_pose_tangents: J (6, 4, H, W) fp32, every element written: J[k] = (dC_r, dC_g, dC_b, dD) / dxi_k of the
 * forward's colour and depth. A pixel without a depth hit, or in a never-rendered or masked-out tile, has depth tangent 0
 * (and, in such a tile, colour tangent 0). Gaussian inputs as in rtg_splat_backward_pose; hit_image = the forward's
 * hit_depth. Validates on the host before any CUDA work. */
int rtg_splat_pose_tangents(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                            const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                            const void *geom_ws, const void *img_ws, const void *bin_ws, int64_t R_cap, const int32_t *counters,
                            const int32_t *hit_image, void *scratch, float *J, void *stream);

/* rtg_splat_pose_gn_step: one damped Gauss-Newton step of the pose on the device. With the pixel sets of rtg_loss_l1 (S_c:
 * the render_mask pixels, or all; S_d: hit_depth != -1, gt_depth > 0, depth - gt_depth < depth_error_max (signed), in the
 * mask), N_c = 3 |S_c|, N_d = |S_d|, the objective is
 *   E = 1/2 [ color_weight / N_c sum_{S_c} sum_ch (C - C^)^2 + depth_weight / N_d sum_{S_d} (D - D^)^2 ]
 * (an empty set contributes 0). H = sum w J^T J and g = sum w J^T r are formed in double with a fixed summation order
 * (identical inputs give bit-identical sums), damped as the ICP step, H + damping * trace(H) * I, solved xi = -H^-1 g and
 * applied as W2C <- exp(xi^) W2C in double; viewmatrix, projmatrix and campos are rewritten in place. A singular system,
 * N_c + N_d = 0 or an overflowed forward leaves the pose and the arrays unchanged. `report` (RTG_POSE_GN_REPORT doubles,
 * device) receives E before the step, its colour and depth parts, N_c, N_d, |rho|, |phi| and the status. Nothing is read
 * back to the host. Validates on the host before any CUDA work. */
#define RTG_POSE_GN_REPORT_LEN 8
enum { RTG_POSE_GN_OK = 0, RTG_POSE_GN_SINGULAR = 1, RTG_POSE_GN_EMPTY = 2, RTG_POSE_GN_OVERFLOW = 3 };
typedef struct RtgPoseGN {
    double *pose;                                       /* 16, W2C row-major, updated in place */
    const float *projection;                            /* 16 */
    float *viewmatrix, *projmatrix, *campos;            /* 16, 16, 3: rewritten from the pose */
    const float *render, *depth;                        /* (3, H, W), (H, W): the forward's colour and depth */
    const int32_t *hit_depth;                           /* (H, W): the forward's depth hit map */
    const float *gt_color, *gt_depth;                   /* (3, H, W) or (H, W, 3) (gt_channels_last), (H, W) */
    const uint8_t *render_mask;                         /* (H, W) or NULL */
    void *scratch;                                      /* rtg_splat_pose_gn_scratch_bytes(P, H, W) */
    double *report;                                     /* RTG_POSE_GN_REPORT_LEN */
    float color_weight, depth_weight, depth_error_max, damping;
    int32_t gt_channels_last, _pad;
} RtgPoseGN;
int rtg_splat_pose_gn_step(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                           const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                           const void *geom_ws, const void *img_ws, const void *bin_ws, int64_t R_cap, const int32_t *counters,
                           const RtgPoseGN *s, void *stream);

/* rtg_splat_pose_gn_step_robust: rtg_splat_pose_gn_step with a robust loss on each residual r (a colour channel, or the
 * depth). With rho(r) = r^2 / 2 for |r| <= delta and delta |r| - delta^2 / 2 otherwise (Huber), the objective is
 *   E = color_weight / N_c sum_{S_c} sum_ch rho_cd(C - C^) + depth_weight / N_d sum_{S_d} rho_dd(D - D^)
 * over the same pixel sets and counts. It is minimised by iteratively reweighted least squares: each residual gets the
 * weight w = 1 (|r| <= delta) or delta / |r|, computed in float from the float residual, H = sum w J^T J and g = sum w J^T r
 * (g is the gradient of E); the damping, the solve, the update, the camera arrays and the report are those of
 * rtg_splat_pose_gn_step, with the report's E, E_colour and E_depth the robust ones. RTG_ROBUST_NONE launches exactly what
 * rtg_splat_pose_gn_step launches. Rejects a NULL `robust`, an unknown kernel and, for RTG_ROBUST_HUBER, a delta that is
 * not positive and finite, on the host before any CUDA work (and validates the rest as rtg_splat_pose_gn_step). */
enum { RTG_ROBUST_NONE = 0, RTG_ROBUST_HUBER = 1 };
typedef struct RtgPoseRobust {
    int32_t kernel;                                     /* RTG_ROBUST_NONE or RTG_ROBUST_HUBER */
    float color_delta, depth_delta;                     /* Huber thresholds: colour units, map units */
    int32_t _pad;
} RtgPoseRobust;
int rtg_splat_pose_gn_step_robust(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                                  const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                                  const void *geom_ws, const void *img_ws, const void *bin_ws, int64_t R_cap, const int32_t *counters,
                                  const RtgPoseGN *s, const RtgPoseRobust *robust, void *stream);

/* rtg_splat_pose_gn_step_exposure: the step of rtg_splat_pose_gn_step_robust with the frame's exposure estimated with the
 * pose. The camera's pixel values are modelled as C^ = e^a C + b (one gain and one offset per frame, shared by the three
 * channels; (0, 0) = none), the colour residual of a selected pixel and channel is r = e^a C + b - C^, and with the
 * unknowns x = (rho, phi, a, b) its Jacobian row is (e^a dC/dxi, e^a C, 1). Depth residuals, the pixel sets, the counts,
 * the weights and the Huber rule are those of rtg_splat_pose_gn_step[_robust], applied to the new r:
 *   E = 1/2 [ color_weight / N_c sum_{S_c} sum_ch r^2 + depth_weight / N_d sum_{S_d} (D - D^)^2 ]    (RTG_ROBUST_NONE)
 *   E = color_weight / N_c sum_{S_c} sum_ch rho_cd(r) + depth_weight / N_d sum_{S_d} rho_dd(D - D^)     (RTG_ROBUST_HUBER)
 * H (8x8, the depth block in its leading 6x6) and g are summed in double in a fixed order (identical inputs give
 * bit-identical sums). Damping: the six pose diagonals get damping * trace(H[0:6, 0:6]), as rtg_splat_pose_gn_step's, so
 * that the pose step with the exposure columns removed is that entry's; the exposure diagonals are scaled, H_aa (1 +
 * damping) and H_bb (1 + damping): the pose trace is of order (focal length * image gradient)^2 while H_bb =
 * color_weight, so adding it there would freeze the exposure. x = -H^-1 g; W2C <- exp(xi^) W2C, a += x_6, b += x_7 in
 * double in `exposure->ab`, and the camera arrays are rewritten. `report` as rtg_splat_pose_gn_step's, E the objective
 * with the exposure before the step.
 * Degenerate cases: with N_c = 0 or color_weight = 0 the exposure columns are empty; the 6x6 pose system is solved alone,
 * (a, b) is left unchanged and the status stays RTG_POSE_GN_OK. A singular system, N_c + N_d = 0 or an overflowed forward
 * leaves the pose, the arrays and (a, b) unchanged.
 * `s->scratch` holds rtg_splat_pose_gn_exposure_scratch_bytes(P, H, W) bytes (the tangent rows and RTG_GN_EXP_ALL = 75
 * doubles per tile); rtg_splat_pose_gn_scratch_bytes keeps its value. `robust->kernel` may be RTG_ROBUST_NONE. Rejects a
 * NULL `exposure`, a NULL or misaligned `ab` and everything rtg_splat_pose_gn_step_robust rejects, on the host before any
 * CUDA work. */
typedef struct RtgPoseExposure {
    double *ab;                                         /* 2 doubles on the device: (a, b), updated in place by the step */
} RtgPoseExposure;
size_t rtg_splat_pose_gn_exposure_scratch_bytes(int32_t P, int32_t H, int32_t W);
int rtg_splat_pose_gn_step_exposure(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                                    const float *colors_precomp, const float *scales, const float *rotations,
                                    const float *cov3D_precomp, const void *geom_ws, const void *img_ws, const void *bin_ws,
                                    int64_t R_cap, const int32_t *counters, const RtgPoseGN *s, const RtgPoseRobust *robust,
                                    const RtgPoseExposure *exposure, void *stream);

/* Expected depth. With the pairs the forward blends (positions < n_contrib of the tile list, alpha past 1/255, the
 * forward's own decisions), w_i = alpha_i T_i and z_i the view-space z of Gaussian i's centre, per pixel
 *   m1 = sum w_i (coverage),  m0 = sum w_i z_i,  D = m0 / m1 (0 where m1 = 0),
 * the map rtg_splat_features composites for F = (z_view, 1), summed in the same order. Its tangents, with dz_i/dxi =
 * (0, 0, 1, p_y, -p_x, 0): dm1 = sum dw_i, dm0 = sum (dw_i z_i + w_i dz_i), dD = (dm0 - D dm1) / m1.
 *
 * rtg_splat_pose_tangents_expected: rtg_splat_pose_tangents with dD/dxi_k in channel 3 of J (0 where m1 = 0), and
 * `expected` (2, H, W) fp32 = (D, m1), both written everywhere (0 in a never-rendered or masked-out tile). It takes no
 * hit map. `scratch` holds rtg_splat_pose_gn_scratch_bytes(P, H, W) bytes. Validates on the host before any CUDA work. */
int rtg_splat_pose_tangents_expected(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                                     const float *colors_precomp, const float *scales, const float *rotations,
                                     const float *cov3D_precomp, const void *geom_ws, const void *img_ws, const void *bin_ws,
                                     int64_t R_cap, const int32_t *counters, void *scratch, float *J, float *expected,
                                     void *stream);

/* rtg_splat_pose_gn_step_expected: the step of rtg_splat_pose_gn_step[_robust|_exposure] with the expected depth in place
 * of the hit depth. The depth residual is D - D^ over S_e: in the render mask, m1 >= min_coverage, gt_depth > 0 and
 * D - gt_depth < depth_error_max (signed); N_d = |S_e|. The colour rows, the weights, the Huber rule, the objective, the
 * damping, the solve, the update and the report are those of the entry point the arguments select: `robust->kernel`
 * RTG_ROBUST_NONE or RTG_ROBUST_HUBER, and `exposure` NULL (six unknowns, scratch rtg_splat_pose_gn_scratch_bytes) or
 * the device exposure (eight unknowns, scratch rtg_splat_pose_gn_exposure_scratch_bytes). `s->depth` and `s->hit_depth`
 * are validated as there but not read. Rejects min_coverage outside (0, 1], a NULL `robust`, a NULL or misaligned
 * `exposure->ab` and everything rtg_splat_pose_gn_step_robust rejects, on the host before any CUDA work. */
int rtg_splat_pose_gn_step_expected(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                                    const float *colors_precomp, const float *scales, const float *rotations,
                                    const float *cov3D_precomp, const void *geom_ws, const void *img_ws, const void *bin_ws,
                                    int64_t R_cap, const int32_t *counters, const RtgPoseGN *s, const RtgPoseRobust *robust,
                                    const RtgPoseExposure *exposure, float min_coverage, void *stream);

/* ---- per-Gaussian contributions to a frame (no reference counterpart) ----------------------------------------------
 * rtg_splat_contributions: what each Gaussian added to the render of one rtg_splat_forward (its view, workspaces, R_cap
 * and counters; the view's flags must be the forward's). The pairs (p, g) that add colour are those the forward blends and
 * the backward replays: p a pixel of a rendered tile, g at a position < n_contrib(p) of p's tile list, alpha past the
 * 1/255 cut-off (the forward's decision, its recheck band included). Such a pair has the weight w(p, g) = alpha T, T the
 * transmittance in front of g at p (the forward's colour weight). Per Gaussian g the call ADDS
 *   n_pixels[g] += #{p : (p, g) adds colour}               (int32, at most H*W per call: exact),
 *   weight[g]   += sum_p w(p, g),
 *   error[g]    += sum_p w(p, g) pixel_error(p)           (only when pixel_error, (H, W) fp32 device, is given),
 * so repeated calls sum over several frames. Culled Gaussians, masked-out and empty tiles and an overflowed forward
 * (counters[RTG_CNT_OVERFLOW] != 0) add nothing. Summed over g, weight is sum_p (1 - T_map(p)) over the rendered pixels;
 * error is the colour intermediate of rtg_splat_backward under dL/dcolor = (pixel_error, 0, 0). The float sums are
 * accumulated with atomics in a varying order (not bit-reproducible); the counts are. No Gaussian parameter array is read.
 * n_pixels, weight, error: P rows, device, 4-byte aligned; n_pixels and weight are required when P > 0; error and
 * pixel_error are both NULL or both given. Validates on the host before any CUDA work; P == 0 does no work. */
int rtg_splat_contributions(const RtgSplatView *view, int32_t P, const void *geom_ws, const void *img_ws, const void *bin_ws,
                            int64_t R_cap, const int32_t *counters, const float *pixel_error, int32_t *n_pixels, float *weight,
                            float *error, void *stream);

/* ---- per-Gaussian feature maps (no reference counterpart) ---------------------------------------------------------
 * rtg_splat_features: a C-channel image of per-Gaussian features composited with the blend weights of one
 * rtg_splat_forward (its view, workspaces, R_cap and counters; the view's flags must be the forward's). With w(p, g) =
 * alpha T, the forward's colour weight of the pairs it blends (as in rtg_splat_contributions),
 *   out[c, p] = sum_g w(p, g) features[g, c]        features (P, C) row-major, out (C, H, W), both fp32 device.
 * Every pixel of out is written: 0 on masked-out and empty tiles and everywhere when the forward overflowed
 * (counters[RTG_CNT_OVERFLOW] != 0). There is no background term (T_map is the remainder). With features = the forward's
 * colours this is its colour image without the background; with features = 1 it is 1 - T_map.
 * rtg_splat_features_backward: the transpose with the weights held fixed,
 *   dL_dfeatures[g, c] = sum_p w(p, g) dL_dout[c, p]   dL_dout (C, H, W), dL_dfeatures (P, C), overwritten.
 * Rows the frame never blends (culled Gaussians among them) are 0, and so is every row after an overflowed forward. The
 * sums are accumulated with atomics in a varying order (not bit-reproducible); the forward map is. No Gaussian parameter
 * array is read. 1 <= C <= RTG_FEATURES_MAX. Both validate on the host before any CUDA work; with P == 0 the forward only
 * zeroes out and the backward does nothing. */
enum { RTG_FEATURES_MAX = 128 };
int rtg_splat_features(const RtgSplatView *view, int32_t P, const void *geom_ws, const void *img_ws, const void *bin_ws,
                       int64_t R_cap, const int32_t *counters, int32_t C, const float *features, float *out, void *stream);
int rtg_splat_features_backward(const RtgSplatView *view, int32_t P, const void *geom_ws, const void *img_ws,
                                const void *bin_ws, int64_t R_cap, const int32_t *counters, int32_t C, const float *dL_dout,
                                float *dL_dfeatures, void *stream);
/* rtg_splat_features_backward_geometry: the other half of the feature map's gradient, through its blend weights. With
 * h_i = sum_c dL_dout[c, p] features[i, c] and S_i = sum_{j > i} w_j h_j over the pixel's blended entries,
 *   dL/dalpha_i = T_i h_i - S_i / (1 - alpha_i),
 * taken through alpha to the same per-Gaussian gradients rtg_splat_backward gives (its colour backward with colours_precomp
 * = features, bg = 0 and dL_ddepth = 0, summed over channel triples): dL_dmeans3D (P,3), dL_dopacity (P,1), and
 * dL_dscales (P,3) + dL_drotations (P,4, 16-byte aligned) or dL_dcov3D (P,6), overwritten (culled rows 0, or unwritten
 * with visible_rows_only != 0; radii is needed otherwise); with dL_dcamera (35 floats: view 16, proj 16, campos 3) and
 * camera_scratch (rtg_splat_camera_scratch_bytes(P), 8-byte aligned) also the camera gradient, as
 * rtg_splat_backward_camera. With every per-Gaussian output NULL and dL_dcamera given only the camera gradient is
 * computed (rtg_splat_backward_pose's per-Gaussian half). means3D, scales / rotations or cov3D_precomp: the forward's
 * inputs (no SH row and no opacity is read: opacities come from the forward's records). grad2d_scratch: P * 16 floats,
 * zero on entry and on exit, as for every backward. dL/dfeatures comes from rtg_splat_features_backward. An overflowed
 * forward gives zero gradients; P == 0 writes only dL_dcamera (zeros). Validates on the host before any CUDA work. */
int rtg_splat_features_backward_geometry(const RtgSplatView *view, int32_t P, const float *means3D, const float *scales,
                                         const float *rotations, const float *cov3D_precomp, const int32_t *radii,
                                         const void *geom_ws, const void *img_ws, const void *bin_ws, int64_t R_cap,
                                         const int32_t *counters, int32_t C, const float *features, const float *dL_dout,
                                         float *grad2d_scratch, float *dL_dmeans3D, float *dL_dopacity, float *dL_dscales,
                                         float *dL_drotations, float *dL_dcov3D, int32_t visible_rows_only, float *dL_dcamera,
                                         void *camera_scratch, void *stream);

/* Replaces CudaRasterizer::Rasterizer::markVisible (rasterizer.h:21-26, rasterizer_impl.cu:145-157). */
int rtg_splat_mark_visible(int32_t P, const float *means3D, const float *viewmatrix, const float *projmatrix,
                           uint8_t *present, void *stream);

/* ---- optimizer step ------------------------------------------------------------------------
 * Replaces torch.optim.Adam(l, lr=0.0, eps=1e-15).step() over the parameter groups built by
 * GaussianPointCloud.parametrize (SLAM/gaussian_pointcloud.py:245-284; SLAM/multiprocess/
 * mapper.py:156,452): one launch for all groups, bias-corrected Adam, no weight decay, no amsgrad. */
#define RTG_ADAM_MAX_GROUPS 8
typedef struct RtgAdamGroup {
    float *param;
    const float *grad;
    float *exp_avg;
    float *exp_avg_sq;
    int64_t numel;
    float lr;
    float _pad;
} RtgAdamGroup;
int rtg_adam_step(const RtgAdamGroup *groups, int32_t n_groups, float beta1, float beta2, float eps, int32_t step,
                  void *stream);

/* ---- fused map-parameter step ---------------------------------------------------------------
 * One pass over the Gaussian map that replaces, per optimisation iteration of Mapping.loss_update
 * (SLAM/multiprocess/mapper.py:376-468):
 *   - the activation backward of get_scaling / get_rotation / get_opacity (torch.exp, F.normalize, torch.sigmoid;
 *     SLAM/gaussian_pointcloud.py:16-25,511-523,574-581) and the slice backward of get_features' torch.cat,
 *   - the gradient of the "attach" regulariser 1000 * (l2(_scaling) + l2(_xyz) + l2(_rotation)) on the rows with
 *     attach_mask (mapper.py:384-401; l2_loss = mean of squares, utils/loss_utils.py:34-36),
 *   - torch.optim.Adam(l, lr=0.0, eps=1e-15).step() over the six groups of parametrize (gaussian_pointcloud.py:245-284),
 *   - `_confidence[(f_dc.grad.abs() != 0).any(-1)] += 1` (mapper.py:455-456),
 *   - the activation forward (and get_normal, gaussian_pointcloud.py:539-550) for the next iteration's render.
 * Gradients are the rasterizer's, i.e. with respect to the ACTIVATED tensors. With `radii` (the forward's output)
 * rows with radii <= 0 are treated as zero gradient and never read, so the backward may be
 * rtg_splat_backward_visible, which skips the zero fill of those rows. `sh` is ONE (P,16,3) block whose [:,0:1] /
 * [:,1:] slices are _features_dc / _features_rest (no torch.cat). All pointers device memory; optional ones may be
 * NULL: radii, attach_mask (+ xyz0, scaling0, rotation0), confidence, normal_out. */
typedef struct RtgMapStep {
    int32_t P;
    int32_t step;                 /* Adam step number, >= 1 */
    float *xyz, *sh, *opacity_raw, *scaling_raw, *rotation_raw;                 /* raw parameters, updated in place */
    float *m_xyz, *m_sh, *m_opacity, *m_scaling, *m_rotation;                   /* exp_avg */
    float *v_xyz, *v_sh, *v_opacity, *v_scaling, *v_rotation;                   /* exp_avg_sq */
    const float *g_means3D, *g_sh, *g_opacity, *g_scales, *g_rotations;         /* rasterizer gradients */
    const int32_t *radii;
    const uint8_t *attach_mask;
    const float *xyz0, *scaling0, *rotation0;                                   /* init_stat: _xyz, _scaling, _rotation (raw) */
    float attach_weight;          /* 1000 in the reference */
    int32_t attach_count;         /* number of rows with attach_mask (the means' denominators) */
    float lr_xyz, lr_f_dc, lr_f_rest, lr_opacity, lr_scaling, lr_rotation;
    float beta1, beta2, eps;
    float *scales_out, *rotations_out, *opacities_out;                          /* activated values after the update */
    float *normal_out;            /* (P,3) get_normal after the update */
    float *confidence;            /* (P) float */
} RtgMapStep;
int rtg_map_adam_step(const RtgMapStep *step, void *stream);
/* Activation forward only (initialisation): scales_out = exp(scaling_raw), rotations_out = normalize(rotation_raw),
 * opacities_out = sigmoid(opacity_raw), normal_out = get_normal (may be NULL). */
int rtg_map_activate(int32_t P, const float *scaling_raw, const float *rotation_raw, const float *opacity_raw,
                     float *scales_out, float *rotations_out, float *opacities_out, float *normal_out, void *stream);

/* Mapping.history_merge (SLAM/multiprocess/mapper.py:212-250) with slerp of SLAM/utils.py:593-652: after an optimisation
 * call, pull the raw parameters back towards their pre-optimisation values (`history_stat`, mapper.py:146-155):
 *   w = max_weight * hist_confidence / (confidence + 1e-6)                                  per Gaussian,
 *   _xyz          <- hist_xyz * w + (1 - w) * _xyz,
 *   _features_dc, _features_rest, _scaling  <- hist * w[0] + (1 - w[0]) * current    (the reference indexes
 *                    `history_weight[0]`: the FIRST Gaussian's weight for every row -- kept),
 *   _rotation     <- slerp(hist_rotation, normalize(_rotation), 1 - w)   (linear where |dot| > 0.9995 or NaN).
 * One launch instead of ~45 eager kernels; all updates in place. hist_rotation is get_rotation before the optimisation
 * (normalised); rotation_raw is `_rotation` (16-byte aligned). features_dc / features_rest rows start every
 * `*_stride` floats (3 / 45 for separate contiguous tensors, 48 for the two slices of one (P,16,3) block);
 * hist arrays are contiguous. max_weight <= 0 or P == 0: nothing is done (mapper.py:213-214). */
typedef struct RtgHistoryMerge {
    int32_t P;
    float max_weight;             /* history_merge_max_weight, configs/base.yaml:54 */
    const float *hist_confidence, *confidence;          /* (P) */
    const float *hist_xyz;      float *xyz;             /* (P,3) */
    const float *hist_features_dc;   float *features_dc;    /* rows of 3 */
    const float *hist_features_rest; float *features_rest;  /* rows of features_rest_width (45 for SH degree 3) */
    const float *hist_scaling;  float *scaling;         /* (P,3) */
    const float *hist_rotation; float *rotation_raw;    /* (P,4) */
    int32_t features_dc_stride, features_rest_stride, features_rest_width;
    int32_t _pad;
} RtgHistoryMerge;
int rtg_map_history_merge(const RtgHistoryMerge *merge, void *stream);

/* ---- projective point-to-plane ICP ---------------------------------------------------------
 * Pyramid level: replaces nn.MaxPool2d(pool) (SLAM/icp.py:343-345,374) + compute_vertex_map
 * (SLAM/utils.py:65-75) + compute_normal_map (SLAM/utils.py:100-122). `depth`: (H,W) full
 * resolution; outputs (H/pool, W/pool, 3) channels-last. fx..cy are the level intrinsics
 * (K*downscale, SLAM/utils.py:517-519). `ws`: rtg_icp_workspace_bytes() bytes. */
size_t rtg_icp_workspace_bytes(int32_t H, int32_t W);
int rtg_icp_build_level(const float *depth, int32_t H, int32_t W, int32_t pool, float fx, float fy, float cx, float cy,
                        float *vertex_out, float *normal_out, void *ws, void *stream);

/* `iters` Gauss-Newton iterations on one level: replaces the loop of ICP.icp (SLAM/icp.py:33-48):
 * compute_residuals_jacobian (:52-104), compute_jtj/jtr (:107-119), lev_mar_H (:248),
 * least_square_solve/invH (:313-333), exp_se3 (:271), forward_update_pose (:259). "0" is the
 * current frame, "1" the previous/model frame, as inside icp(). `pose`: device, 16 floats
 * row-major, updated in place. `valid_ratio`: device float (may be NULL). */
int rtg_icp_solve_level(const float *vertex0, const float *normal0, const float *vertex1, const float *normal1,
                        int32_t H, int32_t W, float fx, float fy, float cx, float cy, float distance_threshold,
                        float normal_cos_threshold, float damping, int32_t iters, float *pose, float *valid_ratio,
                        void *ws, void *stream);

/* point2plane_loss(p_t0, p_t1 @ R^T + t, n_t0, "mean") (SLAM/icp.py:7-13,444-447); `loss`: device float. */
int rtg_icp_point2plane_loss(const float *vertex_t0, const float *vertex_t1, const float *normal_t0, int32_t H, int32_t W,
                             const float *pose, float *loss, void *ws, void *stream);

/* IcpTracker.update_last_status depth filling (SLAM/icp.py:397-415): in place on render_depth. */
int rtg_icp_fill_model_depth(float *render_depth, const float *frame_depth, const float *render_normal,
                             const float *frame_normal, int32_t H, int32_t W, float distance_threshold,
                             float normal_threshold, void *stream);

/* Whole pyramid in one launch: build_vertex_pyramid + build_normal_pyramid (SLAM/utils.py:511-527) as IcpTracker.
 * update_curr_status / predict_pose call them (SLAM/icp.py:385-395,423-425). Level l max-pools `depth` (H,W) by pools[l]
 * and back-projects with the level intrinsics {fx,fy,cx,cy}[l] (K*downscale, SLAM/utils.py:517-519); vertex_out[l] /
 * normal_out[l] are device (H/pools[l], W/pools[l], 3) buffers. 1 <= n_levels <= 4. One cooperative launch (max-pool +
 * vertices of all levels, grid barrier for the per-level depth extremes, normals). */
int rtg_icp_build_pyramid(const float *depth, int32_t H, int32_t W, int32_t n_levels, const int32_t *pools, const float *fx,
                          const float *fy, const float *cx, const float *cy, float *const *vertex_out, float *const *normal_out,
                          void *ws, void *stream);

/* IcpTracker.predict_pose (SLAM/icp.py:417-452) in one cooperative launch: for every level (coarse to fine) `iters`
 * Gauss-Newton iterations as in rtg_icp_solve_level, the pose carried from level to level starting at pose_init (device,
 * 16 floats; NULL = identity), then point2plane_loss of the final pose on (p2p_vertex_t0, p2p_vertex_t1, p2p_normal_t0),
 * each (p2p_H, p2p_W, 3). In every level "0" is the CURRENT frame and "1" the previous / model frame (the argument swap of
 * SLAM/icp.py:438-441). out: 18 device floats = pose (row-major 4x4), loss, valid ratio of the last iteration; out_host
 * (may be NULL): the same 18 floats written straight into mapped pinned host memory by the kernel, valid once work
 * enqueued after this call on `stream` has been reached (record an event and wait for it) -- the only read-back of a
 * predict_pose. */
typedef struct RtgIcpLevel {
    const float *vertex0, *normal0, *vertex1, *normal1; /* (H,W,3) channels-last, device */
    int32_t H, W;
    float fx, fy, cx, cy;
    int32_t iters;
    int32_t _pad;
} RtgIcpLevel;
int rtg_icp_predict_pose(const RtgIcpLevel *levels, int32_t n_levels, float distance_threshold, float normal_cos_threshold,
                         float damping, const float *pose_init, const float *p2p_vertex_t0, const float *p2p_vertex_t1,
                         const float *p2p_normal_t0, int32_t p2p_H, int32_t p2p_W, float *out, float *out_host, void *ws,
                         void *stream);

/* Intensity pyramid of the photometric ICP term, all levels in one launch. `color`: device float32, (H,W,3) if
 * channels_last else (3,H,W). Level l, intensity_out[l] (device, (H/pools[l], W/pools[l]) floats), holds per pixel the mean
 * of Y = 0.299 R + 0.587 G + 0.114 B over the pools[l] x pools[l] block whose maximum rtg_icp_build_pyramid takes for the
 * depth: the same pixel grid and level intrinsics. 1 <= n_levels <= 4. Validated on the host before any CUDA work. */
int rtg_icp_build_intensity_pyramid(const float *color, int32_t H, int32_t W, int32_t channels_last, int32_t n_levels,
                                    const int32_t *pools, float *const *intensity_out, void *stream);

/* rtg_icp_predict_pose with a photometric term (RGB-D odometry), one cooperative launch as well. For every pixel whose
 * geometric row is valid, the row r = I1(u,v) - I0[q] is added: I1 is the bilinear interpolation of the previous frame's
 * level intensity intensity1[l] at the projection (u,v) of the geometric row, I0 = intensity0[l] the current frame's;
 * J = (v' x a, a) with a = dr/dv' through the exact derivative of the interpolant. H = sum_geo J^T J +
 * photometric_weight * sum_photo J^T J, g likewise; damping, solve and update as in rtg_icp_predict_pose. intensity0[l] /
 * intensity1[l]: device, (levels[l].H, levels[l].W) floats (rtg_icp_build_intensity_pyramid). photometric_weight: m^2 per
 * squared intensity unit, finite and >= 0; with 0 the 18 leading floats are rtg_icp_predict_pose's, bit for bit.
 * out / out_host: 20 floats = the 18 of rtg_icp_predict_pose, then the photometric ratio (count / (H*W) of the level) and
 * RMS residual (0 without rows) of the last iteration. Arguments are validated on the host before any CUDA work. */
int rtg_icp_predict_pose_rgbd(const RtgIcpLevel *levels, const float *const *intensity0, const float *const *intensity1,
                              int32_t n_levels, float distance_threshold, float normal_cos_threshold, float damping,
                              float photometric_weight, const float *pose_init, const float *p2p_vertex_t0,
                              const float *p2p_vertex_t1, const float *p2p_normal_t0, int32_t p2p_H, int32_t p2p_W, float *out,
                              float *out_host, void *ws, void *stream);

/* ---- image-space glue between the rasterizer forward and backward (SURVEY.md section 8(f) #1) -------------
 * Fused masked L1 colour + depth loss of Mapping.loss_update (SLAM/multiprocess/mapper.py:402-431,444-451, with
 * l1_loss of utils/loss_utils.py:27-31) and its gradients w.r.t. the rendered colour and depth:
 *   colour = mean |render - gt_color| over the render_mask pixels (NULL = all) x 3 channels,
 *   depth  = mean |depth - gt_depth| over pixels with depth_index != -1, gt_depth > 0, depth - gt_depth <
 *            depth_error_max and the render mask,  loss = color_weight*colour + depth_weight*depth.
 * render (3,H,W), depth (1,H,W), depth_index (1,H,W) are rasterizer outputs; gt_color is (H,W,3) if
 * gt_channels_last else (3,H,W); gt_depth (H,W); render_mask (H,W) bytes. loss_out: 4 device floats
 * {loss, colour, depth, n_depth}. An empty selection contributes 0 (torch's mean of an empty tensor is NaN). The sums are
 * formed in double from per-block partial sums added in a fixed order (no atomics): identical inputs give bit-identical
 * outputs. ws: rtg_loss_workspace_bytes() bytes (about 66 KB), 8-byte aligned; one workspace serves all three losses.
 * Rejects a NULL pointer (render_mask may be NULL), H, W <= 0 and a misaligned ws on the host before any CUDA work. */
size_t rtg_loss_workspace_bytes(void);
int rtg_loss_l1(const float *render, const float *depth, const int32_t *depth_index, const float *gt_color, const float *gt_depth,
                const uint8_t *render_mask, int32_t H, int32_t W, int32_t gt_channels_last, float color_weight, float depth_weight,
                float depth_error_max, float *dL_dcolor, float *dL_ddepth, float *loss_out, void *ws, void *stream);

/* rtg_loss_l1_exposure: rtg_loss_l1 of a render seen under a frame exposure (a, b) = `exposure` (2 device floats): the colour
 * term is the mean of |r|, r = e^a render + b - gt_color, over the same pixels; the depth term is unchanged. Written:
 *   dL_dcolor = color_weight / N_c e^a sgn(r),  dL_ddepth as rtg_loss_l1,
 *   dL_dexposure (2 device floats) = color_weight / N_c (sum sgn(r) e^a render, sum sgn(r)),  N_c = 3 x selected pixels,
 * and loss_out as rtg_loss_l1. exposure = (0, 0) gives rtg_loss_l1's loss_out and gradients bit for bit. Sums, workspace and
 * validation as rtg_loss_l1 (rtg_loss_l1_exposure_workspace_bytes() == rtg_loss_workspace_bytes()); exposure and
 * dL_dexposure must not be NULL. */
size_t rtg_loss_l1_exposure_workspace_bytes(void);
int rtg_loss_l1_exposure(const float *render, const float *depth, const int32_t *depth_index, const float *gt_color,
                         const float *gt_depth, const uint8_t *render_mask, int32_t H, int32_t W, int32_t gt_channels_last,
                         float color_weight, float depth_weight, float depth_error_max, const float *exposure, float *dL_dcolor,
                         float *dL_ddepth, float *dL_dexposure, float *loss_out, void *ws, void *stream);

/* The same loss with the cosine normal term of Mapping.loss_update (mapper.py:433-442):
 *   normal = mean of 1 - cosine_similarity(render_normal, gt_normal) over pixels with render_mask, depth_index != -1 and
 *            gt_normal != 0,  loss = color_weight*colour + depth_weight*depth + normal_weight*normal.
 * render_normal (3,H,W) is Renderer.render's "normal"; gt_normal (H,W,3); dL_dnormal (3,H,W). With normal_weight == 0 the
 * three normal pointers may be NULL. loss_out: 8 device floats {loss, colour, depth, n_depth, normal, n_normal, 0, 0}:
 * everything Mapping.loss_update reports (mapper.py:459-466) in one buffer, one read-back instead of six .item() calls.
 * Sums, workspace and validation as rtg_loss_l1. */
int rtg_loss_mapping(const float *render, const float *depth, const float *render_normal, const int32_t *depth_index,
                     const float *gt_color, const float *gt_depth, const float *gt_normal, const uint8_t *render_mask, int32_t H, int32_t W,
                     int32_t gt_channels_last, float color_weight, float depth_weight, float normal_weight, float depth_error_max,
                     float *dL_dcolor, float *dL_ddepth, float *dL_dnormal, float *loss_out, void *ws, void *stream);

/* rtg_loss_mapping_exposure: rtg_loss_mapping of a render seen under an exposure (a, b) = `exposure` (2 device floats), as
 * rtg_loss_l1_exposure is rtg_loss_l1's: the colour residual is r = e^a render + b - gt_color, the depth and normal terms are
 * unchanged, and
 *   dL_dcolor = color_weight / N_c e^a sgn(r),
 *   dL_dexposure (2 device floats) = color_weight / N_c (sum sgn(r) e^a render, sum sgn(r)),  N_c = 3 x selected pixels.
 * loss_out keeps rtg_loss_mapping's 8 floats. exposure = (0, 0) gives rtg_loss_mapping's loss_out and gradients bit for bit.
 * Sums, workspace (rtg_loss_workspace_bytes()) and validation as rtg_loss_mapping; exposure and dL_dexposure must not be
 * NULL. */
int rtg_loss_mapping_exposure(const float *render, const float *depth, const float *render_normal, const int32_t *depth_index,
                              const float *gt_color, const float *gt_depth, const float *gt_normal, const uint8_t *render_mask,
                              int32_t H, int32_t W, int32_t gt_channels_last, float color_weight, float depth_weight,
                              float normal_weight, float depth_error_max, const float *exposure, float *dL_dcolor, float *dL_ddepth,
                              float *dL_dnormal, float *dL_dexposure, float *loss_out, void *ws, void *stream);

/* SSIM term of Mapping.loss_update (mapper.py:411-415: ssim_loss = 1 - ssim(render, gt), evaluated only without a render
 * mask) with ssim of utils/loss_utils.py:40-100: 11x11 Gaussian window (sigma 1.5, one per channel), zero padding,
 * C1 = 0.01^2, C2 = 0.03^2, mean over all C*H*W entries of the ssim map. img1, img2: (C,H,W).
 * loss_out: 2 device floats {1 - mean(ssim_map), mean(ssim_map)}; dL_dimg1 (C,H,W) = d loss_out[0] / d img1, or NULL for the
 * value only. Replaces five grouped 11x11 convolutions, ~15 elementwise kernels and their autograd twins by three launches;
 * the mean is reduced in a fixed order (bit-reproducible). ws: rtg_ssim_workspace_bytes(C, H, W) bytes. */
size_t rtg_ssim_workspace_bytes(int32_t C, int32_t H, int32_t W);
int rtg_ssim_loss(const float *img1, const float *img2, int32_t C, int32_t H, int32_t W, float *dL_dimg1, float *loss_out, void *ws,
                  void *stream);

/* rtg_ssim_loss_exposure: 1 - ssim(e^a img1 + b, img2) with (a, b) = `exposure` (2 device floats): img1 seen under the
 * exposure, then rtg_ssim_loss. Written: loss_out as rtg_ssim_loss; dL_dimg1 (C,H,W) = e^a dL/dx^ with x^ = e^a img1 + b;
 * dL_dexposure (2 device floats) = (sum dL/dx^ e^a img1, sum dL/dx^), from per-CTA double partials added in a fixed order
 * (bit-reproducible). dL_dimg1 and dL_dexposure may each be NULL; with both NULL only the value is computed.
 * ws: rtg_ssim_exposure_workspace_bytes(C, H, W) bytes (rtg_ssim_workspace_bytes plus the exposure partials), 8-byte
 * aligned. Rejects NULL img1 / img2 / exposure / loss_out / ws, C outside [1, 65535], H or W < 1 and ceil(H / 16) > 65535
 * on the host before any CUDA work. exposure = (0, 0) gives rtg_ssim_loss's loss_out and dL_dimg1 bit for bit. */
size_t rtg_ssim_exposure_workspace_bytes(int32_t C, int32_t H, int32_t W);
int rtg_ssim_loss_exposure(const float *img1, const float *img2, int32_t C, int32_t H, int32_t W, const float *exposure,
                           float *dL_dimg1, float *dL_dexposure, float *loss_out, void *ws, void *stream);

/* render_normal of Renderer.render (SLAM/render.py:130-133): out (3,H,W) = normal[depth_index] where the index is
 * > -1, zeros elsewhere; normal is (P,3). */
int rtg_normal_map(const float *normal, const int32_t *depth_index, int32_t H, int32_t W, float *out, void *stream);

/* ---- tracker-side preprocessing of an incoming depth frame (SURVEY.md section 8(f) #3) --------------------------
 * Tracker.map_preprocess (SLAM/multiprocess/tracker.py:97-132): optional bilateral depth filter (bilateralFilter_torch,
 * SLAM/utils.py:550-589; taps with i^2+j^2 <= radius^2, zero padding, zero-depth neighbours ignored), valid-range mask
 * (min_depth, max_depth) exclusive, vertex map and Sobel normal map (compute_vertex_map / compute_normal_map,
 * SLAM/utils.py:65-122), confidence = |cos(normal, pixel ray)| (compute_confidence_map, SLAM/utils.py:125-138), and the
 * invalid-confidence masking: where the normal is zero or the confidence is below the threshold, depth, vertex, normal
 * and confidence are set to 0 and invalid_mask_out (may be NULL) to 1. depth_in / depth_out (H,W); vertex, normal
 * (H,W,3) channels-last; confidence (H,W). depth_in == depth_out is allowed only without the filter. With vertex_out,
 * normal_out, confidence_out and invalid_mask_out all NULL only the filter and the range mask run.
 * ws: rtg_icp_workspace_bytes() bytes. */
int rtg_frame_preprocess(const float *depth_in, int32_t H, int32_t W, int32_t depth_filter, int32_t radius, float sigma_color,
                         float sigma_space, float min_depth, float max_depth, float fx, float fy, float cx, float cy,
                         float invalid_confidence_thresh, float *depth_out, float *vertex_out, float *normal_out,
                         float *confidence_out, uint8_t *invalid_mask_out, void *ws, void *stream);

/* rtg_frame_downsample: level `scale` (>= 2) of a measured frame for coarse-to-fine tracking, in one launch. Coarse pixel
 * (i, j) covers the fine block [s i, s i + s) x [s j, s j + s); the coarse size is Hs = H / s, Ws = W / s (integer division:
 * a trailing partial row or column is dropped). color (3, H, W) or (H, W, 3) (color_channels_last) -> color_out (3, Hs, Ws):
 * the block mean per channel. depth (H, W) -> depth_out (Hs, Ws): the block mean when all s^2 depths are > 0, else 0.
 * render_mask (H, W) uint8, optional -> mask_out (Hs, Ws): 1 when all s^2 pixels are nonzero, else 0. tile_mask, optional, in
 * the rasterizer's layout (ceil(H/16), ceil(W/16)) int32 -> tile_mask_out (ceil(Hs/16), ceil(Ws/16)): 1 when any fine tile
 * of [s tx, s tx + s) x [s ty, s ty + s), clipped to the fine grid, is nonzero. The camera of the coarse level is the
 * caller's (tracking.level_camera). Validates on the host before any CUDA work: sizes, scale, NULL pointers, and that
 * mask_out / tile_mask_out are given exactly when render_mask / tile_mask are. */
int rtg_frame_downsample(const float *color, const float *depth, const uint8_t *render_mask, const int32_t *tile_mask, int32_t H,
                         int32_t W, int32_t scale, int32_t color_channels_last, float *color_out, float *depth_out,
                         uint8_t *mask_out, int32_t *tile_mask_out, void *stream);

/* ---- per-frame consumers of the rasterizer's index / transmittance maps (SURVEY.md section 8(f) #2) ---------
 * accumulate_gaussian_error of submodules/cuda_utils (cuda_utils.cu:17-60, map_process.cu:33-245), called by
 * Mapping.error_gaussians_remove (SLAM/multiprocess/mapper.py:546-559): for every pixel, the colour error goes to the
 * Gaussian named by color_index, the depth and normal errors to the one named by depth_index (indices outside [0,P)
 * are skipped); per Gaussian the maximum (check_max) or the mean of its pixels; rescale_counter counts the pixels
 * whose colour / depth / normal error exceeds its threshold (as a float, like the reference). All inputs (H*W), all
 * outputs (P); outputs need not be initialised. counters: 2*P int32 of scratch, only used when !check_max. */
int rtg_accumulate_gaussian_error(int32_t H, int32_t W, int32_t P, const float *screen_color_error, const float *screen_depth_error,
                                  const float *screen_normal_error, const int32_t *screen_color_index,
                                  const int32_t *screen_depth_index, float color_threshold, float depth_threshold,
                                  float normal_threshold, int32_t check_max, float *gs_color_error, float *gs_depth_error,
                                  float *gs_normal_error, float *gs_rescale_counter, int32_t *counters, void *stream);

/* 16x16 average pooling of an (H,W) float image with zero padding, as F.avg_pool2d is used by transmission2tilemask /
 * colorerror2tilemask (SLAM/utils.py:695-734): tile_mean (tiles_y, tiles_x) and / or tile_mask = (mean > ratio), either
 * may be NULL. */
int rtg_tile_mean(int32_t H, int32_t W, const float *pixels, float ratio, float *tile_mean, int32_t *tile_mask, void *stream);

/* render_mask = (T_map != 1) and tile_mask = transmission2tilemask(render_mask, 16, ratio) in one pass
 * (Mapping.evaluate_render_range, mapper.py:503-505). render_mask (H,W) bytes, may be NULL. */
int rtg_transmission_tile_mask(int32_t H, int32_t W, const float *T_map, float ratio, uint8_t *render_mask, int32_t *tile_mask,
                               void *stream);

/* colour error image of mapper.py:481-487: sum over channels of |render - gt|, 0 where the rendered pixel is black;
 * render, gt (3,H,W), out (H,W). */
int rtg_color_error(int32_t H, int32_t W, const float *render, const float *gt, float *out, void *stream);

/* ---- map surgery on the Gaussian SoA and nearest neighbours (SURVEY.md section 8(f) #4) ----------------------------
 * rtg_soa_compact: GaussianPointCloud.delete / remove (SLAM/gaussian_pointcloud.py:195-235) -- keep the rows whose mask
 * byte is non-zero (invert = 0) or zero (invert = 1; `delete(mask)` keeps ~mask) of n_arrays attribute arrays that share the
 * row index; array a has words_per_row[a] 4-byte words per row (xyz 3, features_rest 45, rotation 4, counters 1, ...).
 * One scan of the mask, one gather launch for all arrays; rows keep their order. out[a] must hold P rows; n_kept (device
 * uint32) and n_kept_host (mapped pinned uint32, may be NULL) receive the number of rows kept. n_arrays <= 16.
 * ws: rtg_soa_compact_workspace_bytes(P) bytes. in / out: host arrays of device pointers. */
#define RTG_SOA_MAX_ARRAYS 16
size_t rtg_soa_compact_workspace_bytes(int64_t P);
int rtg_soa_compact(const uint8_t *mask, int32_t invert, int64_t P, int32_t n_arrays, const void *const *in, void *const *out,
                    const int32_t *words_per_row, uint32_t *n_kept, uint32_t *n_kept_host, void *ws, void *stream);

/* rtg_knn: exact K nearest reference points of every query point, 1 <= K <= 8, squared Euclidean distances ascending.
 * Replaces distCUDA2 of submodules/simple-knn (simple_knn.cu:169-251; spatial.cu) as GaussianPointCloud.update_geometry
 * uses it (gaussian_pointcloud.py:376: query == ref, K = 3, skip_self = 1, out_mean = (d0+d1+d2)/3 and out_idx) and
 * pytorch3d.ops.knn_points as Mapping.temp_points_filter / gaussians_isolated call it (mapper.py:812-819,903-910:
 * skip_self = 0). query (n_query,3), ref (n_ref,3) fp32; out_d2 (n_query,K), out_idx (n_query,K) int32, out_mean (n_query)
 * -- each may be NULL. With fewer than K candidates the missing slots hold FLT_MAX / INT_MAX (simple-knn's sentinels).
 * Uniform-grid search sized on the device from the bounding box of `ref`; no host synchronisation.
 * ws: rtg_knn_workspace_bytes(n_ref) bytes. */
size_t rtg_knn_workspace_bytes(int64_t n_ref);
int rtg_knn(const float *query, int64_t n_query, const float *ref, int64_t n_ref, int32_t K, int32_t skip_self, float *out_d2,
            int32_t *out_idx, float *out_mean, void *ws, void *stream);

/* ---- the map follows corrected camera poses (no reference counterpart) --------------------------------------------
 * rtg_map_transform: move every Gaussian rigidly with the correction of its anchor frame, in place. Anchor k has the
 * camera-to-world poses old_c2w[k] and new_c2w[k] (K x 16 doubles, row-major 4x4, device). Once per anchor, in float64:
 * q_delta = the unit quaternion (w >= 0) of R_new R_old^T, R = its rotation matrix, t = p_new - R p_old. Every row i with
 * 0 <= anchor[i] < K whose anchor's two poses differ bitwise becomes
 *   xyz' = R xyz + t,  rotation' = q_delta (x) rotation (Hamilton product, (w,x,y,z), the raw magnitude is kept),
 *   normal' = R normal,  features_rest' band l = D^l(R) band l for l = 1..3 and each colour channel,
 * where D^l is the rotation of band l of the rasterizer's real SH basis (computeColorFromSH, forward.cu:104-155):
 * sh(f', R d) = sh(f, d) for every direction d. features_dc, scaling, opacity and every other attribute are untouched.
 * Rows with anchor -1, or whose anchor's poses are bitwise equal, are not written; rows with any other anchor outside
 * [0, K) are not written either and are counted in *n_skipped (device int64, set by the call). No host synchronisation.
 * xyz (P,3), rotation (P,4), normal (P,3) or NULL, features_rest (P, sh_rest, 3) with sh_rest in {0, 3, 8, 15} (NULL iff
 * sh_rest == 0), anchor (P) int32: device, fp32 / int32, contiguous. ws: rtg_map_transform_workspace_bytes(K) bytes,
 * 16-byte aligned. P == 0: nothing is read and *n_skipped is set to 0. K == 0: no row is written, and *n_skipped counts
 * every anchor other than -1 (old_c2w, new_c2w and ws may then be NULL). Validates on the host before any CUDA call: a
 * NULL struct, a NULL required pointer, negative sizes and sh_rest outside the set are rejected. */
typedef struct RtgMapTransform {
    int32_t P, K, sh_rest, _pad;
    const int32_t *anchor;                 /* (P) frame index per Gaussian (_add_tick), -1 = not anchored */
    const double *old_c2w, *new_c2w;       /* (K,4,4) */
    float *xyz, *rotation, *normal, *features_rest;
    int64_t *n_skipped;                    /* rows whose anchor lies outside [-1, K) and != -1 */
} RtgMapTransform;
size_t rtg_map_transform_workspace_bytes(int32_t K);
int rtg_map_transform(const RtgMapTransform *xf, void *ws, void *stream);

/* ---- a surface from the map: TSDF fusion and marching tetrahedra (no reference counterpart) ------------------------
 * RtgTsdfVolume describes a dense voxel grid owned by the caller: voxel (i,j,k) has its centre at origin + voxel_size *
 * (i,j,k); tsdf, weight and color are structure-of-arrays, x fastest (linear index i + nx*(j + ny*k)), float32, with
 * color as three planes of nx*ny*nz floats (R, G, B) or NULL. A fresh volume holds tsdf = 1, weight = 0, color = 0.
 * nx, ny, nz >= 1 and nx*ny*nz < 2^31; voxel_size > 0; trunc > 0 in map units.
 *
 * rtg_tsdf_integrate folds one depth frame into the volume. For every voxel, with p_c = R p + t of the W2C `w2c`:
 *   skip if z <= 0; (u, v) = (fx x/z + cx, fy y/z + cy), pixel (rint(u), rint(v)) with rounding half to even, skip if
 *   outside the image; d = depth[pixel], skip if d <= 0 (0 = no reading / no hit); sdf = d - z, skip if sdf < -trunc;
 *   f = min(1, sdf / trunc); tsdf <- (tsdf w + f)/(w + 1), color <- (color w + c_pixel)/(w + 1), w <- w + 1.
 * depth (H,W) float32; color (3,H,W), or (H,W,3) with color_channels_last = 1, given exactly when the volume has color;
 * w2c: 16 row-major doubles (w2c_is_double = 1) or floats (0) in device memory, read on the device. Arithmetic is float64.
 * A voxel is written only when it is updated; there are no atomics, so equal call sequences give equal bits, and no host
 * synchronisation.
 *
 * Extraction (marching tetrahedra on the Kuhn decomposition: cell (i,j,k), i < nx-1 etc., splits into six tetrahedra,
 * one per axis permutation p in lexicographic order, c -> c+e_p0 -> c+e_p0+e_p1 -> c+(1,1,1)). Voxel a owns the edges to
 * a + (1,0,0), (0,1,0), (0,0,1), (1,1,0), (0,1,1), (1,0,1), (1,1,1) (slots 0..6). An edge (a, b) carries a vertex when both
 * weights are > 0 and exactly one of its tsdf values is < 0; it lies at a + tau (b - a), tau = f_a / (f_a - f_b), in world
 * units, with the colour interpolated with the same tau. A tetrahedron whose four weights are > 0 emits one triangle
 * with one or three negative corners and two with two; winding is right-handed, the normal pointing from negative to
 * positive tsdf. Vertices are ordered by (owning voxel, slot), triangles by (cell, tetrahedron, triangle 0..1).
 *   rtg_tsdf_extract_count: one counting pass and two exclusive scans; writes counts[0] = vertices, counts[1] =
 *     triangles (device uint32[2]) and keeps the offsets in ws (rtg_tsdf_extract_workspace_bytes(nx, ny, nz) bytes).
 *   rtg_tsdf_extract_emit: with the same ws and an unchanged volume, writes vertices (V,3) float32, vertex_colors (V,3)
 *     float32 (may be NULL; ignored without volume color) and faces (F,3) int32. Writes stay inside the counted ranges.
 * Extraction needs 12 * nx*ny*nz < 2^32 (at most 12 triangles per cell, uint32 offsets).
 * Every entry point validates on the host before any CUDA call: a NULL descriptor or required pointer, non-positive sizes,
 * voxel_size or trunc, and a voxel count at or above the limit are rejected. */
typedef struct RtgTsdfVolume {
    int32_t nx, ny, nz;
    float voxel_size, trunc;
    float origin[3];
    float *tsdf, *weight, *color;
} RtgTsdfVolume;
int rtg_tsdf_integrate(const RtgTsdfVolume *vol, const float *depth, const float *color, int32_t H, int32_t W,
                       int32_t color_channels_last, float fx, float fy, float cx, float cy, const void *w2c, int32_t w2c_is_double,
                       void *stream);
/* rtg_tsdf_raycast renders the surface extraction emits, seen from the W2C `w2c` (16 row-major doubles or floats in
 * device memory, read on the device; arithmetic in float64, outputs rounded once to float32). Pixel (u, v) has the ray
 * o + t d, o = -R^T t_w2c, d = R^T ((u - cx)/fx, (v - cy)/fy, 1), so t is camera z; it starts at t > 0 and ends where it
 * leaves the cell region [origin, origin + voxel_size (n - 1)]. The field is the piecewise-linear interpolant on the Kuhn
 * tetrahedra of extraction (not trilinear): in cell c with local u in [0,1]^3, the tetrahedron of the permutation p that
 * orders u decreasingly has the weights 1 - u_p1, u_p1 - u_p2, u_p2 - u_p3, u_p3 on c, c+e_p1, c+e_p1+e_p2, c+(1,1,1);
 * only tetrahedra whose four weights are > 0 take part. Cells are walked in ray order, each cut at the planes u_a = u_b
 * into pieces of one tetrahedron; along a piece the field is linear and its zero is t* = t_s + (t_e - t_s) f_s/(f_s - f_e).
 * The first piece whose field changes sign (sign test f < 0) decides: from >= 0 to < 0 it is a hit, with depth t*,
 * normal the tetrahedron's unit gradient (world space, towards free space: the face normal of the mesh triangle) and
 * colour interpolated with the tetrahedron's weights (the mesh's vertex colours interpolated over the triangle); from < 0
 * to >= 0 it is a back face and the ray ends without a hit. Pixels without a hit get depth 0, normal 0 and colour 0.
 * depth (H,W) float32; normal (3,H,W) float32; color (3,H,W) float32, given exactly when the volume has color.
 * One thread per pixel; no atomics (repeats give equal bits) and no host synchronisation. Validated like
 * rtg_tsdf_integrate: volume (nx*ny*nz < 2^31), H, W >= 1, NULL pointers, colour against the volume, finite intrinsics
 * with fx, fy != 0. */
int rtg_tsdf_raycast(const RtgTsdfVolume *vol, const void *w2c, int32_t w2c_is_double, int32_t H, int32_t W, float fx, float fy,
                     float cx, float cy, float *depth, float *normal, float *color, void *stream);
size_t rtg_tsdf_extract_workspace_bytes(int32_t nx, int32_t ny, int32_t nz);
int rtg_tsdf_extract_count(const RtgTsdfVolume *vol, void *ws, uint32_t *counts, void *stream);
int rtg_tsdf_extract_emit(const RtgTsdfVolume *vol, const void *ws, float *vertices, float *vertex_colors, int32_t *faces,
                          void *stream);

/* ---- measurement hook (no reference counterpart) ---------------------------------------------
 * When enabled, every kernel launch of this library is bracketed by CUDA events on its launching stream.
 * rtg_profile_read synchronises the device and returns, per kernel id, the summed duration (ms) and the number
 * of launches since the last reset. bench.py uses it for the roofline line and the launch count. */
int rtg_profile_enable(int32_t on);
int rtg_profile_kernel_count(void);
const char *rtg_profile_kernel_name(int32_t id);
int rtg_profile_read(double *total_ms, int64_t *launches, int32_t reset);

#ifdef __cplusplus
}
#endif
#endif /* RTG_SPLAT_B200_H */
