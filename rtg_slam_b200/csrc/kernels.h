// Host-side launch entry points of the kernels (internal; the public surface is include/rtg_splat_b200.h).
#pragma once
#include "common.cuh"

struct RtgMapTransform;
struct RtgTsdfVolume;

namespace rtg {

void launch_preprocess_fwd(const ViewParams &vp, int P, int M, const float *means, const float *scales, const float *rots,
                           const float *opac, const float *shs, const float *colors_precomp, const float *cov3D_precomp,
                           const int *tile_mask, const GeomState &g, int *radii, uint32_t *tile_count, uint32_t *tile_touched,
                           uint32_t *vis_count, int p_begin, cudaStream_t s);
void launch_mark_visible(int P, const float *means, const float *view, const float *proj, uint8_t *present, cudaStream_t s);
void launch_bwd_zero(int p_begin, int P, int M, bool has_sh, bool has_sr, const int *radii, float *dL_dmeans, float *dL_dsh,
                     float *dL_dcolors, float *dL_dopacity, float *dL_dscales, float *dL_drot, float *dL_dcov3D, float *dL_dmeans2D,
                     cudaStream_t s);
void launch_preprocess_bwd(const ViewParams &vp, int P, int M, const float *means, const float *scales, const float *rots,
                           const float *shs, const float *cov3D_precomp, const GeomState &g, const uint32_t *vis_count, float *rec,
                           float *dL_dmeans, float *dL_dsh, float *dL_dcolors, float *dL_dopacity, float *dL_dscales, float *dL_drot,
                           float *dL_dcov3D, float *dL_dmeans2D, cudaStream_t s);
// launch_preprocess_bwd that also writes dL/d(viewmatrix 16, projmatrix 16, campos 3) to `dL_dcamera` (35 floats, device);
// `camera_scratch`: camera_scratch_bytes(P) bytes of device memory for the block partials
size_t camera_scratch_bytes(int P);
void launch_preprocess_bwd_camera(const ViewParams &vp, int P, int M, const float *means, const float *scales, const float *rots,
                                  const float *shs, const float *cov3D_precomp, const GeomState &g, const uint32_t *vis_count,
                                  float *rec, float *dL_dmeans, float *dL_dsh, float *dL_dcolors, float *dL_dopacity,
                                  float *dL_dscales, float *dL_drot, float *dL_dcov3D, float *dL_dmeans2D, float *dL_dcamera,
                                  void *camera_scratch, cudaStream_t s);
// the camera gradient alone (frozen map): the records are consumed and cleared, no per-Gaussian gradient is written
void launch_preprocess_bwd_pose(const ViewParams &vp, int P, int M, const float *means, const float *scales, const float *rots,
                                const float *shs, const float *cov3D_precomp, const GeomState &g, const uint32_t *vis_count,
                                float *rec, float *dL_dcamera, void *camera_scratch, cudaStream_t s);

// forward-mode pose tangents of the visible Gaussians (RTG_TAN_ROW float4 per row, indexed by Gaussian id)
void launch_preprocess_tangent(const ViewParams &vp, int P, int M, const float *means, const float *scales, const float *rots,
                               const float *shs, const float *cov3D_precomp, const GeomState &g, const uint32_t *vis_count,
                               float4 *tan, cudaStream_t s);

// binning.cu
void launch_tile_histogram(const ViewParams &vp, int P, const GeomState &g, const int *radii, const int *tile_mask, const BinState &b,
                           cudaStream_t s);
void launch_tile_scan(const BinState &b, int T, int64_t R_cap, int32_t *counters, int32_t *counters_host, cudaStream_t s);
void launch_scatter(const ViewParams &vp, int P, const GeomState &g, const int *radii, const int *tile_mask, const BinState &b,
                    int64_t R_cap, const int32_t *counters, cudaStream_t s);
void launch_tile_sort(const BinState &b, int T, const int32_t *counters, cudaStream_t s);

// render.cu
void launch_render_fwd(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img, const int32_t *counters,
                       float *out_color, float *out_depth, int *out_hit_color, int *out_hit_depth, float *out_hcw,
                       float *out_hdw, float *out_T, cudaStream_t s);
void launch_render_bwd(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img, const int32_t *counters,
                       const float *final_T, const int *hit_image, const float *dL_dcolor, const float *dL_ddepth, float *rec,
                       cudaStream_t s, const float *dL_dT = nullptr);  // dL_dT: (H, W) dL/dT_map, or NULL
// pose Gauss-Newton: scratch = the tangent rows (read) and the per-tile partial sums
size_t pose_gn_scratch_bytes(int P, int H, int W);
size_t pose_gn_exposure_scratch_bytes(int P, int H, int W);  // the per-tile rows hold RTG_GN_EXP_ALL terms
void launch_render_tangent_images(const ViewParams &vp, int P, const GeomState &g, const BinState &b, const ImgState &img,
                                  const int32_t *counters, const int *hit_image, void *scratch, float *J, cudaStream_t s);
// the same with the expected depth in channel 3 of J, and its (D, m1) map in `expected` (2, H, W)
void launch_render_tangent_expected_images(const ViewParams &vp, int P, const GeomState &g, const BinState &b, const ImgState &img,
                                           const int32_t *counters, void *scratch, float *J, float *expected, cudaStream_t s);
// per-Gaussian pixel counts, weight sums and (pixel_error != NULL) weighted error of the forward, added into the outputs
void launch_render_contributions(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img,
                                 const int32_t *counters, const float *pixel_error, int32_t *n_pixels, float *weight, float *error,
                                 cudaStream_t s);
// the forward's blend weights applied to C per-Gaussian features: out (C, H, W) written everywhere; and its transpose,
// dL_dfeatures (P, C) added into (the caller zeroes it)
void launch_render_features(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img,
                            const int32_t *counters, int C, const float *features, float *out, cudaStream_t s);
void launch_render_features_bwd(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img,
                                const int32_t *counters, int C, const float *dL_dout, float *dL_dfeatures, cudaStream_t s);
// the feature map's gradient through its blend weights: the six alpha moments added into the (zeroed) gradient record
void launch_render_features_grad(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img,
                                 const int32_t *counters, int C, const float *features, const float *dL_dout, float *rec,
                                 cudaStream_t s);

// mapstats.cu
void launch_gs_error(int H, int W, int P, const float *color_err, const float *depth_err, const float *normal_err,
                     const int *color_index, const int *depth_index, float thr_c, float thr_d, float thr_n, bool check_max,
                     float *gs_color, float *gs_depth, float *gs_normal, float *rescale, int *counters, cudaStream_t s);
void launch_tile_pool(int H, int W, const float *pixels, int mode, float ratio, uint8_t *pixel_mask, float *tile_mean, int *tile_mask,
                      cudaStream_t s);
void launch_color_error(int H, int W, const float *render, const float *gt, float *err, cudaStream_t s);

// frameprep.cu
void launch_frame_preprocess(const float *depth_in, int H, int W, int filter, int radius, float sigma_color, float sigma_space,
                             float min_depth, float max_depth, float fx, float fy, float cx, float cy, float conf_thresh,
                             float *depth_out, float *vertex, float *normal, float *confidence, uint8_t *invalid, void *ws,
                             cudaStream_t s);

// icp.cu: persistent (cooperative) kernels
#define RTG_ICP_MAX_LEVELS 4
struct IcpLevel {
    const float *v0, *n0, *v1, *n1;  // "0" = current frame, "1" = previous / model frame
    int H, W;
    float fx, fy, cx, cy;
    int iters;
};
struct IcpPredict {
    IcpLevel lv[RTG_ICP_MAX_LEVELS];
    int n_levels;
    float dist_thr, cos_thr, damping;
    const float *pose_in;
    const float *p2p_v_t0, *p2p_v_t1, *p2p_n_t0;
    int p2p_HW;
    float *out, *out_host;
};
// photometric term of icp_predict_kernel<true>: per-level intensities of the current ("0") and previous ("1") frame,
// each (H, W) of its level, and the weight of the photometric normal equations (out then holds 20 floats)
struct IcpPhoto {
    const float *I0[RTG_ICP_MAX_LEVELS], *I1[RTG_ICP_MAX_LEVELS];
    float w;
};
struct IcpIntensity {
    const float *color;  // (H, W, 3) if channels_last, else (3, H, W)
    int H, W, channels_last, n_levels;
    int pool[RTG_ICP_MAX_LEVELS];
    int start[RTG_ICP_MAX_LEVELS];  // first thread of each level
    int total;                      // level pixels of all levels
    float *out[RTG_ICP_MAX_LEVELS];
};
struct IcpPyramid {
    const float *depth;
    int H, W, n_levels;
    int pool[RTG_ICP_MAX_LEVELS];
    float fx[RTG_ICP_MAX_LEVELS], fy[RTG_ICP_MAX_LEVELS], cx[RTG_ICP_MAX_LEVELS], cy[RTG_ICP_MAX_LEVELS];
    float *vertex[RTG_ICP_MAX_LEVELS], *normal[RTG_ICP_MAX_LEVELS];
};
cudaError_t launch_icp_predict(const IcpPredict &prm, void *ws, cudaStream_t s);
cudaError_t launch_icp_predict_rgbd(const IcpPredict &prm, const IcpPhoto &ph, void *ws, cudaStream_t s);
cudaError_t launch_icp_pyramid(const IcpPyramid &prm, void *ws, cudaStream_t s);
void launch_icp_intensity_pyramid(const IcpIntensity &prm, cudaStream_t s);

// mapsurgery.cu
#ifndef RTG_SOA_MAX_ARRAYS
#define RTG_SOA_MAX_ARRAYS 16
#endif
size_t soa_compact_ws_bytes(int64_t P);
void launch_soa_compact(const uint8_t *mask, int invert, int64_t P, int n_arrays, const void *const *in, void *const *out,
                        const int32_t *words_per_row, uint32_t *n_kept, uint32_t *n_kept_host, void *ws, cudaStream_t s);
// out[i] = sum of in[0..i) (out may be in: each element is read before it is overwritten); sums: scratch of
// exclusive_scan_sums_words(n) words; total (device) / total_host (mapped) may be NULL
size_t exclusive_scan_sums_words(uint32_t n);
void exclusive_scan_u32(const uint32_t *in, uint32_t n, uint32_t *out, uint32_t *sums, uint32_t *total, uint32_t *total_host,
                        cudaStream_t s);
size_t knn_ws_bytes(int64_t n_ref);
int launch_knn(const float *query, int64_t n_query, const float *ref, int64_t n_ref, int K, int skip_self, float *out_d2, int32_t *out_idx,
               float *out_mean, void *ws, cudaStream_t s);

// maptransform.cu
size_t map_transform_ws_bytes(int64_t K);
void launch_map_transform(const RtgMapTransform &m, void *ws, cudaStream_t s);

// tsdf.cu
void launch_tsdf_integrate(const RtgTsdfVolume &v, const float *depth, const float *color, int H, int W, int channels_last, float fx,
                           float fy, float cx, float cy, const void *w2c, bool w2c_double, cudaStream_t s);
void launch_tsdf_raycast(const RtgTsdfVolume &v, const void *w2c, bool w2c_double, int H, int W, float fx, float fy, float cx,
                         float cy, float *depth, float *normal, float *color, cudaStream_t s);
size_t tsdf_extract_ws_bytes(int64_t n);
void launch_tsdf_extract_count(const RtgTsdfVolume &v, void *ws, uint32_t *counts, cudaStream_t s);
void launch_tsdf_extract_emit(const RtgTsdfVolume &v, const void *ws, float *vertices, float *vertex_colors, int32_t *faces,
                              cudaStream_t s);

// adam.cu and the per-level icp.cu entry points are declared in their own sections of capi.cu
}  // namespace rtg
