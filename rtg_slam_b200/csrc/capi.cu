// C ABI of librtg_splat_b200.so -- see include/rtg_splat_b200.h for the contract of every entry point.
#include <cstdio>
#include <cstring>
#include <cmath>
#include <string>

#include "../../include/rtg_splat_b200.h"
#include "common.cuh"
#include "kernels.h"
#include "prof.h"
#include <vector>
#include <mutex>
#include <utility>

namespace rtg {
int launch_adam(const RtgAdamGroup *groups, int n_groups, float beta1, float beta2, float eps, int step, cudaStream_t s);
void launch_pose_adam_step(const RtgPoseAdam &st, cudaStream_t s);
void launch_pose_gn_normal_eq_step(const ViewParams &vp, int P, const GeomState &g, const BinState &b, const ImgState &img,
                                   const int32_t *counters, const RtgPoseGN &st, const RtgPoseRobust &robust, cudaStream_t s);
void launch_pose_gn_exposure_step(const ViewParams &vp, int P, const GeomState &g, const BinState &b, const ImgState &img,
                                  const int32_t *counters, const RtgPoseGN &st, const RtgPoseRobust &robust, double *ab,
                                  cudaStream_t s);
void launch_pose_gn_expected_step(const ViewParams &vp, int P, const GeomState &g, const BinState &b, const ImgState &img,
                                  const int32_t *counters, const RtgPoseGN &st, const RtgPoseRobust &robust, double *ab,
                                  float min_cov, cudaStream_t s);
void launch_frame_downsample(const float *color, const float *depth, const uint8_t *render_mask, const int32_t *tile_mask, int H,
                             int W, int scale, int channels_last, float *color_out, float *depth_out, uint8_t *mask_out,
                             int32_t *tile_mask_out, cudaStream_t s);
void launch_map_adam_step(const RtgMapStep &st, cudaStream_t s);
void launch_history_merge(const RtgHistoryMerge &m, cudaStream_t s);
void launch_map_activate(int P, const float *scaling_raw, const float *rotation_raw, const float *opacity_raw, float *scales_out,
                         float *rotations_out, float *opacities_out, float *normal_out, cudaStream_t s);
size_t icp_ws_bytes();
void launch_icp_build_level(const float *depth, int H, int W, int pool, float fx, float fy, float cx, float cy, float *vertex,
                            float *normal, void *ws, cudaStream_t s);
void launch_icp_solve_level(const float *v0, const float *n0, const float *v1, const float *n1, int H, int W, float fx, float fy,
                            float cx, float cy, float dist_thr, float cos_thr, float damping, int iters, float *pose,
                            float *valid_ratio, void *ws, cudaStream_t s);
void launch_icp_p2p(const float *v_t0, const float *v_t1, const float *n_t0, int H, int W, const float *pose, float *loss,
                    void *ws, cudaStream_t s);
size_t loss_ws_bytes();
size_t ssim_ws_bytes(int C, int H, int W);
void launch_ssim_loss(const float *img1, const float *img2, int C, int H, int W, float *dL_dimg1, float *loss_out, void *ws,
                      cudaStream_t s);
void launch_loss_l1(const float *render, const float *depth, const int *depth_index, const float *gt_color, const float *gt_depth,
                    const uint8_t *mask, int H, int W, int channels_last, float color_weight, float depth_weight,
                    float depth_error_max, float *dL_dcolor, float *dL_ddepth, float *loss_out, void *ws, cudaStream_t s);
void launch_loss_mapping(const float *render, const float *depth, const float *render_normal, const int *depth_index,
                         const float *gt_color, const float *gt_depth, const float *gt_normal, const uint8_t *mask, int H, int W,
                         int channels_last, float color_weight, float depth_weight, float normal_weight, float depth_error_max,
                         float *dL_dcolor, float *dL_ddepth, float *dL_dnormal, float *loss_out, void *ws, cudaStream_t s);
void launch_loss_l1_exposure(const float *render, const float *depth, const int *depth_index, const float *gt_color,
                             const float *gt_depth, const uint8_t *mask, int H, int W, int channels_last, float color_weight,
                             float depth_weight, float depth_error_max, const float *exposure, float *dL_dcolor, float *dL_ddepth,
                             float *dL_dexposure, float *loss_out, void *ws, cudaStream_t s);
void launch_loss_mapping_exposure(const float *render, const float *depth, const float *render_normal, const int *depth_index,
                                  const float *gt_color, const float *gt_depth, const float *gt_normal, const uint8_t *mask, int H,
                                  int W, int channels_last, float color_weight, float depth_weight, float normal_weight,
                                  float depth_error_max, const float *exposure, float *dL_dcolor, float *dL_ddepth,
                                  float *dL_dnormal, float *dL_dexposure, float *loss_out, void *ws, cudaStream_t s);
size_t ssim_exposure_ws_bytes(int C, int H, int W);
void launch_ssim_loss_exposure(const float *img1, const float *img2, int C, int H, int W, const float *exposure, float *dL_dimg1,
                               float *dL_dexposure, float *loss_out, void *ws, cudaStream_t s);
void launch_normal_map(const float *normal, const int *depth_index, int H, int W, float *out, cudaStream_t s);
void launch_icp_fill(float *render_depth, const float *frame_depth, const float *rn, const float *fn, int H, int W, float dthr,
                     float nthr, cudaStream_t s);
}  // namespace rtg


// ---------------------------------------------------------------- event profiler
namespace rtg {
struct ProfRec { int id; cudaEvent_t a, b; };
static bool g_prof_on = false;
static std::mutex g_prof_mu;
static std::vector<cudaEvent_t> g_prof_pool;
static std::vector<ProfRec> g_prof_recs;
static thread_local cudaEvent_t t_open[K_COUNT];

static cudaEvent_t prof_get_event() {
    if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}
void prof_begin(int id, cudaStream_t s) {
    if (!g_prof_on) return;
    std::lock_guard<std::mutex> lk(g_prof_mu);
    cudaEvent_t e = prof_get_event();
    cudaEventRecord(e, s);
    t_open[id] = e;
}
void prof_end(int id, cudaStream_t s) {
    if (!g_prof_on) return;
    std::lock_guard<std::mutex> lk(g_prof_mu);
    cudaEvent_t e = prof_get_event();
    cudaEventRecord(e, s);
    g_prof_recs.push_back({id, t_open[id], e});
}
static const char *kKernelNames[K_COUNT] = {"preprocess_fwd", "tile_scan", "scatter", "tile_sort", "render_fwd", "render_bwd",
                                            "preprocess_bwd", "adam", "icp_build_level", "icp_iter", "image_glue", "bwd_zero",
                                            "tsdf_integrate", "tsdf_extract", "tsdf_raycast"};
}  // namespace rtg

static thread_local std::string g_err;

// one non-blocking side stream (+ fork / join events) per device, created on first use
struct SideStream {
    cudaStream_t stream;
    cudaEvent_t fork, join;
    std::mutex use;  // held across record(fork) .. wait(join): two host threads running a backward on the same device must not
                     // re-record the shared events between another thread's record and wait
};
static SideStream *side_stream() {
    static std::mutex mu;
    static SideStream table[64];
    static bool made[64] = {false};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    std::lock_guard<std::mutex> lk(mu);
    if (!made[dev]) {
        if (cudaStreamCreateWithFlags(&table[dev].stream, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
        cudaEventCreateWithFlags(&table[dev].fork, cudaEventDisableTiming);
        cudaEventCreateWithFlags(&table[dev].join, cudaEventDisableTiming);
        made[dev] = true;
    }
    return &table[dev];
}

static int fail(int code, const std::string &msg) {
    g_err = msg;
    return code;
}

static int check_launch(const char *what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(RTG_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
    return RTG_OK;
}

static rtg::ViewParams make_view(const RtgSplatView *v) {
    rtg::ViewParams p;
    p.H = v->image_height;
    p.W = v->image_width;
    p.tiles_x = (p.W + RTG_TILE - 1) / RTG_TILE;
    p.tiles_y = (p.H + RTG_TILE - 1) / RTG_TILE;
    p.tanfovx = v->tanfovx;
    p.tanfovy = v->tanfovy;
    // rasterizer_impl.cu:244-245
    p.focal_y = p.H / (2.0f * v->tanfovy);
    p.focal_x = p.W / (2.0f * v->tanfovx);
    p.cx = v->cx;
    p.cy = v->cy;
    p.scale_modifier = v->scale_modifier;
    p.color_sigma = v->color_sigma;
    p.opaque_thr = v->opaque_threshold;
    p.depth_thr = v->depth_threshold;
    p.normal_thr = v->normal_threshold;
    p.T_thr = v->T_threshold;
    p.sh_degree = v->sh_degree;
    p.prefiltered = v->prefiltered & RTG_VIEW_PREFILTERED;
    p.antialiased = (v->prefiltered & RTG_VIEW_ANTIALIASED) ? 1 : 0;
    p.view = v->viewmatrix;
    p.proj = v->projmatrix;
    p.campos = v->campos;
    p.bg = v->bg;
    p.row_begin = 0;
    p.row_end = p.tiles_y;
    return p;
}

// rows of a LOCAL parameter array addressed with the global Gaussian id: base - p_begin rows (integer arithmetic: the
// shifted value is only ever dereferenced at ids >= p_begin)
template <typename T>
static const T *shift_rows(const T *base, int64_t p_begin, size_t elems_per_row) {
    return base ? reinterpret_cast<const T *>(reinterpret_cast<uintptr_t>(base) - (uintptr_t)p_begin * elems_per_row * sizeof(T)) : nullptr;
}
template <typename T>
static T *shift_rows(T *base, int64_t p_begin, size_t elems_per_row) {
    return base ? reinterpret_cast<T *>(reinterpret_cast<uintptr_t>(base) - (uintptr_t)p_begin * elems_per_row * sizeof(T)) : nullptr;
}

extern "C" {

const char *rtg_last_error(void) { return g_err.c_str(); }
int rtg_version(void) { return 100; }

int rtg_splat_workspace_bytes(int32_t P, int32_t H, int32_t W, int64_t R_cap, size_t *geom_bytes, size_t *img_bytes,
                              size_t *bin_bytes) {
    if (P < 0 || H <= 0 || W <= 0 || R_cap < 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_workspace_bytes: bad sizes");
    const size_t T = (size_t)((W + RTG_TILE - 1) / RTG_TILE) * ((H + RTG_TILE - 1) / RTG_TILE);
    size_t g = 0, i = 0, b = 0;
    rtg::geom_from(nullptr, (size_t)P, &g);
    rtg::img_from(nullptr, (size_t)H * W, &i);
    rtg::bin_from(nullptr, T, (size_t)R_cap, &b);
    if (geom_bytes) *geom_bytes = g + 256;
    if (img_bytes) *img_bytes = i + 256;
    if (bin_bytes) *bin_bytes = b + 256;
    return RTG_OK;
}

static int validate_view(const RtgSplatView *v, const char *who) {
    if (!v) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": view is NULL");
    if (v->image_height <= 0 || v->image_width <= 0) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": bad image size");
    if (!v->viewmatrix || !v->projmatrix || !v->campos || !v->bg)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": view matrices / campos / bg must be device pointers");
    if (v->sh_degree < 0 || v->sh_degree > 3) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": sh_degree must be 0..3");
    if (v->prefiltered & ~RTG_VIEW_FLAGS)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": unknown bits in the view flags (prefiltered): " +
                                                  std::to_string(v->prefiltered));
    return RTG_OK;
}

static int validate_inputs(const char *who, const RtgSplatView *view, int32_t n, int32_t M, const float *means3D, const float *shs,
                           const float *colors_precomp, const float *opacities, const float *scales, const float *rotations,
                           const float *cov3D_precomp, const int32_t *radii) {
    if (n <= 0) return RTG_OK;
    if (!means3D || !opacities || !radii) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL means3D / opacities / radii");
    // same exactly-one-of rules as GaussianRasterizer.forward (__init__.py:335-347)
    if ((shs == nullptr) == (colors_precomp == nullptr))
        return fail(RTG_ERR_INVALID_ARGUMENT, "Please provide excatly one of either SHs or precomputed colors!");
    if (((scales == nullptr || rotations == nullptr) && cov3D_precomp == nullptr) ||
        ((scales != nullptr || rotations != nullptr) && cov3D_precomp != nullptr))
        return fail(RTG_ERR_INVALID_ARGUMENT, "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
    if (shs && (M < (view->sh_degree + 1) * (view->sh_degree + 1) || M > 16))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": M must hold (sh_degree+1)^2 coefficients and be <= 16");
    if ((((uintptr_t)rotations) & 15) || (M == 16 && (((uintptr_t)shs) & 15)))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": rotations / shs must be 16-byte aligned");
    return RTG_OK;
}

// clear of the binning counters + forward preprocess of the Gaussians [p_begin, p_end); `fused_histogram`: the tile
// histogram of these Gaussians is built in the same pass (single-GPU forward)
static int forward_preprocess(const rtg::ViewParams &vp, int32_t p_begin, int32_t p_end, int32_t M, const float *means3D,
                              const float *shs, const float *colors_precomp, const float *opacities, const float *scales,
                              const float *rotations, const float *cov3D_precomp, const int32_t *tile_mask, const rtg::GeomState &g,
                              const rtg::BinState &b, int32_t *radii, bool fused_histogram, cudaStream_t s) {
    // tile_count, tile_fill, tile_touched and vis_count are adjacent (bin_from): one clear
    cudaError_t e = cudaMemsetAsync(b.tile_count, 0, (size_t)((char *)b.tile_offset - (char *)b.tile_count), s);
    if (e != cudaSuccess) return fail(RTG_ERR_CUDA, std::string("rtg_splat_forward memset: ") + cudaGetErrorString(e));
    rtg::launch_preprocess_fwd(vp, p_end, M, means3D, scales, rotations, opacities, shs, colors_precomp, cov3D_precomp, tile_mask, g,
                               radii, fused_histogram ? b.tile_count : nullptr, b.tile_touched, b.vis_count, p_begin, s);
    return RTG_OK;
}

// scan -> scatter -> sort -> compositing over the records of all P Gaussians
static int forward_bin_render(const rtg::ViewParams &vp, int32_t P, const int32_t *tile_mask, const rtg::GeomState &g,
                              const rtg::ImgState &img, const rtg::BinState &b, int64_t R_cap, float *out_color, float *out_depth,
                              int32_t *out_hit_color, int32_t *out_hit_depth, float *out_hit_color_weight, float *out_hit_depth_weight,
                              float *out_T, const int32_t *radii, int32_t *counters, int32_t *counters_host, void *scan_done_event,
                              cudaStream_t s) {
    const int T = vp.tiles_x * vp.tiles_y;
    rtg::launch_tile_scan(b, T, R_cap, counters, counters_host, s);
    if (scan_done_event) {
        cudaError_t e = cudaEventRecord(reinterpret_cast<cudaEvent_t>(scan_done_event), s);
        if (e != cudaSuccess) return fail(RTG_ERR_CUDA, std::string("rtg_splat_forward event: ") + cudaGetErrorString(e));
    }
    rtg::launch_scatter(vp, P, g, radii, tile_mask, b, R_cap, counters, s);
    rtg::launch_tile_sort(b, T, counters, s);
    rtg::launch_render_fwd(vp, g, b, img, counters, out_color, out_depth, out_hit_color, out_hit_depth, out_hit_color_weight,
                           out_hit_depth_weight, out_T, s);
    return RTG_OK;
}

int rtg_splat_forward(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                      const float *colors_precomp, const float *opacities, const float *scales, const float *rotations,
                      const float *cov3D_precomp, const int32_t *tile_mask, void *geom_ws, void *img_ws, void *bin_ws,
                      int64_t R_cap, float *out_color, float *out_depth, int32_t *out_hit_color, int32_t *out_hit_depth,
                      float *out_hit_color_weight, float *out_hit_depth_weight, float *out_T, int32_t *radii, int32_t *counters,
                      int32_t *counters_host, void *scan_done_event, void *stream) {
    int rc = validate_view(view, "rtg_splat_forward");
    if (rc) return rc;
    if (P < 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_forward: P < 0");
    if (!out_color || !out_depth || !out_hit_color || !out_hit_depth || !out_hit_color_weight || !out_hit_depth_weight || !out_T ||
        !counters || !geom_ws || !img_ws || !bin_ws || !tile_mask)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_forward: NULL output / workspace / tile_mask pointer");
    rc = validate_inputs("rtg_splat_forward", view, P, M, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, radii);
    if (rc) return rc;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const rtg::ViewParams vp = make_view(view);
    const int T = vp.tiles_x * vp.tiles_y;
    rtg::GeomState g = rtg::geom_from(geom_ws, (size_t)P);
    rtg::ImgState img = rtg::img_from(img_ws, (size_t)vp.H * vp.W);
    rtg::BinState b = rtg::bin_from(bin_ws, (size_t)T, (size_t)R_cap);
    rc = forward_preprocess(vp, 0, P, M, means3D, shs, colors_precomp, opacities, scales, rotations, cov3D_precomp, tile_mask, g, b, radii,
                            true, s);
    if (rc) return rc;
    rc = forward_bin_render(vp, P, tile_mask, g, img, b, R_cap, out_color, out_depth, out_hit_color, out_hit_depth, out_hit_color_weight,
                            out_hit_depth_weight, out_T, radii, counters, counters_host, scan_done_event, s);
    if (rc) return rc;
    return check_launch("rtg_splat_forward");
}

int rtg_splat_geom_layout(int32_t P, size_t *splat_offset, size_t *rgb_offset, size_t *hit_offset, size_t *vis_list_offset) {
    if (P < 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_geom_layout: P < 0");
    rtg::GeomState g = rtg::geom_from(nullptr, (size_t)P);
    if (splat_offset) *splat_offset = (size_t)reinterpret_cast<char *>(g.splat);
    if (rgb_offset) *rgb_offset = (size_t)reinterpret_cast<char *>(g.rgb_flags);
    if (hit_offset) *hit_offset = (size_t)reinterpret_cast<char *>(g.hit);
    if (vis_list_offset) *vis_list_offset = (size_t)reinterpret_cast<char *>(g.vis_list);
    return RTG_OK;
}

int rtg_splat_forward_preprocess(const RtgSplatView *view, int32_t P, int32_t p_begin, int32_t p_end, int32_t M, const float *means3D,
                                 const float *shs, const float *colors_precomp, const float *opacities, const float *scales,
                                 const float *rotations, const float *cov3D_precomp, void *geom_ws, void *bin_ws, int64_t R_cap,
                                 int32_t *radii, void *stream) {
    int rc = validate_view(view, "rtg_splat_forward_preprocess");
    if (rc) return rc;
    if (P < 0 || p_begin < 0 || p_end < p_begin || p_end > P) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_forward_preprocess: bad range");
    if (!geom_ws || !bin_ws || (P > 0 && !radii)) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_forward_preprocess: NULL workspace / radii");
    rc = validate_inputs("rtg_splat_forward_preprocess", view, p_end - p_begin, M, means3D, shs, colors_precomp, opacities, scales,
                         rotations, cov3D_precomp, radii);
    if (rc) return rc;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const rtg::ViewParams vp = make_view(view);
    const int T = vp.tiles_x * vp.tiles_y;
    rtg::GeomState g = rtg::geom_from(geom_ws, (size_t)P);
    rtg::BinState b = rtg::bin_from(bin_ws, (size_t)T, (size_t)R_cap);
    rc = forward_preprocess(vp, p_begin, p_end, M, shift_rows(means3D, p_begin, 3), shift_rows(shs, p_begin, (size_t)3 * M),
                            shift_rows(colors_precomp, p_begin, 3), shift_rows(opacities, p_begin, 1), shift_rows(scales, p_begin, 3),
                            shift_rows(rotations, p_begin, 4), shift_rows(cov3D_precomp, p_begin, 6), nullptr, g, b, radii, false, s);
    if (rc) return rc;
    return check_launch("rtg_splat_forward_preprocess");
}

int rtg_splat_forward_render(const RtgSplatView *view, int32_t P, const int32_t *tile_mask, void *geom_ws, void *img_ws, void *bin_ws,
                             int64_t R_cap, float *out_color, float *out_depth, int32_t *out_hit_color, int32_t *out_hit_depth,
                             float *out_hit_color_weight, float *out_hit_depth_weight, float *out_T, const int32_t *radii,
                             int32_t *counters, int32_t *counters_host, void *scan_done_event, int32_t tile_row_begin,
                             int32_t tile_row_end, void *stream) {
    int rc = validate_view(view, "rtg_splat_forward_render");
    if (rc) return rc;
    if (P < 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_forward_render: P < 0");
    if (!out_color || !out_depth || !out_hit_color || !out_hit_depth || !out_hit_color_weight || !out_hit_depth_weight || !out_T ||
        !counters || !geom_ws || !img_ws || !bin_ws || !tile_mask || (P > 0 && !radii))
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_forward_render: NULL output / workspace / tile_mask / radii pointer");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    rtg::ViewParams vp = make_view(view);
    if (tile_row_end > tile_row_begin) {  // the rows that hold this rank's tiles: rectangles are clipped to them before expansion
        vp.row_begin = tile_row_begin < 0 ? 0 : tile_row_begin;
        vp.row_end = tile_row_end > vp.tiles_y ? vp.tiles_y : tile_row_end;
    }
    const int T = vp.tiles_x * vp.tiles_y;
    rtg::GeomState g = rtg::geom_from(geom_ws, (size_t)P);
    rtg::ImgState img = rtg::img_from(img_ws, (size_t)vp.H * vp.W);
    rtg::BinState b = rtg::bin_from(bin_ws, (size_t)T, (size_t)R_cap);
    // a re-run after a capacity overflow must start from a clean histogram / cursors (vis_count stays)
    cudaError_t e = cudaMemsetAsync(b.tile_count, 0, (size_t)((char *)b.vis_count - (char *)b.tile_count), s);
    if (e != cudaSuccess) return fail(RTG_ERR_CUDA, std::string("rtg_splat_forward_render memset: ") + cudaGetErrorString(e));
    rtg::launch_tile_histogram(vp, P, g, radii, tile_mask, b, s);
    rc = forward_bin_render(vp, P, tile_mask, g, img, b, R_cap, out_color, out_depth, out_hit_color, out_hit_depth, out_hit_color_weight,
                            out_hit_depth_weight, out_T, radii, counters, counters_host, scan_done_event, s);
    if (rc) return rc;
    return check_launch("rtg_splat_forward_render");
}

// phase: 0 = whole backward, 1 = zero-fill + compositing backward (fills the gradient records), 2 = per-Gaussian backward
static int splat_backward_impl(int phase, int32_t p_begin, int32_t p_end, const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                       const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                       const int32_t *radii, const void *geom_ws, const void *img_ws, const void *bin_ws, int64_t R_cap,
                       const int32_t *counters, const float *final_T, const int32_t *hit_image, const float *dL_dcolor, const float *dL_ddepth, float *grad2d_scratch,
                       float *dL_dmeans3D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity, float *dL_dscales,
                       float *dL_drotations, float *dL_dcov3D, float *dL_dmeans2D, void *stream, float *dL_dcamera = nullptr,
                       void *camera_scratch = nullptr, const float *dL_dT = nullptr) {
    int rc = validate_view(view, "rtg_splat_backward");
    if (rc) return rc;
    if (P < 0 || p_begin < 0 || p_end < p_begin || p_end > P) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_backward: bad P / range");
    if (P == 0) {
        if (!dL_dcamera) return RTG_OK;
        // nothing visible: the camera gradient is zero
        cudaError_t e = cudaMemsetAsync(dL_dcamera, 0, 35 * sizeof(float), reinterpret_cast<cudaStream_t>(stream));
        if (e != cudaSuccess) return fail(RTG_ERR_CUDA, std::string("rtg_splat_backward_camera memset: ") + cudaGetErrorString(e));
        return RTG_OK;
    }
    if (!means3D || !radii || !geom_ws || !img_ws || !bin_ws || !counters || !final_T || !hit_image || !dL_dcolor || !dL_ddepth ||
        !grad2d_scratch || !dL_dmeans3D || !dL_dopacity)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_backward: NULL pointer");
    if ((shs == nullptr) == (colors_precomp == nullptr))
        return fail(RTG_ERR_INVALID_ARGUMENT, "Please provide excatly one of either SHs or precomputed colors!");
    if (shs && !dL_dsh) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_backward: dL_dsh is NULL");
    if (colors_precomp && !dL_dcolors_precomp) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_backward: dL_dcolors_precomp is NULL");
    if (cov3D_precomp == nullptr && (!scales || !rotations || !dL_dscales || !dL_drotations))
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_backward: scales / rotations and their gradients are required");
    if (cov3D_precomp != nullptr && !dL_dcov3D) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_backward: dL_dcov3D is NULL");
    if ((((uintptr_t)grad2d_scratch) & 15) || (((uintptr_t)dL_drotations) & 15) || (M == 16 && (((uintptr_t)dL_dsh) & 15)))
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_backward: scratch / dL_drotations / dL_dsh must be 16-byte aligned");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const rtg::ViewParams vp = make_view(view);
    const int T = vp.tiles_x * vp.tiles_y;
    rtg::GeomState g = rtg::geom_from(const_cast<void *>(geom_ws), (size_t)P);
    rtg::ImgState img = rtg::img_from(const_cast<void *>(img_ws), (size_t)vp.H * vp.W);
    rtg::BinState b = rtg::bin_from(const_cast<void *>(bin_ws), (size_t)T, (size_t)R_cap);
    // counters live in the scan output: recompute the overflow word location is not needed -- the
    // backward reads the same device counters the forward wrote.
    // fork: the zero-fill of the culled rows only depends on the forward; it streams to HBM on a side stream while
    // the compute-bound render backward runs, and joins before the call's work on `s` ends
    if (phase == 3) {  // visible rows only: no zero fill
        rtg::launch_render_bwd(vp, g, b, img, counters, final_T, hit_image, dL_dcolor, dL_ddepth, grad2d_scratch, s, dL_dT);
    } else if (phase != 2) {
        SideStream *ss = side_stream();
        std::unique_lock<std::mutex> side_lock;
        if (ss) side_lock = std::unique_lock<std::mutex>(ss->use);
        cudaError_t e = ss ? cudaEventRecord(ss->fork, s) : cudaErrorUnknown;
        if (e == cudaSuccess) e = cudaStreamWaitEvent(ss->stream, ss->fork, 0);
        const bool forked = (e == cudaSuccess);
        rtg::launch_bwd_zero(p_begin, p_end, M, shs != nullptr, cov3D_precomp == nullptr, radii, shift_rows(dL_dmeans3D, p_begin, 3),
                             shift_rows(dL_dsh, p_begin, (size_t)3 * M), shift_rows(dL_dcolors_precomp, p_begin, 3),
                             shift_rows(dL_dopacity, p_begin, 1), shift_rows(dL_dscales, p_begin, 3), shift_rows(dL_drotations, p_begin, 4),
                             shift_rows(dL_dcov3D, p_begin, 6), shift_rows(dL_dmeans2D, p_begin, 3), forked ? ss->stream : s);
        if (forked) cudaEventRecord(ss->join, ss->stream);
        rtg::launch_render_bwd(vp, g, b, img, counters, final_T, hit_image, dL_dcolor, dL_ddepth, grad2d_scratch, s, dL_dT);
        if (forked) cudaStreamWaitEvent(s, ss->join, 0);  // enqueued after both: the zero-fill still overlaps render_bwd
    }
    if (dL_dcamera)  // whole map only (p_begin == 0): the per-Gaussian backward that also reduces the camera terms
        rtg::launch_preprocess_bwd_camera(vp, P, M, means3D, scales, rotations, shs, cov3D_precomp, g, b.vis_count, grad2d_scratch,
                                          dL_dmeans3D, dL_dsh, dL_dcolors_precomp, dL_dopacity, dL_dscales, dL_drotations, dL_dcov3D,
                                          dL_dmeans2D, dL_dcamera, camera_scratch, s);
    else if (phase != 1)  // walks the compact visible list, which holds only Gaussians of [p_begin, p_end)
        rtg::launch_preprocess_bwd(vp, p_end - p_begin, M, shift_rows(means3D, p_begin, 3), shift_rows(scales, p_begin, 3),
                                   shift_rows(rotations, p_begin, 4), shift_rows(shs, p_begin, (size_t)3 * M),
                                   shift_rows(cov3D_precomp, p_begin, 6), g, b.vis_count, grad2d_scratch,
                                   shift_rows(dL_dmeans3D, p_begin, 3), shift_rows(dL_dsh, p_begin, (size_t)3 * M),
                                   shift_rows(dL_dcolors_precomp, p_begin, 3), shift_rows(dL_dopacity, p_begin, 1),
                                   shift_rows(dL_dscales, p_begin, 3), shift_rows(dL_drotations, p_begin, 4),
                                   shift_rows(dL_dcov3D, p_begin, 6), shift_rows(dL_dmeans2D, p_begin, 3), s);
    return check_launch("rtg_splat_backward");
}

#define RTG_BWD_PARAMS                                                                                                             \
    const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs, const float *colors_precomp,          \
        const float *scales, const float *rotations, const float *cov3D_precomp, const int32_t *radii, const void *geom_ws,        \
        const void *img_ws, const void *bin_ws, int64_t R_cap, const int32_t *counters, const float *final_T,                     \
        const int32_t *hit_image, const float *dL_dcolor, const float *dL_ddepth, float *grad2d_scratch, float *dL_dmeans3D,       \
        float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity, float *dL_dscales, float *dL_drotations, float *dL_dcov3D,  \
        float *dL_dmeans2D, void *stream
#define RTG_BWD_ARGS                                                                                                               \
    view, P, M, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, radii, geom_ws, img_ws, bin_ws, R_cap, counters,  \
        final_T, hit_image, dL_dcolor, dL_ddepth, grad2d_scratch, dL_dmeans3D, dL_dsh, dL_dcolors_precomp, dL_dopacity, dL_dscales, \
        dL_drotations, dL_dcov3D, dL_dmeans2D, stream
int rtg_splat_backward(RTG_BWD_PARAMS) { return splat_backward_impl(0, 0, P, RTG_BWD_ARGS); }
int rtg_splat_backward_visible(RTG_BWD_PARAMS) { return splat_backward_impl(3, 0, P, RTG_BWD_ARGS); }
int rtg_splat_backward_render(RTG_BWD_PARAMS) { return splat_backward_impl(1, 0, P, RTG_BWD_ARGS); }
int rtg_splat_backward_finish(RTG_BWD_PARAMS) { return splat_backward_impl(2, 0, P, RTG_BWD_ARGS); }
size_t rtg_splat_camera_scratch_bytes(int32_t P) { return P < 0 ? 0 : rtg::camera_scratch_bytes(P); }

int rtg_splat_backward_camera(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                              const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                              const int32_t *radii, const void *geom_ws, const void *img_ws, const void *bin_ws, int64_t R_cap,
                              const int32_t *counters, const float *final_T, const int32_t *hit_image, const float *dL_dcolor,
                              const float *dL_ddepth, float *grad2d_scratch, float *dL_dmeans3D, float *dL_dsh,
                              float *dL_dcolors_precomp, float *dL_dopacity, float *dL_dscales, float *dL_drotations,
                              float *dL_dcov3D, float *dL_dmeans2D, int32_t visible_rows_only, float *dL_dcamera,
                              void *camera_scratch, void *stream) {
    int rc = validate_view(view, "rtg_splat_backward_camera");
    if (rc) return rc;
    if (P < 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_backward_camera: P < 0");
    if (!dL_dcamera || !camera_scratch)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_backward_camera: dL_dcamera / camera_scratch is NULL");
    if (((uintptr_t)camera_scratch) & 7)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_backward_camera: camera_scratch must be 8-byte aligned");
    return splat_backward_impl(visible_rows_only ? 3 : 0, 0, P, RTG_BWD_ARGS, dL_dcamera, camera_scratch);
}

int rtg_splat_backward_render_shard(int32_t p_begin, int32_t p_end, RTG_BWD_PARAMS) {
    return splat_backward_impl(1, p_begin, p_end, RTG_BWD_ARGS);
}
int rtg_splat_backward_finish_shard(int32_t p_begin, int32_t p_end, RTG_BWD_PARAMS) {
    return splat_backward_impl(2, p_begin, p_end, RTG_BWD_ARGS);
}

// rtg_splat_backward's argument list with dL_dT (H, W) after dL_ddepth
#define RTG_BWD_DT_PARAMS                                                                                                          \
    const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs, const float *colors_precomp,          \
        const float *scales, const float *rotations, const float *cov3D_precomp, const int32_t *radii, const void *geom_ws,        \
        const void *img_ws, const void *bin_ws, int64_t R_cap, const int32_t *counters, const float *final_T,                     \
        const int32_t *hit_image, const float *dL_dcolor, const float *dL_ddepth, const float *dL_dT, float *grad2d_scratch,      \
        float *dL_dmeans3D, float *dL_dsh, float *dL_dcolors_precomp, float *dL_dopacity, float *dL_dscales, float *dL_drotations, \
        float *dL_dcov3D, float *dL_dmeans2D

static int validate_dT(const char *who, const RtgSplatView *view, int32_t P, const float *dL_dT) {
    int rc = validate_view(view, who);
    if (rc) return rc;
    if (P < 0) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": P < 0");
    if (((uintptr_t)dL_dT) & 3) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": dL_dT must be 4-byte aligned");
    return RTG_OK;
}

int rtg_splat_backward_dt(RTG_BWD_DT_PARAMS, int32_t visible_rows_only, float *dL_dcamera, void *camera_scratch, void *stream) {
    int rc = validate_dT("rtg_splat_backward_dt", view, P, dL_dT);
    if (rc) return rc;
    if (dL_dcamera && !camera_scratch) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_backward_dt: camera_scratch is NULL");
    if (dL_dcamera && (((uintptr_t)camera_scratch) & 7))
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_backward_dt: camera_scratch must be 8-byte aligned");
    return splat_backward_impl(visible_rows_only ? 3 : 0, 0, P, RTG_BWD_ARGS, dL_dcamera, dL_dcamera ? camera_scratch : nullptr,
                               dL_dT);
}

int rtg_splat_backward_render_dt(int32_t p_begin, int32_t p_end, RTG_BWD_DT_PARAMS, void *stream) {
    int rc = validate_dT("rtg_splat_backward_render_dt", view, P, dL_dT);
    if (rc) return rc;
    if (p_begin < 0 || p_end < p_begin || p_end > P) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_backward_render_dt: bad range");
    return splat_backward_impl(1, p_begin, p_end, RTG_BWD_ARGS, nullptr, nullptr, dL_dT);
}

int rtg_splat_backward_pose(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                            const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                            const int32_t *radii, const void *geom_ws, const void *img_ws, const void *bin_ws, int64_t R_cap,
                            const int32_t *counters, const float *final_T, const int32_t *hit_image, const float *dL_dcolor,
                            const float *dL_ddepth, const float *dL_dT, float *grad2d_scratch, float *dL_dcamera,
                            void *camera_scratch, void *stream) {
    const char *who = "rtg_splat_backward_pose";
    int rc = validate_dT(who, view, P, dL_dT);
    if (rc) return rc;
    if (!dL_dcamera || !camera_scratch)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": dL_dcamera / camera_scratch is NULL");
    if (((uintptr_t)camera_scratch) & 7)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": camera_scratch must be 8-byte aligned");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (P == 0) {  // nothing visible: the camera gradient is zero
        cudaError_t e = cudaMemsetAsync(dL_dcamera, 0, 35 * sizeof(float), s);
        if (e != cudaSuccess) return fail(RTG_ERR_CUDA, std::string(who) + " memset: " + cudaGetErrorString(e));
        return RTG_OK;
    }
    if (!means3D || !radii || !geom_ws || !img_ws || !bin_ws || !counters || !final_T || !hit_image || !dL_dcolor || !dL_ddepth ||
        !grad2d_scratch)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL pointer");
    if ((shs == nullptr) == (colors_precomp == nullptr))
        return fail(RTG_ERR_INVALID_ARGUMENT, "Please provide excatly one of either SHs or precomputed colors!");
    if (((scales == nullptr || rotations == nullptr) && cov3D_precomp == nullptr) ||
        ((scales != nullptr || rotations != nullptr) && cov3D_precomp != nullptr))
        return fail(RTG_ERR_INVALID_ARGUMENT, "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
    if (shs && (M < (view->sh_degree + 1) * (view->sh_degree + 1) || M > 16))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": M must hold (sh_degree+1)^2 coefficients and be <= 16");
    if ((((uintptr_t)grad2d_scratch) & 15) || (((uintptr_t)rotations) & 15) || (M == 16 && (((uintptr_t)shs) & 15)))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": grad2d_scratch / rotations / shs must be 16-byte aligned");
    const rtg::ViewParams vp = make_view(view);
    const int T = vp.tiles_x * vp.tiles_y;
    rtg::GeomState g = rtg::geom_from(const_cast<void *>(geom_ws), (size_t)P);
    rtg::ImgState img = rtg::img_from(const_cast<void *>(img_ws), (size_t)vp.H * vp.W);
    rtg::BinState b = rtg::bin_from(const_cast<void *>(bin_ws), (size_t)T, (size_t)R_cap);
    rtg::launch_render_bwd(vp, g, b, img, counters, final_T, hit_image, dL_dcolor, dL_ddepth, grad2d_scratch, s, dL_dT);
    rtg::launch_preprocess_bwd_pose(vp, P, M, means3D, scales, rotations, shs, cov3D_precomp, g, b.vis_count, grad2d_scratch,
                                    dL_dcamera, camera_scratch, s);
    return check_launch(who);
}

size_t rtg_splat_pose_gn_scratch_bytes(int32_t P, int32_t H, int32_t W) {
    return (P < 0 || H <= 0 || W <= 0) ? 0 : rtg::pose_gn_scratch_bytes(P, H, W);
}

// Checks shared by the two tangent entry points: the forward's state and the Gaussian inputs it was rendered from.
static int validate_pose_tangent_inputs(const char *who, const RtgSplatView *view, int32_t P, int32_t M, const float *means3D,
                                        const float *shs, const float *colors_precomp, const float *scales, const float *rotations,
                                        const float *cov3D_precomp, const void *geom_ws, const void *img_ws, const void *bin_ws,
                                        int64_t R_cap, const int32_t *counters, const int32_t *hit_image, const void *scratch,
                                        bool need_hit = true) {
    int rc = validate_view(view, who);
    if (rc) return rc;
    if (P < 1) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": P must be >= 1");
    if (R_cap < 0) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": R_cap < 0");
    if (!means3D || !geom_ws || !img_ws || !bin_ws || !counters || (need_hit && !hit_image) || !scratch)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL pointer");
    if ((shs == nullptr) == (colors_precomp == nullptr))
        return fail(RTG_ERR_INVALID_ARGUMENT, "Please provide excatly one of either SHs or precomputed colors!");
    if (((scales == nullptr || rotations == nullptr) && cov3D_precomp == nullptr) ||
        ((scales != nullptr || rotations != nullptr) && cov3D_precomp != nullptr))
        return fail(RTG_ERR_INVALID_ARGUMENT, "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
    if (shs && (M < (view->sh_degree + 1) * (view->sh_degree + 1) || M > 16))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": M must hold (sh_degree+1)^2 coefficients and be <= 16");
    if ((((uintptr_t)scratch) & 15) || (((uintptr_t)rotations) & 15) || (M == 16 && (((uintptr_t)shs) & 15)))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": scratch / rotations / shs must be 16-byte aligned");
    return RTG_OK;
}

int rtg_splat_pose_tangents(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                            const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                            const void *geom_ws, const void *img_ws, const void *bin_ws, int64_t R_cap, const int32_t *counters,
                            const int32_t *hit_image, void *scratch, float *J, void *stream) {
    const char *who = "rtg_splat_pose_tangents";
    int rc = validate_pose_tangent_inputs(who, view, P, M, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, geom_ws,
                                          img_ws, bin_ws, R_cap, counters, hit_image, scratch);
    if (rc) return rc;
    if (!J) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": J is NULL");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const rtg::ViewParams vp = make_view(view);
    const int T = vp.tiles_x * vp.tiles_y;
    rtg::GeomState g = rtg::geom_from(const_cast<void *>(geom_ws), (size_t)P);
    rtg::ImgState img = rtg::img_from(const_cast<void *>(img_ws), (size_t)vp.H * vp.W);
    rtg::BinState b = rtg::bin_from(const_cast<void *>(bin_ws), (size_t)T, (size_t)R_cap);
    rtg::launch_preprocess_tangent(vp, P, M, means3D, scales, rotations, shs, cov3D_precomp, g, b.vis_count,
                                   reinterpret_cast<float4 *>(scratch), s);
    rtg::launch_render_tangent_images(vp, P, g, b, img, counters, hit_image, scratch, J, s);
    return check_launch(who);
}

int rtg_splat_pose_tangents_expected(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                                     const float *colors_precomp, const float *scales, const float *rotations,
                                     const float *cov3D_precomp, const void *geom_ws, const void *img_ws, const void *bin_ws,
                                     int64_t R_cap, const int32_t *counters, void *scratch, float *J, float *expected,
                                     void *stream) {
    const char *who = "rtg_splat_pose_tangents_expected";
    int rc = validate_pose_tangent_inputs(who, view, P, M, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, geom_ws,
                                          img_ws, bin_ws, R_cap, counters, nullptr, scratch, false);
    if (rc) return rc;
    if (!J || !expected) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": J / expected is NULL");
    if ((((uintptr_t)J) | ((uintptr_t)expected)) & 3)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": J / expected must be 4-byte aligned");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const rtg::ViewParams vp = make_view(view);
    const int T = vp.tiles_x * vp.tiles_y;
    rtg::GeomState g = rtg::geom_from(const_cast<void *>(geom_ws), (size_t)P);
    rtg::ImgState img = rtg::img_from(const_cast<void *>(img_ws), (size_t)vp.H * vp.W);
    rtg::BinState b = rtg::bin_from(const_cast<void *>(bin_ws), (size_t)T, (size_t)R_cap);
    rtg::launch_preprocess_tangent(vp, P, M, means3D, scales, rotations, shs, cov3D_precomp, g, b.vis_count,
                                   reinterpret_cast<float4 *>(scratch), s);
    rtg::launch_render_tangent_expected_images(vp, P, g, b, img, counters, scratch, J, expected, s);
    return check_launch(who);
}

int rtg_splat_contributions(const RtgSplatView *view, int32_t P, const void *geom_ws, const void *img_ws, const void *bin_ws,
                            int64_t R_cap, const int32_t *counters, const float *pixel_error, int32_t *n_pixels, float *weight,
                            float *error, void *stream) {
    const char *who = "rtg_splat_contributions";
    int rc = validate_view(view, who);
    if (rc) return rc;
    if (P < 0) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": P < 0");
    if (R_cap < 0) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": R_cap < 0");
    if (!geom_ws || !img_ws || !bin_ws || !counters)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL workspace / counters");
    if (P > 0 && (!n_pixels || !weight)) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL n_pixels / weight");
    if ((error == nullptr) != (pixel_error == nullptr))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": error and pixel_error must be given together");
    if ((((uintptr_t)n_pixels) | ((uintptr_t)weight) | ((uintptr_t)error) | ((uintptr_t)pixel_error)) & 3)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": outputs / pixel_error must be 4-byte aligned");
    if (P == 0) return RTG_OK;  // no Gaussian, no tile list entry
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const rtg::ViewParams vp = make_view(view);
    const int T = vp.tiles_x * vp.tiles_y;
    rtg::GeomState g = rtg::geom_from(const_cast<void *>(geom_ws), (size_t)P);
    rtg::ImgState img = rtg::img_from(const_cast<void *>(img_ws), (size_t)vp.H * vp.W);
    rtg::BinState b = rtg::bin_from(const_cast<void *>(bin_ws), (size_t)T, (size_t)R_cap);
    rtg::launch_render_contributions(vp, g, b, img, counters, pixel_error, n_pixels, weight, error, s);
    return check_launch(who);
}

// The checks the two feature entry points share; `in` is the (P, C) features or the (C, H, W) upstream gradient, `out` the
// other one.
static int validate_features(const char *who, const RtgSplatView *view, int32_t P, const void *geom_ws, const void *img_ws,
                             const void *bin_ws, int64_t R_cap, const int32_t *counters, int32_t C, const float *in,
                             const float *out, bool out_needed) {
    int rc = validate_view(view, who);
    if (rc) return rc;
    if (P < 0) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": P < 0");
    if (R_cap < 0) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": R_cap < 0");
    if (C < 1 || C > RTG_FEATURES_MAX)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": C must be 1.." + std::to_string(RTG_FEATURES_MAX) +
                                                  ", got " + std::to_string(C));
    if (P > 0 && (!geom_ws || !img_ws || !bin_ws || !counters))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL workspace / counters");
    if ((P > 0 || out_needed) && !out) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL output");
    if (P > 0 && !in) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL input");
    if ((((uintptr_t)in) | ((uintptr_t)out)) & 3)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": input / output must be 4-byte aligned");
    return RTG_OK;
}

int rtg_splat_features(const RtgSplatView *view, int32_t P, const void *geom_ws, const void *img_ws, const void *bin_ws,
                       int64_t R_cap, const int32_t *counters, int32_t C, const float *features, float *out, void *stream) {
    const char *who = "rtg_splat_features";
    int rc = validate_features(who, view, P, geom_ws, img_ws, bin_ws, R_cap, counters, C, features, out, true);
    if (rc) return rc;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const rtg::ViewParams vp = make_view(view);
    if (P == 0) {  // no Gaussian: an empty map
        cudaError_t e = cudaMemsetAsync(out, 0, (size_t)C * vp.H * vp.W * sizeof(float), s);
        if (e != cudaSuccess) return fail(RTG_ERR_CUDA, std::string(who) + " memset: " + cudaGetErrorString(e));
        return RTG_OK;
    }
    const int T = vp.tiles_x * vp.tiles_y;
    rtg::GeomState g = rtg::geom_from(const_cast<void *>(geom_ws), (size_t)P);
    rtg::ImgState img = rtg::img_from(const_cast<void *>(img_ws), (size_t)vp.H * vp.W);
    rtg::BinState b = rtg::bin_from(const_cast<void *>(bin_ws), (size_t)T, (size_t)R_cap);
    rtg::launch_render_features(vp, g, b, img, counters, C, features, out, s);
    return check_launch(who);
}

int rtg_splat_features_backward(const RtgSplatView *view, int32_t P, const void *geom_ws, const void *img_ws, const void *bin_ws,
                                int64_t R_cap, const int32_t *counters, int32_t C, const float *dL_dout, float *dL_dfeatures,
                                void *stream) {
    const char *who = "rtg_splat_features_backward";
    int rc = validate_features(who, view, P, geom_ws, img_ws, bin_ws, R_cap, counters, C, dL_dout, dL_dfeatures, false);
    if (rc) return rc;
    if (P == 0) return RTG_OK;  // no row to write
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const rtg::ViewParams vp = make_view(view);
    cudaError_t e = cudaMemsetAsync(dL_dfeatures, 0, (size_t)P * C * sizeof(float), s);  // rows the frame never blends
    if (e != cudaSuccess) return fail(RTG_ERR_CUDA, std::string(who) + " memset: " + cudaGetErrorString(e));
    const int T = vp.tiles_x * vp.tiles_y;
    rtg::GeomState g = rtg::geom_from(const_cast<void *>(geom_ws), (size_t)P);
    rtg::ImgState img = rtg::img_from(const_cast<void *>(img_ws), (size_t)vp.H * vp.W);
    rtg::BinState b = rtg::bin_from(const_cast<void *>(bin_ws), (size_t)T, (size_t)R_cap);
    rtg::launch_render_features_bwd(vp, g, b, img, counters, C, dL_dout, dL_dfeatures, s);
    return check_launch(who);
}

int rtg_splat_features_backward_geometry(const RtgSplatView *view, int32_t P, const float *means3D, const float *scales,
                                         const float *rotations, const float *cov3D_precomp, const int32_t *radii,
                                         const void *geom_ws, const void *img_ws, const void *bin_ws, int64_t R_cap,
                                         const int32_t *counters, int32_t C, const float *features, const float *dL_dout,
                                         float *grad2d_scratch, float *dL_dmeans3D, float *dL_dopacity, float *dL_dscales,
                                         float *dL_drotations, float *dL_dcov3D, int32_t visible_rows_only, float *dL_dcamera,
                                         void *camera_scratch, void *stream) {
    const char *who = "rtg_splat_features_backward_geometry";
    auto bad = [&](const std::string &msg) { return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": " + msg); };
    int rc = validate_view(view, who);
    if (rc) return rc;
    if (P < 0) return bad("P < 0");
    if (R_cap < 0) return bad("R_cap < 0");
    if (C < 1 || C > RTG_FEATURES_MAX)
        return bad("C must be 1.." + std::to_string(RTG_FEATURES_MAX) + ", got " + std::to_string(C));
    const bool per_gaussian = dL_dmeans3D || dL_dopacity || dL_dscales || dL_drotations || dL_dcov3D;
    if (!per_gaussian && !dL_dcamera) return bad("no output: give the per-Gaussian gradients, dL_dcamera or both");
    if (dL_dcamera && !camera_scratch) return bad("camera_scratch is NULL");
    if (((uintptr_t)camera_scratch) & 7) return bad("camera_scratch must be 8-byte aligned");
    if ((dL_dscales || dL_drotations) && (!scales || !rotations)) return bad("dL_dscales / dL_drotations without scales / rotations");
    if (dL_dcov3D && !cov3D_precomp) return bad("dL_dcov3D without cov3D_precomp");
    if ((((uintptr_t)features) | ((uintptr_t)dL_dout) | ((uintptr_t)dL_dmeans3D) | ((uintptr_t)dL_dopacity) |
         ((uintptr_t)dL_dscales) | ((uintptr_t)dL_dcov3D) | ((uintptr_t)dL_dcamera)) & 3)
        return bad("features / dL_dout / gradients must be 4-byte aligned");
    if ((((uintptr_t)grad2d_scratch) | ((uintptr_t)rotations) | ((uintptr_t)dL_drotations)) & 15)
        return bad("grad2d_scratch / rotations / dL_drotations must be 16-byte aligned");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (P == 0) {  // nothing visible: the camera gradient is zero, and there is no row to write
        if (!dL_dcamera) return RTG_OK;
        cudaError_t e = cudaMemsetAsync(dL_dcamera, 0, 35 * sizeof(float), s);
        if (e != cudaSuccess) return fail(RTG_ERR_CUDA, std::string(who) + " memset: " + cudaGetErrorString(e));
        return RTG_OK;
    }
    if (!geom_ws || !img_ws || !bin_ws || !counters) return bad("NULL workspace / counters");
    if (!means3D || !features || !dL_dout || !grad2d_scratch) return bad("NULL means3D / features / dL_dout / grad2d_scratch");
    if (((scales == nullptr || rotations == nullptr) && cov3D_precomp == nullptr) ||
        ((scales != nullptr || rotations != nullptr) && cov3D_precomp != nullptr))
        return fail(RTG_ERR_INVALID_ARGUMENT, "Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!");
    if (per_gaussian) {
        if (!dL_dmeans3D || !dL_dopacity) return bad("dL_dmeans3D / dL_dopacity is NULL");
        if (scales && (!dL_dscales || !dL_drotations)) return bad("dL_dscales / dL_drotations is NULL");
        if (cov3D_precomp && !dL_dcov3D) return bad("dL_dcov3D is NULL");
        if (!visible_rows_only && !radii) return bad("radii is NULL (the culled rows are zero-filled from it)");
    }
    const rtg::ViewParams vp = make_view(view);
    const int T = vp.tiles_x * vp.tiles_y;
    rtg::GeomState g = rtg::geom_from(const_cast<void *>(geom_ws), (size_t)P);
    rtg::ImgState img = rtg::img_from(const_cast<void *>(img_ws), (size_t)vp.H * vp.W);
    rtg::BinState b = rtg::bin_from(const_cast<void *>(bin_ws), (size_t)T, (size_t)R_cap);
    rtg::launch_render_features_grad(vp, g, b, img, counters, C, features, dL_dout, grad2d_scratch, s);
    // the record holds moments only (no colour, no depth path): the per-Gaussian pass reads no SH row and writes no
    // colour gradient
    if (!per_gaussian) {
        rtg::launch_preprocess_bwd_pose(vp, P, 0, means3D, scales, rotations, nullptr, cov3D_precomp, g, b.vis_count, grad2d_scratch,
                                        dL_dcamera, camera_scratch, s);
        return check_launch(who);
    }
    if (!visible_rows_only)
        rtg::launch_bwd_zero(0, P, 0, false, cov3D_precomp == nullptr, radii, dL_dmeans3D, nullptr, nullptr, dL_dopacity, dL_dscales,
                             dL_drotations, dL_dcov3D, nullptr, s);
    if (dL_dcamera)
        rtg::launch_preprocess_bwd_camera(vp, P, 0, means3D, scales, rotations, nullptr, cov3D_precomp, g, b.vis_count, grad2d_scratch,
                                          dL_dmeans3D, nullptr, nullptr, dL_dopacity, dL_dscales, dL_drotations, dL_dcov3D, nullptr,
                                          dL_dcamera, camera_scratch, s);
    else
        rtg::launch_preprocess_bwd(vp, P, 0, means3D, scales, rotations, nullptr, cov3D_precomp, g, b.vis_count, grad2d_scratch,
                                   dL_dmeans3D, nullptr, nullptr, dL_dopacity, dL_dscales, dL_drotations, dL_dcov3D, nullptr, s);
    return check_launch(who);
}

// The step of the Gauss-Newton entry points: `robust` selects the normal-equation rows (RTG_ROBUST_NONE: the plain ones),
// `ab` (the device exposure, or nullptr) the eight-unknown step, `expected` the expected-depth residual on S_e(min_cov).
static int pose_gn_step(const char *who, const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                        const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                        const void *geom_ws, const void *img_ws, const void *bin_ws, int64_t R_cap, const int32_t *counters,
                        const RtgPoseGN *st, const RtgPoseRobust &robust, double *ab, void *stream, bool expected = false,
                        float min_cov = 0.f) {
    int rc = validate_pose_tangent_inputs(who, view, P, M, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, geom_ws,
                                          img_ws, bin_ws, R_cap, counters, st->hit_depth, st->scratch);
    if (rc) return rc;
    if (!st->pose || !st->projection || !st->viewmatrix || !st->projmatrix || !st->campos || !st->report)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL pose / projection / camera array / report");
    if (!st->render || !st->depth || !st->gt_color || !st->gt_depth)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL render / depth / gt_color / gt_depth");
    if ((((uintptr_t)st->pose) | ((uintptr_t)st->report)) & 7)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": pose / report must be 8-byte aligned");
    if (!(st->damping >= 0.f) || !(st->color_weight >= 0.f) || !(st->depth_weight >= 0.f))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": damping and weights must be >= 0");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const rtg::ViewParams vp = make_view(view);
    const int T = vp.tiles_x * vp.tiles_y;
    rtg::GeomState g = rtg::geom_from(const_cast<void *>(geom_ws), (size_t)P);
    rtg::ImgState img = rtg::img_from(const_cast<void *>(img_ws), (size_t)vp.H * vp.W);
    rtg::BinState b = rtg::bin_from(const_cast<void *>(bin_ws), (size_t)T, (size_t)R_cap);
    rtg::launch_preprocess_tangent(vp, P, M, means3D, scales, rotations, shs, cov3D_precomp, g, b.vis_count,
                                   reinterpret_cast<float4 *>(st->scratch), s);
    if (expected) rtg::launch_pose_gn_expected_step(vp, P, g, b, img, counters, *st, robust, ab, min_cov, s);
    else if (ab) rtg::launch_pose_gn_exposure_step(vp, P, g, b, img, counters, *st, robust, ab, s);
    else rtg::launch_pose_gn_normal_eq_step(vp, P, g, b, img, counters, *st, robust, s);
    return check_launch(who);
}

int rtg_splat_pose_gn_step(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                           const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                           const void *geom_ws, const void *img_ws, const void *bin_ws, int64_t R_cap, const int32_t *counters,
                           const RtgPoseGN *st, void *stream) {
    const char *who = "rtg_splat_pose_gn_step";
    if (!st) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": state is NULL");
    const RtgPoseRobust none{RTG_ROBUST_NONE, 0.f, 0.f, 0};
    return pose_gn_step(who, view, P, M, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, geom_ws, img_ws, bin_ws,
                        R_cap, counters, st, none, nullptr, stream);
}

static int validate_pose_robust(const char *who, const RtgPoseGN *st, const RtgPoseRobust *robust) {
    if (!st) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": state is NULL");
    if (!robust) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": robust is NULL");
    if (robust->kernel != RTG_ROBUST_NONE && robust->kernel != RTG_ROBUST_HUBER)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": unknown robust kernel");
    if (robust->kernel == RTG_ROBUST_HUBER &&
        !(std::isfinite(robust->color_delta) && robust->color_delta > 0.f && std::isfinite(robust->depth_delta) &&
          robust->depth_delta > 0.f))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": color_delta and depth_delta must be positive and finite");
    return RTG_OK;
}

int rtg_splat_pose_gn_step_robust(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                                  const float *colors_precomp, const float *scales, const float *rotations, const float *cov3D_precomp,
                                  const void *geom_ws, const void *img_ws, const void *bin_ws, int64_t R_cap, const int32_t *counters,
                                  const RtgPoseGN *st, const RtgPoseRobust *robust, void *stream) {
    const char *who = "rtg_splat_pose_gn_step_robust";
    int rc = validate_pose_robust(who, st, robust);
    if (rc) return rc;
    return pose_gn_step(who, view, P, M, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, geom_ws, img_ws, bin_ws,
                        R_cap, counters, st, *robust, nullptr, stream);
}

size_t rtg_splat_pose_gn_exposure_scratch_bytes(int32_t P, int32_t H, int32_t W) {
    return (P < 0 || H <= 0 || W <= 0) ? 0 : rtg::pose_gn_exposure_scratch_bytes(P, H, W);
}

int rtg_splat_pose_gn_step_exposure(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                                    const float *colors_precomp, const float *scales, const float *rotations,
                                    const float *cov3D_precomp, const void *geom_ws, const void *img_ws, const void *bin_ws,
                                    int64_t R_cap, const int32_t *counters, const RtgPoseGN *st, const RtgPoseRobust *robust,
                                    const RtgPoseExposure *exposure, void *stream) {
    const char *who = "rtg_splat_pose_gn_step_exposure";
    int rc = validate_pose_robust(who, st, robust);
    if (rc) return rc;
    if (!exposure) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": exposure is NULL");
    if (!exposure->ab) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": exposure ab is NULL");
    if (((uintptr_t)exposure->ab) & 7) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": exposure ab must be 8-byte aligned");
    return pose_gn_step(who, view, P, M, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, geom_ws, img_ws, bin_ws,
                        R_cap, counters, st, *robust, exposure->ab, stream);
}

int rtg_splat_pose_gn_step_expected(const RtgSplatView *view, int32_t P, int32_t M, const float *means3D, const float *shs,
                                    const float *colors_precomp, const float *scales, const float *rotations,
                                    const float *cov3D_precomp, const void *geom_ws, const void *img_ws, const void *bin_ws,
                                    int64_t R_cap, const int32_t *counters, const RtgPoseGN *st, const RtgPoseRobust *robust,
                                    const RtgPoseExposure *exposure, float min_coverage, void *stream) {
    const char *who = "rtg_splat_pose_gn_step_expected";
    int rc = validate_pose_robust(who, st, robust);
    if (rc) return rc;
    if (!(min_coverage > 0.f && min_coverage <= 1.f))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": min_coverage must be in (0, 1]");
    double *ab = nullptr;
    if (exposure) {
        if (!exposure->ab) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": exposure ab is NULL");
        if (((uintptr_t)exposure->ab) & 7)
            return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": exposure ab must be 8-byte aligned");
        ab = exposure->ab;
    }
    return pose_gn_step(who, view, P, M, means3D, shs, colors_precomp, scales, rotations, cov3D_precomp, geom_ws, img_ws, bin_ws,
                        R_cap, counters, st, *robust, ab, stream, true, min_coverage);
}

int rtg_pose_adam_step(const RtgPoseAdam *st, void *stream) {
    if (!st) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_pose_adam_step: state is NULL");
    if (!st->pose || !st->exp_avg || !st->exp_avg_sq)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_pose_adam_step: NULL pose / exp_avg / exp_avg_sq");
    if (!st->projection || !st->viewmatrix || !st->projmatrix || !st->campos)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_pose_adam_step: NULL projection / viewmatrix / projmatrix / campos");
    if (((uintptr_t)st->pose) & 7) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_pose_adam_step: pose must be 8-byte aligned");
    if (st->step < 1) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_pose_adam_step: step must be >= 1");
    rtg::launch_pose_adam_step(*st, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_pose_adam_step");
}

int rtg_splat_mark_visible(int32_t P, const float *means3D, const float *viewmatrix, const float *projmatrix, uint8_t *present,
                           void *stream) {
    if (P < 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_mark_visible: P < 0");
    if (P == 0) return RTG_OK;
    if (!means3D || !viewmatrix || !projmatrix || !present) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_splat_mark_visible: NULL pointer");
    rtg::launch_mark_visible(P, means3D, viewmatrix, projmatrix, present, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_splat_mark_visible");
}

int rtg_adam_step(const RtgAdamGroup *groups, int32_t n_groups, float beta1, float beta2, float eps, int32_t step, void *stream) {
    if (!groups || n_groups <= 0 || n_groups > RTG_ADAM_MAX_GROUPS) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_adam_step: bad groups");
    if (step < 1) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_adam_step: step must be >= 1");
    for (int i = 0; i < n_groups; i++)
        if (groups[i].grad && (!groups[i].param || !groups[i].exp_avg || !groups[i].exp_avg_sq))
            return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_adam_step: NULL param / state pointer");
    rtg::launch_adam(groups, n_groups, beta1, beta2, eps, step, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_adam_step");
}

int rtg_map_adam_step(const RtgMapStep *st, void *stream) {
    if (!st) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_adam_step: NULL step");
    if (st->P < 0 || st->step < 1) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_adam_step: P must be >= 0 and step >= 1");
    if (st->P == 0) return RTG_OK;
    const void *need[] = {st->xyz, st->sh, st->opacity_raw, st->scaling_raw, st->rotation_raw, st->m_xyz, st->m_sh, st->m_opacity,
                          st->m_scaling, st->m_rotation, st->v_xyz, st->v_sh, st->v_opacity, st->v_scaling, st->v_rotation,
                          st->g_means3D, st->g_sh, st->g_opacity, st->g_scales, st->g_rotations, st->scales_out, st->rotations_out,
                          st->opacities_out};
    for (const void *q : need)
        if (!q) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_adam_step: NULL parameter / state / gradient / output pointer");
    const void *al16[] = {st->sh, st->m_sh, st->v_sh, st->g_sh, st->rotation_raw, st->m_rotation, st->v_rotation, st->g_rotations,
                          st->rotations_out, st->rotation0};
    for (const void *q : al16)
        if (((uintptr_t)q) & 15) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_adam_step: sh / rotation tensors must be 16-byte aligned");
    if (st->attach_mask && (!st->xyz0 || !st->scaling0 || !st->rotation0))
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_adam_step: attach_mask needs xyz0, scaling0 and rotation0");
    if (st->attach_mask && st->attach_count < 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_adam_step: attach_count < 0");
    rtg::launch_map_adam_step(*st, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_map_adam_step");
}

int rtg_map_activate(int32_t P, const float *scaling_raw, const float *rotation_raw, const float *opacity_raw, float *scales_out,
                     float *rotations_out, float *opacities_out, float *normal_out, void *stream) {
    if (P < 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_activate: P < 0");
    if (P == 0) return RTG_OK;
    if (!scaling_raw || !rotation_raw || !opacity_raw || !scales_out || !rotations_out || !opacities_out)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_activate: NULL pointer");
    if ((((uintptr_t)rotation_raw) | ((uintptr_t)rotations_out)) & 15)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_activate: rotation tensors must be 16-byte aligned");
    rtg::launch_map_activate(P, scaling_raw, rotation_raw, opacity_raw, scales_out, rotations_out, opacities_out, normal_out,
                             reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_map_activate");
}

int rtg_map_history_merge(const RtgHistoryMerge *m, void *stream) {
    if (!m) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_history_merge: merge is NULL");
    if (m->P < 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_history_merge: P < 0");
    if (m->P == 0 || !(m->max_weight > 0.f)) return RTG_OK;
    if (!m->hist_confidence || !m->confidence || !m->hist_xyz || !m->xyz || !m->hist_features_dc || !m->features_dc ||
        !m->hist_features_rest || !m->features_rest || !m->hist_scaling || !m->scaling || !m->hist_rotation || !m->rotation_raw)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_history_merge: NULL pointer");
    if (m->features_rest_width < 0 || m->features_dc_stride < 3 || m->features_rest_stride < m->features_rest_width)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_history_merge: bad feature strides");
    if ((((uintptr_t)m->hist_rotation) | ((uintptr_t)m->rotation_raw)) & 15)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_history_merge: rotation tensors must be 16-byte aligned");
    rtg::launch_history_merge(*m, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_map_history_merge");
}

size_t rtg_icp_workspace_bytes(int32_t H, int32_t W) {
    (void)H; (void)W;
    return rtg::icp_ws_bytes();
}

int rtg_icp_build_level(const float *depth, int32_t H, int32_t W, int32_t pool, float fx, float fy, float cx, float cy,
                        float *vertex_out, float *normal_out, void *ws, void *stream) {
    if (!depth || !vertex_out || !normal_out || !ws || H <= 0 || W <= 0 || pool < 1 || H / pool < 1 || W / pool < 1)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_icp_build_level: bad arguments");
    rtg::launch_icp_build_level(depth, H, W, pool, fx, fy, cx, cy, vertex_out, normal_out, ws, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_icp_build_level");
}

int rtg_icp_solve_level(const float *vertex0, const float *normal0, const float *vertex1, const float *normal1, int32_t H, int32_t W,
                        float fx, float fy, float cx, float cy, float distance_threshold, float normal_cos_threshold, float damping,
                        int32_t iters, float *pose, float *valid_ratio, void *ws, void *stream) {
    if (!vertex0 || !normal0 || !vertex1 || !normal1 || !pose || !ws || H <= 0 || W <= 0 || iters < 0)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_icp_solve_level: bad arguments");
    rtg::launch_icp_solve_level(vertex0, normal0, vertex1, normal1, H, W, fx, fy, cx, cy, distance_threshold, normal_cos_threshold,
                                damping, iters, pose, valid_ratio, ws, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_icp_solve_level");
}

int rtg_icp_build_pyramid(const float *depth, int32_t H, int32_t W, int32_t n_levels, const int32_t *pools, const float *fx,
                          const float *fy, const float *cx, const float *cy, float *const *vertex_out, float *const *normal_out,
                          void *ws, void *stream) {
    if (!depth || !pools || !fx || !fy || !cx || !cy || !vertex_out || !normal_out || !ws || H <= 0 || W <= 0 || n_levels < 1 ||
        n_levels > RTG_ICP_MAX_LEVELS)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_icp_build_pyramid: bad arguments");
    rtg::IcpPyramid p;
    p.depth = depth; p.H = H; p.W = W; p.n_levels = n_levels;
    for (int l = 0; l < n_levels; l++) {
        if (pools[l] < 1 || H / pools[l] < 1 || W / pools[l] < 1 || !vertex_out[l] || !normal_out[l])
            return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_icp_build_pyramid: bad level");
        p.pool[l] = pools[l]; p.fx[l] = fx[l]; p.fy[l] = fy[l]; p.cx[l] = cx[l]; p.cy[l] = cy[l];
        p.vertex[l] = vertex_out[l]; p.normal[l] = normal_out[l];
    }
    // the grid is sized for the finest level: order the levels so that the last one has the smallest pool
    int finest = 0;
    for (int l = 1; l < n_levels; l++)
        if (p.pool[l] < p.pool[finest]) finest = l;
    if (finest != n_levels - 1) {
        std::swap(p.pool[finest], p.pool[n_levels - 1]); std::swap(p.fx[finest], p.fx[n_levels - 1]);
        std::swap(p.fy[finest], p.fy[n_levels - 1]); std::swap(p.cx[finest], p.cx[n_levels - 1]);
        std::swap(p.cy[finest], p.cy[n_levels - 1]); std::swap(p.vertex[finest], p.vertex[n_levels - 1]);
        std::swap(p.normal[finest], p.normal[n_levels - 1]);
    }
    cudaError_t e = rtg::launch_icp_pyramid(p, ws, reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(RTG_ERR_CUDA, std::string("rtg_icp_build_pyramid: ") + cudaGetErrorString(e));
    return check_launch("rtg_icp_build_pyramid");
}

int rtg_icp_predict_pose(const RtgIcpLevel *levels, int32_t n_levels, float distance_threshold, float normal_cos_threshold,
                         float damping, const float *pose_init, const float *p2p_vertex_t0, const float *p2p_vertex_t1,
                         const float *p2p_normal_t0, int32_t p2p_H, int32_t p2p_W, float *out, float *out_host, void *ws,
                         void *stream) {
    if (!levels || n_levels < 1 || n_levels > RTG_ICP_MAX_LEVELS || !p2p_vertex_t0 || !p2p_vertex_t1 || !p2p_normal_t0 || p2p_H <= 0 ||
        p2p_W <= 0 || !out || !ws)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_icp_predict_pose: bad arguments");
    rtg::IcpPredict p;
    p.n_levels = n_levels;
    for (int l = 0; l < n_levels; l++) {
        const RtgIcpLevel &L = levels[l];
        if (!L.vertex0 || !L.normal0 || !L.vertex1 || !L.normal1 || L.H <= 0 || L.W <= 0 || L.iters < 0)
            return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_icp_predict_pose: bad level");
        p.lv[l] = rtg::IcpLevel{L.vertex0, L.normal0, L.vertex1, L.normal1, L.H, L.W, L.fx, L.fy, L.cx, L.cy, L.iters};
    }
    p.dist_thr = distance_threshold; p.cos_thr = normal_cos_threshold; p.damping = damping;
    p.pose_in = pose_init;
    p.p2p_v_t0 = p2p_vertex_t0; p.p2p_v_t1 = p2p_vertex_t1; p.p2p_n_t0 = p2p_normal_t0; p.p2p_HW = p2p_H * p2p_W;
    p.out = out; p.out_host = out_host;
    cudaError_t e = rtg::launch_icp_predict(p, ws, reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(RTG_ERR_CUDA, std::string("rtg_icp_predict_pose: ") + cudaGetErrorString(e));
    return check_launch("rtg_icp_predict_pose");
}

int rtg_icp_build_intensity_pyramid(const float *color, int32_t H, int32_t W, int32_t channels_last, int32_t n_levels,
                                    const int32_t *pools, float *const *intensity_out, void *stream) {
    if (!color || !pools || !intensity_out || H <= 0 || W <= 0 || n_levels < 1 || n_levels > RTG_ICP_MAX_LEVELS)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_icp_build_intensity_pyramid: bad arguments");
    rtg::IcpIntensity p;
    p.color = color; p.H = H; p.W = W; p.channels_last = channels_last ? 1 : 0; p.n_levels = n_levels;
    int64_t total = 0;
    for (int l = 0; l < n_levels; l++) {
        if (pools[l] < 1 || H / pools[l] < 1 || W / pools[l] < 1 || !intensity_out[l])
            return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_icp_build_intensity_pyramid: bad level");
        p.pool[l] = pools[l]; p.out[l] = intensity_out[l]; p.start[l] = (int)total;
        total += (int64_t)(H / pools[l]) * (W / pools[l]);
    }
    if (total > INT32_MAX) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_icp_build_intensity_pyramid: frame too large");
    for (int l = n_levels; l < RTG_ICP_MAX_LEVELS; l++) { p.pool[l] = 1; p.out[l] = nullptr; p.start[l] = (int)total; }
    p.total = (int)total;
    rtg::launch_icp_intensity_pyramid(p, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_icp_build_intensity_pyramid");
}

int rtg_icp_predict_pose_rgbd(const RtgIcpLevel *levels, const float *const *intensity0, const float *const *intensity1,
                              int32_t n_levels, float distance_threshold, float normal_cos_threshold, float damping,
                              float photometric_weight, const float *pose_init, const float *p2p_vertex_t0,
                              const float *p2p_vertex_t1, const float *p2p_normal_t0, int32_t p2p_H, int32_t p2p_W, float *out,
                              float *out_host, void *ws, void *stream) {
    if (!levels || !intensity0 || !intensity1 || n_levels < 1 || n_levels > RTG_ICP_MAX_LEVELS || !p2p_vertex_t0 ||
        !p2p_vertex_t1 || !p2p_normal_t0 || p2p_H <= 0 || p2p_W <= 0 || !out || !ws)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_icp_predict_pose_rgbd: bad arguments");
    if (!(photometric_weight >= 0.f) || !std::isfinite(photometric_weight))
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_icp_predict_pose_rgbd: photometric_weight must be finite and >= 0");
    rtg::IcpPredict p;
    rtg::IcpPhoto ph{};
    p.n_levels = n_levels;
    for (int l = 0; l < n_levels; l++) {
        const RtgIcpLevel &L = levels[l];
        if (!L.vertex0 || !L.normal0 || !L.vertex1 || !L.normal1 || L.H <= 0 || L.W <= 0 || L.iters < 0 || !intensity0[l] ||
            !intensity1[l])
            return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_icp_predict_pose_rgbd: bad level");
        p.lv[l] = rtg::IcpLevel{L.vertex0, L.normal0, L.vertex1, L.normal1, L.H, L.W, L.fx, L.fy, L.cx, L.cy, L.iters};
        ph.I0[l] = intensity0[l]; ph.I1[l] = intensity1[l];
    }
    ph.w = photometric_weight;
    p.dist_thr = distance_threshold; p.cos_thr = normal_cos_threshold; p.damping = damping;
    p.pose_in = pose_init;
    p.p2p_v_t0 = p2p_vertex_t0; p.p2p_v_t1 = p2p_vertex_t1; p.p2p_n_t0 = p2p_normal_t0; p.p2p_HW = p2p_H * p2p_W;
    p.out = out; p.out_host = out_host;
    cudaError_t e = rtg::launch_icp_predict_rgbd(p, ph, ws, reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) return fail(RTG_ERR_CUDA, std::string("rtg_icp_predict_pose_rgbd: ") + cudaGetErrorString(e));
    return check_launch("rtg_icp_predict_pose_rgbd");
}

int rtg_icp_point2plane_loss(const float *vertex_t0, const float *vertex_t1, const float *normal_t0, int32_t H, int32_t W,
                             const float *pose, float *loss, void *ws, void *stream) {
    if (!vertex_t0 || !vertex_t1 || !normal_t0 || !pose || !loss || !ws || H <= 0 || W <= 0)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_icp_point2plane_loss: bad arguments");
    rtg::launch_icp_p2p(vertex_t0, vertex_t1, normal_t0, H, W, pose, loss, ws, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_icp_point2plane_loss");
}

int rtg_icp_fill_model_depth(float *render_depth, const float *frame_depth, const float *render_normal, const float *frame_normal,
                             int32_t H, int32_t W, float distance_threshold, float normal_threshold, void *stream) {
    if (!render_depth || !frame_depth || !render_normal || !frame_normal || H <= 0 || W <= 0)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_icp_fill_model_depth: bad arguments");
    rtg::launch_icp_fill(render_depth, frame_depth, render_normal, frame_normal, H, W, distance_threshold, normal_threshold,
                         reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_icp_fill_model_depth");
}

// The checks shared by the three frame losses; `ws` holds doubles.
static int validate_loss(const char *who, const float *render, const float *depth, const int32_t *depth_index,
                         const float *gt_color, const float *gt_depth, int32_t H, int32_t W, const float *dL_dcolor,
                         const float *dL_ddepth, const float *loss_out, const void *ws) {
    if (H <= 0 || W <= 0) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": H and W must be >= 1");
    if (!render || !depth || !depth_index || !gt_color || !gt_depth || !dL_dcolor || !dL_ddepth || !loss_out || !ws)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL pointer");
    if (((uintptr_t)ws) & 7) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": ws must be 8-byte aligned");
    return RTG_OK;
}

size_t rtg_loss_workspace_bytes(void) { return rtg::loss_ws_bytes(); }

int rtg_loss_l1(const float *render, const float *depth, const int32_t *depth_index, const float *gt_color, const float *gt_depth,
                const uint8_t *render_mask, int32_t H, int32_t W, int32_t gt_channels_last, float color_weight, float depth_weight,
                float depth_error_max, float *dL_dcolor, float *dL_ddepth, float *loss_out, void *ws, void *stream) {
    const char *who = "rtg_loss_l1";
    int rc = validate_loss(who, render, depth, depth_index, gt_color, gt_depth, H, W, dL_dcolor, dL_ddepth, loss_out, ws);
    if (rc) return rc;
    rtg::launch_loss_l1(render, depth, depth_index, gt_color, gt_depth, render_mask, H, W, gt_channels_last, color_weight, depth_weight,
                        depth_error_max, dL_dcolor, dL_ddepth, loss_out, ws, reinterpret_cast<cudaStream_t>(stream));
    return check_launch(who);
}

size_t rtg_loss_l1_exposure_workspace_bytes(void) { return rtg::loss_ws_bytes(); }

int rtg_loss_l1_exposure(const float *render, const float *depth, const int32_t *depth_index, const float *gt_color,
                         const float *gt_depth, const uint8_t *render_mask, int32_t H, int32_t W, int32_t gt_channels_last,
                         float color_weight, float depth_weight, float depth_error_max, const float *exposure, float *dL_dcolor,
                         float *dL_ddepth, float *dL_dexposure, float *loss_out, void *ws, void *stream) {
    const char *who = "rtg_loss_l1_exposure";
    int rc = validate_loss(who, render, depth, depth_index, gt_color, gt_depth, H, W, dL_dcolor, dL_ddepth, loss_out, ws);
    if (rc) return rc;
    if (!exposure || !dL_dexposure) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL exposure / dL_dexposure");
    rtg::launch_loss_l1_exposure(render, depth, depth_index, gt_color, gt_depth, render_mask, H, W, gt_channels_last, color_weight,
                                 depth_weight, depth_error_max, exposure, dL_dcolor, dL_ddepth, dL_dexposure, loss_out, ws,
                                 reinterpret_cast<cudaStream_t>(stream));
    return check_launch(who);
}

int rtg_loss_mapping(const float *render, const float *depth, const float *render_normal, const int32_t *depth_index,
                     const float *gt_color, const float *gt_depth, const float *gt_normal, const uint8_t *render_mask, int32_t H, int32_t W,
                     int32_t gt_channels_last, float color_weight, float depth_weight, float normal_weight, float depth_error_max,
                     float *dL_dcolor, float *dL_ddepth, float *dL_dnormal, float *loss_out, void *ws, void *stream) {
    const char *who = "rtg_loss_mapping";
    int rc = validate_loss(who, render, depth, depth_index, gt_color, gt_depth, H, W, dL_dcolor, dL_ddepth, loss_out, ws);
    if (rc) return rc;
    if (normal_weight > 0.f && (!render_normal || !gt_normal || !dL_dnormal))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": normal_weight > 0 needs render_normal, gt_normal and dL_dnormal");
    rtg::launch_loss_mapping(render, depth, render_normal, depth_index, gt_color, gt_depth, gt_normal, render_mask, H, W, gt_channels_last,
                             color_weight, depth_weight, normal_weight, depth_error_max, dL_dcolor, dL_ddepth, dL_dnormal, loss_out, ws,
                             reinterpret_cast<cudaStream_t>(stream));
    return check_launch(who);
}

int rtg_loss_mapping_exposure(const float *render, const float *depth, const float *render_normal, const int32_t *depth_index,
                              const float *gt_color, const float *gt_depth, const float *gt_normal, const uint8_t *render_mask,
                              int32_t H, int32_t W, int32_t gt_channels_last, float color_weight, float depth_weight,
                              float normal_weight, float depth_error_max, const float *exposure, float *dL_dcolor, float *dL_ddepth,
                              float *dL_dnormal, float *dL_dexposure, float *loss_out, void *ws, void *stream) {
    const char *who = "rtg_loss_mapping_exposure";
    int rc = validate_loss(who, render, depth, depth_index, gt_color, gt_depth, H, W, dL_dcolor, dL_ddepth, loss_out, ws);
    if (rc) return rc;
    if (!exposure || !dL_dexposure) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL exposure / dL_dexposure");
    if (normal_weight > 0.f && (!render_normal || !gt_normal || !dL_dnormal))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": normal_weight > 0 needs render_normal, gt_normal and dL_dnormal");
    rtg::launch_loss_mapping_exposure(render, depth, render_normal, depth_index, gt_color, gt_depth, gt_normal, render_mask, H, W,
                                      gt_channels_last, color_weight, depth_weight, normal_weight, depth_error_max, exposure, dL_dcolor,
                                      dL_ddepth, dL_dnormal, dL_dexposure, loss_out, ws, reinterpret_cast<cudaStream_t>(stream));
    return check_launch(who);
}

size_t rtg_ssim_workspace_bytes(int32_t C, int32_t H, int32_t W) {
    if (C <= 0 || H <= 0 || W <= 0) return 0;
    return rtg::ssim_ws_bytes(C, H, W);
}

int rtg_ssim_loss(const float *img1, const float *img2, int32_t C, int32_t H, int32_t W, float *dL_dimg1, float *loss_out, void *ws,
                  void *stream) {
    if (!img1 || !img2 || !loss_out || !ws || C <= 0 || C > 65535 || H <= 0 || W <= 0 || (H + 15) / 16 > 65535)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_ssim_loss: bad arguments");
    rtg::launch_ssim_loss(img1, img2, C, H, W, dL_dimg1, loss_out, ws, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_ssim_loss");
}

size_t rtg_ssim_exposure_workspace_bytes(int32_t C, int32_t H, int32_t W) {
    if (C <= 0 || H <= 0 || W <= 0) return 0;
    return rtg::ssim_exposure_ws_bytes(C, H, W);
}

int rtg_ssim_loss_exposure(const float *img1, const float *img2, int32_t C, int32_t H, int32_t W, const float *exposure,
                           float *dL_dimg1, float *dL_dexposure, float *loss_out, void *ws, void *stream) {
    const char *who = "rtg_ssim_loss_exposure";
    if (!img1 || !img2 || !exposure || !loss_out || !ws) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL pointer");
    if (C <= 0 || C > 65535 || H <= 0 || W <= 0 || (H + 15) / 16 > 65535)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": bad size (C in [1, 65535], H and W >= 1, ceil(H / 16) <= 65535)");
    if (((uintptr_t)ws) & 7) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": ws must be 8-byte aligned");
    rtg::launch_ssim_loss_exposure(img1, img2, C, H, W, exposure, dL_dimg1, dL_dexposure, loss_out, ws,
                                   reinterpret_cast<cudaStream_t>(stream));
    return check_launch(who);
}

int rtg_normal_map(const float *normal, const int32_t *depth_index, int32_t H, int32_t W, float *out, void *stream) {
    if (!normal || !depth_index || !out || H <= 0 || W <= 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_normal_map: bad arguments");
    rtg::launch_normal_map(normal, depth_index, H, W, out, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_normal_map");
}

int rtg_frame_preprocess(const float *depth_in, int32_t H, int32_t W, int32_t depth_filter, int32_t radius, float sigma_color,
                         float sigma_space, float min_depth, float max_depth, float fx, float fy, float cx, float cy,
                         float invalid_confidence_thresh, float *depth_out, float *vertex_out, float *normal_out,
                         float *confidence_out, uint8_t *invalid_mask_out, void *ws, void *stream) {
    const bool maps = vertex_out || normal_out || confidence_out || invalid_mask_out;
    if (!depth_in || !depth_out || H <= 0 || W <= 0 || (maps && (!vertex_out || !normal_out || !confidence_out || !ws)))
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_frame_preprocess: bad arguments");
    if (depth_filter && (radius < 0 || radius > 15 || !(sigma_color > 0.f) || !(sigma_space > 0.f)))
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_frame_preprocess: bad filter parameters");
    if (depth_in == depth_out && depth_filter) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_frame_preprocess: the filter is not in-place");
    rtg::launch_frame_preprocess(depth_in, H, W, depth_filter, radius, sigma_color, sigma_space, min_depth, max_depth, fx, fy, cx, cy,
                                 invalid_confidence_thresh, depth_out, vertex_out, normal_out, confidence_out, invalid_mask_out, ws,
                                 reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_frame_preprocess");
}

int rtg_frame_downsample(const float *color, const float *depth, const uint8_t *render_mask, const int32_t *tile_mask, int32_t H,
                         int32_t W, int32_t scale, int32_t color_channels_last, float *color_out, float *depth_out,
                         uint8_t *mask_out, int32_t *tile_mask_out, void *stream) {
    const char *who = "rtg_frame_downsample";
    if (scale < 2) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": scale must be >= 2");
    if (H <= 0 || W <= 0 || H / scale < 1 || W / scale < 1)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": H and W must be >= scale");
    if (color_channels_last != 0 && color_channels_last != 1)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": color_channels_last must be 0 or 1");
    if (!color || !depth || !color_out || !depth_out) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL pointer");
    if ((render_mask == nullptr) != (mask_out == nullptr))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": mask_out must be given exactly when render_mask is");
    if ((tile_mask == nullptr) != (tile_mask_out == nullptr))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": tile_mask_out must be given exactly when tile_mask is");
    rtg::launch_frame_downsample(color, depth, render_mask, tile_mask, H, W, scale, color_channels_last, color_out, depth_out,
                                 mask_out, tile_mask_out, reinterpret_cast<cudaStream_t>(stream));
    return check_launch(who);
}

int rtg_accumulate_gaussian_error(int32_t H, int32_t W, int32_t P, const float *screen_color_error, const float *screen_depth_error,
                                  const float *screen_normal_error, const int32_t *screen_color_index,
                                  const int32_t *screen_depth_index, float color_threshold, float depth_threshold,
                                  float normal_threshold, int32_t check_max, float *gs_color_error, float *gs_depth_error,
                                  float *gs_normal_error, float *gs_rescale_counter, int32_t *counters, void *stream) {
    if (H < 0 || W < 0 || P < 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_accumulate_gaussian_error: negative size");
    if (P == 0) return RTG_OK;
    if (!gs_color_error || !gs_depth_error || !gs_normal_error || !gs_rescale_counter || (!check_max && !counters))
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_accumulate_gaussian_error: NULL output");
    if ((size_t)H * W > 0 && (!screen_color_error || !screen_depth_error || !screen_normal_error || !screen_color_index ||
                              !screen_depth_index))
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_accumulate_gaussian_error: NULL input");
    rtg::launch_gs_error(H, W, P, screen_color_error, screen_depth_error, screen_normal_error, screen_color_index, screen_depth_index,
                         color_threshold, depth_threshold, normal_threshold, check_max != 0, gs_color_error, gs_depth_error,
                         gs_normal_error, gs_rescale_counter, counters, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_accumulate_gaussian_error");
}

int rtg_tile_mean(int32_t H, int32_t W, const float *pixels, float ratio, float *tile_mean, int32_t *tile_mask, void *stream) {
    if (!pixels || H <= 0 || W <= 0 || (!tile_mean && !tile_mask)) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_tile_mean: bad arguments");
    rtg::launch_tile_pool(H, W, pixels, 0, ratio, nullptr, tile_mean, tile_mask, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_tile_mean");
}

int rtg_transmission_tile_mask(int32_t H, int32_t W, const float *T_map, float ratio, uint8_t *render_mask, int32_t *tile_mask,
                               void *stream) {
    if (!T_map || !tile_mask || H <= 0 || W <= 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_transmission_tile_mask: bad arguments");
    rtg::launch_tile_pool(H, W, T_map, 1, ratio, render_mask, nullptr, tile_mask, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_transmission_tile_mask");
}

int rtg_color_error(int32_t H, int32_t W, const float *render, const float *gt, float *out, void *stream) {
    if (!render || !gt || !out || H <= 0 || W <= 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_color_error: bad arguments");
    rtg::launch_color_error(H, W, render, gt, out, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_color_error");
}

size_t rtg_soa_compact_workspace_bytes(int64_t P) { return rtg::soa_compact_ws_bytes(P < 0 ? 0 : P); }

int rtg_soa_compact(const uint8_t *mask, int32_t invert, int64_t P, int32_t n_arrays, const void *const *in, void *const *out,
                    const int32_t *words_per_row, uint32_t *n_kept, uint32_t *n_kept_host, void *ws, void *stream) {
    if (P < 0 || P > 0x7fffffffLL || n_arrays < 0 || n_arrays > RTG_SOA_MAX_ARRAYS || !n_kept)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_soa_compact: bad sizes");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (P == 0) {
        cudaMemsetAsync(n_kept, 0, 4, s);
        if (n_kept_host) *n_kept_host = 0;
        return check_launch("rtg_soa_compact");
    }
    if (!mask || !ws || (n_arrays > 0 && (!in || !out || !words_per_row))) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_soa_compact: NULL pointer");
    for (int i = 0; i < n_arrays; i++)
        if (!in[i] || !out[i] || words_per_row[i] < 1 || in[i] == out[i])
            return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_soa_compact: bad array (NULL, in place, or words_per_row < 1)");
    rtg::launch_soa_compact(mask, invert, P, n_arrays, in, out, words_per_row, n_kept, n_kept_host, ws, s);
    return check_launch("rtg_soa_compact");
}

size_t rtg_knn_workspace_bytes(int64_t n_ref) { return rtg::knn_ws_bytes(n_ref < 0 ? 0 : n_ref); }

int rtg_knn(const float *query, int64_t n_query, const float *ref, int64_t n_ref, int32_t K, int32_t skip_self, float *out_d2,
            int32_t *out_idx, float *out_mean, void *ws, void *stream) {
    if (n_query < 0 || n_ref < 0 || n_query > 0x7fffffffLL || n_ref > 0x7fffffffLL || K < 1 || K > 8)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_knn: bad sizes (1 <= K <= 8)");
    if (n_query == 0) return RTG_OK;
    if (!query || !ws || (n_ref > 0 && !ref)) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_knn: NULL pointer");
    if (skip_self && (n_query != n_ref)) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_knn: skip_self needs query == ref");
    if (rtg::launch_knn(query, n_query, ref, n_ref, K, skip_self, out_d2, out_idx, out_mean, ws, reinterpret_cast<cudaStream_t>(stream)))
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_knn: unsupported K");
    return check_launch("rtg_knn");
}

size_t rtg_map_transform_workspace_bytes(int32_t K) { return rtg::map_transform_ws_bytes(K); }

int rtg_map_transform(const RtgMapTransform *xf, void *ws, void *stream) {
    if (!xf) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_transform: xf is NULL");
    if (xf->P < 0 || xf->K < 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_transform: bad sizes (P, K >= 0)");
    if (xf->sh_rest != 0 && xf->sh_rest != 3 && xf->sh_rest != 8 && xf->sh_rest != 15)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_transform: sh_rest must be 0, 3, 8 or 15");
    if (!xf->n_skipped) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_transform: NULL pointer (n_skipped)");
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    if (xf->P == 0) {
        cudaMemsetAsync(xf->n_skipped, 0, sizeof(int64_t), s);
        return check_launch("rtg_map_transform");
    }
    if (!xf->anchor || !xf->xyz || !xf->rotation)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_transform: NULL pointer (anchor, xyz or rotation)");
    if (xf->K > 0 && (!xf->old_c2w || !xf->new_c2w || !ws))
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_transform: NULL pointer (old_c2w, new_c2w or ws)");
    if ((xf->sh_rest == 0) != (xf->features_rest == nullptr))
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_transform: features_rest must be NULL exactly when sh_rest == 0");
    if (reinterpret_cast<uintptr_t>(ws) & 15) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_map_transform: ws must be 16-byte aligned");
    rtg::launch_map_transform(*xf, ws, s);
    return check_launch("rtg_map_transform");
}

// the voxel count, or -1 when the sizes are not positive or nx*ny*nz >= limit
static int64_t tsdf_voxels(int32_t nx, int32_t ny, int32_t nz, int64_t limit) {
    if (nx <= 0 || ny <= 0 || nz <= 0) return -1;
    if ((int64_t)nx * ny >= limit) return -1;  // then nx*ny < 2^32 and the full product fits int64
    const int64_t n = (int64_t)nx * ny * nz;
    return n >= limit ? -1 : n;
}

static int validate_tsdf_volume(const char *who, const RtgTsdfVolume *v, int64_t limit) {
    if (!v) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": vol is NULL");
    if (tsdf_voxels(v->nx, v->ny, v->nz, limit) < 0)
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": bad dims (each >= 1, nx*ny*nz below the limit)");
    if (!(v->voxel_size > 0.f) || !(v->trunc > 0.f) || !std::isfinite(v->voxel_size) || !std::isfinite(v->trunc))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": voxel_size and trunc must be finite and > 0");
    if (!std::isfinite(v->origin[0]) || !std::isfinite(v->origin[1]) || !std::isfinite(v->origin[2]))
        return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": origin must be finite");
    if (!v->tsdf || !v->weight) return fail(RTG_ERR_INVALID_ARGUMENT, std::string(who) + ": NULL pointer (tsdf or weight)");
    return RTG_OK;
}

static const int64_t kTsdfMaxVoxels = 0x80000000LL;            // 2^31
static const int64_t kTsdfMaxExtractVoxels = 0x100000000LL / 12;  // 12 triangles per cell must fit uint32 offsets

int rtg_tsdf_integrate(const RtgTsdfVolume *vol, const float *depth, const float *color, int32_t H, int32_t W,
                       int32_t color_channels_last, float fx, float fy, float cx, float cy, const void *w2c, int32_t w2c_is_double,
                       void *stream) {
    if (int rc = validate_tsdf_volume("rtg_tsdf_integrate", vol, kTsdfMaxVoxels)) return rc;
    if (H <= 0 || W <= 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_tsdf_integrate: bad image size (H, W >= 1)");
    if (!depth || !w2c) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_tsdf_integrate: NULL pointer (depth or w2c)");
    if ((vol->color == nullptr) != (color == nullptr))
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_tsdf_integrate: color must be given exactly when the volume has color");
    if (!std::isfinite(fx) || !std::isfinite(fy) || !std::isfinite(cx) || !std::isfinite(cy) || fx == 0.f || fy == 0.f)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_tsdf_integrate: intrinsics must be finite with fx, fy != 0");
    rtg::launch_tsdf_integrate(*vol, depth, color, H, W, color_channels_last != 0, fx, fy, cx, cy, w2c, w2c_is_double != 0,
                               reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_tsdf_integrate");
}

int rtg_tsdf_raycast(const RtgTsdfVolume *vol, const void *w2c, int32_t w2c_is_double, int32_t H, int32_t W, float fx, float fy,
                     float cx, float cy, float *depth, float *normal, float *color, void *stream) {
    if (int rc = validate_tsdf_volume("rtg_tsdf_raycast", vol, kTsdfMaxVoxels)) return rc;
    if (H <= 0 || W <= 0) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_tsdf_raycast: bad image size (H, W >= 1)");
    if (!w2c || !depth || !normal) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_tsdf_raycast: NULL pointer (w2c, depth or normal)");
    if ((vol->color == nullptr) != (color == nullptr))
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_tsdf_raycast: color must be given exactly when the volume has color");
    if (!std::isfinite(fx) || !std::isfinite(fy) || !std::isfinite(cx) || !std::isfinite(cy) || fx == 0.f || fy == 0.f)
        return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_tsdf_raycast: intrinsics must be finite with fx, fy != 0");
    rtg::launch_tsdf_raycast(*vol, w2c, w2c_is_double != 0, H, W, fx, fy, cx, cy, depth, normal, color,
                             reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_tsdf_raycast");
}

size_t rtg_tsdf_extract_workspace_bytes(int32_t nx, int32_t ny, int32_t nz) {
    const int64_t n = tsdf_voxels(nx, ny, nz, kTsdfMaxExtractVoxels);
    return n < 0 ? 0 : rtg::tsdf_extract_ws_bytes(n);
}

int rtg_tsdf_extract_count(const RtgTsdfVolume *vol, void *ws, uint32_t *counts, void *stream) {
    if (int rc = validate_tsdf_volume("rtg_tsdf_extract_count", vol, kTsdfMaxExtractVoxels)) return rc;
    if (!ws || !counts) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_tsdf_extract_count: NULL pointer (ws or counts)");
    rtg::launch_tsdf_extract_count(*vol, ws, counts, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_tsdf_extract_count");
}

int rtg_tsdf_extract_emit(const RtgTsdfVolume *vol, const void *ws, float *vertices, float *vertex_colors, int32_t *faces,
                          void *stream) {
    if (int rc = validate_tsdf_volume("rtg_tsdf_extract_emit", vol, kTsdfMaxExtractVoxels)) return rc;
    if (!ws || !vertices || !faces) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_tsdf_extract_emit: NULL pointer (ws, vertices or faces)");
    rtg::launch_tsdf_extract_emit(*vol, ws, vertices, vertex_colors, faces, reinterpret_cast<cudaStream_t>(stream));
    return check_launch("rtg_tsdf_extract_emit");
}

int rtg_profile_enable(int32_t on) {
    std::lock_guard<std::mutex> lk(rtg::g_prof_mu);
    rtg::g_prof_on = on != 0;
    return RTG_OK;
}

int rtg_profile_kernel_count(void) { return rtg::K_COUNT; }

const char *rtg_profile_kernel_name(int32_t id) { return (id >= 0 && id < rtg::K_COUNT) ? rtg::kKernelNames[id] : ""; }

int rtg_profile_read(double *total_ms, int64_t *launches, int32_t reset) {
    if (!total_ms || !launches) return fail(RTG_ERR_INVALID_ARGUMENT, "rtg_profile_read: NULL output");
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return fail(RTG_ERR_CUDA, std::string("rtg_profile_read: ") + cudaGetErrorString(e));
    std::lock_guard<std::mutex> lk(rtg::g_prof_mu);
    for (int i = 0; i < rtg::K_COUNT; i++) { total_ms[i] = 0.0; launches[i] = 0; }
    for (auto &r : rtg::g_prof_recs) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) { total_ms[r.id] += ms; launches[r.id] += 1; }
    }
    if (reset) {
        for (auto &r : rtg::g_prof_recs) { rtg::g_prof_pool.push_back(r.a); rtg::g_prof_pool.push_back(r.b); }
        rtg::g_prof_recs.clear();
    }
    return RTG_OK;
}

}  // extern "C"
