// Fused image-space kernels that sit between the rasterizer forward and backward in the mapping loop
// (SURVEY.md section 8(f) #1): the masked L1 colour + depth loss with its gradients, and the per-pixel normal map.
//
// Reference arithmetic (eager PyTorch, ~25 kernels incl. autograd and two boolean-mask compactions):
//   SLAM/multiprocess/mapper.py:402-431,444-451  loss_update (colour L1 on render_mask, depth L1 on the valid mask)
//   utils/loss_utils.py:27-31                     l1_loss = abs(a - b).mean()
//   SLAM/render.py:130-133                        render_normal[:, idx > -1] = normal[idx[idx > -1]]
#include "common.cuh"
#include "prof.h"

namespace rtg {

// ---- the frame loss, one kernel family for its three forms:
//   rtg_loss_l1          <false, false>  colour L1 on the render mask + depth L1 on frame_depth_pixel's pixels
//   rtg_loss_mapping     <true,  false>  + the cosine normal term of Mapping.loss_update (mapper.py:433-442):
//                        mean over {render_mask & depth_index != -1 & gt_normal != 0} of 1 - cosine_similarity(normal,
//                        gt_normal) (F.cosine_similarity: x.y / (max(|x|, 1e-8) * max(|y|, 1e-8))); render_normal (3,H,W),
//                        gt_normal (H,W,3)
//   rtg_loss_l1_exposure <false, true>   the colour residual under a frame exposure (a, b): r = e^a C + b - C^
//   rtg_loss_mapping_exposure <true, true>  both: the mapping loss of a keyframe seen under its exposure
// Terms, in this order: sum |r|, n_colour, sum |e|, n_depth, [normal] sum (1 - cos), n_normal, [exposure] sum sgn(r) e^a C,
// sum sgn(r) (the last two give dL/da and dL/db). Every block of the reduce kernel writes its partial sums (no atomics); the
// one-block final kernel adds them in a fixed order, so two calls on the same inputs give the same bits. The grad kernel's
// scales depend on the counts only.
#define RTG_LOSS_MAX_TERMS 8
#define RTG_LOSS_MAX_BLOCKS (RTG_NUM_SMS * 8)  // grid of the reduce and grad kernels: min(ceil(N / 256), this)
constexpr int loss_terms(const bool normal, const bool exposure) { return 4 + (normal ? 2 : 0) + (exposure ? 2 : 0); }

struct LossWs {
    double total[RTG_LOSS_MAX_TERMS];
    double partial[RTG_LOSS_MAX_BLOCKS * RTG_LOSS_MAX_TERMS];  // block b's terms at [b * loss_terms(...)]
};

__device__ __forceinline__ float sgn(float x) { return (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f); }

// channel c of the colour residual of pixel p (render (3,H,W)); (ea, eb) = (e^a, b) is read with exposure only
template <bool EXPOSURE>
__device__ __forceinline__ float color_residual(const float *__restrict__ render, const float *__restrict__ gt_color,
                                                int channels_last, int N, int p, int c, float ea, float eb) {
    const float g = frame_color(gt_color, channels_last, N, p, c);
    if constexpr (EXPOSURE) return fmaf(ea, render[(size_t)c * N + p], eb) - g;
    else return render[(size_t)c * N + p] - g;
}

__device__ __forceinline__ bool normal_term(const float *__restrict__ nrm, const float *__restrict__ gtn, int N, int p, float &cosv,
                                            float &x0, float &x1, float &x2, float &y0, float &y1, float &y2, float &nx, float &ny) {
    y0 = gtn[3 * (size_t)p]; y1 = gtn[3 * (size_t)p + 1]; y2 = gtn[3 * (size_t)p + 2];
    if (y0 == 0.f && y1 == 0.f && y2 == 0.f) return false;
    x0 = nrm[p]; x1 = nrm[(size_t)N + p]; x2 = nrm[2 * (size_t)N + p];
    nx = fmaxf(sqrtf(x0 * x0 + x1 * x1 + x2 * x2), 1e-8f);
    ny = fmaxf(sqrtf(y0 * y0 + y1 * y1 + y2 * y2), 1e-8f);
    cosv = (x0 * y0 + x1 * y1 + x2 * y2) / (nx * ny);
    return true;
}

// gt_color: (H,W,3) if channels_last else (3,H,W); gt_depth: (H,W); mask: (H,W) bytes or NULL; nrm: NULL = no normal term
template <bool NORMAL, bool EXPOSURE>
__global__ void __launch_bounds__(256) loss_reduce_kernel(const float *__restrict__ render, const float *__restrict__ depth,
                                                          const float *__restrict__ nrm, const int *__restrict__ depth_index,
                                                          const float *__restrict__ gt_color, const float *__restrict__ gt_depth,
                                                          const float *__restrict__ gt_normal, const uint8_t *__restrict__ mask, int N,
                                                          int channels_last, float depth_error_max, const float *__restrict__ exposure,
                                                          LossWs *ws) {
    constexpr int NT = loss_terms(NORMAL, EXPOSURE), XE = NORMAL ? 6 : 4;
    float ea = 1.f, eb = 0.f;
    if constexpr (EXPOSURE) { ea = expf(exposure[0]); eb = exposure[1]; }
    double a[NT];
#pragma unroll
    for (int k = 0; k < NT; k++) a[k] = 0.0;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        if (mask && mask[p] == 0) continue;
        float s = 0.f, sa = 0.f, sb = 0.f;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const float r = color_residual<EXPOSURE>(render, gt_color, channels_last, N, p, c, ea, eb);
            s += fabsf(r);
            if constexpr (EXPOSURE) { sa += sgn(r) * (ea * render[(size_t)c * N + p]); sb += sgn(r); }
        }
        a[0] += (double)s;
        a[1] += 1.0;
        if constexpr (EXPOSURE) { a[XE] += (double)sa; a[XE + 1] += (double)sb; }
        const float gd = gt_depth[p];
        const float e = depth[p] - gd;
        const int hit = depth_index[p];
        if (frame_depth_pixel(hit, gd, e, depth_error_max)) { a[2] += (double)fabsf(e); a[3] += 1.0; }
        if constexpr (NORMAL) {
            float cosv, x0, x1, x2, y0, y1, y2, nx, ny;
            if (nrm && hit != -1 && normal_term(nrm, gt_normal, N, p, cosv, x0, x1, x2, y0, y1, y2, nx, ny)) {
                a[4] += (double)(1.f - cosv);
                a[5] += 1.0;
            }
        }
    }
#pragma unroll
    for (int k = 0; k < NT; k++)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a[k] += __shfl_xor_sync(0xffffffffu, a[k], o);
    __shared__ double s_p[8][NT];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < NT; k++) s_p[w][k] = a[k];
    __syncthreads();
    if (threadIdx.x < NT) {
        double t = 0.0;
        for (int k = 0; k < 8; k++) t += s_p[k][threadIdx.x];
        ws->partial[blockIdx.x * NT + threadIdx.x] = t;
    }
}

// One block: warp k adds term k over the blocks' partial sums (fixed lane stride, fixed butterfly); thread 0 writes the
// totals, loss_out (4 floats, 8 with the normal term) and dL/d(a, b).
template <bool NORMAL, bool EXPOSURE>
__global__ void __launch_bounds__(32 * RTG_LOSS_MAX_TERMS) loss_final_kernel(int nb, float color_weight, float depth_weight,
                                                                             float normal_weight, LossWs *ws,
                                                                             float *__restrict__ dL_dexposure,
                                                                             float *__restrict__ loss_out) {
    constexpr int NT = loss_terms(NORMAL, EXPOSURE), XE = NORMAL ? 6 : 4;
    __shared__ double s_t[NT];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    double acc = 0.0;
    for (int k = lane; k < nb; k += 32) acc += ws->partial[k * NT + w];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) s_t[w] = acc;
    __syncthreads();
    if (threadIdx.x != 0) return;
#pragma unroll
    for (int k = 0; k < NT; k++) ws->total[k] = s_t[k];
    const double nc = s_t[1], nd = s_t[3];
    const double cl = nc > 0.0 ? s_t[0] / (3.0 * nc) : 0.0, dl = nd > 0.0 ? s_t[2] / nd : 0.0;
    if constexpr (NORMAL) {
        const double nn = s_t[5], nl = nn > 0.0 ? s_t[4] / nn : 0.0;
        loss_out[0] = (float)((double)color_weight * cl + (double)depth_weight * dl + (double)normal_weight * nl);
        loss_out[4] = (float)nl; loss_out[5] = (float)nn; loss_out[6] = 0.f; loss_out[7] = 0.f;
    } else {
        loss_out[0] = (float)((double)color_weight * cl + (double)depth_weight * dl);
    }
    loss_out[1] = (float)cl;
    loss_out[2] = (float)dl;
    loss_out[3] = (float)nd;
    if constexpr (EXPOSURE) {
        const double gcs = nc > 0.0 ? (double)color_weight / (3.0 * nc) : 0.0;
        dL_dexposure[0] = (float)(gcs * s_t[XE]);
        dL_dexposure[1] = (float)(gcs * s_t[XE + 1]);
    }
}

template <bool NORMAL, bool EXPOSURE>
__global__ void __launch_bounds__(256) loss_grad_kernel(const float *__restrict__ render, const float *__restrict__ depth,
                                                        const float *__restrict__ nrm, const int *__restrict__ depth_index,
                                                        const float *__restrict__ gt_color, const float *__restrict__ gt_depth,
                                                        const float *__restrict__ gt_normal, const uint8_t *__restrict__ mask, int N,
                                                        int channels_last, float depth_error_max, const float *__restrict__ exposure,
                                                        float color_weight, float depth_weight, float normal_weight, const LossWs *ws,
                                                        float *__restrict__ dL_dcolor, float *__restrict__ dL_ddepth,
                                                        float *__restrict__ dL_dnormal) {
    const double nc = ws->total[1], nd = ws->total[3];
    float ea = 1.f, eb = 0.f;
    if constexpr (EXPOSURE) { ea = expf(exposure[0]); eb = exposure[1]; }
    float gcs = nc > 0.0 ? (float)((double)color_weight / (3.0 * nc)) : 0.f;  // mean over 3 * n_colour elements
    if constexpr (EXPOSURE) gcs *= ea;  // e^0 = 1 leaves rtg_loss_l1's scale bit-equal
    const float gds = nd > 0.0 ? (float)((double)depth_weight / nd) : 0.f;
    float gns = 0.f;
    if constexpr (NORMAL) {
        const double nn = ws->total[5];
        gns = nn > 0.0 ? (float)((double)normal_weight / nn) : 0.f;
    }
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        const bool m = mask ? (mask[p] != 0) : true;
        float g[3] = {0.f, 0.f, 0.f}, gd_ = 0.f, n0 = 0.f, n1 = 0.f, n2 = 0.f;
        if (m) {
            // the depth loads first: issued before the colour branch on channels_last, all loads are in flight at once
            const float gd = gt_depth[p];
            const float e = depth[p] - gd;
            const int hit = depth_index[p];
#pragma unroll
            for (int c = 0; c < 3; c++) g[c] = gcs * sgn(color_residual<EXPOSURE>(render, gt_color, channels_last, N, p, c, ea, eb));
            if (frame_depth_pixel(hit, gd, e, depth_error_max)) gd_ = gds * sgn(e);
            if constexpr (NORMAL) {
                float cosv, x0, x1, x2, y0, y1, y2, nx, ny;
                if (nrm && hit != -1 && normal_term(nrm, gt_normal, N, p, cosv, x0, x1, x2, y0, y1, y2, nx, ny)) {
                    // d(1 - cos)/dx = -( y / (|x||y|) - cos * x / |x|^2 )
                    const float a = 1.f / (nx * ny), bq = cosv / (nx * nx);
                    n0 = -gns * (y0 * a - x0 * bq); n1 = -gns * (y1 * a - x1 * bq); n2 = -gns * (y2 * a - x2 * bq);
                }
            }
        }
        dL_dcolor[p] = g[0]; dL_dcolor[(size_t)N + p] = g[1]; dL_dcolor[2 * (size_t)N + p] = g[2];
        dL_ddepth[p] = gd_;
        if constexpr (NORMAL)
            if (dL_dnormal) { dL_dnormal[p] = n0; dL_dnormal[(size_t)N + p] = n1; dL_dnormal[2 * (size_t)N + p] = n2; }
    }
}

template <bool NORMAL, bool EXPOSURE>
static void launch_loss(const float *render, const float *depth, const float *nrm, const int *depth_index, const float *gt_color,
                        const float *gt_depth, const float *gt_normal, const uint8_t *mask, int H, int W, int channels_last,
                        float color_weight, float depth_weight, float normal_weight, float depth_error_max, const float *exposure,
                        float *dL_dcolor, float *dL_ddepth, float *dL_dnormal, float *dL_dexposure, float *loss_out, void *ws,
                        cudaStream_t s) {
    ProfScope ps(K_ICP_MISC, s);
    LossWs *w = reinterpret_cast<LossWs *>(ws);
    const int N = H * W;
    int nb = (N + 255) / 256;
    if (nb > RTG_LOSS_MAX_BLOCKS) nb = RTG_LOSS_MAX_BLOCKS;
    loss_reduce_kernel<NORMAL, EXPOSURE><<<nb, 256, 0, s>>>(render, depth, nrm, depth_index, gt_color, gt_depth, gt_normal, mask, N,
                                                            channels_last, depth_error_max, exposure, w);
    loss_final_kernel<NORMAL, EXPOSURE><<<1, 32 * loss_terms(NORMAL, EXPOSURE), 0, s>>>(nb, color_weight, depth_weight, normal_weight,
                                                                                        w, dL_dexposure, loss_out);
    loss_grad_kernel<NORMAL, EXPOSURE><<<nb, 256, 0, s>>>(render, depth, nrm, depth_index, gt_color, gt_depth, gt_normal, mask, N,
                                                          channels_last, depth_error_max, exposure, color_weight, depth_weight,
                                                          normal_weight, w, dL_dcolor, dL_ddepth, dL_dnormal);
}

size_t loss_ws_bytes() { return sizeof(LossWs); }

void launch_loss_l1(const float *render, const float *depth, const int *depth_index, const float *gt_color, const float *gt_depth,
                    const uint8_t *mask, int H, int W, int channels_last, float color_weight, float depth_weight,
                    float depth_error_max, float *dL_dcolor, float *dL_ddepth, float *loss_out, void *ws, cudaStream_t s) {
    launch_loss<false, false>(render, depth, nullptr, depth_index, gt_color, gt_depth, nullptr, mask, H, W, channels_last, color_weight,
                              depth_weight, 0.f, depth_error_max, nullptr, dL_dcolor, dL_ddepth, nullptr, nullptr, loss_out, ws, s);
}

void launch_loss_l1_exposure(const float *render, const float *depth, const int *depth_index, const float *gt_color,
                             const float *gt_depth, const uint8_t *mask, int H, int W, int channels_last, float color_weight,
                             float depth_weight, float depth_error_max, const float *exposure, float *dL_dcolor, float *dL_ddepth,
                             float *dL_dexposure, float *loss_out, void *ws, cudaStream_t s) {
    launch_loss<false, true>(render, depth, nullptr, depth_index, gt_color, gt_depth, nullptr, mask, H, W, channels_last, color_weight,
                             depth_weight, 0.f, depth_error_max, exposure, dL_dcolor, dL_ddepth, nullptr, dL_dexposure, loss_out, ws, s);
}

void launch_loss_mapping(const float *render, const float *depth, const float *render_normal, const int *depth_index,
                         const float *gt_color, const float *gt_depth, const float *gt_normal, const uint8_t *mask, int H, int W,
                         int channels_last, float color_weight, float depth_weight, float normal_weight, float depth_error_max,
                         float *dL_dcolor, float *dL_ddepth, float *dL_dnormal, float *loss_out, void *ws, cudaStream_t s) {
    const float *nrm = (normal_weight > 0.f) ? render_normal : nullptr;
    launch_loss<true, false>(render, depth, nrm, depth_index, gt_color, gt_depth, gt_normal, mask, H, W, channels_last, color_weight,
                             depth_weight, normal_weight, depth_error_max, nullptr, dL_dcolor, dL_ddepth, dL_dnormal, nullptr, loss_out,
                             ws, s);
}

void launch_loss_mapping_exposure(const float *render, const float *depth, const float *render_normal, const int *depth_index,
                                  const float *gt_color, const float *gt_depth, const float *gt_normal, const uint8_t *mask, int H,
                                  int W, int channels_last, float color_weight, float depth_weight, float normal_weight,
                                  float depth_error_max, const float *exposure, float *dL_dcolor, float *dL_ddepth,
                                  float *dL_dnormal, float *dL_dexposure, float *loss_out, void *ws, cudaStream_t s) {
    const float *nrm = (normal_weight > 0.f) ? render_normal : nullptr;
    launch_loss<true, true>(render, depth, nrm, depth_index, gt_color, gt_depth, gt_normal, mask, H, W, channels_last, color_weight,
                            depth_weight, normal_weight, depth_error_max, exposure, dL_dcolor, dL_ddepth, dL_dnormal, dL_dexposure,
                            loss_out, ws, s);
}

// out (3,H,W) = normal[idx] where idx > -1, zeros elsewhere
__global__ void __launch_bounds__(256) normal_map_kernel(const float *__restrict__ normal, const int *__restrict__ depth_index, int N,
                                                         float *__restrict__ out) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= N) return;
    const int id = depth_index[p];
    float x = 0.f, y = 0.f, z = 0.f;
    if (id > -1) { x = normal[3 * (size_t)id]; y = normal[3 * (size_t)id + 1]; z = normal[3 * (size_t)id + 2]; }
    out[p] = x; out[(size_t)N + p] = y; out[2 * (size_t)N + p] = z;
}

void launch_normal_map(const float *normal, const int *depth_index, int H, int W, float *out, cudaStream_t s) {
    ProfScope ps(K_ICP_MISC, s);
    const int N = H * W;
    normal_map_kernel<<<(N + 255) / 256, 256, 0, s>>>(normal, depth_index, N, out);
}

}  // namespace rtg
