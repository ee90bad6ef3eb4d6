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

struct LossStats {  // device scratch, 4 doubles: sum|dC|, n_colour_pixels, sum|dd|, n_depth_pixels
    double v[4];
};

__device__ __forceinline__ float sgn(float x) { return (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f); }

__global__ void loss_init_kernel(LossStats *st) {
    if (threadIdx.x < 4) st->v[threadIdx.x] = 0.0;
}

// gt_color: (H,W,3) if channels_last else (3,H,W); gt_depth: (H,W); mask: (H,W) bytes or NULL
__global__ void __launch_bounds__(256) loss_reduce_kernel(const float *__restrict__ render, const float *__restrict__ depth,
                                                          const int *__restrict__ depth_index, const float *__restrict__ gt_color,
                                                          const float *__restrict__ gt_depth, const uint8_t *__restrict__ mask,
                                                          int N, int channels_last, float depth_error_max, LossStats *st) {
    double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        const bool m = mask ? (mask[p] != 0) : true;
        if (m) {
            float s = 0.f;
#pragma unroll
            for (int c = 0; c < 3; c++) {
                const float g = channels_last ? gt_color[3 * (size_t)p + c] : gt_color[(size_t)c * N + p];
                s += fabsf(render[(size_t)c * N + p] - g);
            }
            a0 += (double)s;
            a1 += 1.0;
            const float gd = gt_depth[p];
            const float e = depth[p] - gd;
            if (depth_index[p] != -1 && gd > 0.f && e < depth_error_max) { a2 += (double)fabsf(e); a3 += 1.0; }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a0 += __shfl_xor_sync(0xffffffffu, a0, o); a1 += __shfl_xor_sync(0xffffffffu, a1, o);
        a2 += __shfl_xor_sync(0xffffffffu, a2, o); a3 += __shfl_xor_sync(0xffffffffu, a3, o);
    }
    __shared__ double s_p[8][4];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) { s_p[w][0] = a0; s_p[w][1] = a1; s_p[w][2] = a2; s_p[w][3] = a3; }
    __syncthreads();
    if (threadIdx.x < 4) {
        double t = 0.0;
        for (int k = 0; k < 8; k++) t += s_p[k][threadIdx.x];
        atomicAdd(&st->v[threadIdx.x], t);
    }
}

__global__ void __launch_bounds__(256) loss_grad_kernel(const float *__restrict__ render, const float *__restrict__ depth,
                                                        const int *__restrict__ depth_index, const float *__restrict__ gt_color,
                                                        const float *__restrict__ gt_depth, const uint8_t *__restrict__ mask,
                                                        int N, int channels_last, float depth_error_max, float color_weight,
                                                        float depth_weight, const LossStats *st, float *__restrict__ dL_dcolor,
                                                        float *__restrict__ dL_ddepth, float *__restrict__ loss_out) {
    const double nc = st->v[1], nd = st->v[3];
    const float gcs = nc > 0.0 ? (float)((double)color_weight / (3.0 * nc)) : 0.f;  // mean over 3 * n_colour elements
    const float gds = nd > 0.0 ? (float)((double)depth_weight / nd) : 0.f;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const double cl = nc > 0.0 ? st->v[0] / (3.0 * nc) : 0.0, dl = nd > 0.0 ? st->v[2] / nd : 0.0;
        loss_out[0] = (float)((double)color_weight * cl + (double)depth_weight * dl);
        loss_out[1] = (float)cl;
        loss_out[2] = (float)dl;
        loss_out[3] = (float)nd;
    }
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        const bool m = mask ? (mask[p] != 0) : true;
        float g0 = 0.f, g1 = 0.f, g2 = 0.f, gd_ = 0.f;
        if (m) {
            const float t0 = channels_last ? gt_color[3 * (size_t)p + 0] : gt_color[p];
            const float t1 = channels_last ? gt_color[3 * (size_t)p + 1] : gt_color[(size_t)N + p];
            const float t2 = channels_last ? gt_color[3 * (size_t)p + 2] : gt_color[2 * (size_t)N + p];
            g0 = gcs * sgn(render[p] - t0);
            g1 = gcs * sgn(render[(size_t)N + p] - t1);
            g2 = gcs * sgn(render[2 * (size_t)N + p] - t2);
            const float gd = gt_depth[p];
            const float e = depth[p] - gd;
            if (depth_index[p] != -1 && gd > 0.f && e < depth_error_max) gd_ = gds * sgn(e);
        }
        dL_dcolor[p] = g0; dL_dcolor[(size_t)N + p] = g1; dL_dcolor[2 * (size_t)N + p] = g2;
        dL_ddepth[p] = gd_;
    }
}

// ---- the L1 loss under a frame exposure (a, b): the colour residual is r = e^a C + b - C^, the depth term is unchanged.
// Besides the four statistics, sum sgn(r) e^a C and sum sgn(r) give dL/da and dL/db. Every block writes its six partial
// sums (no atomics); one block adds them in a fixed order, so two calls on the same inputs give the same bits.
#define RTG_LOSS_EXP_TERMS 6
struct LossExposureWs {
    LossStats st;
    double partial[RTG_NUM_SMS * 8][RTG_LOSS_EXP_TERMS];
};

__global__ void __launch_bounds__(256) loss_exposure_reduce_kernel(const float *__restrict__ render, const float *__restrict__ depth,
                                                                   const int *__restrict__ depth_index,
                                                                   const float *__restrict__ gt_color,
                                                                   const float *__restrict__ gt_depth, const uint8_t *__restrict__ mask,
                                                                   int N, int channels_last, float depth_error_max,
                                                                   const float *__restrict__ exposure, LossExposureWs *ws) {
    const float ea = expf(exposure[0]), eb = exposure[1];
    double a[RTG_LOSS_EXP_TERMS] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        const bool m = mask ? (mask[p] != 0) : true;
        if (m) {
            float s = 0.f, sa = 0.f, sb = 0.f;
#pragma unroll
            for (int c = 0; c < 3; c++) {
                const float g = channels_last ? gt_color[3 * (size_t)p + c] : gt_color[(size_t)c * N + p];
                const float C = render[(size_t)c * N + p], ec = ea * C;
                const float r = fmaf(ea, C, eb) - g;  // the expression of loss_exposure_grad_kernel
                s += fabsf(r);
                sa += sgn(r) * ec;
                sb += sgn(r);
            }
            a[0] += (double)s;
            a[1] += 1.0;
            a[4] += (double)sa;
            a[5] += (double)sb;
            const float gd = gt_depth[p];
            const float e = depth[p] - gd;
            if (depth_index[p] != -1 && gd > 0.f && e < depth_error_max) { a[2] += (double)fabsf(e); a[3] += 1.0; }
        }
    }
#pragma unroll
    for (int k = 0; k < RTG_LOSS_EXP_TERMS; k++)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a[k] += __shfl_xor_sync(0xffffffffu, a[k], o);
    __shared__ double s_p[8][RTG_LOSS_EXP_TERMS];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < RTG_LOSS_EXP_TERMS; k++) s_p[w][k] = a[k];
    __syncthreads();
    if (threadIdx.x < RTG_LOSS_EXP_TERMS) {
        double t = 0.0;
        for (int k = 0; k < 8; k++) t += s_p[k][threadIdx.x];
        ws->partial[blockIdx.x][threadIdx.x] = t;
    }
}

// One block: warp k adds term k over the blocks' partial sums (fixed lane stride, fixed butterfly); thread 0 writes the
// statistics loss_grad's scales are made of, the loss parts and dL/d(a, b).
__global__ void __launch_bounds__(32 * RTG_LOSS_EXP_TERMS) loss_exposure_final_kernel(int nb, float color_weight, float depth_weight,
                                                                                      LossExposureWs *ws,
                                                                                      float *__restrict__ dL_dexposure,
                                                                                      float *__restrict__ loss_out) {
    __shared__ double s_t[RTG_LOSS_EXP_TERMS];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    double acc = 0.0;
    for (int k = lane; k < nb; k += 32) acc += ws->partial[k][w];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) s_t[w] = acc;
    __syncthreads();
    if (threadIdx.x != 0) return;
#pragma unroll
    for (int k = 0; k < 4; k++) ws->st.v[k] = s_t[k];
    const double nc = s_t[1], nd = s_t[3];
    const double cl = nc > 0.0 ? s_t[0] / (3.0 * nc) : 0.0, dl = nd > 0.0 ? s_t[2] / nd : 0.0;
    loss_out[0] = (float)((double)color_weight * cl + (double)depth_weight * dl);
    loss_out[1] = (float)cl;
    loss_out[2] = (float)dl;
    loss_out[3] = (float)nd;
    const double gcs = nc > 0.0 ? (double)color_weight / (3.0 * nc) : 0.0;
    dL_dexposure[0] = (float)(gcs * s_t[4]);
    dL_dexposure[1] = (float)(gcs * s_t[5]);
}

__global__ void __launch_bounds__(256) loss_exposure_grad_kernel(const float *__restrict__ render, const float *__restrict__ depth,
                                                                 const int *__restrict__ depth_index, const float *__restrict__ gt_color,
                                                                 const float *__restrict__ gt_depth, const uint8_t *__restrict__ mask,
                                                                 int N, int channels_last, float depth_error_max, float color_weight,
                                                                 float depth_weight, const float *__restrict__ exposure,
                                                                 const LossExposureWs *ws, float *__restrict__ dL_dcolor,
                                                                 float *__restrict__ dL_ddepth) {
    const double nc = ws->st.v[1], nd = ws->st.v[3];
    const float ea = expf(exposure[0]), eb = exposure[1];
    // the scale of rtg_loss_l1 times e^a (e^0 = 1 leaves it bit-equal)
    const float gcs = (nc > 0.0 ? (float)((double)color_weight / (3.0 * nc)) : 0.f) * ea;
    const float gds = nd > 0.0 ? (float)((double)depth_weight / nd) : 0.f;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        const bool m = mask ? (mask[p] != 0) : true;
        float g0 = 0.f, g1 = 0.f, g2 = 0.f, gd_ = 0.f;
        if (m) {
            const float t0 = channels_last ? gt_color[3 * (size_t)p + 0] : gt_color[p];
            const float t1 = channels_last ? gt_color[3 * (size_t)p + 1] : gt_color[(size_t)N + p];
            const float t2 = channels_last ? gt_color[3 * (size_t)p + 2] : gt_color[2 * (size_t)N + p];
            g0 = gcs * sgn(fmaf(ea, render[p], eb) - t0);
            g1 = gcs * sgn(fmaf(ea, render[(size_t)N + p], eb) - t1);
            g2 = gcs * sgn(fmaf(ea, render[2 * (size_t)N + p], eb) - t2);
            const float gd = gt_depth[p];
            const float e = depth[p] - gd;
            if (depth_index[p] != -1 && gd > 0.f && e < depth_error_max) gd_ = gds * sgn(e);
        }
        dL_dcolor[p] = g0; dL_dcolor[(size_t)N + p] = g1; dL_dcolor[2 * (size_t)N + p] = g2;
        dL_ddepth[p] = gd_;
    }
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

// ---- the same loss with the cosine normal term of Mapping.loss_update (mapper.py:433-442):
//   normal_loss = mean over {render_mask & depth_index != -1 & gt_normal != 0} of 1 - cosine_similarity(normal, gt_normal)
// (F.cosine_similarity: x.y / (max(|x|, 1e-8) * max(|y|, 1e-8))). render_normal (3,H,W), gt_normal (H,W,3).
struct LossStats2 {
    double v[8];  // sum|dC|, n_colour, sum|dd|, n_depth, sum(1-cos), n_normal
};

__global__ void loss2_init_kernel(LossStats2 *st) {
    if (threadIdx.x < 8) st->v[threadIdx.x] = 0.0;
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

__global__ void __launch_bounds__(256) loss2_reduce_kernel(const float *__restrict__ render, const float *__restrict__ depth,
                                                           const float *__restrict__ nrm, const int *__restrict__ depth_index,
                                                           const float *__restrict__ gt_color, const float *__restrict__ gt_depth,
                                                           const float *__restrict__ gt_normal, const uint8_t *__restrict__ mask, int N,
                                                           int channels_last, float depth_error_max, LossStats2 *st) {
    double a[6] = {0, 0, 0, 0, 0, 0};
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        const bool m = mask ? (mask[p] != 0) : true;
        if (!m) continue;
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const float g = channels_last ? gt_color[3 * (size_t)p + c] : gt_color[(size_t)c * N + p];
            s += fabsf(render[(size_t)c * N + p] - g);
        }
        a[0] += (double)s; a[1] += 1.0;
        const float gd = gt_depth[p];
        const float e = depth[p] - gd;
        const bool has = depth_index[p] != -1;
        if (has && gd > 0.f && e < depth_error_max) { a[2] += (double)fabsf(e); a[3] += 1.0; }
        if (nrm && has) {
            float cosv, x0, x1, x2, y0, y1, y2, nx, ny;
            if (normal_term(nrm, gt_normal, N, p, cosv, x0, x1, x2, y0, y1, y2, nx, ny)) { a[4] += (double)(1.f - cosv); a[5] += 1.0; }
        }
    }
#pragma unroll
    for (int k = 0; k < 6; k++)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a[k] += __shfl_xor_sync(0xffffffffu, a[k], o);
    __shared__ double s_p[8][6];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0)
        for (int k = 0; k < 6; k++) s_p[w][k] = a[k];
    __syncthreads();
    if (threadIdx.x < 6) {
        double t = 0.0;
        for (int k = 0; k < 8; k++) t += s_p[k][threadIdx.x];
        atomicAdd(&st->v[threadIdx.x], t);
    }
}

__global__ void __launch_bounds__(256) loss2_grad_kernel(const float *__restrict__ render, const float *__restrict__ depth,
                                                         const float *__restrict__ nrm, const int *__restrict__ depth_index,
                                                         const float *__restrict__ gt_color, const float *__restrict__ gt_depth,
                                                         const float *__restrict__ gt_normal, const uint8_t *__restrict__ mask, int N,
                                                         int channels_last, float depth_error_max, float color_weight, float depth_weight,
                                                         float normal_weight, const LossStats2 *st, float *__restrict__ dL_dcolor,
                                                         float *__restrict__ dL_ddepth, float *__restrict__ dL_dnormal,
                                                         float *__restrict__ loss_out) {
    const double nc = st->v[1], nd = st->v[3], nn = st->v[5];
    const float gcs = nc > 0.0 ? (float)((double)color_weight / (3.0 * nc)) : 0.f;
    const float gds = nd > 0.0 ? (float)((double)depth_weight / nd) : 0.f;
    const float gns = nn > 0.0 ? (float)((double)normal_weight / nn) : 0.f;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const double cl = nc > 0.0 ? st->v[0] / (3.0 * nc) : 0.0, dl = nd > 0.0 ? st->v[2] / nd : 0.0, nl = nn > 0.0 ? st->v[4] / nn : 0.0;
        loss_out[0] = (float)((double)color_weight * cl + (double)depth_weight * dl + (double)normal_weight * nl);
        loss_out[1] = (float)cl; loss_out[2] = (float)dl; loss_out[3] = (float)nd; loss_out[4] = (float)nl; loss_out[5] = (float)nn;
        loss_out[6] = 0.f; loss_out[7] = 0.f;
    }
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        const bool m = mask ? (mask[p] != 0) : true;
        float g0 = 0.f, g1 = 0.f, g2 = 0.f, gd_ = 0.f, n0 = 0.f, n1 = 0.f, n2 = 0.f;
        if (m) {
            const float t0 = channels_last ? gt_color[3 * (size_t)p + 0] : gt_color[p];
            const float t1 = channels_last ? gt_color[3 * (size_t)p + 1] : gt_color[(size_t)N + p];
            const float t2 = channels_last ? gt_color[3 * (size_t)p + 2] : gt_color[2 * (size_t)N + p];
            g0 = gcs * sgn(render[p] - t0);
            g1 = gcs * sgn(render[(size_t)N + p] - t1);
            g2 = gcs * sgn(render[2 * (size_t)N + p] - t2);
            const float gd = gt_depth[p];
            const float e = depth[p] - gd;
            const bool has = depth_index[p] != -1;
            if (has && gd > 0.f && e < depth_error_max) gd_ = gds * sgn(e);
            if (nrm && has) {
                float cosv, x0, x1, x2, y0, y1, y2, nx, ny;
                if (normal_term(nrm, gt_normal, N, p, cosv, x0, x1, x2, y0, y1, y2, nx, ny)) {
                    // d(1 - cos)/dx = -( y / (|x||y|) - cos * x / |x|^2 )
                    const float a = 1.f / (nx * ny), bq = cosv / (nx * nx);
                    n0 = -gns * (y0 * a - x0 * bq); n1 = -gns * (y1 * a - x1 * bq); n2 = -gns * (y2 * a - x2 * bq);
                }
            }
        }
        dL_dcolor[p] = g0; dL_dcolor[(size_t)N + p] = g1; dL_dcolor[2 * (size_t)N + p] = g2;
        dL_ddepth[p] = gd_;
        if (dL_dnormal) { dL_dnormal[p] = n0; dL_dnormal[(size_t)N + p] = n1; dL_dnormal[2 * (size_t)N + p] = n2; }
    }
}

size_t loss_ws_bytes() { return sizeof(LossStats2); }

void launch_loss_mapping(const float *render, const float *depth, const float *render_normal, const int *depth_index,
                         const float *gt_color, const float *gt_depth, const float *gt_normal, const uint8_t *mask, int H, int W,
                         int channels_last, float color_weight, float depth_weight, float normal_weight, float depth_error_max,
                         float *dL_dcolor, float *dL_ddepth, float *dL_dnormal, float *loss_out, void *ws, cudaStream_t s) {
    ProfScope ps(K_ICP_MISC, s);
    LossStats2 *st = reinterpret_cast<LossStats2 *>(ws);
    const int N = H * W;
    int nb = (N + 255) / 256;
    if (nb > RTG_NUM_SMS * 8) nb = RTG_NUM_SMS * 8;
    const float *nrm = (normal_weight > 0.f) ? render_normal : nullptr;
    loss2_init_kernel<<<1, 32, 0, s>>>(st);
    loss2_reduce_kernel<<<nb, 256, 0, s>>>(render, depth, nrm, depth_index, gt_color, gt_depth, gt_normal, mask, N, channels_last,
                                           depth_error_max, st);
    loss2_grad_kernel<<<nb, 256, 0, s>>>(render, depth, nrm, depth_index, gt_color, gt_depth, gt_normal, mask, N, channels_last,
                                         depth_error_max, color_weight, depth_weight, normal_weight, st, dL_dcolor, dL_ddepth,
                                         dL_dnormal, loss_out);
}

void launch_loss_l1(const float *render, const float *depth, const int *depth_index, const float *gt_color, const float *gt_depth,
                    const uint8_t *mask, int H, int W, int channels_last, float color_weight, float depth_weight,
                    float depth_error_max, float *dL_dcolor, float *dL_ddepth, float *loss_out, void *ws, cudaStream_t s) {
    ProfScope ps(K_ICP_MISC, s);
    LossStats *st = reinterpret_cast<LossStats *>(ws);
    const int N = H * W;
    int nb = (N + 255) / 256;
    if (nb > RTG_NUM_SMS * 8) nb = RTG_NUM_SMS * 8;
    loss_init_kernel<<<1, 32, 0, s>>>(st);
    loss_reduce_kernel<<<nb, 256, 0, s>>>(render, depth, depth_index, gt_color, gt_depth, mask, N, channels_last, depth_error_max, st);
    loss_grad_kernel<<<nb, 256, 0, s>>>(render, depth, depth_index, gt_color, gt_depth, mask, N, channels_last, depth_error_max,
                                        color_weight, depth_weight, st, dL_dcolor, dL_ddepth, loss_out);
}

size_t loss_exposure_ws_bytes() { return sizeof(LossExposureWs); }

void launch_loss_l1_exposure(const float *render, const float *depth, const int *depth_index, const float *gt_color,
                             const float *gt_depth, const uint8_t *mask, int H, int W, int channels_last, float color_weight,
                             float depth_weight, float depth_error_max, const float *exposure, float *dL_dcolor, float *dL_ddepth,
                             float *dL_dexposure, float *loss_out, void *ws, cudaStream_t s) {
    ProfScope ps(K_ICP_MISC, s);
    LossExposureWs *w = reinterpret_cast<LossExposureWs *>(ws);
    const int N = H * W;
    int nb = (N + 255) / 256;
    if (nb > RTG_NUM_SMS * 8) nb = RTG_NUM_SMS * 8;
    loss_exposure_reduce_kernel<<<nb, 256, 0, s>>>(render, depth, depth_index, gt_color, gt_depth, mask, N, channels_last,
                                                   depth_error_max, exposure, w);
    loss_exposure_final_kernel<<<1, 32 * RTG_LOSS_EXP_TERMS, 0, s>>>(nb, color_weight, depth_weight, w, dL_dexposure, loss_out);
    loss_exposure_grad_kernel<<<nb, 256, 0, s>>>(render, depth, depth_index, gt_color, gt_depth, mask, N, channels_last,
                                                 depth_error_max, color_weight, depth_weight, exposure, w, dL_dcolor, dL_ddepth);
}

void launch_normal_map(const float *normal, const int *depth_index, int H, int W, float *out, cudaStream_t s) {
    ProfScope ps(K_ICP_MISC, s);
    const int N = H * W;
    normal_map_kernel<<<(N + 255) / 256, 256, 0, s>>>(normal, depth_index, N, out);
}

}  // namespace rtg
