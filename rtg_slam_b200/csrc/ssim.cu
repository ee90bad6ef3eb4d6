// Fused SSIM term of the mapping loss (SURVEY.md section 8(f) #1): value and gradient in three launches.
//
// Reference arithmetic (eager PyTorch: five grouped 11x11 convolutions + ~15 elementwise kernels, and autograd builds the
// transposed convolutions again in the backward):
//   utils/loss_utils.py:40-60    gaussian(11, 1.5), create_window (outer product, one window per channel), ssim
//   utils/loss_utils.py:63-100   _ssim: mu = conv(img), sigma = conv(img*img) - mu^2, zero padding 5, C1 = 0.01^2, C2 = 0.03^2,
//                                ssim_map.mean()
//   SLAM/multiprocess/mapper.py:411-415   ssim_loss = 1 - ssim(render, gt) (only without a render mask)
//
// Design: the window is an outer product, so every 11x11 convolution is two 11-tap passes through shared memory. One CTA
// owns a 16x16 tile of one channel (26x26 with the halo). The forward pass also leaves the three partial-derivative maps
//   dS/dmu1, dS/dE[x^2], dS/dE[xy]      (S = ssim_map, all five window means treated as independent variables)
// and the backward pass is the same separable convolution over those maps:
//   dS_total/dx_p = sum_q w(q - p) * (dS_q/dmu1 + 2 x_p dS_q/dE[x^2] + y_p dS_q/dE[xy])
// (zero padding in the forward = maps that are zero outside the image in the backward; the window is symmetric).
// The mean is a deterministic two-stage reduction in double (per-CTA partials, one CTA sums them in a fixed order).
#include "common.cuh"
#include "prof.h"

namespace rtg {

#define SSIM_T 16                     // output tile edge
#define SSIM_R 5                      // window radius
#define SSIM_K (2 * SSIM_R + 1)       // 11 taps
#define SSIM_E (SSIM_T + 2 * SSIM_R)  // tile + halo

struct SsimWindow {
    float g[SSIM_K];
};

// one CTA (256 threads) = one 16x16 tile of channel blockIdx.z. EXPOSURE: img1 is read as e^a img1 + b, (ea, eb) =
// (e^a, b) (zero padding stays zero: the padded image is the exposed one).
template <bool EXPOSURE>
__global__ void __launch_bounds__(256) ssim_fwd_kernel(const float *__restrict__ img1, const float *__restrict__ img2, int H, int W,
                                                       const SsimWindow win, float *__restrict__ d_mu1, float *__restrict__ d_e11,
                                                       float *__restrict__ d_e12, double *__restrict__ partial,
                                                       const float *__restrict__ exposure) {
    __shared__ float s_x[SSIM_E][SSIM_E + 1];
    __shared__ float s_y[SSIM_E][SSIM_E + 1];
    __shared__ float s_h[5][SSIM_E][SSIM_T];
    __shared__ double s_sum[8];
    const int tid = threadIdx.x;
    const int x0 = blockIdx.x * SSIM_T, y0 = blockIdx.y * SSIM_T;
    const size_t plane = (size_t)blockIdx.z * (size_t)H * (size_t)W;
    float ea = 1.f, eb = 0.f;
    if constexpr (EXPOSURE) { ea = expf(exposure[0]); eb = exposure[1]; }

    for (int k = tid; k < SSIM_E * SSIM_E; k += 256) {
        const int r = k / SSIM_E, q = k - r * SSIM_E;
        const int gy = y0 + r - SSIM_R, gx = x0 + q - SSIM_R;
        float a = 0.f, b = 0.f;  // zero padding (F.conv2d(..., padding=5))
        if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
            const size_t o = plane + (size_t)gy * W + gx;
            if constexpr (EXPOSURE) a = fmaf(ea, img1[o], eb);
            else a = img1[o];
            b = img2[o];
        }
        s_x[r][q] = a;
        s_y[r][q] = b;
    }
    __syncthreads();
    // horizontal pass: 26 rows x 16 columns, five window sums each
    for (int k = tid; k < SSIM_E * SSIM_T; k += 256) {
        const int r = k / SSIM_T, q = k - r * SSIM_T;
        float m1 = 0.f, m2 = 0.f, e11 = 0.f, e22 = 0.f, e12 = 0.f;
#pragma unroll
        for (int t = 0; t < SSIM_K; t++) {
            const float g = win.g[t], a = s_x[r][q + t], b = s_y[r][q + t];
            m1 = fmaf(g, a, m1);
            m2 = fmaf(g, b, m2);
            e11 = fmaf(g, a * a, e11);
            e22 = fmaf(g, b * b, e22);
            e12 = fmaf(g, a * b, e12);
        }
        s_h[0][r][q] = m1; s_h[1][r][q] = m2; s_h[2][r][q] = e11; s_h[3][r][q] = e22; s_h[4][r][q] = e12;
    }
    __syncthreads();
    // vertical pass: one output pixel per thread
    const int tx = tid & (SSIM_T - 1), ty = tid >> 4;
    float m1 = 0.f, m2 = 0.f, e11 = 0.f, e22 = 0.f, e12 = 0.f;
#pragma unroll
    for (int t = 0; t < SSIM_K; t++) {
        const float g = win.g[t];
        m1 = fmaf(g, s_h[0][ty + t][tx], m1);
        m2 = fmaf(g, s_h[1][ty + t][tx], m2);
        e11 = fmaf(g, s_h[2][ty + t][tx], e11);
        e22 = fmaf(g, s_h[3][ty + t][tx], e22);
        e12 = fmaf(g, s_h[4][ty + t][tx], e12);
    }
    const int gx = x0 + tx, gy = y0 + ty;
    float S = 0.f;
    if (gx < W && gy < H) {
        const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
        const float mu1_sq = m1 * m1, mu2_sq = m2 * m2, mu12 = m1 * m2;
        const float A1 = 2.f * mu12 + C1, A2 = 2.f * (e12 - mu12) + C2;
        const float B1 = mu1_sq + mu2_sq + C1, B2 = (e11 - mu1_sq) + (e22 - mu2_sq) + C2;
        const float inv = 1.f / (B1 * B2);
        S = A1 * A2 * inv;
        if (d_mu1) {
            const size_t o = plane + (size_t)gy * W + gx;
            d_mu1[o] = 2.f * m2 * (A2 - A1) * inv - 2.f * m1 * S * (1.f / B1 - 1.f / B2);
            d_e11[o] = -S / B2;
            d_e12[o] = 2.f * A1 * inv;
        }
    }
    double v = (double)S;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((tid & 31) == 0) s_sum[tid >> 5] = v;
    __syncthreads();
    if (tid == 0) {
        double t = 0.0;
        for (int k = 0; k < 8; k++) t += s_sum[k];
        partial[((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = t;
    }
}

// loss_out = {1 - mean(ssim_map), mean(ssim_map)}; partials summed in a fixed order (bit-reproducible)
__global__ void __launch_bounds__(256) ssim_final_kernel(const double *__restrict__ partial, int n, double inv_count,
                                                         float *__restrict__ loss_out) {
    __shared__ double s[256];
    double a = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) a += partial[i];
    s[threadIdx.x] = a;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const double m = s[0] * inv_count;
        loss_out[0] = (float)(1.0 - m);
        loss_out[1] = (float)m;
    }
}

// dL/dimg1 for L = 1 - mean(ssim_map): scale = -1 / (C*H*W). EXPOSURE: with x^ = e^a img1 + b the exposed image,
// dL/dx^ is the expression below evaluated on x^, dL/dimg1 = e^a dL/dx^ (dL_dimg1 may then be NULL), and the CTA writes the
// double partials (sum dL/dx^ e^a img1, sum dL/dx^) of dL/da and dL/db to exposure_partial[2 * CTA + {0, 1}].
template <bool EXPOSURE>
__global__ void __launch_bounds__(256) ssim_bwd_kernel(const float *__restrict__ img1, const float *__restrict__ img2, int H, int W,
                                                       const SsimWindow win, const float *__restrict__ d_mu1,
                                                       const float *__restrict__ d_e11, const float *__restrict__ d_e12, float scale,
                                                       float *__restrict__ dL_dimg1, const float *__restrict__ exposure,
                                                       double *__restrict__ exposure_partial) {
    __shared__ float s_d[3][SSIM_E][SSIM_E + 1];
    __shared__ float s_h[3][SSIM_E][SSIM_T];
    const int tid = threadIdx.x;
    const int x0 = blockIdx.x * SSIM_T, y0 = blockIdx.y * SSIM_T;
    const size_t plane = (size_t)blockIdx.z * (size_t)H * (size_t)W;
    for (int k = tid; k < SSIM_E * SSIM_E; k += 256) {
        const int r = k / SSIM_E, q = k - r * SSIM_E;
        const int gy = y0 + r - SSIM_R, gx = x0 + q - SSIM_R;
        float a = 0.f, b = 0.f, c = 0.f;  // pixels outside the image have no ssim_map entry
        if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
            const size_t o = plane + (size_t)gy * W + gx;
            a = d_mu1[o];
            b = d_e11[o];
            c = d_e12[o];
        }
        s_d[0][r][q] = a; s_d[1][r][q] = b; s_d[2][r][q] = c;
    }
    __syncthreads();
    for (int k = tid; k < SSIM_E * SSIM_T; k += 256) {
        const int r = k / SSIM_T, q = k - r * SSIM_T;
        float a = 0.f, b = 0.f, c = 0.f;
#pragma unroll
        for (int t = 0; t < SSIM_K; t++) {
            const float g = win.g[t];
            a = fmaf(g, s_d[0][r][q + t], a);
            b = fmaf(g, s_d[1][r][q + t], b);
            c = fmaf(g, s_d[2][r][q + t], c);
        }
        s_h[0][r][q] = a; s_h[1][r][q] = b; s_h[2][r][q] = c;
    }
    __syncthreads();
    const int tx = tid & (SSIM_T - 1), ty = tid >> 4;
    float a = 0.f, b = 0.f, c = 0.f;
#pragma unroll
    for (int t = 0; t < SSIM_K; t++) {
        const float g = win.g[t];
        a = fmaf(g, s_h[0][ty + t][tx], a);
        b = fmaf(g, s_h[1][ty + t][tx], b);
        c = fmaf(g, s_h[2][ty + t][tx], c);
    }
    const int gx = x0 + tx, gy = y0 + ty;
    if constexpr (EXPOSURE) {
        __shared__ double s_e[2][8];
        const float ea = expf(exposure[0]), eb = exposure[1];
        double va = 0.0, vb = 0.0;
        if (gx < W && gy < H) {
            const size_t o = plane + (size_t)gy * W + gx;
            const float x = img1[o], ex = ea * x;
            const float g = scale * (a + 2.f * fmaf(ea, x, eb) * b + img2[o] * c);
            if (dL_dimg1) dL_dimg1[o] = ea * g;
            va = (double)g * (double)ex;
            vb = (double)g;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            va += __shfl_xor_sync(0xffffffffu, va, o);
            vb += __shfl_xor_sync(0xffffffffu, vb, o);
        }
        if ((tid & 31) == 0) { s_e[0][tid >> 5] = va; s_e[1][tid >> 5] = vb; }
        __syncthreads();
        if (tid < 2) {
            double t = 0.0;
            for (int k = 0; k < 8; k++) t += s_e[tid][k];
            exposure_partial[2 * (((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) + tid] = t;
        }
    } else if (gx < W && gy < H) {
        const size_t o = plane + (size_t)gy * W + gx;
        dL_dimg1[o] = scale * (a + 2.f * img1[o] * b + img2[o] * c);
    }
}

// dL_dexposure = (sum of the CTAs' dL/da partials, sum of their dL/db partials), added in a fixed order (bit-reproducible)
__global__ void __launch_bounds__(256) ssim_exposure_final_kernel(const double *__restrict__ exposure_partial, int n,
                                                                  float *__restrict__ dL_dexposure) {
    __shared__ double s[2][256];
    double a = 0.0, b = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) { a += exposure_partial[2 * i]; b += exposure_partial[2 * i + 1]; }
    s[0][threadIdx.x] = a;
    s[1][threadIdx.x] = b;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) { s[0][threadIdx.x] += s[0][threadIdx.x + o]; s[1][threadIdx.x] += s[1][threadIdx.x + o]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { dL_dexposure[0] = (float)s[0][0]; dL_dexposure[1] = (float)s[1][0]; }
}

static inline size_t ssim_tiles(int C, int H, int W) {
    return (size_t)C * (size_t)((H + SSIM_T - 1) / SSIM_T) * (size_t)((W + SSIM_T - 1) / SSIM_T);
}

static inline size_t ssim_partial_bytes(int C, int H, int W) { return (ssim_tiles(C, H, W) * sizeof(double) + 255) & ~(size_t)255; }

// per-CTA partial sums (double) + the three derivative maps
size_t ssim_ws_bytes(int C, int H, int W) { return ssim_partial_bytes(C, H, W) + 3 * (size_t)C * H * W * sizeof(float); }

// ssim_ws_bytes rounded up to 256 bytes (the derivative maps end on any 4-byte boundary), then the per-CTA double partials
// of the two exposure sums
static inline size_t ssim_exposure_partial_offset(int C, int H, int W) { return (ssim_ws_bytes(C, H, W) + 255) & ~(size_t)255; }
size_t ssim_exposure_ws_bytes(int C, int H, int W) { return ssim_exposure_partial_offset(C, H, W) + 2 * ssim_partial_bytes(C, H, W); }

// gaussian(11, 1.5) of utils/loss_utils.py:40-47: fp32 values of exp(-(x-5)^2 / (2 sigma^2)), normalised in fp32
static SsimWindow ssim_window() {
    SsimWindow win;
    float sum = 0.f;
    for (int x = 0; x < SSIM_K; x++) {
        win.g[x] = (float)exp(-(double)((x - SSIM_R) * (x - SSIM_R)) / (2.0 * 1.5 * 1.5));
        sum += win.g[x];
    }
    for (int x = 0; x < SSIM_K; x++) win.g[x] /= sum;
    return win;
}

void launch_ssim_loss(const float *img1, const float *img2, int C, int H, int W, float *dL_dimg1, float *loss_out, void *ws,
                      cudaStream_t s) {
    ProfScope ps(K_ICP_MISC, s);
    const SsimWindow win = ssim_window();
    double *partial = reinterpret_cast<double *>(ws);
    const size_t n_px = (size_t)C * H * W;
    float *d_mu1 = dL_dimg1 ? reinterpret_cast<float *>(reinterpret_cast<char *>(ws) + ssim_partial_bytes(C, H, W)) : nullptr;
    float *d_e11 = dL_dimg1 ? d_mu1 + n_px : nullptr, *d_e12 = dL_dimg1 ? d_mu1 + 2 * n_px : nullptr;
    const dim3 grid((W + SSIM_T - 1) / SSIM_T, (H + SSIM_T - 1) / SSIM_T, C);
    ssim_fwd_kernel<false><<<grid, 256, 0, s>>>(img1, img2, H, W, win, d_mu1, d_e11, d_e12, partial, nullptr);
    ssim_final_kernel<<<1, 256, 0, s>>>(partial, (int)ssim_tiles(C, H, W), 1.0 / (double)n_px, loss_out);
    if (dL_dimg1)
        ssim_bwd_kernel<false><<<grid, 256, 0, s>>>(img1, img2, H, W, win, d_mu1, d_e11, d_e12, (float)(-1.0 / (double)n_px), dL_dimg1,
                                                    nullptr, nullptr);
}

// Workspace: [value partials | derivative maps | exposure partials] (ssim_exposure_ws_bytes). The backward runs when either
// gradient is wanted; the derivative maps are written only then.
void launch_ssim_loss_exposure(const float *img1, const float *img2, int C, int H, int W, const float *exposure, float *dL_dimg1,
                               float *dL_dexposure, float *loss_out, void *ws, cudaStream_t s) {
    ProfScope ps(K_ICP_MISC, s);
    const SsimWindow win = ssim_window();
    double *partial = reinterpret_cast<double *>(ws);
    const size_t n_px = (size_t)C * H * W;
    const bool grad = dL_dimg1 || dL_dexposure;
    char *base = reinterpret_cast<char *>(ws);
    float *d_mu1 = grad ? reinterpret_cast<float *>(base + ssim_partial_bytes(C, H, W)) : nullptr;
    float *d_e11 = grad ? d_mu1 + n_px : nullptr, *d_e12 = grad ? d_mu1 + 2 * n_px : nullptr;
    double *exposure_partial = reinterpret_cast<double *>(base + ssim_exposure_partial_offset(C, H, W));
    const int tiles = (int)ssim_tiles(C, H, W);
    const dim3 grid((W + SSIM_T - 1) / SSIM_T, (H + SSIM_T - 1) / SSIM_T, C);
    ssim_fwd_kernel<true><<<grid, 256, 0, s>>>(img1, img2, H, W, win, d_mu1, d_e11, d_e12, partial, exposure);
    ssim_final_kernel<<<1, 256, 0, s>>>(partial, tiles, 1.0 / (double)n_px, loss_out);
    if (!grad) return;
    ssim_bwd_kernel<true><<<grid, 256, 0, s>>>(img1, img2, H, W, win, d_mu1, d_e11, d_e12, (float)(-1.0 / (double)n_px), dL_dimg1,
                                               exposure, exposure_partial);
    if (dL_dexposure) ssim_exposure_final_kernel<<<1, 256, 0, s>>>(exposure_partial, tiles, dL_dexposure);
}

}  // namespace rtg
