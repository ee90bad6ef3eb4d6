// Projective point-to-plane ICP on the device, no host round trips.
//
// The reference (SLAM/icp.py) runs ~40 eager PyTorch ops per Gauss-Newton iteration, materialises an
// (HW,3,3) skew tensor and an (HW,6,6) outer-product tensor, inverts the 6x6 system on the CPU and
// rebuilds small tensors from device scalars (>= 3 host syncs per iteration). Here one kernel per
// iteration computes the per-pixel residual and Jacobian row, reduces the 27 unique normal-equation
// terms (+ valid count) by a transposing warp butterfly and per-block double partials, and the last
// block to finish solves the damped 6x6 system, applies exp_se3 and updates the pose in place.
// icp_predict_kernel<true> adds a photometric row (RGB-D odometry) to the same normal equations.
#include "common.cuh"
#include "kernels.h"
#include "prof.h"
#include "../../include/rtg_splat_b200.h"

namespace rtg {

#define ICP_THREADS 256
#define ICP_MAX_BLOCKS (RTG_NUM_SMS * 4)
#define ICP_TERMS 32        // 21 (JtJ upper) + 6 (Jtr) + 1 (valid) [+ 2 (photometric count, sum r^2)] padded to 32

#define ICP_MAX_LEVELS RTG_ICP_MAX_LEVELS
struct IcpWs {
    int minmax[2];       // ordered-int encoded min / max depth of the level being built
    unsigned int ticket; // blocks-finished counter for the last-block reduction
    unsigned int barrier;               // arrival counter of the grid barrier of the persistent kernels
    int level_minmax[2 * ICP_MAX_LEVELS];
    double partial[ICP_MAX_BLOCKS * ICP_TERMS];
    double partial2[ICP_MAX_BLOCKS * ICP_TERMS];  // second buffer: iteration k+1 writes while slow blocks still read k
};

__device__ __forceinline__ int float_to_ordered(float f) {
    const int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ordered_to_float(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

__global__ void icp_ws_init_kernel(IcpWs *ws) {
    ws->minmax[0] = 0x7fffffff;
    ws->minmax[1] = (int)0x80000000;
    ws->ticket = 0;
}

// max-pool + back-projection (MaxPool2d k=stride=pool: SLAM/icp.py:343-345; compute_vertex_map: SLAM/utils.py:65-75)
__global__ void __launch_bounds__(256) icp_vertex_kernel(const float *__restrict__ depth, int H, int W, int pool, int Hs, int Ws,
                                                         float fx, float fy, float cx, float cy, float *__restrict__ vertex,
                                                         IcpWs *ws) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    float d = 0.f;
    const bool ok = idx < Hs * Ws;
    if (ok) {
        const int ys = idx / Ws, xs = idx % Ws;
        d = -INFINITY;
        for (int a = 0; a < pool; a++)
            for (int c = 0; c < pool; c++) d = fmaxf(d, depth[(size_t)(ys * pool + a) * W + xs * pool + c]);
        float *v = vertex + 3 * (size_t)idx;
        v[0] = (((float)xs - cx) / fx) * d;
        v[1] = (((float)ys - cy) / fy) * d;
        v[2] = 1.0f * d;
    }
    float mn = ok ? d : INFINITY, mx = ok ? d : -INFINITY;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMin(&ws->minmax[0], float_to_ordered(mn));
        atomicMax(&ws->minmax[1], float_to_ordered(mx));
    }
}

// Sobel normals with replicate padding, normalised, zeroed at the global depth extremes
// (compute_normal_map + feature_gradient: SLAM/utils.py:77-122)
__global__ void __launch_bounds__(256) icp_normal_kernel(const float *__restrict__ vertex, int Hs, int Ws, float *__restrict__ normal,
                                                         const IcpWs *ws) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= Hs * Ws) return;
    const int y = idx / Ws, x = idx % Ws;
    const int ym = max(y - 1, 0), yp = min(y + 1, Hs - 1), xm = max(x - 1, 0), xp = min(x + 1, Ws - 1);
    float dx[3], dy[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        const float a00 = vertex[3 * ((size_t)ym * Ws + xm) + c], a01 = vertex[3 * ((size_t)ym * Ws + x) + c], a02 = vertex[3 * ((size_t)ym * Ws + xp) + c];
        const float a10 = vertex[3 * ((size_t)y * Ws + xm) + c], a12 = vertex[3 * ((size_t)y * Ws + xp) + c];
        const float a20 = vertex[3 * ((size_t)yp * Ws + xm) + c], a21 = vertex[3 * ((size_t)yp * Ws + x) + c], a22 = vertex[3 * ((size_t)yp * Ws + xp) + c];
        dx[c] = -a00 + a02 - 2.f * a10 + 2.f * a12 - a20 + a22;
        dy[c] = -a00 - 2.f * a01 - a02 + a20 + 2.f * a21 + a22;
    }
    // normal = cross(img_dy, img_dx)
    float nx = dy[1] * dx[2] - dy[2] * dx[1];
    float ny = dy[2] * dx[0] - dy[0] * dx[2];
    float nz = dy[0] * dx[1] - dy[1] * dx[0];
    const float mag = sqrtf(nx * nx + ny * ny + nz * nz);
    const float inv = 1.0f / (mag + 1e-8f);
    nx *= inv; ny *= inv; nz *= inv;
    const float d = vertex[3 * (size_t)idx + 2];
    const float dmin = ordered_to_float(ws->minmax[0]), dmax = ordered_to_float(ws->minmax[1]);
    if (d <= dmin || d >= dmax) { nx = 0.f; ny = 0.f; nz = 0.f; }
    float *n = normal + 3 * (size_t)idx;
    n[0] = nx; n[1] = ny; n[2] = nz;
}

// Sum 32 per-lane values across the warp; afterwards lane k holds the total of value k.
__device__ __forceinline__ float warp_transpose_reduce32(float v[32], const int lane) {
#pragma unroll
    for (int i = 0; i < 16; i++) {
        const bool hi = lane & 16;
        const float send = hi ? v[i] : v[i + 16];
        const float keep = hi ? v[i + 16] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const bool hi = lane & 8;
        const float send = hi ? v[i] : v[i + 8];
        const float keep = hi ? v[i + 8] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const bool hi = lane & 4;
        const float send = hi ? v[i] : v[i + 4];
        const float keep = hi ? v[i + 4] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
    }
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const bool hi = lane & 2;
        const float send = hi ? v[i] : v[i + 2];
        const float keep = hi ? v[i + 2] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
    }
    {
        const bool hi = lane & 1;
        const float send = hi ? v[0] : v[1];
        const float keep = hi ? v[1] : v[0];
        v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 1);
    }
    return v[0];  // lane L holds value index bitrev-free: (b4<<4|b3<<3|b2<<2|b1<<1|b0) == L
}

// exp_se3 (SLAM/icp.py:271-310) and pose <- exp(xi) @ pose (forward_update_pose :259-268). Every loop has a
// compile-time trip count and is unrolled: the small matrices live in registers (the serial tail of every iteration
// runs on one thread; with dynamically indexed local arrays it cost more than the per-pixel pass of the coarse levels).
__device__ __forceinline__ void se3_update(const double xi[6], float *pose) {
    const double w0 = xi[0], w1 = xi[1], w2 = xi[2];
    const double Wh[3][3] = {{0.0, -w2, w1}, {w2, 0.0, -w0}, {-w1, w0, 0.0}};
    double W2[3][3];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) W2[i][j] = Wh[i][0] * Wh[0][j] + Wh[i][1] * Wh[1][j] + Wh[i][2] * Wh[2][j];
    const double theta = sqrt(w0 * w0 + w1 * w1 + w2 * w2);
    double E[3][3], J[3][3];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) { E[i][j] = (i == j); J[i][j] = (i == j); }
    if (!(theta <= 1e-8)) {
        const double th2 = theta * theta, th3 = th2 * theta, sn = sin(theta), cs = cos(theta);
        const double k1 = (1.0 - cs) / th2, k2 = (theta - sn) / th3;
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) {
                E[i][j] += Wh[i][j] * sn / theta + W2[i][j] * (1.0 - cs) / th2;
                J[i][j] += k1 * Wh[i][j] + k2 * W2[i][j];
            }
    }
    double Tm[3][4];
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
        for (int j = 0; j < 3; j++) Tm[i][j] = E[i][j];
        Tm[i][3] = J[i][0] * xi[3] + J[i][1] * xi[4] + J[i][2] * xi[5];
    }
    double P[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) P[i][j] = (double)pose[4 * i + j];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 4; j++)
            pose[4 * i + j] = (float)(Tm[i][0] * P[0][j] + Tm[i][1] * P[1][j] + Tm[i][2] * P[2][j] + Tm[i][3] * P[3][j]);
    // the last row of exp(xi) is (0, 0, 0, 1): the pose's last row is unchanged
}

// (solve6, the damped 6x6 Cholesky solve: common.cuh)

// One Gauss-Newton iteration (compute_residuals_jacobian + compute_jtj/jtr + GN_solver, SLAM/icp.py:52-130).
__global__ void __launch_bounds__(ICP_THREADS) icp_iter_kernel(const float *__restrict__ vertex0, const float *__restrict__ normal0,
                                                               const float *__restrict__ vertex1, const float *__restrict__ normal1,
                                                               int H, int W, float fx, float fy, float cx, float cy, float dist_thr,
                                                               float cos_thr, float damping, float *pose, float *valid_ratio,
                                                               IcpWs *ws) {
    __shared__ float s_red[ICP_THREADS / 32][ICP_TERMS];
    __shared__ bool s_last;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    float Rm[9], tv[3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
        for (int j = 0; j < 3; j++) Rm[3 * i + j] = pose[4 * i + j];
        tv[i] = pose[4 * i + 3];
    }
    float acc[ICP_TERMS];
#pragma unroll
    for (int k = 0; k < ICP_TERMS; k++) acc[k] = 0.f;
    const int HW = H * W;
    const float Wm1 = (float)(W - 1), Hm1 = (float)(H - 1);
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
        const float v0x = vertex0[3 * (size_t)p], v0y = vertex0[3 * (size_t)p + 1], v0z = vertex0[3 * (size_t)p + 2];
        const bool mask0 = v0z > 0.0f;
        const float n0x = normal0[3 * (size_t)p], n0y = normal0[3 * (size_t)p + 1], n0z = normal0[3 * (size_t)p + 2];
        const float x = Rm[0] * v0x + Rm[1] * v0y + Rm[2] * v0z + tv[0];
        const float y = Rm[3] * v0x + Rm[4] * v0y + Rm[5] * v0z + tv[1];
        const float z = Rm[6] * v0x + Rm[7] * v0y + Rm[8] * v0z + tv[2];
        const float nx = Rm[0] * n0x + Rm[1] * n0y + Rm[2] * n0z;
        const float ny = Rm[3] * n0x + Rm[4] * n0y + Rm[5] * n0z;
        const float nz = Rm[6] * n0x + Rm[7] * n0y + Rm[8] * n0z;
        const float u = (x / z) * fx + cx, v = (y / z) * fy + cy;
        const bool inview = (u > 0.f) && (u < Wm1) && (v > 0.f) && (v < Hm1);
        // warp_features: grid_sample(nearest, border, align_corners=True) (SLAM/icp.py:132-148)
        const float un = u / (Wm1 / 2.f) - 1.f, vn = v / (Hm1 / 2.f) - 1.f;
        float ix = ((un + 1.f) / 2.f) * Wm1, iy = ((vn + 1.f) / 2.f) * Hm1;
        ix = fminf(Wm1, fmaxf(ix, 0.f));
        iy = fminf(Hm1, fmaxf(iy, 0.f));
        int xi = (int)nearbyintf(ix), yi = (int)nearbyintf(iy);
        xi = min(W - 1, max(0, xi));
        yi = min(H - 1, max(0, yi));
        const size_t q = (size_t)yi * W + xi;
        const float rx = vertex1[3 * q], ry = vertex1[3 * q + 1], rz = vertex1[3 * q + 2];
        const float mx = normal1[3 * q], my = normal1[3 * q + 1], mz = normal1[3 * q + 2];
        const bool mask1 = rz > 0.f;
        const float dx = x - rx, dy = y - ry, dz = z - rz;
        const bool normal_ok = (nx * mx + ny * my + nz * mz) > cos_thr;
        const bool occ = !inview || (sqrtf(dx * dx + dy * dy + dz * dz) > dist_thr);
        const bool valid = !(occ || !mask0 || !mask1 || !normal_ok);
        if (valid) {
            const float res = mx * dx + my * dy + mz * dz;
            // J = [ -(n1^T [v']x) , n1^T ] = [ v' x n1 , n1 ]
            float J[6];
            J[0] = -(my * z - mz * y);
            J[1] = -(mz * x - mx * z);
            J[2] = -(mx * y - my * x);
            J[3] = mx; J[4] = my; J[5] = mz;
            int k = 0;
#pragma unroll
            for (int a = 0; a < 6; a++)
#pragma unroll
                for (int c = a; c < 6; c++) acc[k++] += J[a] * J[c];
#pragma unroll
            for (int a = 0; a < 6; a++) acc[21 + a] += J[a] * res;
            acc[27] += 1.f;
        }
    }
    const float tot = warp_transpose_reduce32(acc, lane);
    s_red[wid][lane] = tot;
    __syncthreads();
    if (wid == 0) {
        double sacc = 0.0;
#pragma unroll
        for (int w = 0; w < ICP_THREADS / 32; w++) sacc += (double)s_red[w][lane];
        ws->partial[(size_t)blockIdx.x * ICP_TERMS + lane] = sacc;
        __threadfence();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int done = atomicAdd(&ws->ticket, 1u);
        s_last = (done == gridDim.x - 1);
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (wid == 0) {
        double sacc = 0.0;
        for (unsigned int bidx = 0; bidx < gridDim.x; bidx++) sacc += ws->partial[(size_t)bidx * ICP_TERMS + lane];
        __shared__ double s_tot[ICP_TERMS];
        s_tot[lane] = sacc;
        __syncwarp();
        if (lane == 0) {
            double A[6][6], bvec[6], xi[6];
#pragma unroll
            for (int a = 0; a < 6; a++)
#pragma unroll
                for (int c = a; c < 6; c++) { const double v = s_tot[a * 6 - a * (a - 1) / 2 + (c - a)]; A[a][c] = v; A[c][a] = v; }
            double trace = 0.0;
#pragma unroll
            for (int a = 0; a < 6; a++) trace += A[a][a];
#pragma unroll
            for (int a = 0; a < 6; a++) { A[a][a] += trace * (double)damping; bvec[a] = -s_tot[21 + a]; }
            if (solve6(A, bvec, xi)) se3_update(xi, pose);
            if (valid_ratio) *valid_ratio = (float)(s_tot[27] / (double)H / (double)W);
            ws->ticket = 0;
        }
    }
}

// point2plane_loss(p_t0, p_t1 @ R^T + t, n_t0, "mean") (SLAM/icp.py:7-13,444-447)
__global__ void __launch_bounds__(256) icp_p2p_kernel(const float *__restrict__ v_t0, const float *__restrict__ v_t1,
                                                      const float *__restrict__ n_t0, int HW, const float *__restrict__ pose,
                                                      float *loss, IcpWs *ws) {
    __shared__ double s_w[8];
    __shared__ bool s_last;
    float Rm[9], tv[3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
        for (int j = 0; j < 3; j++) Rm[3 * i + j] = pose[4 * i + j];
        tv[i] = pose[4 * i + 3];
    }
    double acc = 0.0;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
        const float ax = v_t1[3 * (size_t)p], ay = v_t1[3 * (size_t)p + 1], az = v_t1[3 * (size_t)p + 2];
        const float x = Rm[0] * ax + Rm[1] * ay + Rm[2] * az + tv[0];
        const float y = Rm[3] * ax + Rm[4] * ay + Rm[5] * az + tv[1];
        const float z = Rm[6] * ax + Rm[7] * ay + Rm[8] * az + tv[2];
        const float l = (x - v_t0[3 * (size_t)p]) * n_t0[3 * (size_t)p] + (y - v_t0[3 * (size_t)p + 1]) * n_t0[3 * (size_t)p + 1] +
                        (z - v_t0[3 * (size_t)p + 2]) * n_t0[3 * (size_t)p + 2];
        acc += (double)(l * l);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < 8; w++) t += s_w[w];
        ws->partial[blockIdx.x] = t;
        __threadfence();
        const unsigned int done = atomicAdd(&ws->ticket, 1u);
        s_last = (done == gridDim.x - 1);
    }
    __syncthreads();
    if (!s_last || threadIdx.x != 0) return;
    __threadfence();
    double t = 0.0;
    for (unsigned int bidx = 0; bidx < gridDim.x; bidx++) t += ws->partial[bidx];
    *loss = (float)(t / (double)HW);
    ws->ticket = 0;
}

// IcpTracker.update_last_status depth filling (SLAM/icp.py:397-415)
__global__ void __launch_bounds__(256) icp_fill_kernel(float *__restrict__ render_depth, const float *__restrict__ frame_depth,
                                                       const float *__restrict__ rn, const float *__restrict__ fn, int HW, float dthr,
                                                       float nthr) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= HW) return;
    const float ax = rn[3 * (size_t)p], ay = rn[3 * (size_t)p + 1], az = rn[3 * (size_t)p + 2];
    const float bx = fn[3 * (size_t)p], by = fn[3 * (size_t)p + 1], bz = fn[3 * (size_t)p + 2];
    // F.cosine_similarity: x.y / (max(|x|,eps) * max(|y|,eps)), eps = 1e-8
    const float na = fmaxf(sqrtf(ax * ax + ay * ay + az * az), 1e-8f), nb = fmaxf(sqrtf(bx * bx + by * by + bz * bz), 1e-8f);
    const float cosv = (ax * bx + ay * by + az * bz) / (na * nb);
    const bool normal_mask = (1.f - cosv) > nthr;
    const float rd = render_depth[p], fd = frame_depth[p];
    const bool fill = ((fabsf(rd - fd) > dthr) || (rd == 0.f) || normal_mask) && (fd > 0.f);
    if (fill) render_depth[p] = fd;
}

// ------------------------------------------------------------------ persistent kernels (one launch per predict_pose)
// Grid barrier of a cooperative launch (all blocks co-resident): arrival counter, released when it reaches
// generation * gridDim.x. The counter is zeroed by the host before the launch.
__device__ __forceinline__ void grid_barrier(unsigned int *counter, unsigned int &generation) {
    __syncthreads();
    if (threadIdx.x == 0) {
        generation++;
        __threadfence();
        atomicAdd(counter, 1u);
        const unsigned int target = generation * gridDim.x;
        unsigned int seen;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(counter) : "memory");
        } while (seen < target);
    }
    __syncthreads();
}

// Per-pixel residual and Jacobian row of one iteration, accumulated into the 28 normal-equation terms (same arithmetic
// as icp_iter_kernel above; `pose` in shared memory). With RGBD, every pixel with a valid geometric row also adds the
// photometric row: r = I1(u, v) - I0[p], bilinear in the previous frame's level intensity at the projection the
// geometric row already computed, with J = (v' x a, a), a = dr/dv' through the exact derivative of the interpolant. Its
// terms enter the same 27 slots scaled by photo_w (after the geometric ones, so photo_w = 0 leaves every slot's bits
// unchanged); slots 28 and 29 take its count and its sum of r^2.
template <bool RGBD>
__device__ __forceinline__ void icp_accumulate(const IcpLevel &L, const float *pose, const float dist_thr, const float cos_thr,
                                               float acc[ICP_TERMS], const float *__restrict__ inten0 = nullptr,
                                               const float *__restrict__ inten1 = nullptr, const float photo_w = 0.f) {
    float Rm[9], tv[3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
        for (int j = 0; j < 3; j++) Rm[3 * i + j] = pose[4 * i + j];
        tv[i] = pose[4 * i + 3];
    }
    const int H = L.H, W = L.W, HW = H * W;
    const float fx = L.fx, fy = L.fy, cx = L.cx, cy = L.cy;
    const float Wm1 = (float)(W - 1), Hm1 = (float)(H - 1);
    const float *__restrict__ vertex0 = L.v0, *__restrict__ normal0 = L.n0, *__restrict__ vertex1 = L.v1, *__restrict__ normal1 = L.n1;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < HW; p += gridDim.x * blockDim.x) {
        const float v0x = vertex0[3 * (size_t)p], v0y = vertex0[3 * (size_t)p + 1], v0z = vertex0[3 * (size_t)p + 2];
        const bool mask0 = v0z > 0.0f;
        const float n0x = normal0[3 * (size_t)p], n0y = normal0[3 * (size_t)p + 1], n0z = normal0[3 * (size_t)p + 2];
        const float x = Rm[0] * v0x + Rm[1] * v0y + Rm[2] * v0z + tv[0];
        const float y = Rm[3] * v0x + Rm[4] * v0y + Rm[5] * v0z + tv[1];
        const float z = Rm[6] * v0x + Rm[7] * v0y + Rm[8] * v0z + tv[2];
        const float nx = Rm[0] * n0x + Rm[1] * n0y + Rm[2] * n0z;
        const float ny = Rm[3] * n0x + Rm[4] * n0y + Rm[5] * n0z;
        const float nz = Rm[6] * n0x + Rm[7] * n0y + Rm[8] * n0z;
        const float u = (x / z) * fx + cx, v = (y / z) * fy + cy;
        const bool inview = (u > 0.f) && (u < Wm1) && (v > 0.f) && (v < Hm1);
        const float un = u / (Wm1 / 2.f) - 1.f, vn = v / (Hm1 / 2.f) - 1.f;
        float ix = ((un + 1.f) / 2.f) * Wm1, iy = ((vn + 1.f) / 2.f) * Hm1;
        ix = fminf(Wm1, fmaxf(ix, 0.f));
        iy = fminf(Hm1, fmaxf(iy, 0.f));
        int xi = (int)nearbyintf(ix), yi = (int)nearbyintf(iy);
        xi = min(W - 1, max(0, xi));
        yi = min(H - 1, max(0, yi));
        const size_t q = (size_t)yi * W + xi;
        const float rx = vertex1[3 * q], ry = vertex1[3 * q + 1], rz = vertex1[3 * q + 2];
        const float mx = normal1[3 * q], my = normal1[3 * q + 1], mz = normal1[3 * q + 2];
        const bool mask1 = rz > 0.f;
        const float dx = x - rx, dy = y - ry, dz = z - rz;
        const bool normal_ok = (nx * mx + ny * my + nz * mz) > cos_thr;
        const bool occ = !inview || (sqrtf(dx * dx + dy * dy + dz * dz) > dist_thr);
        const bool valid = !(occ || !mask0 || !mask1 || !normal_ok);
        if (valid) {
            const float res = mx * dx + my * dy + mz * dz;
            float J[6];
            J[0] = -(my * z - mz * y);
            J[1] = -(mz * x - mx * z);
            J[2] = -(mx * y - my * x);
            J[3] = mx; J[4] = my; J[5] = mz;
            int k = 0;
#pragma unroll
            for (int a = 0; a < 6; a++)
#pragma unroll
                for (int c = a; c < 6; c++) acc[k++] += J[a] * J[c];
#pragma unroll
            for (int a = 0; a < 6; a++) acc[21 + a] += J[a] * res;
            acc[27] += 1.f;
            if constexpr (RGBD) {
                // 0 < u < W-1 and 0 < v < H-1 (inview): the four taps exist
                const float fu = floorf(u), fv = floorf(v);
                const float al = u - fu, be = v - fv;
                const size_t t = (size_t)(int)fv * W + (int)fu;
                const float i00 = inten1[t], i10 = inten1[t + 1], i01 = inten1[t + W], i11 = inten1[t + W + 1];
                const float I = (1.f - be) * ((1.f - al) * i00 + al * i10) + be * ((1.f - al) * i01 + al * i11);
                const float r = I - inten0[p];
                const float gu = (1.f - be) * (i10 - i00) + be * (i11 - i01);
                const float gv = (1.f - al) * (i01 - i00) + al * (i11 - i10);
                const float iz = 1.f / z;
                const float a0 = gu * fx * iz, a1 = gv * fy * iz, a2 = -(a0 * x + a1 * y) * iz;
                float Jp[6];
                Jp[0] = y * a2 - z * a1;
                Jp[1] = z * a0 - x * a2;
                Jp[2] = x * a1 - y * a0;
                Jp[3] = a0; Jp[4] = a1; Jp[5] = a2;
                float Jw[6];
#pragma unroll
                for (int a = 0; a < 6; a++) Jw[a] = photo_w * Jp[a];
                int kp = 0;
#pragma unroll
                for (int a = 0; a < 6; a++)
#pragma unroll
                    for (int c = a; c < 6; c++) acc[kp++] += Jw[a] * Jp[c];
#pragma unroll
                for (int a = 0; a < 6; a++) acc[21 + a] += Jw[a] * r;
                acc[28] += 1.f;
                acc[29] += r * r;
            }
        }
    }
}

// Block-level sum of the warp-reduced terms into this block's row of `partial` (double).
__device__ __forceinline__ void icp_block_partial(float acc[ICP_TERMS], float (*s_red)[ICP_TERMS], double *partial_row) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const float tot = warp_transpose_reduce32(acc, lane);
    s_red[wid][lane] = tot;
    __syncthreads();
    if (wid == 0) {
        double sacc = 0.0;
        for (int w = 0; w < nw; w++) sacc += (double)s_red[w][lane];
        partial_row[lane] = sacc;
    }
}

// Every block sums all blocks' rows in the same order, so every block obtains bit-identical totals (no broadcast).
__device__ __forceinline__ void icp_grid_total(const double *partial, double (*s_part)[ICP_TERMS], double *s_tot) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    double sacc = 0.0;
    for (unsigned int b = wid; b < gridDim.x; b += nw) sacc += __ldcg(partial + (size_t)b * ICP_TERMS + lane);
    s_part[wid][lane] = sacc;
    __syncthreads();
    if (wid == 0) {
        double t = 0.0;
        for (int w = 0; w < nw; w++) t += s_part[w][lane];
        s_tot[lane] = t;
    }
    __syncthreads();
}

#define ICP_P_THREADS 512
// IcpTracker.predict_pose in one cooperative launch (SLAM/icp.py:417-452): for every pyramid level, `iters` Gauss-Newton
// iterations (one grid barrier each: every block reduces the per-block partial sums itself and solves the 6x6 system
// redundantly, so the updated pose needs no broadcast), then the point-to-plane loss of the final pose; pose (16),
// loss and valid ratio go to `out` on the device and, if given, straight into mapped host memory. RGBD adds the
// photometric row (icp_accumulate) and two more result floats: the photometric ratio and RMS residual of the last
// iteration.
template <bool RGBD>
__global__ void __launch_bounds__(ICP_P_THREADS) icp_predict_kernel(const IcpPredict prm, IcpWs *ws, const IcpPhoto ph) {
    __shared__ float s_red[ICP_P_THREADS / 32][ICP_TERMS];
    __shared__ double s_part[ICP_P_THREADS / 32][ICP_TERMS];
    __shared__ double s_tot[ICP_TERMS];
    __shared__ float s_pose[16];
    __shared__ float s_valid;
    __shared__ float s_photo[2];
    unsigned int generation = 0;
    if (threadIdx.x < 16) s_pose[threadIdx.x] = prm.pose_in ? prm.pose_in[threadIdx.x] : ((threadIdx.x % 5 == 0) ? 1.f : 0.f);
    if (threadIdx.x == 0) s_valid = 0.f;
    if constexpr (RGBD) {
        if (threadIdx.x < 2) s_photo[threadIdx.x] = 0.f;
    }
    __syncthreads();
    int it_global = 0;
    for (int l = 0; l < prm.n_levels; l++) {
        const IcpLevel L = prm.lv[l];
        for (int it = 0; it < L.iters; it++, it_global++) {
            float acc[ICP_TERMS];
#pragma unroll
            for (int k = 0; k < ICP_TERMS; k++) acc[k] = 0.f;
            if constexpr (RGBD) {
                // constant indices only, so the intensity pointers stay in the constant bank
                const float *i0 = ph.I0[0], *i1 = ph.I1[0];
#pragma unroll
                for (int j = 1; j < ICP_MAX_LEVELS; j++)
                    if (j == l) { i0 = ph.I0[j]; i1 = ph.I1[j]; }
                icp_accumulate<true>(L, s_pose, prm.dist_thr, prm.cos_thr, acc, i0, i1, ph.w);
            } else
                icp_accumulate<false>(L, s_pose, prm.dist_thr, prm.cos_thr, acc);
            double *partial = (it_global & 1) ? ws->partial2 : ws->partial;
            icp_block_partial(acc, s_red, partial + (size_t)blockIdx.x * ICP_TERMS);
            grid_barrier(&ws->barrier, generation);
            icp_grid_total(partial, s_part, s_tot);
            if (threadIdx.x == 0) {
                double A[6][6], bvec[6], xi[6];
#pragma unroll
                for (int a = 0; a < 6; a++)
#pragma unroll
                    for (int c = a; c < 6; c++) { const double v = s_tot[a * 6 - a * (a - 1) / 2 + (c - a)]; A[a][c] = v; A[c][a] = v; }
                double trace = 0.0;
#pragma unroll
                for (int a = 0; a < 6; a++) trace += A[a][a];
#pragma unroll
                for (int a = 0; a < 6; a++) { A[a][a] += trace * (double)prm.damping; bvec[a] = -s_tot[21 + a]; }
                if (solve6(A, bvec, xi)) se3_update(xi, s_pose);
                s_valid = (float)(s_tot[27] / (double)L.H / (double)L.W);
                if constexpr (RGBD) {
                    s_photo[0] = (float)(s_tot[28] / (double)L.H / (double)L.W);
                    s_photo[1] = s_tot[28] > 0.0 ? (float)sqrt(s_tot[29] / s_tot[28]) : 0.f;
                }
            }
            __syncthreads();
        }
    }
    // point2plane_loss(p_t0, p_t1 @ R^T + t, n_t0, "mean") of the finest level (SLAM/icp.py:444-447)
    {
        float Rm[9], tv[3];
#pragma unroll
        for (int i = 0; i < 3; i++) {
#pragma unroll
            for (int j = 0; j < 3; j++) Rm[3 * i + j] = s_pose[4 * i + j];
            tv[i] = s_pose[4 * i + 3];
        }
        double acc = 0.0;
        const float *__restrict__ v_t0 = prm.p2p_v_t0, *__restrict__ v_t1 = prm.p2p_v_t1, *__restrict__ n_t0 = prm.p2p_n_t0;
        for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < prm.p2p_HW; p += gridDim.x * blockDim.x) {
            const float ax = v_t1[3 * (size_t)p], ay = v_t1[3 * (size_t)p + 1], az = v_t1[3 * (size_t)p + 2];
            const float x = Rm[0] * ax + Rm[1] * ay + Rm[2] * az + tv[0];
            const float y = Rm[3] * ax + Rm[4] * ay + Rm[5] * az + tv[1];
            const float z = Rm[6] * ax + Rm[7] * ay + Rm[8] * az + tv[2];
            const float lq = (x - v_t0[3 * (size_t)p]) * n_t0[3 * (size_t)p] + (y - v_t0[3 * (size_t)p + 1]) * n_t0[3 * (size_t)p + 1] +
                             (z - v_t0[3 * (size_t)p + 2]) * n_t0[3 * (size_t)p + 2];
            acc += (double)(lq * lq);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
        if (lane == 0) s_part[wid][0] = acc;
        __syncthreads();
        double *partial = (it_global & 1) ? ws->partial2 : ws->partial;
        if (threadIdx.x == 0) {
            double t = 0.0;
            for (int w = 0; w < ICP_P_THREADS / 32; w++) t += s_part[w][0];
            partial[blockIdx.x] = t;
        }
        grid_barrier(&ws->barrier, generation);
        if (blockIdx.x == 0 && threadIdx.x < 32) {
            double t = 0.0;
            for (unsigned int b = threadIdx.x; b < gridDim.x; b += 32) t += __ldcg(partial + b);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
            const float loss = (float)(t / (double)prm.p2p_HW);
            if (threadIdx.x < 16) {
                prm.out[threadIdx.x] = s_pose[threadIdx.x];
                if (prm.out_host) prm.out_host[threadIdx.x] = s_pose[threadIdx.x];
            } else if (threadIdx.x == 16) {
                prm.out[16] = loss;
                if (prm.out_host) prm.out_host[16] = loss;
            } else if (threadIdx.x == 17) {
                prm.out[17] = s_valid;
                if (prm.out_host) prm.out_host[17] = s_valid;
            }
            if constexpr (RGBD) {
                if (threadIdx.x == 18 || threadIdx.x == 19) {
                    prm.out[threadIdx.x] = s_photo[threadIdx.x - 18];
                    if (prm.out_host) prm.out_host[threadIdx.x] = s_photo[threadIdx.x - 18];
                }
            }
        }
    }
}

// All levels of build_vertex_pyramid + build_normal_pyramid (SLAM/utils.py:511-527) in one cooperative launch: phase 1
// max-pools and back-projects every level and finds each level's depth extremes, grid barrier, phase 2 the Sobel normals.
__global__ void __launch_bounds__(256) icp_pyramid_kernel(const IcpPyramid prm, IcpWs *ws) {
    unsigned int generation = 0;
    const int gtid = blockIdx.x * blockDim.x + threadIdx.x, gsize = gridDim.x * blockDim.x;
    for (int l = 0; l < prm.n_levels; l++) {
        const int pool = prm.pool[l], Hs = prm.H / pool, Ws = prm.W / pool, W = prm.W;
        const float fx = prm.fx[l], fy = prm.fy[l], cx = prm.cx[l], cy = prm.cy[l];
        float *__restrict__ vertex = prm.vertex[l];
        float mn = INFINITY, mx = -INFINITY;
        for (int idx = gtid; idx < Hs * Ws; idx += gsize) {
            const int ys = idx / Ws, xs = idx % Ws;
            float d = -INFINITY;
            for (int a = 0; a < pool; a++)
                for (int c = 0; c < pool; c++) d = fmaxf(d, prm.depth[(size_t)(ys * pool + a) * W + xs * pool + c]);
            float *v = vertex + 3 * (size_t)idx;
            v[0] = (((float)xs - cx) / fx) * d;
            v[1] = (((float)ys - cy) / fy) * d;
            v[2] = 1.0f * d;
            mn = fminf(mn, d); mx = fmaxf(mx, d);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        }
        if ((threadIdx.x & 31) == 0 && mn <= mx) {
            atomicMin(&ws->level_minmax[2 * l], float_to_ordered(mn));
            atomicMax(&ws->level_minmax[2 * l + 1], float_to_ordered(mx));
        }
    }
    grid_barrier(&ws->barrier, generation);
    for (int l = 0; l < prm.n_levels; l++) {
        const int pool = prm.pool[l], Hs = prm.H / pool, Ws = prm.W / pool;
        const float *__restrict__ vertex = prm.vertex[l];
        float *__restrict__ normal = prm.normal[l];
        const float dmin = ordered_to_float(__ldcg(&ws->level_minmax[2 * l])), dmax = ordered_to_float(__ldcg(&ws->level_minmax[2 * l + 1]));
        for (int idx = gtid; idx < Hs * Ws; idx += gsize) {
            const int y = idx / Ws, x = idx % Ws;
            const int ym = max(y - 1, 0), yp = min(y + 1, Hs - 1), xm = max(x - 1, 0), xp = min(x + 1, Ws - 1);
            float dx[3], dy[3];
#pragma unroll
            for (int c = 0; c < 3; c++) {
                const float a00 = __ldcg(vertex + 3 * ((size_t)ym * Ws + xm) + c), a01 = __ldcg(vertex + 3 * ((size_t)ym * Ws + x) + c),
                            a02 = __ldcg(vertex + 3 * ((size_t)ym * Ws + xp) + c);
                const float a10 = __ldcg(vertex + 3 * ((size_t)y * Ws + xm) + c), a12 = __ldcg(vertex + 3 * ((size_t)y * Ws + xp) + c);
                const float a20 = __ldcg(vertex + 3 * ((size_t)yp * Ws + xm) + c), a21 = __ldcg(vertex + 3 * ((size_t)yp * Ws + x) + c),
                            a22 = __ldcg(vertex + 3 * ((size_t)yp * Ws + xp) + c);
                dx[c] = -a00 + a02 - 2.f * a10 + 2.f * a12 - a20 + a22;
                dy[c] = -a00 - 2.f * a01 - a02 + a20 + 2.f * a21 + a22;
            }
            float nx = dy[1] * dx[2] - dy[2] * dx[1];
            float ny = dy[2] * dx[0] - dy[0] * dx[2];
            float nz = dy[0] * dx[1] - dy[1] * dx[0];
            const float mag = sqrtf(nx * nx + ny * ny + nz * nz);
            const float inv = 1.0f / (mag + 1e-8f);
            nx *= inv; ny *= inv; nz *= inv;
            const float d = __ldcg(vertex + 3 * (size_t)idx + 2);
            if (d <= dmin || d >= dmax) { nx = 0.f; ny = 0.f; nz = 0.f; }
            float *n = normal + 3 * (size_t)idx;
            n[0] = nx; n[1] = ny; n[2] = nz;
        }
    }
}

// Intensity pyramid of the photometric term, all levels in one launch: one thread per level pixel, the mean of
// Y = 0.299 R + 0.587 G + 0.114 B over the pool x pool block whose maximum icp_pyramid_kernel takes for the depth.
__global__ void __launch_bounds__(256) icp_intensity_pyramid_kernel(const IcpIntensity prm) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= prm.total) return;
    // constant indices only, so the parameter arrays stay in the constant bank
    int start = 0, pool = prm.pool[0];
    float *out = prm.out[0];
#pragma unroll
    for (int j = 1; j < RTG_ICP_MAX_LEVELS; j++)
        if (j < prm.n_levels && idx >= prm.start[j]) { start = prm.start[j]; pool = prm.pool[j]; out = prm.out[j]; }
    const int Ws = prm.W / pool, H = prm.H, W = prm.W;
    const int k = idx - start, ys = k / Ws, xs = k % Ws;
    const size_t plane = (size_t)H * W;
    float s = 0.f;
    for (int a = 0; a < pool; a++)
        for (int c = 0; c < pool; c++) {
            const size_t q = (size_t)(ys * pool + a) * W + xs * pool + c;
            float R, G, B;
            if (prm.channels_last) {
                R = prm.color[3 * q]; G = prm.color[3 * q + 1]; B = prm.color[3 * q + 2];
            } else {
                R = prm.color[q]; G = prm.color[plane + q]; B = prm.color[2 * plane + q];
            }
            s += 0.299f * R + 0.587f * G + 0.114f * B;
        }
    out[k] = s / (float)(pool * pool);
}

__global__ void icp_persistent_init_kernel(IcpWs *ws) {
    ws->barrier = 0;
    if (threadIdx.x < ICP_MAX_LEVELS) {
        ws->level_minmax[2 * threadIdx.x] = 0x7fffffff;
        ws->level_minmax[2 * threadIdx.x + 1] = (int)0x80000000;
    }
}

static int sm_count() {
    static int n[64] = {0};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (!n[dev]) cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
    return n[dev] > 0 ? n[dev] : 1;
}

template <bool RGBD>
static cudaError_t launch_icp_predict_t(const IcpPredict &prm, const IcpPhoto &ph, void *ws_, cudaStream_t s) {
    IcpWs *ws = reinterpret_cast<IcpWs *>(ws_);
    ProfScope ps(K_ICP_ITER, s);
    icp_persistent_init_kernel<<<1, 32, 0, s>>>(ws);
    int grid = sm_count();
    if (grid > ICP_MAX_BLOCKS) grid = ICP_MAX_BLOCKS;
    void *args[] = {(void *)&prm, (void *)&ws, (void *)&ph};
    return cudaLaunchCooperativeKernel((const void *)icp_predict_kernel<RGBD>, dim3(grid), dim3(ICP_P_THREADS), args, 0, s);
}

cudaError_t launch_icp_predict(const IcpPredict &prm, void *ws, cudaStream_t s) {
    const IcpPhoto none{};
    return launch_icp_predict_t<false>(prm, none, ws, s);
}

cudaError_t launch_icp_predict_rgbd(const IcpPredict &prm, const IcpPhoto &ph, void *ws, cudaStream_t s) {
    return launch_icp_predict_t<true>(prm, ph, ws, s);
}

void launch_icp_intensity_pyramid(const IcpIntensity &prm, cudaStream_t s) {
    icp_intensity_pyramid_kernel<<<(prm.total + 255) / 256, 256, 0, s>>>(prm);
}

cudaError_t launch_icp_pyramid(const IcpPyramid &prm, void *ws_, cudaStream_t s) {
    IcpWs *ws = reinterpret_cast<IcpWs *>(ws_);
    ProfScope ps(K_ICP_BUILD, s);
    icp_persistent_init_kernel<<<1, 32, 0, s>>>(ws);
    int grid = 2 * sm_count();
    const int need = (prm.H * prm.W / (prm.pool[prm.n_levels - 1] * prm.pool[prm.n_levels - 1]) + 255) / 256;
    if (grid > need) grid = need < 1 ? 1 : need;
    void *args[] = {(void *)&prm, (void *)&ws};
    return cudaLaunchCooperativeKernel((const void *)icp_pyramid_kernel, dim3(grid), dim3(256), args, 0, s);
}

static int icp_blocks(int HW) {
    int b = (HW + ICP_THREADS - 1) / ICP_THREADS;
    return b < 1 ? 1 : (b > ICP_MAX_BLOCKS ? ICP_MAX_BLOCKS : b);
}

size_t icp_ws_bytes() { return sizeof(IcpWs); }

void launch_icp_build_level(const float *depth, int H, int W, int pool, float fx, float fy, float cx, float cy, float *vertex,
                            float *normal, void *ws_, cudaStream_t s) {
    IcpWs *ws = reinterpret_cast<IcpWs *>(ws_);
    const int Hs = H / pool, Ws = W / pool;
    ProfScope ps(K_ICP_BUILD, s);
    icp_ws_init_kernel<<<1, 1, 0, s>>>(ws);
    const int nb = (Hs * Ws + 255) / 256;
    icp_vertex_kernel<<<nb, 256, 0, s>>>(depth, H, W, pool, Hs, Ws, fx, fy, cx, cy, vertex, ws);
    icp_normal_kernel<<<nb, 256, 0, s>>>(vertex, Hs, Ws, normal, ws);
}

void launch_icp_solve_level(const float *v0, const float *n0, const float *v1, const float *n1, int H, int W, float fx, float fy,
                            float cx, float cy, float dist_thr, float cos_thr, float damping, int iters, float *pose,
                            float *valid_ratio, void *ws_, cudaStream_t s) {
    IcpWs *ws = reinterpret_cast<IcpWs *>(ws_);
    icp_ws_init_kernel<<<1, 1, 0, s>>>(ws);
    const int nb = icp_blocks(H * W);
    for (int it = 0; it < iters; it++) {
        ProfScope ps(K_ICP_ITER, s);
        icp_iter_kernel<<<nb, ICP_THREADS, 0, s>>>(v0, n0, v1, n1, H, W, fx, fy, cx, cy, dist_thr, cos_thr, damping, pose,
                                                   valid_ratio, ws);
    }
}

void launch_icp_p2p(const float *v_t0, const float *v_t1, const float *n_t0, int H, int W, const float *pose, float *loss,
                    void *ws_, cudaStream_t s) {
    IcpWs *ws = reinterpret_cast<IcpWs *>(ws_);
    icp_ws_init_kernel<<<1, 1, 0, s>>>(ws);
    icp_p2p_kernel<<<icp_blocks(H * W), 256, 0, s>>>(v_t0, v_t1, n_t0, H * W, pose, loss, ws);
}

void launch_icp_fill(float *render_depth, const float *frame_depth, const float *rn, const float *fn, int H, int W, float dthr,
                     float nthr, cudaStream_t s) {
    icp_fill_kernel<<<(H * W + 255) / 256, 256, 0, s>>>(render_depth, frame_depth, rn, fn, H * W, dthr, nthr);
}

}  // namespace rtg
