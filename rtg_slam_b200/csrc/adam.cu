// One-launch Adam over all parameter groups of the Gaussian map.
//
// Replaces torch.optim.Adam(l, lr=0.0, eps=1e-15).step() over the six groups of
// GaussianPointCloud.parametrize (SLAM/gaussian_pointcloud.py:245-284, SLAM/multiprocess/
// mapper.py:156,452): bias-corrected, no weight decay, no amsgrad. Pure streaming work:
// 28 bytes per parameter (read p,g,m,v; write p,m,v), 128-bit accesses.
#include "common.cuh"
#include "prof.h"
#include "../../include/rtg_splat_b200.h"

namespace rtg {

struct AdamArgs {
    RtgAdamGroup g[RTG_ADAM_MAX_GROUPS];
    int n_groups;
    float beta1, beta2, eps, bc1, bc2_sqrt;
};

__global__ void __launch_bounds__(256) adam_kernel(const AdamArgs a) {
    const RtgAdamGroup grp = a.g[blockIdx.y];
    if (grp.grad == nullptr || grp.numel <= 0) return;
    const float lr_over_bc1 = grp.lr / a.bc1;
    const long long n = grp.numel;
    const bool vec = ((((uintptr_t)grp.param | (uintptr_t)grp.grad | (uintptr_t)grp.exp_avg | (uintptr_t)grp.exp_avg_sq) & 15) == 0);
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (vec) {
        const long long n4 = n >> 2;
        float4 *P4 = reinterpret_cast<float4 *>(grp.param);
        const float4 *G4 = reinterpret_cast<const float4 *>(grp.grad);
        float4 *M4 = reinterpret_cast<float4 *>(grp.exp_avg);
        float4 *V4 = reinterpret_cast<float4 *>(grp.exp_avg_sq);
        for (long long i = tid; i < n4; i += stride) {
            float4 p = P4[i], m = M4[i], v = V4[i];
            const float4 g = __ldg(G4 + i);
            adam_one(p.x, g.x, m.x, v.x, lr_over_bc1, a.beta1, a.beta2, a.eps, a.bc2_sqrt);
            adam_one(p.y, g.y, m.y, v.y, lr_over_bc1, a.beta1, a.beta2, a.eps, a.bc2_sqrt);
            adam_one(p.z, g.z, m.z, v.z, lr_over_bc1, a.beta1, a.beta2, a.eps, a.bc2_sqrt);
            adam_one(p.w, g.w, m.w, v.w, lr_over_bc1, a.beta1, a.beta2, a.eps, a.bc2_sqrt);
            P4[i] = p; M4[i] = m; V4[i] = v;
        }
        for (long long i = (n4 << 2) + tid; i < n; i += stride) {
            float p = grp.param[i], m = grp.exp_avg[i], v = grp.exp_avg_sq[i];
            adam_one(p, grp.grad[i], m, v, lr_over_bc1, a.beta1, a.beta2, a.eps, a.bc2_sqrt);
            grp.param[i] = p; grp.exp_avg[i] = m; grp.exp_avg_sq[i] = v;
        }
    } else {
        for (long long i = tid; i < n; i += stride) {
            float p = grp.param[i], m = grp.exp_avg[i], v = grp.exp_avg_sq[i];
            adam_one(p, grp.grad[i], m, v, lr_over_bc1, a.beta1, a.beta2, a.eps, a.bc2_sqrt);
            grp.param[i] = p; grp.exp_avg[i] = m; grp.exp_avg_sq[i] = v;
        }
    }
}

int launch_adam(const RtgAdamGroup *groups, int n_groups, float beta1, float beta2, float eps, int step, cudaStream_t s) {
    AdamArgs a;
    long long max_n = 0;
    for (int i = 0; i < n_groups; i++) {
        a.g[i] = groups[i];
        if (groups[i].grad != nullptr && groups[i].numel > max_n) max_n = groups[i].numel;
    }
    a.n_groups = n_groups;
    a.beta1 = beta1; a.beta2 = beta2; a.eps = eps;
    // torch computes the bias corrections in python doubles (torch/optim/adam.py, _single_tensor_adam)
    const double bc1 = 1.0 - pow((double)beta1, (double)step);
    const double bc2 = 1.0 - pow((double)beta2, (double)step);
    a.bc1 = (float)bc1;
    a.bc2_sqrt = (float)sqrt(bc2);
    if (max_n == 0) return 0;
    long long blocks = (max_n / 4 + 255) / 256;
    if (blocks < 1) blocks = 1;
    if (blocks > RTG_NUM_SMS * 16) blocks = RTG_NUM_SMS * 16;
    dim3 grid((unsigned)blocks, (unsigned)n_groups);
    ProfScope ps(K_ADAM, s);
    adam_kernel<<<grid, 256, 0, s>>>(a);
    return 0;
}

// ------------------------------------------------------------------ pose step (rtg_pose_adam_step)
// A few hundred double operations with a chain of dependencies: one thread does them all. Not bracketed by the event
// profiler: its ids are fixed, and timing it under `adam` would mix pose steps into the map optimizer's entry.
__global__ void __launch_bounds__(1) pose_adam_kernel(const RtgPoseAdam s, const double bc1, const double bc2_sqrt) {
    double T[4][4];
#pragma unroll
    for (int i = 0; i < 16; i++) T[i / 4][i % 4] = s.pose[i];

    // G = dL/dW2C through viewmatrix = W2C^T, projmatrix = W2C^T @ projection and campos = -R^T t
    double G[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
            double v = s.dL_dviewmatrix ? (double)s.dL_dviewmatrix[4 * j + i] : 0.0;
            if (s.dL_dprojmatrix)
#pragma unroll
                for (int k = 0; k < 4; k++) v += (double)s.projection[4 * i + k] * (double)s.dL_dprojmatrix[4 * j + k];
            G[i][j] = v;
        }
    if (s.dL_dcampos) {
        const double gc[3] = {s.dL_dcampos[0], s.dL_dcampos[1], s.dL_dcampos[2]};
#pragma unroll
        for (int k = 0; k < 3; k++) {
#pragma unroll
            for (int i = 0; i < 3; i++) G[k][i] -= T[k][3] * gc[i];
            G[k][3] -= T[k][0] * gc[0] + T[k][1] * gc[1] + T[k][2] * gc[2];
        }
    }
    // tangent gradient of the left twist at zero: A = G W2C^T
    double A[3][4];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int k = 0; k < 4; k++) A[i][k] = G[i][0] * T[k][0] + G[i][1] * T[k][1] + G[i][2] * T[k][2] + G[i][3] * T[k][3];
    const double grad[6] = {A[0][3], A[1][3], A[2][3], A[2][1] - A[1][2], A[0][2] - A[2][0], A[1][0] - A[0][1]};

    // Adam from xi = 0 (torch.optim.Adam, _single_tensor_adam): xi = -lr / bc1 * m / (sqrt(v) / sqrt(bc2) + eps)
    const double b1 = s.beta1, b2 = s.beta2;
    double xi[6];
#pragma unroll
    for (int k = 0; k < 6; k++) {
        const double m = b1 * (double)s.exp_avg[k] + (1.0 - b1) * grad[k];
        const double v = b2 * (double)s.exp_avg_sq[k] + (1.0 - b2) * grad[k] * grad[k];
        s.exp_avg[k] = (float)m;
        s.exp_avg_sq[k] = (float)v;
        const double lr = k < 3 ? s.lr_trans : s.lr_rot;
        xi[k] = -(lr / bc1) * m / (sqrt(v) / bc2_sqrt + (double)s.eps);
    }

    // W2C <- exp(xi^) W2C and the three camera arrays (common.cuh)
    double E[3][4];
    se3_exp_twist(xi, E);
    pose_left_update(E, T, s.pose, s.projection, s.viewmatrix, s.projmatrix, s.campos);
}

void launch_pose_adam_step(const RtgPoseAdam &st, cudaStream_t s) {
    // bias corrections in double, as rtg_adam_step (torch computes them in python floats)
    const double bc1 = 1.0 - pow((double)st.beta1, (double)st.step);
    const double bc2_sqrt = sqrt(1.0 - pow((double)st.beta2, (double)st.step));
    pose_adam_kernel<<<1, 1, 0, s>>>(st, bc1, bc2_sqrt);
}

}  // namespace rtg
