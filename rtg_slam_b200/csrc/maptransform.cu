// Rigid per-anchor transforms of the Gaussians already in the map: the map follows corrected camera poses.
//
// The reference moves only its Camera objects when the backend corrects the trajectory (Mapping.update_poses,
// SLAM/multiprocess/mapper.py:134-141); the Gaussians stay where the old poses put them. Here every Gaussian row carries
// an anchor (the frame that created it, GaussianPointCloud._add_tick) and is moved with its anchor's correction
//   T_k = new_c2w[k] * old_c2w[k]^-1:   x' = R x + t,  q' = q_delta (x) q,  n' = R n,  f'_l = D^l(R) f_l  (l = 1..3).
//
//  * map_xform_table_kernel: one thread per anchor, float64 arithmetic. q_delta is the unit quaternion (w >= 0) of
//    R_new R_old^T (Shepperd's method, so the nearest rotation even for slightly non-orthonormal input), R is rebuilt from
//    it and t = p_new - R p_old. D^l is the band-l rotation matrix of the rasterizer's real SH basis (computeColorFromSH,
//    forward.cu:104-155, with its signs): sh(f', R d) = sh(f, d) for every direction d, i.e.
//        D^l_mk = integral over the sphere of y_m(e) y_k(R^T e) de,
//    which the 26-point Lebedev rule integrates exactly (the integrand is a polynomial of degree <= 6 on the sphere and
//    the rule is exact to degree 7; the basis is orthonormal). Once per anchor, never per Gaussian.
//  * map_xform_rows_kernel<SH_REST>: one in-place streaming pass. A block stages MX_TILE rows of each array through
//    shared memory with flat, coalesced float4 accesses (the 36 / 96 / 180-byte SH rows are not 16-byte aligned row by
//    row), moves its rows there, and writes back only the words of moved rows. Rows with anchor -1, an unmoved anchor or
//    an anchor outside [0, K) are neither read (beyond the anchor id) nor written; the last kind is counted.
#include "../../include/rtg_splat_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace rtg {

#define MX_TILE 128
#define MX_ROW 104  // floats per anchor in the table (16-byte multiple)
// table row: [0] moved flag (int bits), [1..4] q_delta (w,x,y,z), [5..13] R row-major, [14..16] t,
//            [17..25] D1 (3x3), [26..50] D2 (5x5), [51..99] D3 (7x7), all row-major
#define MX_Q 1
#define MX_R 5
#define MX_T 14
#define MX_D1 17
#define MX_D2 26
#define MX_D3 51

size_t map_transform_ws_bytes(int64_t K) { return align_up((size_t)(K > 0 ? K : 0) * MX_ROW * sizeof(float), 256); }

// 26-point Lebedev rule (degree 7) on the unit sphere: point q = the 6 axes, then the 12 edge midpoints, then the 8 corners
// of the cube; w = 4 pi * weight
__device__ __forceinline__ void lebedev_point(int q, double &x, double &y, double &z, double &w) {
    const double PI4 = 12.566370614359172954, S2 = 0.70710678118654752440, S3 = 0.57735026918962576451;
    if (q < 6) {
        const int ax = q >> 1;
        const double s = (q & 1) ? -1.0 : 1.0;
        x = ax == 0 ? s : 0.0; y = ax == 1 ? s : 0.0; z = ax == 2 ? s : 0.0;
        w = PI4 / 21.0;
    } else if (q < 18) {
        const int e = q - 6, zero = e >> 2;  // the axis the edge midpoint is perpendicular to
        const double s1 = (e & 1) ? -S2 : S2, s2 = (e & 2) ? -S2 : S2;
        x = zero == 0 ? 0.0 : s1;
        y = zero == 1 ? 0.0 : (zero == 0 ? s1 : s2);
        z = zero == 2 ? 0.0 : s2;
        w = PI4 * 4.0 / 105.0;
    } else {
        const int c = q - 18;
        x = (c & 1) ? -S3 : S3; y = (c & 2) ? -S3 : S3; z = (c & 4) ? -S3 : S3;
        w = PI4 * 9.0 / 280.0;
    }
}

// band L of the rasterizer's SH basis at the unit direction (x, y, z), in its coefficient order and signs
template <int L>
__device__ __forceinline__ void sh_band(double x, double y, double z, double (&b)[2 * L + 1]) {
    if (L == 1) {
        const double C1 = 0.4886025119029199;
        b[0] = -C1 * y; b[1] = C1 * z; b[2] = -C1 * x;
    } else if (L == 2) {
        b[0] = 1.0925484305920792 * x * y;
        b[1] = -1.0925484305920792 * y * z;
        b[2] = 0.31539156525252005 * (2 * z * z - x * x - y * y);
        b[3] = -1.0925484305920792 * x * z;
        b[4] = 0.5462742152960396 * (x * x - y * y);
    } else {
        const double xx = x * x, yy = y * y, zz = z * z;
        b[0] = -0.5900435899266435 * y * (3 * xx - yy);
        b[1] = 2.890611442640554 * x * y * z;
        b[2] = -0.4570457994644658 * y * (4 * zz - xx - yy);
        b[3] = 0.3731763325901154 * z * (2 * zz - 3 * xx - 3 * yy);
        b[4] = -0.4570457994644658 * x * (4 * zz - xx - yy);
        b[5] = 1.445305721320277 * z * (xx - yy);
        b[6] = -0.5900435899266435 * x * (xx - 3 * yy);
    }
}

// D^L_mk = sum_q w_q y_m(e_q) y_k(R^T e_q), written as floats to out[(2L+1) m + k]
template <int L>
__device__ void sh_rotation_band(const double (&R)[9], float *__restrict__ out) {
    constexpr int N = 2 * L + 1;
    double D[N][N];
#pragma unroll
    for (int m = 0; m < N; m++)
#pragma unroll
        for (int k = 0; k < N; k++) D[m][k] = 0.0;
    for (int q = 0; q < 26; q++) {
        double ex, ey, ez, w;
        lebedev_point(q, ex, ey, ez, w);
        double a[N], b[N];
        sh_band<L>(ex, ey, ez, a);
        sh_band<L>(R[0] * ex + R[3] * ey + R[6] * ez, R[1] * ex + R[4] * ey + R[7] * ez, R[2] * ex + R[5] * ey + R[8] * ez, b);
#pragma unroll
        for (int m = 0; m < N; m++)
#pragma unroll
            for (int k = 0; k < N; k++) D[m][k] = fma(w * a[m], b[k], D[m][k]);
    }
#pragma unroll
    for (int m = 0; m < N; m++)
#pragma unroll
        for (int k = 0; k < N; k++) out[N * m + k] = (float)D[m][k];
}

__global__ void __launch_bounds__(128) map_xform_table_kernel(const double *__restrict__ old_c2w, const double *__restrict__ new_c2w, int K,
                                                              float *__restrict__ tab) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= K) return;
    const double *o = old_c2w + 16 * (size_t)k, *n = new_c2w + 16 * (size_t)k;
    float *row = tab + (size_t)k * MX_ROW;
    bool moved = false;
    for (int i = 0; i < 16; i++) moved |= __double_as_longlong(o[i]) != __double_as_longlong(n[i]);
    row[0] = __int_as_float(moved ? 1 : 0);
    if (!moved) return;
    // dR = R_new R_old^T
    double M[9];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) M[3 * i + j] = n[4 * i] * o[4 * j] + n[4 * i + 1] * o[4 * j + 1] + n[4 * i + 2] * o[4 * j + 2];
    // Shepperd: the largest of 4w^2, 4x^2, 4y^2, 4z^2 picks the well-conditioned formula
    const double tr = M[0] + M[4] + M[8];
    double qw, qx, qy, qz;
    if (tr >= M[0] && tr >= M[4] && tr >= M[8]) {
        const double s = 2.0 * sqrt(fmax(1.0 + tr, 0.0));
        qw = 0.25 * s; qx = (M[7] - M[5]) / s; qy = (M[2] - M[6]) / s; qz = (M[3] - M[1]) / s;
    } else if (M[0] >= M[4] && M[0] >= M[8]) {
        const double s = 2.0 * sqrt(fmax(1.0 + M[0] - M[4] - M[8], 0.0));
        qw = (M[7] - M[5]) / s; qx = 0.25 * s; qy = (M[1] + M[3]) / s; qz = (M[2] + M[6]) / s;
    } else if (M[4] >= M[8]) {
        const double s = 2.0 * sqrt(fmax(1.0 + M[4] - M[0] - M[8], 0.0));
        qw = (M[2] - M[6]) / s; qx = (M[1] + M[3]) / s; qy = 0.25 * s; qz = (M[5] + M[7]) / s;
    } else {
        const double s = 2.0 * sqrt(fmax(1.0 + M[8] - M[0] - M[4], 0.0));
        qw = (M[3] - M[1]) / s; qx = (M[2] + M[6]) / s; qy = (M[5] + M[7]) / s; qz = 0.25 * s;
    }
    const double inv = (qw < 0.0 ? -1.0 : 1.0) / sqrt(qw * qw + qx * qx + qy * qy + qz * qz);
    qw *= inv; qx *= inv; qy *= inv; qz *= inv;
    const double R[9] = {1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qw * qz),     2 * (qx * qz + qw * qy),
                         2 * (qx * qy + qw * qz),     1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qw * qx),
                         2 * (qx * qz - qw * qy),     2 * (qy * qz + qw * qx),     1 - 2 * (qx * qx + qy * qy)};
    row[MX_Q] = (float)qw; row[MX_Q + 1] = (float)qx; row[MX_Q + 2] = (float)qy; row[MX_Q + 3] = (float)qz;
    for (int i = 0; i < 9; i++) row[MX_R + i] = (float)R[i];
    for (int i = 0; i < 3; i++) row[MX_T + i] = (float)(n[4 * i + 3] - (R[3 * i] * o[3] + R[3 * i + 1] * o[7] + R[3 * i + 2] * o[11]));
    sh_rotation_band<1>(R, row + MX_D1);
    sh_rotation_band<2>(R, row + MX_D2);
    sh_rotation_band<3>(R, row + MX_D3);
}

// Stage the block's rows [row0, row0 + nrows) of a (P, W) float array into shared memory with row stride WS (LOAD), or write
// the words of moved rows back (!LOAD). s_k[r] >= 0 marks a moved row. float4 accesses when the array is 16-byte aligned
// (then so is every block's first row: MX_TILE * W is a multiple of 4); the tail and an unaligned array go word by word.
template <int W, int WS, bool LOAD>
__device__ __forceinline__ void mx_stage(float *__restrict__ g, float *__restrict__ s, int row0, int nrows, const int *__restrict__ s_k) {
    constexpr int N4 = MX_TILE * W / 4;
    float *base = g + (size_t)row0 * W;
    const int n = nrows * W;
    int start = 0;
    if ((reinterpret_cast<uintptr_t>(g) & 15) == 0) {
        const int n4 = n / 4;
        start = 4 * n4;
#pragma unroll
        for (int it = 0; it < (N4 + MX_TILE - 1) / MX_TILE; it++) {
            const int j = it * MX_TILE + threadIdx.x;
            if (j >= n4) break;
            const int w0 = 4 * j, ra = w0 / W, rb = (w0 + 3) / W;
            const bool ma = s_k[ra] >= 0, mb = s_k[rb] >= 0;
            if (!ma && !mb) continue;
            float *p = base + w0;
            if (LOAD) {
                const float4 v = __ldcs(reinterpret_cast<const float4 *>(p));
                const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    const int r = (w0 + c) / W;
                    s[r * WS + (w0 + c - r * W)] = e[c];
                }
            } else {
                float e[4];
#pragma unroll
                for (int c = 0; c < 4; c++) {
                    const int r = (w0 + c) / W;
                    e[c] = s[r * WS + (w0 + c - r * W)];
                }
                if (ma && mb) {
                    __stcs(reinterpret_cast<float4 *>(p), make_float4(e[0], e[1], e[2], e[3]));
                } else {  // a float4 shared with an unmoved row: only this row's words
#pragma unroll
                    for (int c = 0; c < 4; c++)
                        if ((((w0 + c) / W) == ra) == ma) p[c] = e[c];
                }
            }
        }
    }
    for (int j = start + threadIdx.x; j < n; j += MX_TILE) {
        const int r = j / W;
        if (s_k[r] < 0) continue;
        if (LOAD) s[r * WS + (j - r * W)] = base[j];
        else base[j] = s[r * WS + (j - r * W)];
    }
}

template <int L>
__device__ __forceinline__ void mx_rotate_band(const float *__restrict__ D, float *__restrict__ f) {
    constexpr int N = 2 * L + 1;
    float in[N][3], out[N][3];
#pragma unroll
    for (int j = 0; j < N; j++)
#pragma unroll
        for (int c = 0; c < 3; c++) in[j][c] = f[3 * j + c];
#pragma unroll
    for (int m = 0; m < N; m++) {
        out[m][0] = out[m][1] = out[m][2] = 0.f;
#pragma unroll
        for (int j = 0; j < N; j++) {
            const float d = __ldg(D + N * m + j);
#pragma unroll
            for (int c = 0; c < 3; c++) out[m][c] = fmaf(d, in[j][c], out[m][c]);
        }
    }
#pragma unroll
    for (int m = 0; m < N; m++)
#pragma unroll
        for (int c = 0; c < 3; c++) f[3 * m + c] = out[m][c];
}

struct MapXformRows {
    const int32_t *anchor;
    float *xyz, *rotation, *normal, *rest;
    const float *tab;
    unsigned long long *n_skipped;
    int P, K;
};

template <int SH_REST>
__global__ void __launch_bounds__(MX_TILE) map_xform_rows_kernel(const MapXformRows a) {
    constexpr int WR = 3 * SH_REST, WRS = WR | 1;  // odd row stride: conflict-free per-thread rows
    __shared__ __align__(16) float s_xyz[MX_TILE * 3], s_rot[MX_TILE * 4], s_nrm[MX_TILE * 3], s_rest[MX_TILE * WRS];
    __shared__ int s_k[MX_TILE];
    const int row0 = blockIdx.x * MX_TILE, nrows = min(MX_TILE, a.P - row0), t = threadIdx.x;
    int k = -1;
    bool skipped = false;
    if (t < nrows) {
        const int id = __ldcs(a.anchor + row0 + t);
        if (id != -1) {
            if (id < 0 || id >= a.K) skipped = true;
            else if (__float_as_int(__ldg(a.tab + (size_t)id * MX_ROW)) != 0) k = id;
        }
    }
    s_k[t] = k;
    const unsigned n_skip = __syncthreads_count(skipped);
    if (t == 0 && n_skip) atomicAdd(a.n_skipped, (unsigned long long)n_skip);
    if (!__syncthreads_or(k >= 0)) return;
    mx_stage<3, 3, true>(a.xyz, s_xyz, row0, nrows, s_k);
    mx_stage<4, 4, true>(a.rotation, s_rot, row0, nrows, s_k);
    if (a.normal) mx_stage<3, 3, true>(a.normal, s_nrm, row0, nrows, s_k);
    if constexpr (SH_REST > 0) mx_stage<WR, WRS, true>(a.rest, s_rest, row0, nrows, s_k);
    __syncthreads();
    if (k >= 0) {
        const float *T = a.tab + (size_t)k * MX_ROW;
        float R[9], tr[3];
#pragma unroll
        for (int i = 0; i < 9; i++) R[i] = __ldg(T + MX_R + i);
#pragma unroll
        for (int i = 0; i < 3; i++) tr[i] = __ldg(T + MX_T + i);
        float *x = s_xyz + 3 * t;
        const float x0 = x[0], x1 = x[1], x2 = x[2];
#pragma unroll
        for (int i = 0; i < 3; i++) x[i] = fmaf(R[3 * i], x0, fmaf(R[3 * i + 1], x1, fmaf(R[3 * i + 2], x2, tr[i])));
        const float4 q = reinterpret_cast<const float4 *>(s_rot)[t];
        const float dw = __ldg(T + MX_Q), dx = __ldg(T + MX_Q + 1), dy = __ldg(T + MX_Q + 2), dz = __ldg(T + MX_Q + 3);
        reinterpret_cast<float4 *>(s_rot)[t] = make_float4(dw * q.x - dx * q.y - dy * q.z - dz * q.w, dw * q.y + dx * q.x + dy * q.w - dz * q.z,
                                                           dw * q.z - dx * q.w + dy * q.x + dz * q.y, dw * q.w + dx * q.z - dy * q.y + dz * q.x);
        if (a.normal) {
            float *nm = s_nrm + 3 * t;
            const float n0 = nm[0], n1 = nm[1], n2 = nm[2];
#pragma unroll
            for (int i = 0; i < 3; i++) nm[i] = fmaf(R[3 * i], n0, fmaf(R[3 * i + 1], n1, R[3 * i + 2] * n2));
        }
        float *f = s_rest + WRS * t;
        if constexpr (SH_REST >= 3) mx_rotate_band<1>(T + MX_D1, f);
        if constexpr (SH_REST >= 8) mx_rotate_band<2>(T + MX_D2, f + 9);
        if constexpr (SH_REST >= 15) mx_rotate_band<3>(T + MX_D3, f + 24);
    }
    __syncthreads();
    mx_stage<3, 3, false>(a.xyz, s_xyz, row0, nrows, s_k);
    mx_stage<4, 4, false>(a.rotation, s_rot, row0, nrows, s_k);
    if (a.normal) mx_stage<3, 3, false>(a.normal, s_nrm, row0, nrows, s_k);
    if constexpr (SH_REST > 0) mx_stage<WR, WRS, false>(a.rest, s_rest, row0, nrows, s_k);
}

void launch_map_transform(const RtgMapTransform &m, void *ws, cudaStream_t s) {
    float *tab = reinterpret_cast<float *>(ws);
    cudaMemsetAsync(m.n_skipped, 0, sizeof(int64_t), s);
    // K == 0: no table; every anchor other than -1 is out of range, so the row pass only counts them
    if (m.K > 0) map_xform_table_kernel<<<(m.K + 127) / 128, 128, 0, s>>>(m.old_c2w, m.new_c2w, m.K, tab);
    MapXformRows a;
    a.anchor = m.anchor; a.xyz = m.xyz; a.rotation = m.rotation; a.normal = m.normal; a.rest = m.features_rest;
    a.tab = tab; a.n_skipped = reinterpret_cast<unsigned long long *>(m.n_skipped); a.P = m.P; a.K = m.K;
    const unsigned nb = (unsigned)((m.P + MX_TILE - 1) / MX_TILE);
    switch (m.sh_rest) {
        case 0: map_xform_rows_kernel<0><<<nb, MX_TILE, 0, s>>>(a); break;
        case 3: map_xform_rows_kernel<3><<<nb, MX_TILE, 0, s>>>(a); break;
        case 8: map_xform_rows_kernel<8><<<nb, MX_TILE, 0, s>>>(a); break;
        default: map_xform_rows_kernel<15><<<nb, MX_TILE, 0, s>>>(a); break;
    }
}

}  // namespace rtg
