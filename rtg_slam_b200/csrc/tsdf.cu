// A surface from the map: truncated signed distance fusion of depth frames into a dense voxel grid, and marching
// tetrahedra on the grid (no reference counterpart; the reference evaluates meshes with trimesh / open3d on the host).
//
//  * tsdf_integrate_kernel<POSE>: one thread per voxel (grid-stride, x fastest). The voxel centre is projected with the
//    W2C read on the device (float64 or float32, arithmetic in float64), the nearest pixel is taken with rint (half to
//    even: integer pixel coordinates are the sample points) and the voxel is updated with weight 1 when the pixel has
//    depth and the signed distance is above -trunc. A voxel that is not updated is neither read nor written, and no
//    voxel is written by two threads: no atomics, bit-identical repeats.
//  * tsdf_count_kernel / tsdf_emit_kernel: the Kuhn decomposition splits cell (i,j,k) into six tetrahedra, one per axis
//    permutation p (lexicographic order): c, c+e_p0, c+e_p0+e_p1, c+(1,1,1). Every tetrahedron edge joins a corner to one
//    with a superset of its offset bits, so each grid voxel owns the seven edges to +x, +y, +z, +x+y, +y+z, +x+z, +x+y+z
//    (slots 0..6). The count pass writes per voxel the bitmask of its edges that carry a vertex and the number of
//    triangles of the cell it anchors; two exclusive scans (the one rtg_soa_compact uses) give the output offsets; the
//    emit pass writes vertex owner_offset + popc(mask & ((1 << slot) - 1)) and the cell's triangles in (tetrahedron,
//    triangle) order. No hashing, no atomics.
#include "../../include/rtg_splat_b200.h"
#include "common.cuh"
#include "kernels.h"
#include "prof.h"

namespace rtg {

// triangles of a positively oriented tetrahedron per case (bit q = corner q has tsdf < 0), as edge ids into kTetEdge,
// -1 = none; normal from the negative corners to the positive ones. Derived, and compared with this table, by
// oracle/tsdf_oracle.py:tet_table.
__constant__ int8_t kTetTriangles[16][2][3] = {
    {{-1, -1, -1}, {-1, -1, -1}}, {{0, 1, 2}, {-1, -1, -1}}, {{0, 4, 3}, {-1, -1, -1}}, {{1, 2, 4}, {1, 4, 3}},
    {{1, 3, 5}, {-1, -1, -1}},    {{2, 0, 3}, {2, 3, 5}},    {{0, 4, 5}, {0, 5, 1}},    {{2, 4, 5}, {-1, -1, -1}},
    {{2, 5, 4}, {-1, -1, -1}},    {{0, 1, 5}, {0, 5, 4}},    {{3, 0, 2}, {3, 2, 5}},    {{1, 5, 3}, {-1, -1, -1}},
    {{1, 3, 4}, {1, 4, 2}},       {{0, 3, 4}, {-1, -1, -1}}, {{0, 2, 1}, {-1, -1, -1}}, {{-1, -1, -1}, {-1, -1, -1}}};
// tetrahedron edge e joins path corners kTetEdge[e][0] < kTetEdge[e][1]
__constant__ int8_t kTetEdge[6][2] = {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}};
// cell corner (bit 0 = +x, bit 1 = +y, bit 2 = +z) of the path corners 1 and 2 of tetrahedron t; corner 0 is 0, corner 3 is 7
__constant__ uint8_t kTetPath[6][2] = {{1, 3}, {1, 5}, {2, 3}, {2, 6}, {4, 5}, {4, 6}};
// edge slot of a corner offset (bits as above), and back
__constant__ int8_t kSlotOfOffset[8] = {-1, 0, 1, 3, 2, 5, 4, 6};
__constant__ uint8_t kOffsetOfSlot[7] = {1, 2, 4, 3, 6, 5, 7};

struct TsdfGrid {
    int nx, ny, nz;
    uint32_t n;
    double ox, oy, oz, s;
    float trunc;
    float *tsdf, *weight, *color;
};

static TsdfGrid make_grid(const RtgTsdfVolume &v) {
    TsdfGrid g;
    g.nx = v.nx; g.ny = v.ny; g.nz = v.nz;
    g.n = (uint32_t)((int64_t)v.nx * v.ny * v.nz);
    g.ox = v.origin[0]; g.oy = v.origin[1]; g.oz = v.origin[2];
    g.s = v.voxel_size;
    g.trunc = v.trunc;
    g.tsdf = v.tsdf; g.weight = v.weight; g.color = v.color;
    return g;
}

template <typename POSE>
__global__ void __launch_bounds__(256) tsdf_integrate_kernel(const TsdfGrid g, const float *__restrict__ depth,
                                                              const float *__restrict__ color, int H, int W, int channels_last,
                                                              float fx, float fy, float cx, float cy, const POSE *__restrict__ w2c) {
    double P[12];
#pragma unroll
    for (int r = 0; r < 12; r++) P[r] = (double)w2c[r];
    const double tr = g.trunc;
    const size_t HW = (size_t)H * W;
    for (uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x; idx < g.n; idx += gridDim.x * blockDim.x) {
        const uint32_t i = idx % (uint32_t)g.nx, rest = idx / (uint32_t)g.nx;
        const uint32_t j = rest % (uint32_t)g.ny, k = rest / (uint32_t)g.ny;
        const double px = g.ox + g.s * (double)i, py = g.oy + g.s * (double)j, pz = g.oz + g.s * (double)k;
        const double z = P[8] * px + P[9] * py + P[10] * pz + P[11];
        if (!(z > 0.0)) continue;
        const double x = P[0] * px + P[1] * py + P[2] * pz + P[3];
        const double y = P[4] * px + P[5] * py + P[6] * pz + P[7];
        const double ru = rint((double)fx * x / z + (double)cx), rv = rint((double)fy * y / z + (double)cy);
        if (!(ru >= 0.0 && ru <= (double)(W - 1) && rv >= 0.0 && rv <= (double)(H - 1))) continue;
        const size_t pix = (size_t)rv * W + (size_t)ru;
        const float d = depth[pix];
        if (!(d > 0.f)) continue;
        const double sdf = (double)d - z;
        if (sdf < -tr) continue;
        const float f = (float)fmin(1.0, sdf / tr);
        const float w = g.weight[idx], w1 = w + 1.f;
        g.tsdf[idx] = (g.tsdf[idx] * w + f) / w1;
        if (g.color) {
#pragma unroll
            for (int c = 0; c < 3; c++) {
                const float cp = channels_last ? color[pix * 3 + c] : color[(size_t)c * HW + pix];
                float *cv = g.color + (size_t)c * g.n + idx;
                *cv = (*cv * w + cp) / w1;
            }
        }
        g.weight[idx] = w1;
    }
}

// the 8 corners of the cell anchored at voxel (i,j,k), corner q = dx + 2 dy + 4 dz: observed (weight > 0 and inside the
// grid) and negative (tsdf < 0) as bitmasks
struct CellSigns {
    uint32_t obs, neg;
};

__device__ __forceinline__ CellSigns load_signs(const TsdfGrid &g, uint32_t idx, uint32_t i, uint32_t j, uint32_t k) {
    CellSigns c{0u, 0u};
#pragma unroll
    for (int q = 0; q < 8; q++) {
        const uint32_t dx = q & 1, dy = (q >> 1) & 1, dz = (q >> 2) & 1;
        if (i + dx < (uint32_t)g.nx && j + dy < (uint32_t)g.ny && k + dz < (uint32_t)g.nz) {
            const size_t o = (size_t)idx + dx + (size_t)dy * g.nx + (size_t)dz * g.nx * g.ny;
            if (g.weight[o] > 0.f) {
                c.obs |= 1u << q;
                if (g.tsdf[o] < 0.f) c.neg |= 1u << q;
            }
        }
    }
    return c;
}

__device__ __forceinline__ uint32_t edge_mask(const CellSigns &c) {
    uint32_t m = 0;
    if (!(c.obs & 1u)) return 0;
#pragma unroll
    for (int slot = 0; slot < 7; slot++) {
        const uint32_t q = kOffsetOfSlot[slot];
        if ((c.obs >> q & 1u) && ((c.neg & 1u) != (c.neg >> q & 1u))) m |= 1u << slot;
    }
    return m;
}

// case of tetrahedron t (bit q = path corner q negative), or -1 when a corner is unobserved
__device__ __forceinline__ int tet_case(const CellSigns &c, int t, int (&path)[4]) {
    path[0] = 0; path[1] = kTetPath[t][0]; path[2] = kTetPath[t][1]; path[3] = 7;
    const uint32_t corners = 1u | (1u << path[1]) | (1u << path[2]) | 0x80u;
    if ((c.obs & corners) != corners) return -1;
    return (int)((c.neg & 1u) | (c.neg >> path[1] & 1u) << 1 | (c.neg >> path[2] & 1u) << 2 | (c.neg >> 7 & 1u) << 3);
}

__device__ __forceinline__ bool is_cell(const TsdfGrid &g, uint32_t i, uint32_t j, uint32_t k) {
    return i + 1 < (uint32_t)g.nx && j + 1 < (uint32_t)g.ny && k + 1 < (uint32_t)g.nz;
}

__global__ void __launch_bounds__(256) tsdf_count_kernel(const TsdfGrid g, uint8_t *__restrict__ mask, uint32_t *__restrict__ vcount,
                                                          uint32_t *__restrict__ tcount) {
    for (uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x; idx < g.n; idx += gridDim.x * blockDim.x) {
        const uint32_t i = idx % (uint32_t)g.nx, rest = idx / (uint32_t)g.nx;
        const uint32_t j = rest % (uint32_t)g.ny, k = rest / (uint32_t)g.ny;
        const CellSigns c = load_signs(g, idx, i, j, k);
        const uint32_t m = edge_mask(c);
        uint32_t nt = 0;
        if (is_cell(g, i, j, k)) {
            for (int t = 0; t < 6; t++) {
                int path[4];
                const int cs = tet_case(c, t, path);
                if (cs > 0 && cs < 15) nt += __popc(cs) == 2 ? 2u : 1u;
            }
        }
        mask[idx] = (uint8_t)m;
        vcount[idx] = __popc(m);
        tcount[idx] = nt;
    }
}

__global__ void __launch_bounds__(256) tsdf_emit_kernel(const TsdfGrid g, const uint8_t *__restrict__ mask,
                                                         const uint32_t *__restrict__ voff, const uint32_t *__restrict__ toff,
                                                         float *__restrict__ vertices, float *__restrict__ vcolor,
                                                         int32_t *__restrict__ faces) {
    for (uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x; idx < g.n; idx += gridDim.x * blockDim.x) {
        const uint32_t m = mask[idx];
        const uint32_t i = idx % (uint32_t)g.nx, rest = idx / (uint32_t)g.nx;
        const uint32_t j = rest % (uint32_t)g.ny, k = rest / (uint32_t)g.ny;
        const bool cell = is_cell(g, i, j, k);  // then idx + 1 < n
        // this cell's triangle range as counted: nothing is written outside it even if the grid changed since the count
        const uint32_t tbase = toff[idx], tend = cell ? toff[idx + 1] : tbase;
        if (m == 0 && tbase == tend) continue;
        const CellSigns c = load_signs(g, idx, i, j, k);
        // vertices owned by this voxel, slot order
        uint32_t vo = voff[idx];
        for (int slot = 0; slot < 7; slot++) {
            if (!(m >> slot & 1u)) continue;
            const int q = kOffsetOfSlot[slot];
            const uint32_t dx = q & 1, dy = (q >> 1) & 1, dz = (q >> 2) & 1;
            const size_t ob = (size_t)idx + dx + (size_t)dy * g.nx + (size_t)dz * g.nx * g.ny;
            const double fa = g.tsdf[idx], fb = g.tsdf[ob], tau = fa / (fa - fb);
            const double ax = g.ox + g.s * (double)i, ay = g.oy + g.s * (double)j, az = g.oz + g.s * (double)k;
            const double bx = g.ox + g.s * (double)(i + dx), by = g.oy + g.s * (double)(j + dy), bz = g.oz + g.s * (double)(k + dz);
            vertices[3 * (size_t)vo + 0] = (float)(ax + tau * (bx - ax));
            vertices[3 * (size_t)vo + 1] = (float)(ay + tau * (by - ay));
            vertices[3 * (size_t)vo + 2] = (float)(az + tau * (bz - az));
            if (vcolor) {
#pragma unroll
                for (int ch = 0; ch < 3; ch++) {
                    const double ca = g.color[(size_t)ch * g.n + idx], cb = g.color[(size_t)ch * g.n + ob];
                    vcolor[3 * (size_t)vo + ch] = (float)(ca + tau * (cb - ca));
                }
            }
            vo++;
        }
        // triangles of this cell, (tetrahedron, triangle) order
        uint32_t to = tbase;
        for (int t = 0; t < 6 && to < tend; t++) {
            int path[4];
            const int cs = tet_case(c, t, path);
            if (cs <= 0 || cs >= 15) continue;
            const bool odd = t == 1 || t == 2 || t == 5;  // odd permutations give negatively oriented tetrahedra
            for (int r = 0; r < 2 && to < tend; r++) {
                if (kTetTriangles[cs][r][0] < 0) break;
                int32_t id[3];
#pragma unroll
                for (int e = 0; e < 3; e++) {
                    const int edge = kTetTriangles[cs][r][e];
                    const int ca = path[kTetEdge[edge][0]], cb = path[kTetEdge[edge][1]];
                    const uint32_t own = idx + (uint32_t)(ca & 1) + (uint32_t)((ca >> 1) & 1) * (uint32_t)g.nx +
                                         (uint32_t)((ca >> 2) & 1) * (uint32_t)g.nx * (uint32_t)g.ny;
                    const int slot = kSlotOfOffset[ca ^ cb];
                    id[e] = (int32_t)(voff[own] + __popc((uint32_t)mask[own] & ((1u << slot) - 1u)));
                }
                int32_t *out = faces + 3 * (size_t)to;
                out[0] = id[0];
                out[1] = odd ? id[2] : id[1];
                out[2] = odd ? id[1] : id[2];
                to++;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------------ ray-cast
// The surface the ray-cast finds is the extracted mesh: the piecewise-linear interpolant on the same Kuhn tetrahedra, a
// tetrahedron taking part only when its four weights are > 0. Rays walk the cells in grid coordinates (3-D DDA); inside
// a cell the planes u_a = u_b cut the ray into at most four pieces, one tetrahedron each, and along a piece the field is
// linear, so its zero crossing is exact. The first piece whose field changes sign decides: >= 0 to < 0 is a hit, < 0 to
// >= 0 (a back face) ends the ray without one.

// corner q (bit 0 = +x, bit 1 = +y, bit 2 = +z) of the cell anchored at voxel offset `base`
__device__ __forceinline__ size_t raycast_corner(const TsdfGrid &g, size_t base, int q) {
    return base + (size_t)(q & 1) + (size_t)((q >> 1) & 1) * (size_t)g.nx + (size_t)((q >> 2) & 1) * (size_t)g.nx * (size_t)g.ny;
}

__device__ __forceinline__ void raycast_load(const TsdfGrid &g, size_t base, int q, float (&f)[8], uint32_t &obs) {
    const size_t o = raycast_corner(g, base, q);
    const float w = __ldg(g.weight + o);
    f[q] = w > 0.f ? __ldg(g.tsdf + o) : 1.f;
    obs = w > 0.f ? (obs | 1u << q) : (obs & ~(1u << q));
}

// the four corners on side SIDE of axis A
template <int A, int SIDE>
__device__ __forceinline__ void raycast_load_face(const TsdfGrid &g, size_t base, float (&f)[8], uint32_t &obs) {
#pragma unroll
    for (int q = 0; q < 8; q++)
        if ((q >> A & 1) == SIDE) raycast_load(g, base, q, f, obs);
}

// one cell along axis A (up: +1): the four corners the two cells share move across, the four new ones are loaded
template <int A>
__device__ __forceinline__ void raycast_step(const TsdfGrid &g, size_t base, bool up, float (&f)[8], uint32_t &obs) {
    constexpr int sh = 1 << A;
    constexpr uint32_t lo = A == 0 ? 0x55u : (A == 1 ? 0x33u : 0x0Fu);  // corners with bit A clear
    if (up) {
#pragma unroll
        for (int q = 0; q < 8; q++)
            if (!(q >> A & 1)) f[q] = f[q | sh];
        obs = (obs >> sh) & lo;
        raycast_load_face<A, 1>(g, base, f, obs);
    } else {
#pragma unroll
        for (int q = 0; q < 8; q++)
            if (!(q >> A & 1)) f[q | sh] = f[q];
        obs = (obs << sh) & (0xFFu & ~lo);
        raycast_load_face<A, 0>(g, base, f, obs);
    }
}

__device__ __forceinline__ float raycast_pick(const float (&f)[8], int q) {
    float r = f[0];
#pragma unroll
    for (int k = 1; k < 8; k++) r = q == k ? f[k] : r;
    return r;
}

__device__ __forceinline__ double raycast_pick3(const double (&a)[3], int i) { return i == 0 ? a[0] : (i == 1 ? a[1] : a[2]); }

template <typename POSE>
__global__ void __launch_bounds__(128) tsdf_raycast_kernel(const TsdfGrid g, const POSE *__restrict__ w2c, int H, int W, float fx,
                                                           float fy, float cx, float cy, float *__restrict__ depth,
                                                           float *__restrict__ normal, float *__restrict__ color) {
    const int px = blockIdx.x * blockDim.x + threadIdx.x, py = blockIdx.y * blockDim.y + threadIdx.y;
    if (px >= W || py >= H) return;
    const size_t HW = (size_t)H * W, pix = (size_t)py * W + px;
    // the ray o + t d in grid coordinates (voxel (i,j,k) at (i,j,k)); t is camera z
    double l[3], dg[3];
    {
        double P[12];
#pragma unroll
        for (int r = 0; r < 12; r++) P[r] = (double)w2c[r];
        const double dcx = ((double)px - (double)cx) / (double)fx, dcy = ((double)py - (double)cy) / (double)fy;
        const double org[3] = {g.ox, g.oy, g.oz};
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const double o = -(P[a] * P[3] + P[4 + a] * P[7] + P[8 + a] * P[11]);
            const double d = P[a] * dcx + P[4 + a] * dcy + P[8 + a];
            l[a] = (o - org[a]) / g.s;
            dg[a] = d / g.s;
        }
    }
    const int n[3] = {g.nx, g.ny, g.nz};
    float out_t = 0.f, out_n[3] = {0.f, 0.f, 0.f}, out_c[3] = {0.f, 0.f, 0.f};
    // clip to t >= 0 and the cell region [0, n-1]^3
    double t_in = 0.0, t_out = INFINITY;
    bool live = n[0] > 1 && n[1] > 1 && n[2] > 1;
#pragma unroll
    for (int a = 0; a < 3; a++) {
        const double hi = (double)(n[a] - 1);
        if (dg[a] != 0.0) {
            const double ta = -l[a] / dg[a], tb = (hi - l[a]) / dg[a];
            t_in = fmax(t_in, fmin(ta, tb));
            t_out = fmin(t_out, fmax(ta, tb));
        } else if (!(l[a] >= 0.0 && l[a] <= hi)) {
            live = false;
        }
    }
    if (live && t_in < t_out) {
        int c[3];
        double tn[3];
#pragma unroll
        for (int a = 0; a < 3; a++) {
            c[a] = (int)fmin(fmax(floor(l[a] + t_in * dg[a]), 0.0), (double)(n[a] - 2));
            tn[a] = dg[a] > 0.0 ? ((double)(c[a] + 1) - l[a]) / dg[a] : (dg[a] < 0.0 ? ((double)c[a] - l[a]) / dg[a] : INFINITY);
        }
        const size_t sy = (size_t)g.nx, sz = (size_t)g.nx * (size_t)g.ny;
        size_t base = (size_t)c[0] + (size_t)c[1] * sy + (size_t)c[2] * sz;
        float f[8];
        uint32_t obs = 0;
#pragma unroll
        for (int q = 0; q < 8; q++) raycast_load(g, base, q, f, obs);
        double t0 = t_in;
        while (true) {
            const int ax = tn[0] <= tn[1] ? (tn[0] <= tn[2] ? 0 : 2) : (tn[1] <= tn[2] ? 1 : 2);
            const double t1 = fmin(raycast_pick3(tn, ax), t_out);
            uint32_t neg = 0;
#pragma unroll
            for (int q = 0; q < 8; q++) neg |= (f[q] < 0.f ? 1u : 0u) << q;
            neg &= obs;
            // a tetrahedron needs corners 0 and 7; a crossing needs an observed corner of either sign
            if ((obs & 0x81u) == 0x81u && neg != 0 && (obs & ~neg) != 0 && t1 > t0) {
                double u[3];  // local coordinates are u_a(t) = u[a] + t dg[a]
#pragma unroll
                for (int a = 0; a < 3; a++) u[a] = l[a] - (double)c[a];
                double s01 = (u[1] - u[0]) / (dg[0] - dg[1]), s02 = (u[2] - u[0]) / (dg[0] - dg[2]),
                       s12 = (u[2] - u[1]) / (dg[1] - dg[2]);
                if (!(s01 > t0 && s01 < t1)) s01 = t1;
                if (!(s02 > t0 && s02 < t1)) s02 = t1;
                if (!(s12 > t0 && s12 < t1)) s12 = t1;
                // the three in order (min, median, max)
                const double b[5] = {t0, fmin(fmin(s01, s02), s12), fmax(fmin(s01, s02), fmin(fmax(s01, s02), s12)),
                                     fmax(fmax(s01, s02), s12), t1};
                int state = 0;  // 1 = hit, 2 = back face
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const double ta = b[i], tb = b[i + 1];
                    if (state != 0 || !(tb > ta)) continue;
                    const double mid = 0.5 * (ta + tb);
                    const double m0 = u[0] + mid * dg[0], m1 = u[1] + mid * dg[1], m2 = u[2] + mid * dg[2];
                    // the permutation ordering u decreasingly, ties to the lower axis
                    int p1, p2, p3;
                    if (m0 >= m1) {
                        if (m1 >= m2) { p1 = 0; p2 = 1; p3 = 2; }
                        else if (m0 >= m2) { p1 = 0; p2 = 2; p3 = 1; }
                        else { p1 = 2; p2 = 0; p3 = 1; }
                    } else {
                        if (m0 >= m2) { p1 = 1; p2 = 0; p3 = 2; }
                        else if (m1 >= m2) { p1 = 1; p2 = 2; p3 = 0; }
                        else { p1 = 2; p2 = 1; p3 = 0; }
                    }
                    const int q1 = 1 << p1, q2 = q1 | 1 << p2;
                    if (!(obs >> q1 & 1u) || !(obs >> q2 & 1u)) continue;
                    const double f0 = f[0], f1 = raycast_pick(f, q1), f2 = raycast_pick(f, q2), f3 = f[7];
                    const double g1 = f1 - f0, g2 = f2 - f1, g3 = f3 - f2;
                    const double ua1 = raycast_pick3(u, p1), ua2 = raycast_pick3(u, p2), ua3 = raycast_pick3(u, p3);
                    const double d1 = raycast_pick3(dg, p1), d2 = raycast_pick3(dg, p2), d3 = raycast_pick3(dg, p3);
                    const double fa = f0 + g1 * (ua1 + ta * d1) + g2 * (ua2 + ta * d2) + g3 * (ua3 + ta * d3);
                    const double fb = f0 + g1 * (ua1 + tb * d1) + g2 * (ua2 + tb * d2) + g3 * (ua3 + tb * d3);
                    if (fa < 0.0 && fb >= 0.0) state = 2;
                    if (!(fa >= 0.0 && fb < 0.0)) continue;
                    state = 1;
                    const double ts = ta + (tb - ta) * fa / (fa - fb);
                    out_t = (float)ts;
                    const double gx = p1 == 0 ? g1 : (p2 == 0 ? g2 : g3), gy = p1 == 1 ? g1 : (p2 == 1 ? g2 : g3),
                                 gz = p1 == 2 ? g1 : (p2 == 2 ? g2 : g3);
                    const double inv = 1.0 / sqrt(gx * gx + gy * gy + gz * gz);
                    out_n[0] = (float)(gx * inv);
                    out_n[1] = (float)(gy * inv);
                    out_n[2] = (float)(gz * inv);
                    if (color) {
                        const double h1 = ua1 + ts * d1, h2 = ua2 + ts * d2, h3 = ua3 + ts * d3;
                        const double w0 = 1.0 - h1, w1 = h1 - h2, w2 = h2 - h3, w3 = h3;
                        const size_t o0 = base, o1 = raycast_corner(g, base, q1), o2 = raycast_corner(g, base, q2),
                                     o3 = raycast_corner(g, base, 7);
#pragma unroll
                        for (int ch = 0; ch < 3; ch++) {
                            const float *cc = g.color + (size_t)ch * g.n;
                            out_c[ch] = (float)(w0 * (double)__ldg(cc + o0) + w1 * (double)__ldg(cc + o1) + w2 * (double)__ldg(cc + o2) +
                                                w3 * (double)__ldg(cc + o3));
                        }
                    }
                }
                if (state != 0) break;
            }
            if (t1 >= t_out) break;
            t0 = t1;
            if (ax == 0) {
                const bool up = dg[0] > 0.0;
                c[0] += up ? 1 : -1;
                if (c[0] < 0 || c[0] > n[0] - 2) break;
                base = up ? base + 1 : base - 1;
                tn[0] = (up ? (double)(c[0] + 1) - l[0] : (double)c[0] - l[0]) / dg[0];
                raycast_step<0>(g, base, up, f, obs);
            } else if (ax == 1) {
                const bool up = dg[1] > 0.0;
                c[1] += up ? 1 : -1;
                if (c[1] < 0 || c[1] > n[1] - 2) break;
                base = up ? base + sy : base - sy;
                tn[1] = (up ? (double)(c[1] + 1) - l[1] : (double)c[1] - l[1]) / dg[1];
                raycast_step<1>(g, base, up, f, obs);
            } else {
                const bool up = dg[2] > 0.0;
                c[2] += up ? 1 : -1;
                if (c[2] < 0 || c[2] > n[2] - 2) break;
                base = up ? base + sz : base - sz;
                tn[2] = (up ? (double)(c[2] + 1) - l[2] : (double)c[2] - l[2]) / dg[2];
                raycast_step<2>(g, base, up, f, obs);
            }
        }
    }
    depth[pix] = out_t;
#pragma unroll
    for (int a = 0; a < 3; a++) normal[(size_t)a * HW + pix] = out_n[a];
    if (color) {
#pragma unroll
        for (int ch = 0; ch < 3; ch++) color[(size_t)ch * HW + pix] = out_c[ch];
    }
}

static unsigned grid_blocks(uint32_t n) {
    const uint32_t b = (n + 255) / 256;
    return b < RTG_NUM_SMS * 16 ? b : RTG_NUM_SMS * 16;
}

void launch_tsdf_integrate(const RtgTsdfVolume &v, const float *depth, const float *color, int H, int W, int channels_last, float fx,
                           float fy, float cx, float cy, const void *w2c, bool w2c_double, cudaStream_t s) {
    ProfScope ps(K_TSDF_INTEGRATE, s);
    const TsdfGrid g = make_grid(v);
    const unsigned nb = grid_blocks(g.n);
    if (w2c_double)
        tsdf_integrate_kernel<double><<<nb, 256, 0, s>>>(g, depth, g.color ? color : nullptr, H, W, channels_last, fx, fy, cx, cy,
                                                         static_cast<const double *>(w2c));
    else
        tsdf_integrate_kernel<float><<<nb, 256, 0, s>>>(g, depth, g.color ? color : nullptr, H, W, channels_last, fx, fy, cx, cy,
                                                        static_cast<const float *>(w2c));
}

void launch_tsdf_raycast(const RtgTsdfVolume &v, const void *w2c, bool w2c_double, int H, int W, float fx, float fy, float cx,
                         float cy, float *depth, float *normal, float *color, cudaStream_t s) {
    ProfScope ps(K_TSDF_RAYCAST, s);
    const TsdfGrid g = make_grid(v);
    const dim3 block(16, 8), grid((W + 15) / 16, (H + 7) / 8);  // neighbouring rays walk neighbouring cells
    if (w2c_double)
        tsdf_raycast_kernel<double><<<grid, block, 0, s>>>(g, static_cast<const double *>(w2c), H, W, fx, fy, cx, cy, depth, normal,
                                                           g.color ? color : nullptr);
    else
        tsdf_raycast_kernel<float><<<grid, block, 0, s>>>(g, static_cast<const float *>(w2c), H, W, fx, fy, cx, cy, depth, normal,
                                                          g.color ? color : nullptr);
}

size_t tsdf_extract_ws_bytes(int64_t n) {
    const size_t N = (size_t)n;
    return align_up(N, 256) + 2 * align_up(N * 4, 256) + 2 * align_up(exclusive_scan_sums_words((uint32_t)N) * 4, 256) + 256;
}

struct ExtractWs {
    uint8_t *mask;
    uint32_t *voff, *toff, *vsums, *tsums;
};

static ExtractWs carve_extract(void *ws, uint32_t n) {
    char *p = reinterpret_cast<char *>(ws);
    ExtractWs w;
    w.mask = carve<uint8_t>(p, n);
    w.voff = carve<uint32_t>(p, n);
    w.toff = carve<uint32_t>(p, n);
    w.vsums = carve<uint32_t>(p, exclusive_scan_sums_words(n));
    w.tsums = carve<uint32_t>(p, exclusive_scan_sums_words(n));
    return w;
}

void launch_tsdf_extract_count(const RtgTsdfVolume &v, void *ws, uint32_t *counts, cudaStream_t s) {
    ProfScope ps(K_TSDF_EXTRACT, s);
    const TsdfGrid g = make_grid(v);
    const ExtractWs w = carve_extract(ws, g.n);
    tsdf_count_kernel<<<grid_blocks(g.n), 256, 0, s>>>(g, w.mask, w.voff, w.toff);
    // in place: each scan element is read before the same thread overwrites it
    exclusive_scan_u32(w.voff, g.n, w.voff, w.vsums, counts, nullptr, s);
    exclusive_scan_u32(w.toff, g.n, w.toff, w.tsums, counts + 1, nullptr, s);
}

void launch_tsdf_extract_emit(const RtgTsdfVolume &v, const void *ws, float *vertices, float *vertex_colors, int32_t *faces,
                              cudaStream_t s) {
    ProfScope ps(K_TSDF_EXTRACT, s);
    const TsdfGrid g = make_grid(v);
    const ExtractWs w = carve_extract(const_cast<void *>(ws), g.n);
    tsdf_emit_kernel<<<grid_blocks(g.n), 256, 0, s>>>(g, w.mask, w.voff, w.toff, vertices, g.color ? vertex_colors : nullptr, faces);
}

}  // namespace rtg
