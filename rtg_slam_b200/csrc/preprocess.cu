// Per-Gaussian passes: forward preprocess, frustum marking, backward preprocess.
//
// Behaviour follows the reference's preprocessCUDA (RAST/cuda_rasterizer/forward.cu:238-354),
// checkFrustum (rasterizer_impl.cu:54-66), computeCov2DCUDA (backward.cu:273-422) and the backward
// preprocessCUDA (backward.cu:492-548); the structure does not: one fused pass per direction,
// 16-byte splat records for the render kernels, tile histogram by atomics instead of a global
// scan + 64-bit radix sort, view-space surfel normal/centre computed once per Gaussian instead of
// once per (pixel, Gaussian) pair, and the backward consumes + clears a 64-byte gradient record.
#include "common.cuh"
#include "kernels.h"
#include "prof.h"

namespace rtg {

#define SH_C0 0.28209479177387814f
#define SH_C1 0.4886025119029199f
#define SH_C2_0 1.0925484305920792f
#define SH_C2_1 -1.0925484305920792f
#define SH_C2_2 0.31539156525252005f
#define SH_C2_3 -1.0925484305920792f
#define SH_C2_4 0.5462742152960396f
#define SH_C3_0 -0.5900435899266435f
#define SH_C3_1 2.890611442640554f
#define SH_C3_2 -0.4570457994644658f
#define SH_C3_3 0.3731763325901154f
#define SH_C3_4 -0.4570457994644658f
#define SH_C3_5 1.445305721320277f
#define SH_C3_6 -0.5900435899266435f

// Loads the 3*M SH floats of one Gaussian. M == 16 -> twelve 128-bit loads of a 192-byte,
// 64-byte-aligned record.
__device__ __forceinline__ void load_sh(const float *__restrict__ shs, size_t idx, int M, int ncoef, float *sh) {
    if (M == 16) {
        const float4 *p = reinterpret_cast<const float4 *>(shs + idx * 48);
        const int nv = (ncoef * 3 + 3) / 4;
#pragma unroll
        for (int i = 0; i < 12; i++) {
            if (i < nv) {
                float4 v = __ldg(p + i);
                sh[4 * i] = v.x; sh[4 * i + 1] = v.y; sh[4 * i + 2] = v.z; sh[4 * i + 3] = v.w;
            }
        }
    } else {
        const float *p = shs + idx * (size_t)(3 * M);
#pragma unroll
        for (int i = 0; i < 48; i++)
            if (i < 3 * ncoef) sh[i] = __ldg(p + i);
    }
}

__device__ __forceinline__ int sh_ncoef(int deg) { return (deg + 1) * (deg + 1); }

// Sigma = R S S R^T, symmetric 6-vector (computeCov3D, forward.cu:202-235).
__device__ __forceinline__ void cov3d_from(const float3 s, float mod, const float R[3][3], float *c6) {
    const float sx = mod * s.x, sy = mod * s.y, sz = mod * s.z;
    float Mx[3], My[3], Mz[3];
#pragma unroll
    for (int j = 0; j < 3; j++) { Mx[j] = sx * R[j][0]; My[j] = sy * R[j][1]; Mz[j] = sz * R[j][2]; }
    c6[0] = Mx[0] * Mx[0] + My[0] * My[0] + Mz[0] * Mz[0];
    c6[1] = Mx[0] * Mx[1] + My[0] * My[1] + Mz[0] * Mz[1];
    c6[2] = Mx[0] * Mx[2] + My[0] * My[2] + Mz[0] * Mz[2];
    c6[3] = Mx[1] * Mx[1] + My[1] * My[1] + Mz[1] * Mz[1];
    c6[4] = Mx[1] * Mx[2] + My[1] * My[2] + Mz[1] * Mz[2];
    c6[5] = Mx[2] * Mx[2] + My[2] * My[2] + Mz[2] * Mz[2];
}

// A = J * Rw (two live rows) with the 1.3*tanfov clamp of the view-space centre
// (computeCov2D, forward.cu:158-197). t is the clamped view-space centre.
__device__ __forceinline__ void ewa_A(const float3 tv, const float *vm, float fx, float fy, float tanx, float tany,
                                      float A0[3], float A1[3], float3 &t, float &txtz, float &tytz) {
    t = tv;
    const float limx = 1.3f * tanx, limy = 1.3f * tany;
    txtz = t.x / t.z;
    tytz = t.y / t.z;
    t.x = fminf(limx, fmaxf(-limx, txtz)) * t.z;
    t.y = fminf(limy, fmaxf(-limy, tytz)) * t.z;
    const float J00 = fx / t.z, J02 = -(fx * t.x) / (t.z * t.z);
    const float J11 = fy / t.z, J12 = -(fy * t.y) / (t.z * t.z);
#pragma unroll
    for (int k = 0; k < 3; k++) {
        A0[k] = J00 * vm[0 + 4 * k] + J02 * vm[2 + 4 * k];
        A1[k] = J11 * vm[1 + 4 * k] + J12 * vm[2 + 4 * k];
    }
}

__device__ __forceinline__ void cov2d_from(const float A0[3], const float A1[3], const float *c6, float AV0[3], float AV1[3],
                                           float &a, float &b, float &c) {
    // AV = A * Vrk
    AV0[0] = A0[0] * c6[0] + A0[1] * c6[1] + A0[2] * c6[2];
    AV0[1] = A0[0] * c6[1] + A0[1] * c6[3] + A0[2] * c6[4];
    AV0[2] = A0[0] * c6[2] + A0[1] * c6[4] + A0[2] * c6[5];
    AV1[0] = A1[0] * c6[0] + A1[1] * c6[1] + A1[2] * c6[2];
    AV1[1] = A1[0] * c6[1] + A1[1] * c6[3] + A1[2] * c6[4];
    AV1[2] = A1[0] * c6[2] + A1[1] * c6[4] + A1[2] * c6[5];
    a = AV0[0] * A0[0] + AV0[1] * A0[1] + AV0[2] * A0[2] + 0.3f;
    b = AV0[0] * A1[0] + AV0[1] * A1[1] + AV0[2] * A1[2];
    c = AV1[0] * A1[0] + AV1[1] * A1[1] + AV1[2] * A1[2] + 0.3f;
}

__device__ __forceinline__ bool frustum_cull(const float3 p, const float *vm, const float *pm, float3 &p_view, float3 &p_proj) {
    const float4 ph = xform4x4(p, pm);
    const float pw = 1.0f / (ph.w + 0.0000001f);
    p_proj = make_float3(ph.x * pw, ph.y * pw, ph.z * pw);
    p_view = xform4x3(p, vm);
    // in_frustum, auxiliary.h:139-165
    return (p_view.z <= 0.2f || p_proj.x < -1.3f || p_proj.x > 1.3f || p_proj.y < -1.3f || p_proj.y > 1.3f);
}

// Everything of the forward preprocess that concerns one Gaussian. Returns false if it is culled (radii = 0).
// On success the splat / colour / surfel records are written and the tile rectangle is returned.
struct SplatTiles {
    float2 pix;
    float3 conic;
    float q_cut;
    int x0, y0, x1, y1;
};

__device__ __forceinline__ bool preprocess_one(const ViewParams &vp, const int idx, const int M, const float *s_m,
                                               const float *__restrict__ means, const float *__restrict__ scales,
                                               const float *__restrict__ rots, const float *__restrict__ opac,
                                               const float *__restrict__ shs, const float *__restrict__ colors_precomp,
                                               const float *__restrict__ cov3D_precomp, const GeomState &g, int *__restrict__ radii,
                                               SplatTiles &st) {
    const float *vm = s_m, *pm = s_m + 16;

    const float3 p = make_float3(__ldg(means + 3 * (size_t)idx), __ldg(means + 3 * (size_t)idx + 1), __ldg(means + 3 * (size_t)idx + 2));
    // issued before the cull decision is known: one memory round trip less for the Gaussians that survive
    float3 sc_e = make_float3(0.f, 0.f, 0.f);
    float4 q_e = make_float4(1.f, 0.f, 0.f, 0.f);
    if (cov3D_precomp == nullptr) {
        sc_e = make_float3(__ldg(scales + 3 * (size_t)idx), __ldg(scales + 3 * (size_t)idx + 1), __ldg(scales + 3 * (size_t)idx + 2));
        q_e = __ldg(reinterpret_cast<const float4 *>(rots) + idx);
    }
    float3 pv, pp;
    if (frustum_cull(p, vm, pm, pv, pp)) {
        if (vp.prefiltered) __trap();  // the reference traps as well (auxiliary.h:157-161)
        radii[idx] = 0;
        return false;
    }
    if (shs != nullptr) prefetch_l2(shs + (size_t)idx * 3 * M, 12 * M + 64);  // consumed ~300 instructions later

    float c6[6];
    float R[3][3];
    float3 sc = make_float3(0.f, 0.f, 0.f);
    float4 q = make_float4(1.f, 0.f, 0.f, 0.f);
    if (cov3D_precomp != nullptr) {
#pragma unroll
        for (int i = 0; i < 6; i++) c6[i] = __ldg(cov3D_precomp + 6 * (size_t)idx + i);
    } else {
        sc = sc_e; q = q_e;
        quat_to_R(q, R);
        cov3d_from(sc, vp.scale_modifier, R, c6);
    }

    float A0[3], A1[3], AV0[3], AV1[3], ca, cb, cc, txtz, tytz;
    float3 t;
    ewa_A(pv, vm, vp.focal_x, vp.focal_y, vp.tanfovx, vp.tanfovy, A0, A1, t, txtz, tytz);
    cov2d_from(A0, A1, c6, AV0, AV1, ca, cb, cc);
    const float det = ca * cc - cb * cb;
    if (det == 0.0f) { radii[idx] = 0; return false; }
    const float det_inv = 1.f / det;
    const float3 conic = make_float3(cc * det_inv, -cb * det_inv, ca * det_inv);
    const float mid = 0.5f * (ca + cc);
    const float sq = sqrtf(fmaxf(0.1f, mid * mid - det));
    const float lambda1 = mid + sq, lambda2 = mid - sq;
    const float my_radius = ceilf(vp.color_sigma * sqrtf(fmaxf(lambda1, lambda2)));
    // ndc2Pix(v,S,c) = v*S*0.5 + c, evaluated in double by the reference (auxiliary.h:44-47)
    const float2 pix = make_float2((float)((double)(pp.x * (float)vp.W) * 0.5 + (double)vp.cx),
                                   (float)((double)(pp.y * (float)vp.H) * 0.5 + (double)vp.cy));
    int x0, y0, x1, y1;
    tile_rect(pix, (int)my_radius, vp.tiles_x, vp.tiles_y, x0, y0, x1, y1);
    if ((x1 - x0) * (y1 - y0) == 0) { radii[idx] = 0; return false; }

    // colour
    float3 rgb;
    int flags = 0;
    if (colors_precomp != nullptr) {
        rgb = make_float3(__ldg(colors_precomp + 3 * (size_t)idx), __ldg(colors_precomp + 3 * (size_t)idx + 1),
                          __ldg(colors_precomp + 3 * (size_t)idx + 2));
    } else {
        // computeColorFromSH, forward.cu:104-155
        const int deg = vp.sh_degree;
        float sh[48];
        load_sh(shs, idx, M, sh_ncoef(deg), sh);
        float3 dir = make_float3(p.x - s_m[32], p.y - s_m[33], p.z - s_m[34]);
        const float len = sqrtf(dir.x * dir.x + dir.y * dir.y + dir.z * dir.z);
        const float x = dir.x / len, y = dir.y / len, z = dir.z / len;
        float res[3];
#pragma unroll
        for (int ch = 0; ch < 3; ch++) {
#define S(k) sh[(k) * 3 + ch]
            float r = SH_C0 * S(0);
            if (deg > 0) {
                r = r - SH_C1 * y * S(1) + SH_C1 * z * S(2) - SH_C1 * x * S(3);
                if (deg > 1) {
                    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                    r = r + SH_C2_0 * xy * S(4) + SH_C2_1 * yz * S(5) + SH_C2_2 * (2.0f * zz - xx - yy) * S(6) +
                        SH_C2_3 * xz * S(7) + SH_C2_4 * (xx - yy) * S(8);
                    if (deg > 2) {
                        r = r + SH_C3_0 * y * (3.0f * xx - yy) * S(9) + SH_C3_1 * xy * z * S(10) +
                            SH_C3_2 * y * (4.0f * zz - xx - yy) * S(11) + SH_C3_3 * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * S(12) +
                            SH_C3_4 * x * (4.0f * zz - xx - yy) * S(13) + SH_C3_5 * z * (xx - yy) * S(14) +
                            SH_C3_6 * x * (xx - 3.0f * yy) * S(15);
                    }
                }
            }
#undef S
            r += 0.5f;
            if (r < 0.f) flags |= (1 << ch);
            res[ch] = fmaxf(r, 0.0f);
        }
        rgb = make_float3(res[0], res[1], res[2]);
    }

    // surfel normal / centre in view space (computeNormal_ScaleMax, forward.cu:54-74, and the
    // transforms of forward.cu:779-782), once per Gaussian
    float4 h0 = make_float4(0.f, 0.f, 0.f, 0.f), h1 = make_float4(pv.x, pv.y, pv.z, __int_as_float(0));
    if (cov3D_precomp == nullptr) {
        const int na = arg_min3(sc.x, sc.y, sc.z), ma = arg_max3(sc.x, sc.y, sc.z);
        const float3 nw = make_float3(R[0][na], R[1][na], R[2][na]);
        const float3 nc = xvec4x3(nw, vm);
        const float smax = (ma == 0 ? sc.x : (ma == 1 ? sc.y : sc.z)) * vp.scale_modifier;
        h0 = make_float4(nc.x, nc.y, nc.z, smax);
        h1.w = __int_as_float(na);
    }

    const float opacity = __ldg(opac + idx);
    const float q_cut = q_cutoff(opacity);
    radii[idx] = (int)my_radius;
    g.splat[2 * (size_t)idx] = make_float4(pix.x, pix.y, q_cut, opacity);
    g.splat[2 * (size_t)idx + 1] = make_float4(conic.x, conic.y, conic.z, log2f(opacity));  // see pair_alpha (common.cuh)
    g.rgb_flags[idx] = make_float4(rgb.x, rgb.y, rgb.z, __int_as_float(flags));
    g.hit[2 * (size_t)idx] = h0;
    g.hit[2 * (size_t)idx + 1] = h1;

    st.pix = pix; st.conic = conic; st.q_cut = q_cut;
    st.x0 = x0; st.y0 = y0; st.x1 = x1; st.y1 = y1;
    return true;
}

#ifndef PFWD_MIN_BLOCKS
#define PFWD_MIN_BLOCKS 3  // sm_90a: capped at 80 registers, ptxas spills 16 B (stores and loads)
#endif
__global__ void __launch_bounds__(256, PFWD_MIN_BLOCKS) preprocess_fwd_kernel(const ViewParams vp, const int P, const int M,
                                                             const float *__restrict__ means, const float *__restrict__ scales,
                                                             const float *__restrict__ rots, const float *__restrict__ opac,
                                                             const float *__restrict__ shs, const float *__restrict__ colors_precomp,
                                                             const float *__restrict__ cov3D_precomp,
                                                             const int *__restrict__ tile_mask, GeomState g,
                                                             int *__restrict__ radii, uint32_t *__restrict__ tile_count,
                                                             uint32_t *__restrict__ tile_touched, uint32_t *__restrict__ vis_count,
                                                             const int p_begin) {
    __shared__ float s_m[40];
    __shared__ uint32_t s_excl[8][32], s_rect[8][32];
    __shared__ float4 s_ga[8][32], s_gb[8][32];
    if (threadIdx.x < 16) s_m[threadIdx.x] = vp.view[threadIdx.x];
    else if (threadIdx.x < 32) s_m[threadIdx.x] = vp.proj[threadIdx.x - 16];
    else if (threadIdx.x < 35) s_m[threadIdx.x] = vp.campos[threadIdx.x - 32];
    __syncthreads();
    // Gaussians [p_begin, P) of the map: the whole map, or the slice a rank owns (the parameter pointers are then
    // shifted so that they can be indexed with the global id; the records are always indexed with the global id)
    const int idx = p_begin + blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;

    SplatTiles st;
    bool valid = false;
    if (idx < P) valid = preprocess_one(vp, idx, M, s_m, means, scales, rots, opac, shs, colors_precomp, cov3D_precomp, g, radii, st);

    // Tile histogram over the masked-in tiles of the reference's rectangle (forward.cu:344-353), minus the tiles
    // in which no pixel can pass the alpha cut-off (exact test; such entries are skipped by every pixel of the
    // reference's render loop, so dropping them changes no output). Tiles that lose all their entries this way
    // are flagged: the reference still renders them (hit maps -1, colour = background). The (Gaussian, tile)
    // pairs of the warp's 32 Gaussians are shared evenly among its lanes.
    {   // compact list of the surviving Gaussians (used by the backward preprocess); warp-aggregated append
        const uint32_t vb = __ballot_sync(0xffffffffu, valid);
        if (vb) {
            uint32_t basep = 0;
            if (lane == 0) basep = atomicAdd(vis_count, (uint32_t)__popc(vb));
            basep = __shfl_sync(0xffffffffu, basep, 0);
            if (valid) g.vis_list[basep + __popc(vb & ((1u << lane) - 1u))] = (uint32_t)idx;
        }
    }
    if (tile_count == nullptr) return;  // Gaussian-sharded forward: the histogram runs after the exchange of the records
    const int npairs = valid ? (st.x1 - st.x0) * (st.y1 - st.y0) : 0;
    const int incl = warp_incl_scan(npairs, lane);
    const int total = __shfl_sync(0xffffffffu, incl, 31);
    if (total == 0) return;  // warp-uniform
    s_excl[w][lane] = (uint32_t)(incl - npairs);
    if (valid) {
        s_rect[w][lane] = pack_rect(st.x0, st.y0, st.x1 - st.x0);
        const float2 nb = cut_slopes(st.conic.x, st.conic.y, st.conic.z);
        s_ga[w][lane] = make_float4(st.pix.x, st.pix.y, st.q_cut, nb.x);
        s_gb[w][lane] = make_float4(st.conic.x, st.conic.y, st.conic.z, nb.y);
    }
    __syncwarp();
    for (int k = lane; k < total; k += 32) {
        const int o = pair_owner(s_excl[w], (uint32_t)k);
        const uint32_t local = (uint32_t)k - s_excl[w][o], rc = s_rect[w][o];
        const uint32_t rw = rc >> 20;
        int cx, cy;
        rect_cell(local, rw, cx, cy);
        const int x = (int)(rc & 1023u) + cx, y = (int)((rc >> 10) & 1023u) + cy;
        const int tt = y * vp.tiles_x + x;
        if (__ldg(tile_mask + tt)) {
            const float4 ga = s_ga[w][o], gb = s_gb[w][o];
            const float fx0 = (float)(x * RTG_TILE), fy0 = (float)(y * RTG_TILE);
            if (rect_below_cutoff(ga.x, ga.y, gb.x, gb.y, gb.z, ga.z, ga.w, gb.w, fx0, fx0 + (RTG_TILE - 1), fy0, fy0 + (RTG_TILE - 1)))
                tile_touched[tt] = 1u;
            else
                atomicAdd(tile_count + (size_t)tt * RTG_CNT_STRIDE, 1u);
        }
    }
}

__global__ void __launch_bounds__(256) mark_visible_kernel(int P, const float *__restrict__ means, const float *__restrict__ view,
                                                           const float *__restrict__ proj, uint8_t *__restrict__ present) {
    __shared__ float s_m[32];
    if (threadIdx.x < 16) s_m[threadIdx.x] = view[threadIdx.x];
    else if (threadIdx.x < 32) s_m[threadIdx.x] = proj[threadIdx.x - 16];
    __syncthreads();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    const float3 p = make_float3(means[3 * (size_t)idx], means[3 * (size_t)idx + 1], means[3 * (size_t)idx + 2]);
    float3 pv, pp;
    present[idx] = frustum_cull(p, s_m, s_m + 16, pv, pp) ? 0 : 1;
}

// ------------------------------------------------------------------ backward
// One pass per Gaussian: conic -> cov2D -> cov3D -> (scale, quaternion); projection-path and
// SH-path mean gradients; adds the depth-path mean / rotation gradients that the render backward
// left in the record; writes every dense output exactly once (zeros for culled Gaussians) and
// clears the record for the next call.
struct BwdOut {
    float *dL_dmeans, *dL_dsh, *dL_dcolors, *dL_dopacity, *dL_dscales, *dL_drot, *dL_dcov3D, *dL_dmeans2D;
};

// zeros for a culled Gaussian (the reference zero-fills all gradient tensors first, rasterize_points.cu:195-203)
__device__ __forceinline__ void bwd_zero(const int idx, const int M, const bool has_sh, const bool has_sr, const BwdOut &o,
                                         const bool sh_done) {
    const size_t i3 = 3 * (size_t)idx;
    o.dL_dmeans[i3] = 0.f; o.dL_dmeans[i3 + 1] = 0.f; o.dL_dmeans[i3 + 2] = 0.f;
    o.dL_dopacity[idx] = 0.f;
    if (has_sr) {
        o.dL_dscales[i3] = 0.f; o.dL_dscales[i3 + 1] = 0.f; o.dL_dscales[i3 + 2] = 0.f;
        reinterpret_cast<float4 *>(o.dL_drot)[idx] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (has_sh && !sh_done) {
        if (M == 16) {
            float4 *p = reinterpret_cast<float4 *>(o.dL_dsh + (size_t)idx * 48);
#pragma unroll
            for (int i = 0; i < 12; i++) p[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        } else {
            for (int i = 0; i < 3 * M; i++) o.dL_dsh[(size_t)idx * 3 * M + i] = 0.f;
        }
    }
    if (o.dL_dcolors) { o.dL_dcolors[i3] = 0.f; o.dL_dcolors[i3 + 1] = 0.f; o.dL_dcolors[i3 + 2] = 0.f; }
    if (o.dL_dcov3D)
        for (int i = 0; i < 6; i++) o.dL_dcov3D[6 * (size_t)idx + i] = 0.f;
    if (o.dL_dmeans2D) { o.dL_dmeans2D[i3] = 0.f; o.dL_dmeans2D[i3 + 1] = 0.f; o.dL_dmeans2D[i3 + 2] = 0.f; }
}

// SH part of the backward (computeColorFromSH, backward.cu:152-268): dL/dsh and the view-direction term of dL/dmean.
// Inlined, with 128 registers per thread (2 CTAs / SM): the kernel is bound by memory latency, not by occupancy --
// what pays is that all of a thread's independent loads (record, mean, scale, rotation, 12 x 16 B of SH) are in
// flight together. STORE_DSH = false is the store-free form of the pose-only backward: it returns the view-direction
// term alone and leaves dL_dsh (then NULL) untouched.
template <bool STORE_DSH = true>
__device__ __forceinline__ float3 bwd_sh(const int deg, const int idx, const int M, const float3 mean, const float3 campos,
                                      const float dcol0, const float dcol1, const float dcol2, const int flags,
                                      const float *__restrict__ shs, float *__restrict__ dL_dsh) {
    float3 dmean = make_float3(0.f, 0.f, 0.f);
    const float dcol[3] = {dcol0, dcol1, dcol2};
    const float s_m32 = campos.x, s_m33 = campos.y, s_m34 = campos.z;
    {
        float dRGB[3];
#pragma unroll
        for (int ch = 0; ch < 3; ch++) dRGB[ch] = (flags >> ch) & 1 ? 0.f : dcol[ch];
        float sh[48];
        load_sh(shs, idx, M, sh_ncoef(deg), sh);
        const float3 d0 = make_float3(mean.x - s_m32, mean.y - s_m33, mean.z - s_m34);
        const float len = sqrtf(d0.x * d0.x + d0.y * d0.y + d0.z * d0.z);
        const float x = d0.x / len, y = d0.y / len, z = d0.z / len;
        const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
        float w[16];  // dRGB/dsh_k, identical for the three channels
        w[0] = SH_C0;
        w[1] = -SH_C1 * y; w[2] = SH_C1 * z; w[3] = -SH_C1 * x;
        w[4] = SH_C2_0 * xy; w[5] = SH_C2_1 * yz; w[6] = SH_C2_2 * (2.f * zz - xx - yy); w[7] = SH_C2_3 * xz; w[8] = SH_C2_4 * (xx - yy);
        w[9] = SH_C3_0 * y * (3.f * xx - yy); w[10] = SH_C3_1 * xy * z; w[11] = SH_C3_2 * y * (4.f * zz - xx - yy);
        w[12] = SH_C3_3 * z * (2.f * zz - 3.f * xx - 3.f * yy); w[13] = SH_C3_4 * x * (4.f * zz - xx - yy);
        w[14] = SH_C3_5 * z * (xx - yy); w[15] = SH_C3_6 * x * (xx - 3.f * yy);
        const int nc = sh_ncoef(deg);
        // dL/dsh[k][ch] = w[k] * dRGB[ch] for k < (deg+1)^2, zero above; constant indices only (keeps w[] in registers)
        if constexpr (STORE_DSH) {
            if (M == 16) {
                float4 *o4 = reinterpret_cast<float4 *>(dL_dsh + (size_t)idx * 48);
#pragma unroll
                for (int i = 0; i < 12; i++) {
                    float e[4];
#pragma unroll
                    for (int t = 0; t < 4; t++) {
                        const int k = (4 * i + t) / 3, ch = (4 * i + t) % 3;
                        e[t] = (k < nc) ? w[k] * dRGB[ch] : 0.f;
                    }
                    o4[i] = make_float4(e[0], e[1], e[2], e[3]);
                }
            } else {
                float *o1 = dL_dsh + (size_t)idx * 3 * M;
#pragma unroll
                for (int e = 0; e < 48; e++)
                    if (e < 3 * M) o1[e] = (e / 3 < nc) ? w[e / 3] * dRGB[e % 3] : 0.f;
            }
        }
        float3 ddir = make_float3(0.f, 0.f, 0.f);
#pragma unroll
        for (int ch = 0; ch < 3; ch++) {
#define S(k) sh[(k) * 3 + ch]
            float rx = 0.f, ry = 0.f, rz = 0.f;
            if (deg > 0) {
                rx = -SH_C1 * S(3); ry = -SH_C1 * S(1); rz = SH_C1 * S(2);
                if (deg > 1) {
                    rx += SH_C2_0 * y * S(4) + SH_C2_2 * 2.f * -x * S(6) + SH_C2_3 * z * S(7) + SH_C2_4 * 2.f * x * S(8);
                    ry += SH_C2_0 * x * S(4) + SH_C2_1 * z * S(5) + SH_C2_2 * 2.f * -y * S(6) + SH_C2_4 * 2.f * -y * S(8);
                    rz += SH_C2_1 * y * S(5) + SH_C2_2 * 2.f * 2.f * z * S(6) + SH_C2_3 * x * S(7);
                    if (deg > 2) {
                        rx += SH_C3_0 * S(9) * 3.f * 2.f * xy + SH_C3_1 * S(10) * yz + SH_C3_2 * S(11) * -2.f * xy +
                              SH_C3_3 * S(12) * -3.f * 2.f * xz + SH_C3_4 * S(13) * (-3.f * xx + 4.f * zz - yy) +
                              SH_C3_5 * S(14) * 2.f * xz + SH_C3_6 * S(15) * 3.f * (xx - yy);
                        ry += SH_C3_0 * S(9) * 3.f * (xx - yy) + SH_C3_1 * S(10) * xz + SH_C3_2 * S(11) * (-3.f * yy + 4.f * zz - xx) +
                              SH_C3_3 * S(12) * -3.f * 2.f * yz + SH_C3_4 * S(13) * -2.f * xy + SH_C3_5 * S(14) * -2.f * yz +
                              SH_C3_6 * S(15) * -3.f * 2.f * xy;
                        rz += SH_C3_1 * S(10) * xy + SH_C3_2 * S(11) * 4.f * 2.f * yz + SH_C3_3 * S(12) * 3.f * (2.f * zz - xx - yy) +
                              SH_C3_4 * S(13) * 4.f * 2.f * xz + SH_C3_5 * S(14) * (xx - yy);
                    }
                }
            }
#undef S
            ddir.x += rx * dRGB[ch]; ddir.y += ry * dRGB[ch]; ddir.z += rz * dRGB[ch];
        }
        // dnormvdv, auxiliary.h:107-118
        const float sum2 = d0.x * d0.x + d0.y * d0.y + d0.z * d0.z;
        const float inv32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
        dmean.x += ((+sum2 - d0.x * d0.x) * ddir.x - d0.y * d0.x * ddir.y - d0.z * d0.x * ddir.z) * inv32;
        dmean.y += (-d0.x * d0.y * ddir.x + (sum2 - d0.y * d0.y) * ddir.y - d0.z * d0.y * ddir.z) * inv32;
        dmean.z += (-d0.x * d0.z * ddir.x - d0.y * d0.z * ddir.y + (sum2 - d0.z * d0.z) * ddir.z) * inv32;
    
    }
    return dmean;
}

// Camera terms of one Gaussian (CAMERA variant of bwd_visible), RTG_CAM_TERMS floats:
//   [3j+k]      j < 4, k < 3   dL/dviewmatrix[4j+k]          (view[4j+3] is never read: its gradient is 0)
//   [12+3j+c]   j < 4, c < 3   dL/dprojmatrix[4j+{0,1,3}[c]] (proj[4j+2] only feeds the cull and the unused NDC z: 0)
//   [24+i]      i < 3          dL/dcampos[i]
#define RTG_CAM_TERMS 27

// What bwd_visible produces: the per-Gaussian gradients (BWD_GAUSSIAN), those and the camera terms (BWD_CAMERA), or the
// camera terms alone (BWD_POSE: a frozen map, nothing per Gaussian is stored -- only the record is consumed and cleared).
enum BwdMode { BWD_GAUSSIAN, BWD_CAMERA, BWD_POSE };

template <int MODE>
__device__ __forceinline__ void bwd_visible(const ViewParams &vp, const int idx, const int M, const float *s_m,
                                            const float *__restrict__ means, const float *__restrict__ scales,
                                            const float *__restrict__ rots, const float *__restrict__ shs,
                                            const float *__restrict__ cov3D_precomp, const GeomState &g, float *__restrict__ rec,
                                            const BwdOut &o, float *cam) {
    constexpr bool CAMERA = MODE != BWD_GAUSSIAN;   // the camera terms go to cam[]
    constexpr bool GAUSSIANS = MODE != BWD_POSE;    // the per-Gaussian gradients are stored
    const float *vm = s_m, *pj = s_m + 16;
    const size_t i3 = 3 * (size_t)idx;
    const bool has_sh = (shs != nullptr);
    const bool has_sr = (cov3D_precomp == nullptr);
    float *dL_dmeans = o.dL_dmeans, *dL_dsh = o.dL_dsh, *dL_dcolors = o.dL_dcolors, *dL_dopacity = o.dL_dopacity,
          *dL_dscales = o.dL_dscales, *dL_drot = o.dL_drot, *dL_dcov3D = o.dL_dcov3D, *dL_dmeans2D = o.dL_dmeans2D;

    if (has_sh) prefetch_l2(shs + (size_t)idx * 3 * M, 12 * M + 64);  // consumed inside bwd_sh
    // consume + clear the gradient record
    float4 *r4 = reinterpret_cast<float4 *>(rec + (size_t)idx * RTG_REC);
    const float4 ra = r4[0], rb = r4[1], rc = r4[2], rd = r4[3];  // cleared at the very end, see below
    const float dcol[3] = {ra.x, ra.y, ra.z};
    // The compositing backward leaves the six moments of u = opacity*G*dL/dalpha (common.cuh, REC_M*). With
    // dL/dG = opacity*dL/dalpha, d = centre - pixel and the conic (a, b, c), backward.cu:960-995 reads
    //   dL/dmean2D.x = sum dL/dG * (-G dx a - G dy b) * W/2 = -(a Mx + b My) * W/2      (.y: -(c My + b Mx) * H/2)
    //   dL/dconic.{x,y,w} = sum -0.5 G d{x,x,y} d{x,y,y} dL/dG = -0.5 * {Mxx, Mxy, Myy}
    //   dL/dopacity = sum G dL/dalpha = M0 / opacity
    const float4 sp0 = g.splat[2 * (size_t)idx], sp1 = g.splat[2 * (size_t)idx + 1];
    const float m0 = ra.w, mx = rb.x, my = rb.y, mxx = rb.z, mxy = rb.w, myy = rc.x;
    const float g2x = -(sp1.x * mx + sp1.y * my) * (0.5f * (float)vp.W);
    const float g2y = -(sp1.z * my + sp1.y * mx) * (0.5f * (float)vp.H);
    const float dcon[3] = {-0.5f * mxx, -0.5f * mxy, -0.5f * myy};  // conic.x, conic.y, conic.w
    const float dopac = m0 / sp0.w;
    float3 dmean = make_float3(rc.y, rc.z, rc.w);  // depth path
    const float3 dnrm = make_float3(rd.x, rd.y, rd.z);  // depth path: dL/d(surfel normal), world space
    float4 drot = make_float4(0.f, 0.f, 0.f, 0.f);

    const float3 mean = make_float3(means[i3], means[i3 + 1], means[i3 + 2]);
    if (has_sh) {
        const float3 dsh_mean = bwd_sh<GAUSSIANS>(vp.sh_degree, idx, M, mean, make_float3(s_m[32], s_m[33], s_m[34]), dcol[0], dcol[1],
                                                  dcol[2], __float_as_int(g.rgb_flags[idx].w), shs, dL_dsh);
        dmean.x += dsh_mean.x; dmean.y += dsh_mean.y; dmean.z += dsh_mean.z;
        if constexpr (CAMERA) {  // campos enters only through the view direction mean - campos
            cam[24] = -dsh_mean.x; cam[25] = -dsh_mean.y; cam[26] = -dsh_mean.z;
        }
    }
    float3 sc = make_float3(0.f, 0.f, 0.f);
    float4 q = make_float4(1.f, 0.f, 0.f, 0.f);
    float R[3][3];
    float c6[6];
    if (has_sr) {
        sc = make_float3(scales[i3], scales[i3 + 1], scales[i3 + 2]);
        q = reinterpret_cast<const float4 *>(rots)[idx];
        quat_to_R(q, R);
        cov3d_from(sc, vp.scale_modifier, R, c6);
        if constexpr (GAUSSIANS) {
            // depth path: the surfel normal is column argmin(scale) of R(q); d(normal)/dq of propagateRotationGrad
            // (backward.cu:100-148) applied to the accumulated dL/dnormal
            const int axis = arg_min3(sc.x, sc.y, sc.z);
            const float q0 = q.x, q1 = q.y, q2 = q.z, q3 = q.w;
            const float w1 = dnrm.x, w2 = dnrm.y, w3 = dnrm.z;
            if (axis == 0) {
                drot.x = w2 * (2 * q3) + w3 * (-2 * q2);
                drot.y = w2 * (2 * q2) + w3 * (2 * q3);
                drot.z = w1 * (-4 * q2) + w2 * (2 * q1) + w3 * (-2 * q0);
                drot.w = w1 * (-4 * q3) + w2 * (2 * q0) + w3 * (2 * q1);
            } else if (axis == 1) {
                drot.x = w1 * (-2 * q3) + w3 * (2 * q1);
                drot.y = w1 * (2 * q2) + w2 * (-4 * q1) + w3 * (2 * q0);
                drot.z = w1 * (2 * q1) + w3 * (2 * q3);
                drot.w = w1 * (-2 * q0) + w2 * (-4 * q3) + w3 * (2 * q2);
            } else {
                drot.x = w1 * (2 * q2) + w2 * (-2 * q1);
                drot.y = w1 * (2 * q3) + w2 * (-2 * q0) + w3 * (-4 * q1);
                drot.z = w1 * (2 * q0) + w2 * (2 * q3) + w3 * (-4 * q2);
                drot.w = w1 * (2 * q1) + w2 * (2 * q2);
            }
        }
    } else {
#pragma unroll
        for (int i = 0; i < 6; i++) c6[i] = cov3D_precomp[6 * (size_t)idx + i];
    }

    // ---- computeCov2DCUDA, backward.cu:273-422
    float A0[3], A1[3], AV0[3], AV1[3], a, b, c, txtz, tytz;
    float3 t;
    ewa_A(xform4x3(mean, vm), vm, vp.focal_x, vp.focal_y, vp.tanfovx, vp.tanfovy, A0, A1, t, txtz, tytz);
    const float limx = 1.3f * vp.tanfovx, limy = 1.3f * vp.tanfovy;
    const float xg = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
    const float yg = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
    cov2d_from(A0, A1, c6, AV0, AV1, a, b, c);
    const float denom = a * c - b * b;
    float da = 0.f, db = 0.f, dc = 0.f;
    const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
    float dcov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (denom2inv != 0.f) {
        da = denom2inv * (-c * c * dcon[0] + 2 * b * c * dcon[1] + (denom - a * c) * dcon[2]);
        dc = denom2inv * (-a * a * dcon[2] + 2 * a * b * dcon[1] + (denom - a * c) * dcon[0]);
        db = denom2inv * 2 * (b * c * dcon[0] - (denom + 2 * b * b) * dcon[1] + a * b * dcon[2]);
        if constexpr (GAUSSIANS) {
            dcov[0] = A0[0] * A0[0] * da + A0[0] * A1[0] * db + A1[0] * A1[0] * dc;
            dcov[3] = A0[1] * A0[1] * da + A0[1] * A1[1] * db + A1[1] * A1[1] * dc;
            dcov[5] = A0[2] * A0[2] * da + A0[2] * A1[2] * db + A1[2] * A1[2] * dc;
            dcov[1] = 2 * A0[0] * A0[1] * da + (A0[0] * A1[1] + A0[1] * A1[0]) * db + 2 * A1[0] * A1[1] * dc;
            dcov[2] = 2 * A0[0] * A0[2] * da + (A0[0] * A1[2] + A0[2] * A1[0]) * db + 2 * A1[0] * A1[2] * dc;
            dcov[4] = 2 * A0[2] * A0[1] * da + (A0[1] * A1[2] + A0[2] * A1[1]) * db + 2 * A1[1] * A1[2] * dc;
        }
    }
    float dA0[3], dA1[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        dA0[k] = 2 * AV0[k] * da + AV1[k] * db;
        dA1[k] = 2 * AV1[k] * dc + AV0[k] * db;
    }
    const float dJ00 = vm[0] * dA0[0] + vm[4] * dA0[1] + vm[8] * dA0[2];
    const float dJ02 = vm[2] * dA0[0] + vm[6] * dA0[1] + vm[10] * dA0[2];
    const float dJ11 = vm[1] * dA1[0] + vm[5] * dA1[1] + vm[9] * dA1[2];
    const float dJ12 = vm[2] * dA1[0] + vm[6] * dA1[1] + vm[10] * dA1[2];
    const float tz = 1.f / t.z, tz2 = tz * tz, tz3 = tz2 * tz;
    const float hx = vp.focal_x, hy = vp.focal_y;
    const float3 dt = make_float3(xg * -hx * tz2 * dJ02, yg * -hy * tz2 * dJ12,
                                  -hx * tz2 * dJ00 - hy * tz2 * dJ11 + (2 * hx * t.x) * tz3 * dJ02 + (2 * hy * t.y) * tz3 * dJ12);
    const float3 dm_cov = xvec4x3T(dt, vm);
    dmean.x += dm_cov.x; dmean.y += dm_cov.y; dmean.z += dm_cov.z;

    // ---- projection path, backward.cu:516-533
    if constexpr (GAUSSIANS) {
        const float4 mh = xform4x4(mean, pj);
        const float mw = 1.0f / (mh.w + 0.0000001f);
        const float mul1 = (pj[0] * mean.x + pj[4] * mean.y + pj[8] * mean.z + pj[12]) * mw * mw;
        const float mul2 = (pj[1] * mean.x + pj[5] * mean.y + pj[9] * mean.z + pj[13]) * mw * mw;
        dmean.x += (pj[0] * mw - pj[3] * mul1) * g2x + (pj[1] * mw - pj[3] * mul2) * g2y;
        dmean.y += (pj[4] * mw - pj[7] * mul1) * g2x + (pj[5] * mw - pj[7] * mul2) * g2y;
        dmean.z += (pj[8] * mw - pj[11] * mul1) * g2x + (pj[9] * mw - pj[11] * mul2) * g2y;
    }

    // (SH path: bwd_sh, run first)

    // ---- cov3D -> scale, quaternion, backward.cu:426-487
    if (GAUSSIANS && has_sr) {
        const float sv[3] = {vp.scale_modifier * sc.x, vp.scale_modifier * sc.y, vp.scale_modifier * sc.z};
        float Mm[3][3], dS[3][3], dM[3][3], G[3][3];
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) Mm[i][j] = sv[i] * R[j][i];
        dS[0][0] = dcov[0]; dS[0][1] = 0.5f * dcov[1]; dS[0][2] = 0.5f * dcov[2];
        dS[1][0] = 0.5f * dcov[1]; dS[1][1] = dcov[3]; dS[1][2] = 0.5f * dcov[4];
        dS[2][0] = 0.5f * dcov[2]; dS[2][1] = 0.5f * dcov[4]; dS[2][2] = dcov[5];
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) dM[i][j] = 2.0f * (Mm[i][0] * dS[0][j] + Mm[i][1] * dS[1][j] + Mm[i][2] * dS[2][j]);
        float ds[3];
#pragma unroll
        for (int i = 0; i < 3; i++) ds[i] = R[0][i] * dM[i][0] + R[1][i] * dM[i][1] + R[2][i] * dM[i][2];
#pragma unroll
        for (int i = 0; i < 3; i++)
#pragma unroll
            for (int j = 0; j < 3; j++) G[j][i] = sv[i] * dM[i][j];
        const float r = q.x, x = q.y, y = q.z, z = q.w;
        drot.x += 2 * z * (G[1][0] - G[0][1]) + 2 * y * (G[0][2] - G[2][0]) + 2 * x * (G[2][1] - G[1][2]);
        drot.y += 2 * y * (G[0][1] + G[1][0]) + 2 * z * (G[0][2] + G[2][0]) + 2 * r * (G[2][1] - G[1][2]) - 4 * x * (G[2][2] + G[1][1]);
        drot.z += 2 * x * (G[0][1] + G[1][0]) + 2 * r * (G[0][2] - G[2][0]) + 2 * z * (G[2][1] + G[1][2]) - 4 * y * (G[2][2] + G[0][0]);
        drot.w += 2 * r * (G[1][0] - G[0][1]) + 2 * x * (G[0][2] + G[2][0]) + 2 * y * (G[2][1] + G[1][2]) - 4 * z * (G[1][1] + G[0][0]);
        dL_dscales[i3] = ds[0]; dL_dscales[i3 + 1] = ds[1]; dL_dscales[i3 + 2] = ds[2];
        reinterpret_cast<float4 *>(dL_drot)[idx] = drot;
    }

    if constexpr (CAMERA) {
        // The view matrix enters through the view-space centre p = W mean + T (the EWA J path `dt` and the depth path),
        // through W in A = J W, and through the view-space surfel normal W n. The record holds the depth path's view-space
        // gradients pulled back to world space (W^T dpc, W^T dnc, render.cu depth_hit_grad): W^-T (s_m[36..44], row
        // major) recovers them, for any invertible W.
        const float *wi = s_m + 36;
        const float3 dpc = make_float3(wi[0] * rc.y + wi[1] * rc.z + wi[2] * rc.w, wi[3] * rc.y + wi[4] * rc.z + wi[5] * rc.w,
                                       wi[6] * rc.y + wi[7] * rc.z + wi[8] * rc.w);
        const float3 dnc = make_float3(wi[0] * dnrm.x + wi[1] * dnrm.y + wi[2] * dnrm.z, wi[3] * dnrm.x + wi[4] * dnrm.y + wi[5] * dnrm.z,
                                       wi[6] * dnrm.x + wi[7] * dnrm.y + wi[8] * dnrm.z);
        const float vx = dt.x + dpc.x, vy = dt.y + dpc.y, vz = dt.z + dpc.z;
        const float J00 = hx * tz, J02 = -(hx * t.x) * tz2, J11 = hy * tz, J12 = -(hy * t.y) * tz2;
        float n[3] = {0.f, 0.f, 0.f};  // world surfel normal: column argmin(scale) of R(q); none under cov3D_precomp
        if (has_sr) {
            const int axis = arg_min3(sc.x, sc.y, sc.z);
#pragma unroll
            for (int j = 0; j < 3; j++) n[j] = axis == 0 ? R[j][0] : (axis == 1 ? R[j][1] : R[j][2]);
        }
        const float mt[3] = {mean.x, mean.y, mean.z};
#pragma unroll
        for (int j = 0; j < 3; j++) {
            cam[3 * j + 0] = mt[j] * vx + J00 * dA0[j] + n[j] * dnc.x;
            cam[3 * j + 1] = mt[j] * vy + J11 * dA1[j] + n[j] * dnc.y;
            cam[3 * j + 2] = mt[j] * vz + J02 * dA0[j] + J12 * dA1[j] + n[j] * dnc.z;
        }
        cam[9] = vx; cam[10] = vy; cam[11] = vz;
        // projection path: pixel = f(clip.xy / clip.w) with clip = P^T (mean, 1); dL/dclip from dL/dmean2D (g2x, g2y)
        const float4 mh = xform4x4(mean, pj);
        const float mw = 1.0f / (mh.w + 0.0000001f);
        const float dcx = g2x * mw, dcy = g2y * mw, dcw = -(mh.x * g2x + mh.y * g2y) * mw * mw;
#pragma unroll
        for (int j = 0; j < 3; j++) {
            cam[12 + 3 * j] = mt[j] * dcx; cam[13 + 3 * j] = mt[j] * dcy; cam[14 + 3 * j] = mt[j] * dcw;
        }
        cam[21] = dcx; cam[22] = dcy; cam[23] = dcw;
    }

    if constexpr (GAUSSIANS) {
        dL_dmeans[i3] = dmean.x; dL_dmeans[i3 + 1] = dmean.y; dL_dmeans[i3 + 2] = dmean.z;
        dL_dopacity[idx] = dopac;
        if (dL_dcolors) { dL_dcolors[i3] = dcol[0]; dL_dcolors[i3 + 1] = dcol[1]; dL_dcolors[i3 + 2] = dcol[2]; }
        if (dL_dcov3D)
#pragma unroll
            for (int i = 0; i < 6; i++) dL_dcov3D[6 * (size_t)idx + i] = dcov[i];
        if (dL_dmeans2D) { dL_dmeans2D[i3] = g2x; dL_dmeans2D[i3 + 1] = g2y; dL_dmeans2D[i3 + 2] = 0.f; }
    }
    {   // consume-and-clear: the record is cleared only now. A store to a line whose load is still in flight has to
        // wait for it, which would put one more memory round trip into every warp's life.
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        r4[0] = z4; r4[1] = z4; r4[2] = z4; r4[3] = z4;
    }
}


// Zero gradients for the culled Gaussians (the reference zero-fills every gradient tensor first,
// rasterize_points.cu:195-203). Pure streaming stores that depend on the forward only, so the C ABI runs this kernel
// on a side stream, concurrently with the compute-bound render backward.
__global__ void __launch_bounds__(256) bwd_zero_kernel(const int p_begin, const int P, const int M, const bool has_sh, const bool has_sr,
                                                       const int *__restrict__ radii, const BwdOut o) {
    const int idx = p_begin + blockIdx.x * blockDim.x + threadIdx.x;
    const bool culled = idx < P && !(radii[idx] > 0);
    const bool coop_sh = has_sh && (M == 16);
    if (coop_sh) {
        // the warp's 32 dL_dsh rows are one contiguous 6 KB block: zero the culled rows with fully coalesced stores
        const uint32_t cm = __ballot_sync(0xffffffffu, culled);
        if (cm) {
            const int lane = threadIdx.x & 31;
            float4 *blk = reinterpret_cast<float4 *>(o.dL_dsh + (size_t)(idx - lane) * 48);
#pragma unroll
            for (int k = 0; k < 12; k++) {
                const int f = lane + 32 * k, row = f / 12;
                if ((cm >> row) & 1u) blk[f] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
    }
    if (culled) bwd_zero(idx, M, has_sh, has_sr, o, coop_sh);
}

// Full backward for the compact visible list built by the forward preprocess: the register-heavy path runs with full
// warps instead of ~40 % of the lanes. PBWD_MIN_BLOCKS = 2 gives the compiler 128 registers (see bwd_sh).
#define PBWD_THREADS 256
#ifndef PBWD_MIN_BLOCKS
#define PBWD_MIN_BLOCKS 2
#endif
__global__ void __launch_bounds__(PBWD_THREADS, PBWD_MIN_BLOCKS) preprocess_bwd_kernel(const ViewParams vp, const int P, const int M,
                                                                const float *__restrict__ means, const float *__restrict__ scales,
                                                                const float *__restrict__ rots, const float *__restrict__ shs,
                                                                const float *__restrict__ cov3D_precomp, const GeomState g,
                                                                const uint32_t *__restrict__ vis_count, float *__restrict__ rec,
                                                                const BwdOut o) {
    __shared__ float s_m[40];
    if (threadIdx.x < 16) s_m[threadIdx.x] = vp.view[threadIdx.x];
    else if (threadIdx.x < 32) s_m[threadIdx.x] = vp.proj[threadIdx.x - 16];
    else if (threadIdx.x < 35) s_m[threadIdx.x] = vp.campos[threadIdx.x - 32];
    __syncthreads();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t V = *vis_count;
    if ((uint32_t)idx < V) bwd_visible<BWD_GAUSSIAN>(vp,(int)g.vis_list[idx], M, s_m, means, scales, rots, shs, cov3D_precomp, g, rec, o, nullptr);
}

// The same backward that also returns dL/d(viewmatrix, projmatrix, campos): every visible Gaussian's RTG_CAM_TERMS terms
// are summed by a warp butterfly, the block's eight warp sums in double in warp order, and the block partial goes to
// `cam_partial` (double[RTG_CAM_TERMS] per block that holds a visible Gaussian); camera_grad_final_kernel adds the block
// partials in block order. Nothing depends on timing, so identical records give a bit-identical camera gradient.
// The body of the camera and the pose-only kernel; they own the shared arrays s_m[48] and s_red.
template <int MODE>
__device__ __forceinline__ void bwd_camera_block(float *s_m, float (*s_red)[RTG_CAM_TERMS], const ViewParams &vp, const int M,
                                                 const float *__restrict__ means, const float *__restrict__ scales,
                                                 const float *__restrict__ rots, const float *__restrict__ shs,
                                                 const float *__restrict__ cov3D_precomp, const GeomState &g,
                                                 const uint32_t *__restrict__ vis_count, float *__restrict__ rec, const BwdOut &o,
                                                 double *__restrict__ cam_partial) {
    if (threadIdx.x < 16) s_m[threadIdx.x] = vp.view[threadIdx.x];
    else if (threadIdx.x < 32) s_m[threadIdx.x] = vp.proj[threadIdx.x - 16];
    else if (threadIdx.x < 35) s_m[threadIdx.x] = vp.campos[threadIdx.x - 32];
    __syncthreads();
    if (threadIdx.x == 0) {  // W^-T = cofactor matrix / det of the 3x3 block W[i][k] = view[i + 4k]
        const float *v = s_m;
#define W_(i, k) v[(i) + 4 * (k)]
        const float c00 = W_(1, 1) * W_(2, 2) - W_(1, 2) * W_(2, 1), c01 = W_(1, 2) * W_(2, 0) - W_(1, 0) * W_(2, 2),
                    c02 = W_(1, 0) * W_(2, 1) - W_(1, 1) * W_(2, 0);
        const float c10 = W_(0, 2) * W_(2, 1) - W_(0, 1) * W_(2, 2), c11 = W_(0, 0) * W_(2, 2) - W_(0, 2) * W_(2, 0),
                    c12 = W_(0, 1) * W_(2, 0) - W_(0, 0) * W_(2, 1);
        const float c20 = W_(0, 1) * W_(1, 2) - W_(0, 2) * W_(1, 1), c21 = W_(0, 2) * W_(1, 0) - W_(0, 0) * W_(1, 2),
                    c22 = W_(0, 0) * W_(1, 1) - W_(0, 1) * W_(1, 0);
        const float inv_det = 1.f / (W_(0, 0) * c00 + W_(0, 1) * c01 + W_(0, 2) * c02);
#undef W_
        const float c[9] = {c00, c01, c02, c10, c11, c12, c20, c21, c22};
#pragma unroll
        for (int i = 0; i < 9; i++) s_m[36 + i] = c[i] * inv_det;
    }
    __syncthreads();
    const uint32_t V = *vis_count;
    if ((uint32_t)blockIdx.x * blockDim.x >= V) return;  // block-uniform: no visible Gaussian, no partial
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    float cam[RTG_CAM_TERMS];
#pragma unroll
    for (int i = 0; i < RTG_CAM_TERMS; i++) cam[i] = 0.f;
    if ((uint32_t)idx < V) bwd_visible<MODE>(vp, (int)g.vis_list[idx], M, s_m, means, scales, rots, shs, cov3D_precomp, g, rec, o, cam);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < RTG_CAM_TERMS; i++) {
        float v = cam[i];
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
        if (lane == 0) s_red[w][i] = v;
    }
    __syncthreads();
    if (threadIdx.x < RTG_CAM_TERMS) {
        double acc = 0.0;
#pragma unroll
        for (int k = 0; k < PBWD_THREADS / 32; k++) acc += (double)s_red[k][threadIdx.x];
        cam_partial[(size_t)blockIdx.x * RTG_CAM_TERMS + threadIdx.x] = acc;
    }
}

__global__ void __launch_bounds__(PBWD_THREADS, PBWD_MIN_BLOCKS) preprocess_bwd_camera_kernel(const ViewParams vp, const int P, const int M,
                                                                const float *__restrict__ means, const float *__restrict__ scales,
                                                                const float *__restrict__ rots, const float *__restrict__ shs,
                                                                const float *__restrict__ cov3D_precomp, const GeomState g,
                                                                const uint32_t *__restrict__ vis_count, float *__restrict__ rec,
                                                                const BwdOut o, double *__restrict__ cam_partial) {
    __shared__ float s_m[48];
    __shared__ float s_red[PBWD_THREADS / 32][RTG_CAM_TERMS];
    bwd_camera_block<BWD_CAMERA>(s_m, s_red, vp, M, means, scales, rots, shs, cov3D_precomp, g, vis_count, rec, o, cam_partial);
}

// Pose-only backward of a frozen map: the camera kernel's terms and reduction, with no per-Gaussian store (no SH, mean,
// scale, rotation, opacity, colour or covariance gradient) -- each visible Gaussian's record is read and cleared.
__global__ void __launch_bounds__(PBWD_THREADS, PBWD_MIN_BLOCKS) preprocess_bwd_pose_kernel(const ViewParams vp, const int M,
                                                                const float *__restrict__ means, const float *__restrict__ scales,
                                                                const float *__restrict__ rots, const float *__restrict__ shs,
                                                                const float *__restrict__ cov3D_precomp, const GeomState g,
                                                                const uint32_t *__restrict__ vis_count, float *__restrict__ rec,
                                                                double *__restrict__ cam_partial) {
    __shared__ float s_m[48];
    __shared__ float s_red[PBWD_THREADS / 32][RTG_CAM_TERMS];
    const BwdOut none{};
    bwd_camera_block<BWD_POSE>(s_m, s_red, vp, M, means, scales, rots, shs, cov3D_precomp, g, vis_count, rec, none, cam_partial);
}

// One warp per camera term: a fixed-stride double sum over the block partials, a fixed butterfly, one float store. Writes
// all 35 outputs (view 16, proj 16, campos 3), the never-read entries as exact zeros.
__global__ void __launch_bounds__(RTG_CAM_TERMS * 32) camera_grad_final_kernel(const uint32_t *__restrict__ vis_count,
                                                                              const double *__restrict__ cam_partial,
                                                                              float *__restrict__ dL_dcamera) {
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t nb = (*vis_count + PBWD_THREADS - 1) / PBWD_THREADS;
    double acc = 0.0;
    for (uint32_t b = lane; b < nb; b += 32) acc += cam_partial[(size_t)b * RTG_CAM_TERMS + w];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) {
        int slot;
        if (w < 12) slot = 4 * (w / 3) + w % 3;                                    // viewmatrix
        else if (w < 24) slot = 16 + 4 * ((w - 12) / 3) + ((w - 12) % 3 == 2 ? 3 : (w - 12) % 3);  // projmatrix
        else slot = 32 + (w - 24);                                                 // campos
        dL_dcamera[slot] = (float)acc;
    }
    if (threadIdx.x < 4) dL_dcamera[4 * threadIdx.x + 3] = 0.f;
    else if (threadIdx.x < 8) dL_dcamera[16 + 4 * (threadIdx.x - 4) + 2] = 0.f;
}

// ------------------------------------------------------------------ forward-mode pose tangents
// Tangents of one visible Gaussian's splat along the six directions of a left twist xi = (rho, phi) of the pose at zero,
// W2C(xi) = exp(xi^) W2C: the view-space centre moves as dp_c = rho + phi x p_c, the view rotation as dW = [phi]x W and
// the camera centre as -W^T rho. Row `idx` of `tan` (RTG_TAN_ROW float4) holds, for direction k, [2k] = (d pixel x,
// d pixel y, d conic.x, d conic.y), [2k+1] = (d conic.z, d rgb). Not differentiated, as in the reverse-mode gradients: the
// 1.3*tanfov clamp of the EWA Jacobian (a clamped coordinate does not move), the clamped SH channels (bwd_sh zeroes them),
// the cull. The SH colour moves with the view direction only: d rgb_ch = (W g_ch) . rho with g_ch = d rgb_ch / d mean.
__global__ void __launch_bounds__(256) preprocess_tangent_kernel(const ViewParams vp, const int M, const float *__restrict__ means,
                                                                 const float *__restrict__ scales, const float *__restrict__ rots,
                                                                 const float *__restrict__ shs, const float *__restrict__ cov3D_precomp,
                                                                 const GeomState g, const uint32_t *__restrict__ vis_count,
                                                                 float4 *__restrict__ tan) {
    __shared__ float s_m[36];
    if (threadIdx.x < 16) s_m[threadIdx.x] = vp.view[threadIdx.x];
    else if (threadIdx.x < 32) s_m[threadIdx.x] = vp.proj[threadIdx.x - 16];
    else if (threadIdx.x < 35) s_m[threadIdx.x] = vp.campos[threadIdx.x - 32];
    __syncthreads();
    const uint32_t V = *vis_count;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if ((uint32_t)i >= V) return;
    const int idx = (int)g.vis_list[i];
    const float *vm = s_m, *pm = s_m + 16;
    const size_t i3 = 3 * (size_t)idx;
    const float3 mean = make_float3(means[i3], means[i3 + 1], means[i3 + 2]);

    float c6[6];
    if (cov3D_precomp == nullptr) {
        float R[3][3];
        quat_to_R(reinterpret_cast<const float4 *>(rots)[idx], R);
        cov3d_from(make_float3(scales[i3], scales[i3 + 1], scales[i3 + 2]), vp.scale_modifier, R, c6);
    } else {
#pragma unroll
        for (int k = 0; k < 6; k++) c6[k] = cov3D_precomp[6 * (size_t)idx + k];
    }
    const float3 pc = xform4x3(mean, vm);
    float A0[3], A1[3], AV0[3], AV1[3], a, b, c, txtz, tytz;
    float3 t;
    ewa_A(pc, vm, vp.focal_x, vp.focal_y, vp.tanfovx, vp.tanfovy, A0, A1, t, txtz, tytz);
    const float limx = 1.3f * vp.tanfovx, limy = 1.3f * vp.tanfovy;
    const float xg = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
    const float yg = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
    cov2d_from(A0, A1, c6, AV0, AV1, a, b, c);
    const float det_inv = 1.f / (a * c - b * b);
    const float3 conic = make_float3(c * det_inv, -b * det_inv, a * det_inv);
    const float4 clip = xform4x4(mean, pm);
    const float pw = 1.0f / (clip.w + 0.0000001f);
    const float hx = vp.focal_x, hy = vp.focal_y;
    const float tz = 1.f / t.z, tz2 = tz * tz, tz3 = tz2 * tz;
    const float J00 = hx * tz, J02 = -(hx * t.x) * tz2, J11 = hy * tz, J12 = -(hy * t.y) * tz2;

    // colour: d rgb / d rho = W g_ch (rows of W = vm[k + 4j]); none for precomputed colours
    float3 drgb_drho[3] = {make_float3(0.f, 0.f, 0.f), make_float3(0.f, 0.f, 0.f), make_float3(0.f, 0.f, 0.f)};
    if (shs != nullptr) {
        const int flags = __float_as_int(g.rgb_flags[idx].w);
        const float3 cp = make_float3(s_m[32], s_m[33], s_m[34]);
#pragma unroll
        for (int ch = 0; ch < 3; ch++) {
            const float3 gm = bwd_sh<false>(vp.sh_degree, idx, M, mean, cp, ch == 0 ? 1.f : 0.f, ch == 1 ? 1.f : 0.f,
                                            ch == 2 ? 1.f : 0.f, flags, shs, nullptr);
            drgb_drho[ch] = xvec4x3(gm, vm);
        }
    }

    float4 *row = tan + (size_t)idx * RTG_TAN_ROW;
#pragma unroll
    for (int k = 0; k < 6; k++) {
        // twist direction k: rho = e_k (k < 3) or phi = e_{k-3}
        const float3 phi = make_float3(k == 3 ? 1.f : 0.f, k == 4 ? 1.f : 0.f, k == 5 ? 1.f : 0.f);
        const float3 dp = k < 3 ? make_float3(k == 0 ? 1.f : 0.f, k == 1 ? 1.f : 0.f, k == 2 ? 1.f : 0.f)
                                : make_float3(phi.y * pc.z - phi.z * pc.y, phi.z * pc.x - phi.x * pc.z, phi.x * pc.y - phi.y * pc.x);
        // pixel centre: clip = (mean, 1) proj; the world point that moves p_c by dp is W^T dp
        const float3 dw = xvec4x3T(dp, vm);
        const float dcx = dw.x * pm[0] + dw.y * pm[4] + dw.z * pm[8], dcy = dw.x * pm[1] + dw.y * pm[5] + dw.z * pm[9];
        const float dcw = dw.x * pm[3] + dw.y * pm[7] + dw.z * pm[11];
        const float dpx = 0.5f * (float)vp.W * (dcx * pw - clip.x * dcw * pw * pw);
        const float dpy = 0.5f * (float)vp.H * (dcy * pw - clip.y * dcw * pw * pw);
        // EWA Jacobian J(t) and A = J W
        const float dtx = xg * dp.x, dty = yg * dp.y, dtz = dp.z;
        const float dJ00 = -hx * tz2 * dtz, dJ11 = -hy * tz2 * dtz;
        const float dJ02 = -hx * tz2 * dtx + 2.f * hx * t.x * tz3 * dtz, dJ12 = -hy * tz2 * dty + 2.f * hy * t.y * tz3 * dtz;
        float da = 0.f, db = 0.f, dc = 0.f;
#pragma unroll
        for (int j = 0; j < 3; j++) {
            const float3 col = make_float3(vm[4 * j], vm[4 * j + 1], vm[4 * j + 2]);  // column j of W
            const float3 dcol = make_float3(phi.y * col.z - phi.z * col.y, phi.z * col.x - phi.x * col.z, phi.x * col.y - phi.y * col.x);
            const float dA0 = dJ00 * col.x + dJ02 * col.z + J00 * dcol.x + J02 * dcol.z;
            const float dA1 = dJ11 * col.y + dJ12 * col.z + J11 * dcol.y + J12 * dcol.z;
            da += 2.f * dA0 * AV0[j];
            db += dA0 * AV1[j] + dA1 * AV0[j];
            dc += 2.f * dA1 * AV1[j];
        }
        // conic = (c, -b, a) / (a c - b^2)
        const float ddet = da * c + a * dc - 2.f * b * db;
        const float dk0 = (dc - conic.x * ddet) * det_inv, dk1 = (-db - conic.y * ddet) * det_inv, dk2 = (da - conic.z * ddet) * det_inv;
        const float dr = k < 3 ? (k == 0 ? drgb_drho[0].x : (k == 1 ? drgb_drho[0].y : drgb_drho[0].z)) : 0.f;
        const float dg = k < 3 ? (k == 0 ? drgb_drho[1].x : (k == 1 ? drgb_drho[1].y : drgb_drho[1].z)) : 0.f;
        const float dbl = k < 3 ? (k == 0 ? drgb_drho[2].x : (k == 1 ? drgb_drho[2].y : drgb_drho[2].z)) : 0.f;
        row[2 * k] = make_float4(dpx, dpy, dk0, dk1);
        row[2 * k + 1] = make_float4(dk2, dr, dg, dbl);
    }
}

// ------------------------------------------------------------------ launchers
void launch_preprocess_tangent(const ViewParams &vp, int P, int M, const float *means, const float *scales, const float *rots,
                               const float *shs, const float *cov3D_precomp, const GeomState &g, const uint32_t *vis_count,
                               float4 *tan, cudaStream_t s) {
    if (P <= 0) return;
    preprocess_tangent_kernel<<<(P + 255) / 256, 256, 0, s>>>(vp, M, means, scales, rots, shs, cov3D_precomp, g, vis_count, tan);
}

void launch_preprocess_fwd(const ViewParams &vp, int P, int M, const float *means, const float *scales, const float *rots,
                           const float *opac, const float *shs, const float *colors_precomp, const float *cov3D_precomp,
                           const int *tile_mask, const GeomState &g, int *radii, uint32_t *tile_count, uint32_t *tile_touched,
                           uint32_t *vis_count, int p_begin, cudaStream_t s) {
    if (P - p_begin <= 0) return;
    ProfScope ps(K_PREPROCESS_FWD, s);
    preprocess_fwd_kernel<<<(P - p_begin + 255) / 256, 256, 0, s>>>(vp, P, M, means, scales, rots, opac, shs, colors_precomp,
                                                                    cov3D_precomp, tile_mask, g, radii, tile_count, tile_touched,
                                                                    vis_count, p_begin);
}

void launch_mark_visible(int P, const float *means, const float *view, const float *proj, uint8_t *present, cudaStream_t s) {
    if (P <= 0) return;
    mark_visible_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, means, view, proj, present);
}

void launch_bwd_zero(int p_begin, int P, int M, bool has_sh, bool has_sr, const int *radii, float *dL_dmeans, float *dL_dsh,
                     float *dL_dcolors, float *dL_dopacity, float *dL_dscales, float *dL_drot, float *dL_dcov3D, float *dL_dmeans2D,
                     cudaStream_t s) {
    if (P - p_begin <= 0) return;
    ProfScope ps(K_BWD_ZERO, s);
    BwdOut o{dL_dmeans, dL_dsh, dL_dcolors, dL_dopacity, dL_dscales, dL_drot, dL_dcov3D, dL_dmeans2D};
    bwd_zero_kernel<<<(P - p_begin + 255) / 256, 256, 0, s>>>(p_begin, P, M, has_sh, has_sr, radii, o);
}

void launch_preprocess_bwd(const ViewParams &vp, int P, int M, const float *means, const float *scales, const float *rots,
                           const float *shs, const float *cov3D_precomp, const GeomState &g, const uint32_t *vis_count, float *rec,
                           float *dL_dmeans, float *dL_dsh, float *dL_dcolors, float *dL_dopacity, float *dL_dscales, float *dL_drot,
                           float *dL_dcov3D, float *dL_dmeans2D, cudaStream_t s) {
    if (P <= 0) return;
    ProfScope ps(K_PREPROCESS_BWD, s);
    BwdOut o{dL_dmeans, dL_dsh, dL_dcolors, dL_dopacity, dL_dscales, dL_drot, dL_dcov3D, dL_dmeans2D};
    preprocess_bwd_kernel<<<(P + PBWD_THREADS - 1) / PBWD_THREADS, PBWD_THREADS, 0, s>>>(vp, P, M, means, scales, rots, shs, cov3D_precomp, g, vis_count, rec, o);
}

size_t camera_scratch_bytes(int P) {
    const size_t blocks = P > 0 ? (size_t)(P + PBWD_THREADS - 1) / PBWD_THREADS : 1;
    return blocks * RTG_CAM_TERMS * sizeof(double);
}

void launch_preprocess_bwd_camera(const ViewParams &vp, int P, int M, const float *means, const float *scales, const float *rots,
                                  const float *shs, const float *cov3D_precomp, const GeomState &g, const uint32_t *vis_count,
                                  float *rec, float *dL_dmeans, float *dL_dsh, float *dL_dcolors, float *dL_dopacity,
                                  float *dL_dscales, float *dL_drot, float *dL_dcov3D, float *dL_dmeans2D, float *dL_dcamera,
                                  void *camera_scratch, cudaStream_t s) {
    if (P <= 0) return;
    ProfScope ps(K_PREPROCESS_BWD, s);
    BwdOut o{dL_dmeans, dL_dsh, dL_dcolors, dL_dopacity, dL_dscales, dL_drot, dL_dcov3D, dL_dmeans2D};
    double *partial = reinterpret_cast<double *>(camera_scratch);
    preprocess_bwd_camera_kernel<<<(P + PBWD_THREADS - 1) / PBWD_THREADS, PBWD_THREADS, 0, s>>>(vp, P, M, means, scales, rots, shs,
                                                                                                cov3D_precomp, g, vis_count, rec, o,
                                                                                                partial);
    camera_grad_final_kernel<<<1, RTG_CAM_TERMS * 32, 0, s>>>(vis_count, partial, dL_dcamera);
}

void launch_preprocess_bwd_pose(const ViewParams &vp, int P, int M, const float *means, const float *scales, const float *rots,
                                const float *shs, const float *cov3D_precomp, const GeomState &g, const uint32_t *vis_count,
                                float *rec, float *dL_dcamera, void *camera_scratch, cudaStream_t s) {
    if (P <= 0) return;
    ProfScope ps(K_PREPROCESS_BWD, s);
    double *partial = reinterpret_cast<double *>(camera_scratch);
    preprocess_bwd_pose_kernel<<<(P + PBWD_THREADS - 1) / PBWD_THREADS, PBWD_THREADS, 0, s>>>(vp, M, means, scales, rots, shs,
                                                                                              cov3D_precomp, g, vis_count, rec,
                                                                                              partial);
    camera_grad_final_kernel<<<1, RTG_CAM_TERMS * 32, 0, s>>>(vis_count, partial, dL_dcamera);
}

}  // namespace rtg
