// Shared definitions of the sm_90a (H100) splat kernels. Product code: never includes or calls oracle/.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

#define RTG_TILE 16
#define RTG_TILE_PIX 256
#define RTG_REC 16  // floats per Gaussian in the 2-D gradient record
#define RTG_NUM_SMS 132  // H100 SXM: sizes the grid-stride launches (a few resident CTAs per SM)

namespace rtg {

// Gradient record slots (one 64-byte line per Gaussian, filled by render-backward atomics,
// consumed and cleared by preprocess-backward).
// Slots 3..8 hold the six moments  sum u, u dx, u dy, u dx^2, u dx dy, u dy^2  of u = (opacity * G) * dL/dalpha over the
// blended (pixel, Gaussian) pairs (d = centre - pixel): every 2-D gradient of backward.cu:926-995 is a fixed linear
// combination of them (moments_to_grad2d), formed once per Gaussian by the per-Gaussian backward pass.
// Slots 9..11: depth-path dL/dmean (world); 12..14: depth-path dL/d(surfel normal) (world; the quaternion chain is applied
// by the per-Gaussian pass); 15: unused.
enum { REC_COLOR = 0, REC_M0 = 3, REC_MX = 4, REC_MY = 5, REC_MXX = 6, REC_MXY = 7, REC_MYY = 8, REC_DMEAN = 9, REC_DNORMAL = 12 };

// Forward-mode pose tangents (preprocess_tangent_kernel): float4 per Gaussian row, two per twist direction.
#define RTG_TAN_ROW 12
// Gauss-Newton terms of one residual set (colour or depth): 21 entries of J^T J (upper triangle, row by row), 6 of J^T r,
// sum r^2, pixel count. The colour set comes first, then the depth set.
#define RTG_GN_TERMS 29
#define RTG_GN_ALL (2 * RTG_GN_TERMS)
// The same with the frame's exposure (a, b) as unknowns 6 and 7 of the colour set: 36 entries of the 8x8 J^T J (upper
// triangle, row by row), 8 of J^T r, sum 2 rho(r), pixel count. The depth set keeps its RTG_GN_TERMS and follows.
#define RTG_GN_EXP_COLOR 46
#define RTG_GN_EXP_ALL (RTG_GN_EXP_COLOR + RTG_GN_TERMS)

struct ViewParams {
    int H, W, tiles_x, tiles_y;
    float tanfovx, tanfovy, focal_x, focal_y, cx, cy;
    float scale_modifier, color_sigma, opaque_thr, depth_thr, normal_thr, T_thr;
    int sh_degree, prefiltered;
    const float *view, *proj, *campos, *bg;
    int row_begin, row_end;  // tile rows the binning passes expand (a rank's band in the Gaussian-sharded forward); else all
};

// Per-Gaussian state written by the forward preprocess (16-byte records so that every gather in the render
// kernels is one LDG.128; the two halves of `splat` share a 32-byte sector).
struct GeomState {
    float4 *splat;     // [2P]  [2i]   = pixel-space centre (x, y), q_cut, opacity
                       //       [2i+1] = inverse 2-D covariance (a, b, c), log2(opacity)
    float4 *rgb_flags; // [P]   SH colour (clamped at 0) + clamp bits (int in .w)
    float4 *hit;       // [2P]  [2i]   = view-space normal (xyz), scale_max*scale_modifier
                       //       [2i+1] = view-space centre (xyz; z = the view depth of the sort key), normal axis (int in .w)
    uint32_t *vis_list; // [P]  ids of the Gaussians that survived the preprocess (count in BinState::vis_count)
};

struct BinState {
    uint32_t *tile_count;   // [T*RTG_CNT_STRIDE] instances per tile (tile t at t*RTG_CNT_STRIDE)
    uint32_t *tile_fill;    // [T*RTG_CNT_STRIDE] scatter cursors
    uint32_t *tile_touched; // [T]   1 if a Gaussian's rectangle covered the tile but the exact test culled it
    uint32_t *vis_count;    // [1]   number of entries of GeomState::vis_list
    uint32_t *tile_offset;  // [T+1] start of every tile's bucket: exclusive scan of the counts rounded up to RTG_LIST_ALIGN entries
                            //       (16-byte aligned list starts: the lists are staged with TMA bulk copies). The number of
                            //       entries of tile t is tile_count[t * RTG_CNT_STRIDE], NOT the offset difference.
    uint32_t *active;       // [T]   launch order of the tiles: longest list first, empty tiles last
    uint64_t *keys;         // [R_cap] (depth bits << 32 | gaussian id), bucketed by tile
    uint32_t *point_list;   // [R_cap] gaussian ids, per tile front-to-back
};

struct ImgState {
    uint32_t *n_contrib; // [H*W]
};

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

template <typename T>
static inline T *carve(char *&p, size_t n) {
    T *r = reinterpret_cast<T *>(p);
    p += align_up(n * sizeof(T), 256);
    return r;
}

// Words per tile in the tile histogram: counter of tile t is element t * RTG_CNT_STRIDE. L2 atomics on the same 32-byte
// sector serialise, so neighbouring tiles do not share one.
#define RTG_LIST_ALIGN 4    // tile buckets start at multiples of 4 entries (16 bytes)
#define RTG_LIST_SLACK 260  // entries readable past the end of point_list
#ifndef RTG_CNT_STRIDE
#define RTG_CNT_STRIDE 8
#endif

static inline GeomState geom_from(void *ws, size_t P, size_t *bytes = nullptr) {
    char *p = reinterpret_cast<char *>(ws);
    GeomState g;
    g.splat = carve<float4>(p, 2 * P);
    g.rgb_flags = carve<float4>(p, P);
    g.hit = carve<float4>(p, 2 * P);
    g.vis_list = carve<uint32_t>(p, P);
    if (bytes) *bytes = (size_t)(p - reinterpret_cast<char *>(ws));
    return g;
}

static inline BinState bin_from(void *ws, size_t T, size_t R_cap, size_t *bytes = nullptr) {
    char *p = reinterpret_cast<char *>(ws);
    BinState b;
    // tile_count, tile_fill, tile_touched and vis_count are adjacent: one memset clears them all. The two atomic
    // counter arrays keep RTG_CNT_STRIDE words per tile (see the define).
    b.tile_count = carve<uint32_t>(p, T * RTG_CNT_STRIDE);
    b.tile_fill = carve<uint32_t>(p, T * RTG_CNT_STRIDE);
    b.tile_touched = carve<uint32_t>(p, T);
    b.vis_count = carve<uint32_t>(p, 1);
    b.tile_offset = carve<uint32_t>(p, T + 1);
    b.active = carve<uint32_t>(p, T);
    b.keys = carve<uint64_t>(p, R_cap);
    b.point_list = carve<uint32_t>(p, R_cap + RTG_LIST_SLACK);  // a bulk copy of the last list may read up to one batch past it
    if (bytes) *bytes = (size_t)(p - reinterpret_cast<char *>(ws));
    return b;
}

static inline ImgState img_from(void *ws, size_t N, size_t *bytes = nullptr) {
    char *p = reinterpret_cast<char *>(ws);
    ImgState s;
    s.n_contrib = carve<uint32_t>(p, N);
    if (bytes) *bytes = (size_t)(p - reinterpret_cast<char *>(ws));
    return s;
}

// ------------------------------------------------------------------ device helpers
#ifdef __CUDACC__
__device__ __forceinline__ float3 xform4x3(const float3 p, const float *m) {
    return make_float3(m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12], m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
                       m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14]);
}
__device__ __forceinline__ float4 xform4x4(const float3 p, const float *m) {
    return make_float4(m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12], m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
                       m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14], m[3] * p.x + m[7] * p.y + m[11] * p.z + m[15]);
}
__device__ __forceinline__ float3 xvec4x3(const float3 p, const float *m) {
    return make_float3(m[0] * p.x + m[4] * p.y + m[8] * p.z, m[1] * p.x + m[5] * p.y + m[9] * p.z,
                       m[2] * p.x + m[6] * p.y + m[10] * p.z);
}
__device__ __forceinline__ float3 xvec4x3T(const float3 p, const float *m) {
    return make_float3(m[0] * p.x + m[1] * p.y + m[2] * p.z, m[4] * p.x + m[5] * p.y + m[6] * p.z,
                       m[8] * p.x + m[9] * p.y + m[10] * p.z);
}
__device__ __forceinline__ int arg_max3(float a, float b, float c) { return (a >= b && a >= c) ? 0 : ((b >= a && b >= c) ? 1 : 2); }
__device__ __forceinline__ int arg_min3(float a, float b, float c) { return (a <= b && a <= c) ? 0 : ((b <= a && b <= c) ? 1 : 2); }

// ------------------------------------------------------------------ the frame residual's pixel rules
// One definition for the L1 / mapping losses (loss.cu) and the Gauss-Newton tracker's residuals (render.cu).
// Channel c of the measured colour at pixel p of an N-pixel frame: gt_color is (H,W,3) if channels_last else (3,H,W).
__device__ __forceinline__ float frame_color(const float *gt_color, int channels_last, int N, int p, int c) {
    return channels_last ? gt_color[3 * (size_t)p + c] : gt_color[(size_t)c * N + p];
}
// A depth pixel of the loss: the render hit a Gaussian, the frame measured a depth, and the signed error
// err = depth - gt_depth is below depth_error_max.
__device__ __forceinline__ bool frame_depth_pixel(int hit, float gt_depth, float err, float depth_error_max) {
    return hit != -1 && gt_depth > 0.f && err < depth_error_max;
}

// Tile rectangle touched by a splat of integer radius r centred at p (same rounding as the
// reference's getRect, auxiliary.h:49-57).
__device__ __forceinline__ void tile_rect(const float2 p, int r, int gx, int gy, int &x0, int &y0, int &x1, int &y1) {
    x0 = min(gx, max(0, (int)((p.x - r) / RTG_TILE)));
    y0 = min(gy, max(0, (int)((p.y - r) / RTG_TILE)));
    x1 = min(gx, max(0, (int)((p.x + r + RTG_TILE - 1) / RTG_TILE)));
    y1 = min(gy, max(0, (int)((p.y + r + RTG_TILE - 1) / RTG_TILE)));
}

// Unit view ray through integer pixel (px,py) (ndc2ray, forward.cu:92-100).
__device__ __forceinline__ float3 pixel_ray(int px, int py, float fx, float fy, float cx, float cy) {
    float3 ray = make_float3(((float)px - cx) / fx, ((float)py - cy) / fy, 1.0f);
    float n = 1.0f / sqrtf(ray.x * ray.x + ray.y * ray.y + ray.z * ray.z);
    ray.x *= n; ray.y *= n; ray.z *= n;
    return ray;
}

// Standard rotation matrix rows from a quaternion used as given (w,x,y,z); not re-normalised
// (forward.cu:57,211).
__device__ __forceinline__ void quat_to_R(const float4 q, float R[3][3]) {
    const float r = q.x, x = q.y, y = q.z, z = q.w;
    R[0][0] = 1.f - 2.f * (y * y + z * z); R[0][1] = 2.f * (x * y - r * z); R[0][2] = 2.f * (x * z + r * y);
    R[1][0] = 2.f * (x * y + r * z); R[1][1] = 1.f - 2.f * (x * x + z * z); R[1][2] = 2.f * (y * z - r * x);
    R[2][0] = 2.f * (x * z - r * y); R[2][1] = 2.f * (y * z + r * x); R[2][2] = 1.f - 2.f * (x * x + y * y);
}

// Margin (in units of the exponent q = -power) added to ln(255*opacity): a (pixel, Gaussian) pair whose q
// exceeds q_cut has alpha < (1/255)*exp(-Q_MARGIN), i.e. fails the reference's `alpha < 1/255` test with a
// 1 % safety factor against fp32 rounding, so skipping it can never change an output.
#define RTG_Q_MARGIN 0.01f

// q_cut of a Gaussian: pairs with q > q_cut contribute nothing. Negative => contributes nowhere.
__device__ __forceinline__ float q_cutoff(float opacity) {
    const float t = 255.0f * opacity;
    return (t < 0.999f) ? -1.0f : (logf(fmaxf(t, 0.999f)) + RTG_Q_MARGIN);
}

// True if q(d) = 0.5*(a dx^2 + c dy^2) + b dx dy > q_cut for EVERY point of the pixel rectangle
// [x0,x1] x [y0,y1] (d = centre - pixel), i.e. the Gaussian cannot pass the alpha cut-off anywhere in it.
// Exact minimisation of the convex quadratic over the rectangle: with the centre outside, the minimum lies on a
// boundary edge that faces the centre (q decreases along the segment from any point of a far edge towards the
// centre), so two line minimisations suffice: along the vertical line through the rectangle point nearest to the
// centre and along the horizontal one. When the centre is inside the x (y) range, that line passes through the
// nearest point itself and its minimum is dominated by the other line's; with the centre inside the rectangle
// both give 0. Written with explicit round-to-nearest intrinsics so that every kernel that evaluates it
// (histogram, scatter, per-warp masks) takes bit-identical decisions.
// `nb_c` = -b/c and `nb_a` = -b/a (cut_slopes) are per-Gaussian: callers that test many rectangles pass them in.
__device__ __forceinline__ float2 cut_slopes(float a, float b, float c) { return make_float2(__fdiv_rn(-b, c), __fdiv_rn(-b, a)); }
__device__ __forceinline__ float cut_q(float a, float b, float c, float dx, float dy) {
    return __fmaf_rn(__fmul_rn(b, dx), dy, __fmul_rn(0.5f, __fmaf_rn(__fmul_rn(a, dx), dx, __fmul_rn(__fmul_rn(c, dy), dy))));
}
__device__ __forceinline__ bool rect_below_cutoff(float gx, float gy, float a, float b, float c, float q_cut, float nb_c, float nb_a,
                                                  float x0, float x1, float y0, float y1) {
    if (q_cut < 0.f) return true;
    if (!(a > 0.f) || !(c > 0.f)) return false;  // not a proper conic: keep the reference's behaviour
    const float dxl = __fsub_rn(gx, x1), dxh = __fsub_rn(gx, x0), dyl = __fsub_rn(gy, y1), dyh = __fsub_rn(gy, y0);
    const float dxn = fminf(dxh, fmaxf(dxl, 0.f)), dyn = fminf(dyh, fmaxf(dyl, 0.f));  // rectangle point nearest to the centre
    const float qx = cut_q(a, b, c, dxn, fminf(dyh, fmaxf(dyl, __fmul_rn(nb_c, dxn))));
    const float qy = cut_q(a, b, c, fminf(dxh, fmaxf(dxl, __fmul_rn(nb_a, dyn))), dyn);
    // the line minimiser is exact up to rounding; shave a relative 1e-4 so that rounding can only keep, never cull
    return __fmul_rn(fminf(qx, qy), 0.9999f) > q_cut;
}

// ------------------------------------------------------------------ alpha of a (pixel, Gaussian) pair
// The reference evaluates  alpha = min(0.99, opacity * expf(power))  with the accurate expf (forward.cu:764-771,
// backward.cu:940-945). Here the fast path is one FFMA and one MUFU.EX2:  au = 2^(power*log2(e) + log2(opacity)),
// relative error <= 1e-6 (half an ulp of an exponent of magnitude <= 8 twice, plus the 2^-22 of ex2.approx). The only
// discontinuous decision taken on alpha for every pair is `alpha < 1/255`: when the fast value lands within RTG_ALPHA_BAND
// (relative, 4x the error bound) of that threshold the reference expression is evaluated instead, so the decision is the
// reference's. Forward and backward call the same function on the same inputs: they agree bit for bit on which pairs
// blend and with what alpha. `au` is the unclamped opacity * G (the backward's moments are sums of au * dL/dalpha).
#define RTG_ALPHA_BAND 4e-6f
#define RTG_LOG2E 1.4426950408889634f
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// the reference's exponent, same expression in every kernel (forward.cu:757, backward.cu:936)
__device__ __forceinline__ float pair_power(float a, float b, float c, float dx, float dy) {
    return -0.5f * (a * dx * dx + c * dy * dy) - b * dx * dy;
}
// returns false if the pair is skipped (alpha < 1/255)
__device__ __forceinline__ bool pair_alpha(float power, float log2o, float opacity, float &alpha, float &au) {
    au = ex2_approx(fmaf(power, RTG_LOG2E, log2o));
    alpha = fminf(0.99f, au);
    if (alpha < (1.0f / 255.0f) * (1.0f - RTG_ALPHA_BAND)) return false;
    if (alpha < (1.0f / 255.0f) * (1.0f + RTG_ALPHA_BAND)) {  // a few pairs per frame
        au = opacity * expf(power);
        alpha = fminf(0.99f, au);
        return alpha >= 1.0f / 255.0f;
    }
    return true;
}

// The same function split in two for callers that evaluate several pairs per step without a branch in between:
// pair_alpha_fast never branches; when it reports `band` the caller must run pair_alpha_exact on that pair.
__device__ __forceinline__ bool pair_alpha_fast(float power, float log2o, float &alpha, float &au, bool &band) {
    au = ex2_approx(fmaf(power, RTG_LOG2E, log2o));
    alpha = fminf(0.99f, au);
    band = alpha < (1.0f / 255.0f) * (1.0f + RTG_ALPHA_BAND);
    return alpha >= (1.0f / 255.0f) * (1.0f - RTG_ALPHA_BAND);
}
static __device__ __noinline__ float pair_au_exact(float power, float opacity) { return opacity * expf(power); }  // out of line: rare
__device__ __forceinline__ bool pair_alpha_exact(float power, float opacity, float &alpha, float &au) {
    au = pair_au_exact(power, opacity);
    alpha = fminf(0.99f, au);
    return alpha >= 1.0f / 255.0f;
}

// Warp-cooperative expansion of per-lane tile rectangles into (owner lane, tile) pairs, so that the 32 lanes of a
// warp share the pairs evenly instead of each lane looping over its own rectangle. `excl` / `rect` are the warp's
// 32-entry shared arrays: exclusive prefix of the pair counts, and x0 | y0 << 10 | width << 20.
__device__ __forceinline__ uint32_t pack_rect(int x0, int y0, int w) { return (uint32_t)x0 | ((uint32_t)y0 << 10) | ((uint32_t)w << 20); }
// (column, row) of pair `local` inside a rectangle `rw` tiles wide, without an integer division: (local + 0.5) / rw is at
// least 0.5 / rw away from an integer and the quotients are below 2^10, so the fp32 product truncates to the exact row.
__device__ __forceinline__ void rect_cell(uint32_t local, uint32_t rw, int &dx, int &dy) {
    dy = __float2int_rz(((float)local + 0.5f) * __frcp_rn((float)rw));
    dx = (int)local - dy * (int)rw;
}
__device__ __forceinline__ int warp_incl_scan(int v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += n;
    }
    return v;
}
__device__ __forceinline__ int pair_owner(const uint32_t *excl, uint32_t k) {
    int o = 0;
#pragma unroll
    for (int step = 16; step > 0; step >>= 1)
        if (excl[o + step] <= k) o += step;  // o + step <= 31 always
    return o;
}

// L2 prefetch of the 128-byte line(s) holding [p, p + bytes): issued as soon as an index is known, long before the
// data is consumed, to overlap the DRAM latency with the arithmetic in between
__device__ __forceinline__ void prefetch_l2(const void *p, int bytes) {
    const char *c = reinterpret_cast<const char *>(p);
    for (int o = 0; o < bytes; o += 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(c + o));
}

// 16-byte asynchronous global -> shared copy (LDGSTS, bypassing L1) and its group fences
__device__ __forceinline__ void cp_async16(uint32_t smem_dst, const void *gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_dst), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
// ---- TMA bulk copy (cp.async.bulk, SASS: UBLKCP) of a contiguous global range into shared memory, completion on an
// mbarrier. Source address, shared destination and byte count must be multiples of 16.
__device__ __forceinline__ void mbar_init(uint32_t mbar, uint32_t arrivals) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(arrivals) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t mbar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t smem_dst, const void *gsrc, uint32_t bytes, uint32_t mbar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_dst), "l"(gsrc),
                 "r"(bytes), "r"(mbar)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t mbar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done)
                     : "r"(mbar), "r"(parity)
                     : "memory");
    } while (!done);
}
__device__ __forceinline__ void sts32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }

// explicit shared-state-space accesses with a precomputed 32-bit base (keeps address arithmetic out of the loops)
__device__ __forceinline__ uint32_t smem_addr(const void *p) {
    uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
    // opaque to the optimiser: otherwise ptxas re-materialises the address (S2R SR_CgaCtaId + LEA chain) at every use
    asm volatile("" : "+r"(a));
    return a;
}
__device__ __forceinline__ float4 lds128(uint32_t a) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t a) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}

// ------------------------------------------------------------------ 6-dof solve and SE(3) update (double)
// Solve (JtJ + trace*damping*I) xi = -Jtr (the reference inverts the same matrix with torch.inverse on the CPU,
// SLAM/icp.py:248-257,313-333). The damped normal matrix is symmetric positive definite: Cholesky without pivoting, fully
// unrolled (registers only), double precision. Returns false if a pivot is not positive (degenerate view: pose unchanged).
// Shared by the ICP iterations (icp.cu) and the render-based Gauss-Newton pose step (render.cu).
__device__ __forceinline__ bool solve6(const double A[6][6], const double bvec[6], double x[6]) {
    double Lm[6][6];
    bool ok = true;
#pragma unroll
    for (int j = 0; j < 6; j++) {
        double d = A[j][j];
#pragma unroll
        for (int k = 0; k < j; k++) d -= Lm[j][k] * Lm[j][k];
        ok = ok && (d > 0.0);
        const double ljj = sqrt(fmax(d, 1e-300));
        Lm[j][j] = ljj;
        const double inv = 1.0 / ljj;
#pragma unroll
        for (int i = j + 1; i < 6; i++) {
            double v = A[i][j];
#pragma unroll
            for (int k = 0; k < j; k++) v -= Lm[i][k] * Lm[j][k];
            Lm[i][j] = v * inv;
        }
    }
    double y[6];
#pragma unroll
    for (int i = 0; i < 6; i++) {
        double v = bvec[i];
#pragma unroll
        for (int k = 0; k < i; k++) v -= Lm[i][k] * y[k];
        y[i] = v / Lm[i][i];
    }
#pragma unroll
    for (int i = 5; i >= 0; i--) {
        double v = y[i];
#pragma unroll
        for (int k = i + 1; k < 6; k++) v -= Lm[k][i] * x[k];
        x[i] = v / Lm[i][i];
    }
    return ok;
}

// solve6's Cholesky for an N x N symmetric positive definite system (the 8 unknowns of the pose step with exposure). A
// separate function: solve6 and the kernels that call it keep their code.
template <int N>
__device__ __forceinline__ bool solve_n(const double A[N][N], const double bvec[N], double x[N]) {
    double Lm[N][N];
    bool ok = true;
#pragma unroll
    for (int j = 0; j < N; j++) {
        double d = A[j][j];
#pragma unroll
        for (int k = 0; k < j; k++) d -= Lm[j][k] * Lm[j][k];
        ok = ok && (d > 0.0);
        const double ljj = sqrt(fmax(d, 1e-300));
        Lm[j][j] = ljj;
        const double inv = 1.0 / ljj;
#pragma unroll
        for (int i = j + 1; i < N; i++) {
            double v = A[i][j];
#pragma unroll
            for (int k = 0; k < j; k++) v -= Lm[i][k] * Lm[j][k];
            Lm[i][j] = v * inv;
        }
    }
    double y[N];
#pragma unroll
    for (int i = 0; i < N; i++) {
        double v = bvec[i];
#pragma unroll
        for (int k = 0; k < i; k++) v -= Lm[i][k] * y[k];
        y[i] = v / Lm[i][i];
    }
#pragma unroll
    for (int i = N - 1; i >= 0; i--) {
        double v = y[i];
#pragma unroll
        for (int k = i + 1; k < N; k++) v -= Lm[k][i] * x[k];
        x[i] = v / Lm[i][i];
    }
    return ok;
}

// exp(xi^) of a twist xi = (rho, phi) as its top 3x4 block: [[R, V rho]], R = I + a K + b K^2, V = I + b K + c K^2,
// K = [phi]x (closed form; Taylor series for small angles).
__device__ __forceinline__ void se3_exp_twist(const double xi[6], double E[3][4]) {
    const double p0 = xi[3], p1 = xi[4], p2 = xi[5];
    const double th2 = p0 * p0 + p1 * p1 + p2 * p2;
    double a, b, c;
    if (th2 < 1e-4) {  // Taylor series; the first omitted terms are below 1e-16
        a = 1.0 - th2 / 6.0 * (1.0 - th2 / 20.0);
        b = 0.5 - th2 / 24.0 * (1.0 - th2 / 30.0);
        c = 1.0 / 6.0 - th2 / 120.0 * (1.0 - th2 / 42.0);
    } else {
        const double th = sqrt(th2), sn = sin(th), cs = cos(th);
        a = sn / th;
        b = (1.0 - cs) / th2;
        c = (th - sn) / (th2 * th);
    }
    const double K[3][3] = {{0.0, -p2, p1}, {p2, 0.0, -p0}, {-p1, p0, 0.0}};
#pragma unroll
    for (int i = 0; i < 3; i++) {
        double Vr = 0.0;
#pragma unroll
        for (int j = 0; j < 3; j++) {
            const double K2 = K[i][0] * K[0][j] + K[i][1] * K[1][j] + K[i][2] * K[2][j];
            const double I = i == j ? 1.0 : 0.0;
            E[i][j] = I + a * K[i][j] + b * K2;
            Vr += (I + b * K[i][j] + c * K2) * xi[j];
        }
        E[i][3] = Vr;
    }
}

// W2C <- exp(xi^) W2C for the double pose T (row-major in `pose`), then the three arrays the rasterizer reads:
// viewmatrix = W2C^T, projmatrix = viewmatrix @ projection, campos = -R^T t.
__device__ __forceinline__ void pose_left_update(const double E[3][4], const double T[4][4], double *pose, const float *projection,
                                                 float *viewmatrix, float *projmatrix, float *campos) {
    double N[4][4];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) N[i][j] = E[i][0] * T[0][j] + E[i][1] * T[1][j] + E[i][2] * T[2][j] + (j == 3 ? E[i][3] : 0.0);
#pragma unroll
    for (int j = 0; j < 4; j++) N[3][j] = T[3][j];

#pragma unroll
    for (int i = 0; i < 16; i++) pose[i] = N[i / 4][i % 4];
#pragma unroll
    for (int r = 0; r < 4; r++)
#pragma unroll
        for (int q = 0; q < 4; q++) {
            viewmatrix[4 * r + q] = (float)N[q][r];
            double pm = 0.0;
#pragma unroll
            for (int k = 0; k < 4; k++) pm += N[k][r] * (double)projection[4 * k + q];
            projmatrix[4 * r + q] = (float)pm;
        }
#pragma unroll
    for (int i = 0; i < 3; i++) campos[i] = (float)-(N[0][i] * N[0][3] + N[1][i] * N[1][3] + N[2][i] * N[2][3]);
}
#endif

// One Adam update, operation for operation as torch.optim.Adam's single-tensor path (bias-corrected, no weight decay).
__device__ __forceinline__ void adam_one(float &p, const float g, float &m, float &v, const float lr_over_bc1, const float beta1,
                                         const float beta2, const float eps, const float bc2_sqrt) {
    m = m + (g - m) * (1.f - beta1);           // exp_avg.lerp_(grad, 1 - beta1)
    v = v * beta2 + (1.f - beta2) * g * g;     // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
    const float denom = sqrtf(v) / bc2_sqrt + eps;
    p = p - lr_over_bc1 * (m / denom);         // param.addcdiv_(exp_avg, denom, value=-step_size)
}


// The same update with one-instruction square root and reciprocal (MUFU.SQRT / MUFU.RCP, about 1 ulp each; denormal
// inputs kept) and the division by sqrt(1 - beta2^t) folded into a multiplication: ~12 instructions instead of ~40.
// The step differs from adam_one's by a few 1e-7 RELATIVE TO THE STEP (lr-sized), far below the 1e-5 parameter
// tolerance; used where the per-element instruction count, not HBM, would otherwise bound the kernel (mapstep.cu).
__device__ __forceinline__ void adam_one_fast(float &p, const float g, float &m, float &v, const float lr_over_bc1, const float beta1,
                                              const float beta2, const float eps, const float inv_bc2_sqrt) {
    m = fmaf(g - m, 1.f - beta1, m);
    v = fmaf(v, beta2, (1.f - beta2) * g * g);
    float sq, rc;
    asm("sqrt.approx.f32 %0, %1;" : "=f"(sq) : "f"(v));
    asm("rcp.approx.f32 %0, %1;" : "=f"(rc) : "f"(fmaf(sq, inv_bc2_sqrt, eps)));
    p = fmaf(-lr_over_bc1 * m, rc, p);
}

}  // namespace rtg
