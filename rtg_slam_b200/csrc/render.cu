// Tile compositing: forward colour + opaque-surfel depth, and the per-Gaussian backward.
//
// Semantics follow renderCUDA_withMask (RAST/cuda_rasterizer/forward.cu:636-861) and
// renderCUDA_flat (backward.cu:808-1066). What differs by design:
//  * one CTA per tile over a device-resident tile table (no host-side tile compaction); CTAs of
//    empty / masked-out tiles write the reference's initial values (rasterize_points.cu:79-87);
//  * a warp owns an 8x4 pixel patch (the reference: a 16x2 strip). While a batch of 256 list entries is
//    staged into shared memory, the staging thread also computes, once per entry, which of the 8 patches the
//    Gaussian can reach above the alpha cut-off (exact convex minimisation, common.cuh). Each warp then walks
//    only its own entries (ballot + find-first-set), so entries that every lane would skip are never visited;
//  * per pair, alpha comes from one FFMA + one MUFU.EX2 (pair_alpha, common.cuh); the reference's accurate
//    expression is evaluated only when that value is within 4e-6 (relative) of the 1/255 cut, and for the one entry
//    per pixel that decides the opaque hit when it is that close to opaque_threshold;
//  * the plane hit is evaluated lazily, only for the first entry with alpha >= opaque_threshold, from a
//    per-Gaussian view-space record (the reference recomputes quaternion->normal and two 4x3 transforms from
//    global memory for every blended pair, forward.cu:778-790);
//  * the backward walks only the prefix of the tile list that some pixel of the CTA actually blended. Per pair it
//    accumulates three colour terms and six moments of u = opacity*G*dL/dalpha (sum u, u dx, u dy, u dx^2, u dx dy,
//    u dy^2): all 2-D gradients of backward.cu:960-995 are linear in them, so the per-pair work is 9 multiply-adds
//    and the conversion happens once per Gaussian in the per-Gaussian pass. The colour behind a pair enters only
//    through its dot product with dL/dC, so the replay keeps one scalar instead of three channels. The two pixels of a
//    lane are blended without a branch (a skipped pair is a pair with alpha = 0, which leaves the replay state
//    bit-identical). The 9 sums are reduced across the warp with a transposing butterfly (12 shuffles instead of 45)
//    and added with one 9-lane atomic per (warp, Gaussian), instead of 9 atomics per (pixel, Gaussian) pair;
//  * hit_normal_c / hit_point_c are not stored per pixel: they are functions of the hit Gaussian and the pixel
//    ray and are recomputed bit-identically in the backward.
#include "common.cuh"
#include "kernels.h"
#include "prof.h"
#include "../../include/rtg_splat_b200.h"

namespace rtg {

#define BATCH 256
#define FULL 0xffffffffu

// power > 0 is skipped by the reference. (A second cheap rejection, power < -q_cut, is optional: RTG_QCUT_PRETEST.)
#ifdef RTG_QCUT_PRETEST
#define RTG_FWD_PRETEST(power, q_cut) ((power) <= 0.0f && (power) >= -(q_cut))
#else
#define RTG_FWD_PRETEST(power, q_cut) ((power) <= 0.0f)
#endif

// warp w of the CTA owns the 8x4 patch (w & 1, w >> 1) of the 16x16 tile
__device__ __forceinline__ void pixel_of(const ViewParams &vp, int tile, int &px, int &py, bool &inside) {
    const int tx = tile % vp.tiles_x, ty = tile / vp.tiles_x;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    px = tx * RTG_TILE + (w & 1) * 8 + (lane & 7);
    py = ty * RTG_TILE + (w >> 1) * 4 + (lane >> 3);
    inside = px < vp.W && py < vp.H;
}

// bit k set <=> the Gaussian can pass the alpha cut-off somewhere in patch k of the tile at (tx0, ty0)
__device__ __forceinline__ uint32_t patch_mask(const float4 s0, const float4 s1, float tx0, float ty0) {
    uint32_t m = 0;
    const float2 nb = cut_slopes(s1.x, s1.y, s1.z);
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const float x0 = tx0 + (float)((k & 1) * 8), y0 = ty0 + (float)((k >> 1) * 4);
        if (!rect_below_cutoff(s0.x, s0.y, s1.x, s1.y, s1.z, s0.z, nb.x, nb.y, x0, x0 + 7.f, y0, y0 + 3.f)) m |= (1u << k);
    }
    return m;
}

// Plane / centre depth of the first opaque entry (forward.cu:778-809).
__device__ __forceinline__ float surfel_depth(const float4 h0, const float4 h1, const float3 ray, float center_depth,
                                              float depth_thr, float normal_thr) {
    const float3 nc = make_float3(h0.x, h0.y, h0.z);
    const float3 pc = make_float3(h1.x, h1.y, h1.z);
    const float num = pc.x * nc.x + pc.y * nc.y + pc.z * nc.z;
    const float den = ray.x * nc.x + ray.y * nc.y + ray.z * nc.z;
    // the reference adds a double literal here: (float / (float + 1e-8)) is evaluated in double
    const float t = (float)((double)num / ((double)den + 1e-8));
    const float hz = t * ray.z;
    const float angle_distance = fabsf(den);
    const float depth_distance = fabsf(hz - pc.z);
    const bool plane = (depth_distance <= h0.w * depth_thr) && (angle_distance >= normal_thr);
    return plane ? hz : center_depth;
}

__global__ void __launch_bounds__(256) render_fwd_kernel(const ViewParams vp, const GeomState g, const BinState b, ImgState img,
                                                         const int *__restrict__ counters, float *__restrict__ out_color,
                                                         float *__restrict__ out_depth, int *__restrict__ out_hit_color,
                                                         int *__restrict__ out_hit_depth, float *__restrict__ out_hcw,
                                                         float *__restrict__ out_hdw, float *__restrict__ out_T) {
    // two staging buffers: batch i+1 is gathered with cp.async while batch i is composited
    __shared__ float4 s_rec[2 * BATCH * 3];  // one 48-byte record per staged entry: splat half 0, half 1, colour
    __shared__ int s_id[2 * BATCH];
    __shared__ uint32_t s_mask[2 * BATCH];
    // the tile's id list arrives by TMA: one bulk copy (cp.async.bulk -> UBLKCP) per batch of 256 ids, issued by one thread
    // two batches ahead, completion on an mbarrier per buffer
    __shared__ __align__(16) int s_list[2 * BATCH];
    __shared__ __align__(8) unsigned long long s_mbar[2];

    const int tile = (int)b.active[blockIdx.x];  // longest lists first
    int px, py;
    bool inside;
    pixel_of(vp, tile, px, py, inside);
    const int pix_id = vp.W * py + px;
    const int N = vp.H * vp.W;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;

    const bool overflow = counters[2] != 0;
    const uint32_t start = b.tile_offset[tile];  // multiple of RTG_LIST_ALIGN entries: 16-byte aligned list
    const int n = overflow ? 0 : (int)b.tile_count[(size_t)tile * RTG_CNT_STRIDE];
    if (n == 0) {
        if (inside) {
            // never-rendered tile: the wrapper's initial values (hit maps 0). A tile whose entries were all culled by
            // the exact test is still "rendered" by the reference: hit maps -1, colour = background.
            const bool touched = !overflow && b.tile_touched[tile] != 0u;
            out_color[pix_id] = touched ? __ldg(vp.bg) : 0.f;
            out_color[N + pix_id] = touched ? __ldg(vp.bg + 1) : 0.f;
            out_color[2 * N + pix_id] = touched ? __ldg(vp.bg + 2) : 0.f;
            out_depth[pix_id] = 0.f;
            out_hit_color[pix_id] = touched ? -1 : 0;
            out_hit_depth[pix_id] = touched ? -1 : 0;
            out_hcw[pix_id] = 0.f; out_hdw[pix_id] = 0.f;
            out_T[pix_id] = 1.f;
            img.n_contrib[pix_id] = 0u;
        }
        return;
    }

    // A pixel that is finished (or outside the image) moves infinitely far away: every later entry then fails the
    // `power >= -q_cut` test (power = -inf or NaN), so the visit loop needs no separate `done` branch.
    const float FAR = 1e30f;
    float pfx = inside ? (float)px : FAR;
    const float pfy = (float)py;
    const float3 ray = pixel_ray(px, py, vp.focal_x, vp.focal_y, vp.cx, vp.cy);
    const float tx0 = (float)((tile % vp.tiles_x) * RTG_TILE), ty0 = (float)((tile / vp.tiles_x) * RTG_TILE);
    // interleaved records: one address computation per visit instead of three (quarter-warp 128-bit accesses at a
    // 48-byte stride fall into distinct banks)
    const uint32_t a_rec = smem_addr(s_rec), a_id = smem_addr(s_id), a_mask = smem_addr(s_mask);
#define REC_S0(k) (a_rec + (k) * 48)
#define REC_S1(k) (a_rec + (k) * 48 + 16)
#define REC_RGB(k) (a_rec + (k) * 48 + 32)
    const float T_thr = vp.T_thr;
    // lower edge of the band around opaque_threshold; becomes +inf once the pixel has its opaque hit (`!hit &&` folded
    // into the compare)
    float opaque_lo = vp.opaque_thr * (1.0f - RTG_ALPHA_BAND);
    bool done = !inside;

    float T = 1.0f, end_T = 1.0f;
    uint32_t last_contributor = 0;
    float C0 = 0.f, C1 = 0.f, C2 = 0.f;
    float depth_ = 0.f;
    bool hit = false;
    int hit_id = -1, hit_color_id = -1;
    float cw_max = -1.f, hit_dw = 0.f;  // arg-max colour weight (forward.cu:725-726: max starts at -1, the output at 0)

    const int rounds = (n + BATCH - 1) / BATCH;
    // stage(batch, id): asynchronous gather of one list entry per thread into buffer (batch & 1)
    auto stage = [&](const int batch, const int id) {
        const uint32_t slot = (uint32_t)((batch & 1) * BATCH + threadIdx.x);
        cp_async16(REC_S0(slot), g.splat + 2 * (size_t)id);
        cp_async16(REC_S1(slot), g.splat + 2 * (size_t)id + 1);
        cp_async16(REC_RGB(slot), g.rgb_flags + id);
        sts32(a_id + slot * 4, (uint32_t)id);
    };
    const uint32_t a_list = smem_addr(s_list), a_mbar = smem_addr(s_mbar);
    const int n_pad = (n + (RTG_LIST_ALIGN - 1)) & ~(RTG_LIST_ALIGN - 1);
    // ids of batch k -> buffer k & 1 (its mbarrier completes for the (k >> 1)-th time); thread 0 only
    auto issue_ids = [&](const int k) {
        const int ents = min(BATCH, n_pad - k * BATCH);
        if (ents > 0) {
            mbar_expect_tx(a_mbar + (k & 1) * 8, (uint32_t)ents * 4u);
            bulk_g2s(a_list + (uint32_t)((k & 1) * BATCH) * 4u, b.point_list + start + (size_t)k * BATCH, (uint32_t)ents * 4u,
                     a_mbar + (k & 1) * 8);
        }
    };
    auto wait_ids = [&](const int k) { mbar_wait(a_mbar + (k & 1) * 8, (uint32_t)((k >> 1) & 1)); };
    if (threadIdx.x == 0) {
        mbar_init(a_mbar, 1);
        mbar_init(a_mbar + 8, 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) { issue_ids(0); issue_ids(1); }
    wait_ids(0);
    if ((int)threadIdx.x < n) stage(0, (int)lds32(a_list + threadIdx.x * 4));
    cp_async_commit();
    __syncthreads();                                          // buffer 0 has been read by everybody
    if (threadIdx.x == 0) issue_ids(2);
    int consumed = 1;                                         // id batches < consumed have been read
    for (int i = 0; i < rounds; i++) {
        cp_async_wait_all();                                   // this thread's copies of batch i have landed
        if (__syncthreads_count(done) == BATCH) break;          // everybody's have; and batch i-1 is fully consumed
        const uint32_t boff = (uint32_t)((i & 1) * BATCH);
        if (i * BATCH + (int)threadIdx.x < n) {
            const float4 s0 = lds128(REC_S0(boff + threadIdx.x)), s1 = lds128(REC_S1(boff + threadIdx.x));
            sts32(a_mask + (boff + threadIdx.x) * 4, patch_mask(s0, s1, tx0, ty0));
        }
        if ((i + 1) * BATCH < n) {                              // gathers of batch i + 1 overlap the compositing of batch i
            wait_ids(i + 1);
            consumed = i + 2;
            if ((i + 1) * BATCH + (int)threadIdx.x < n)
                stage(i + 1, (int)lds32(a_list + (uint32_t)(((i + 1) & 1) * BATCH + threadIdx.x) * 4));
        }
        cp_async_commit();
        __syncthreads();
        if (threadIdx.x == 0) issue_ids(i + 3);                // its buffer, (i + 1) & 1, has been read by everybody
        const int cnt = min(BATCH, n - i * BATCH);
        if (__all_sync(FULL, done)) continue;  // warp-uniform
        const int chunks = (cnt + 31) >> 5;
        // batch-local bookkeeping, resolved once per batch instead of once per blend: slot of the last colour
        // contribution and of the current arg-max weight (-1 = none in this batch)
        int j_last = -1, j_cmax = -1;
        for (int c = 0; c < chunks; c++) {
            const int e = (c << 5) + lane;
            const uint32_t mm = (e < cnt) ? lds32(a_mask + (boff + e) * 4) : 0u;
            uint32_t bits = __ballot_sync(FULL, (mm >> w) & 1u);
            // everything after the alpha of a (pixel, entry) pair (forward.cu:772-838)
            auto blend = [&](const int j, const uint32_t jb, const float4 s0, const float power, const float alpha) {
                if (alpha >= opaque_lo) {  // at most a few entries per pixel (opaque_lo = +inf after the hit)
                    // inside the band the decision is taken on the reference's own expression
                    const float a_dec = (alpha < vp.opaque_thr * (1.0f + RTG_ALPHA_BAND)) ? fminf(0.99f, s0.w * expf(power)) : alpha;
                    if (a_dec >= vp.opaque_thr) {
                        const int id = (int)lds32(a_id + jb * 4);
                        const float4 h0 = __ldg(g.hit + 2 * (size_t)id), h1 = __ldg(g.hit + 2 * (size_t)id + 1);
                        depth_ = surfel_depth(h0, h1, ray, h1.z, vp.depth_thr, vp.normal_thr);
                        hit_id = id;
                        hit_dw = alpha * T;
                        hit = true;
                        opaque_lo = __int_as_float(0x7f800000);
                    }
                }
                const float test_T = T * (1.f - alpha);
                if (test_T < T_thr) {
                    // no colour is added any more; the pixel keeps scanning until it has an opaque hit
                    if (hit) { done = true; pfx = FAR; }
                    else T = test_T;
                } else {
                    const float cw = alpha * T;
                    const float4 col = lds128(REC_RGB(jb));
                    C0 += col.x * cw; C1 += col.y * cw; C2 += col.z * cw;
                    if (cw > cw_max) { cw_max = cw; j_cmax = j; }
                    j_last = j;
                    end_T = test_T;
                    T = test_T;
                }
            };
#ifndef RTG_FWD_ILP1  // -DRTG_FWD_ILP1: one entry per iteration (a longer dependent chain per entry)
            // two entries in flight per warp: their records, exponents and alphas are independent (only the blend is
            // sequential in T), which halves the dependent latency chain of a warp's walk -- what bounds a heavy tile
            while (bits) {
                const int ja = (c << 5) + __ffs(bits) - 1;
                bits &= bits - 1;
                const bool two = bits != 0u;  // warp-uniform
                const int jc = two ? (c << 5) + __ffs(bits) - 1 : ja;
                if (two) bits &= bits - 1;
                const uint32_t jba = boff + (uint32_t)ja, jbc = boff + (uint32_t)jc;
                const float4 s0a = lds128(REC_S0(jba)), s1a = lds128(REC_S1(jba));
                const float4 s0c = lds128(REC_S0(jbc)), s1c = lds128(REC_S1(jbc));
                const float pwa = pair_power(s1a.x, s1a.y, s1a.z, s0a.x - pfx, s0a.y - pfy);
                const float pwc = pair_power(s1c.x, s1c.y, s1c.z, s0c.x - pfx, s0c.y - pfy);
                float ala, aua, alc, auc;
                bool banda, bandc;
                bool oka = pair_alpha_fast(pwa, s1a.w, ala, aua, banda) && RTG_FWD_PRETEST(pwa, s0a.z);
                bool okc = pair_alpha_fast(pwc, s1c.w, alc, auc, bandc) && RTG_FWD_PRETEST(pwc, s0c.z) && two;
                if ((banda && oka) || (bandc && okc)) {  // a few pairs per frame
                    if (banda && oka) oka = pair_alpha_exact(pwa, s0a.w, ala, aua);
                    if (bandc && okc) okc = pair_alpha_exact(pwc, s0c.w, alc, auc);
                }
                if (oka) blend(ja, jba, s0a, pwa, ala);
                if (okc && !done) blend(jc, jbc, s0c, pwc, alc);  // the pixel may have finished on the first entry
            }
#else
            while (bits) {
                const int j = (c << 5) + __ffs(bits) - 1;
                const uint32_t jb = boff + (uint32_t)j;
                bits &= bits - 1;
                const float4 s0 = lds128(REC_S0(jb)), s1 = lds128(REC_S1(jb));
                const float dx = s0.x - pfx, dy = s0.y - pfy;
                const float power = pair_power(s1.x, s1.y, s1.z, dx, dy);
                // power > 0: skipped by the reference; finished pixel: power = -inf or NaN, never passes
                float alpha, au;
                if (RTG_FWD_PRETEST(power, s0.z) && pair_alpha(power, s1.w, s0.w, alpha, au)) blend(j, jb, s0, power, alpha);
            }
#endif
            if (__all_sync(FULL, done)) break;  // checked once per 32 entries: a finished warp skips visits cheaply
        }
        if (j_last >= 0) last_contributor = (uint32_t)(i * BATCH + j_last + 1);
        if (j_cmax >= 0) hit_color_id = (int)lds32(a_id + (boff + (uint32_t)j_cmax) * 4);
    }

    // bulk copies that were issued for batches this CTA no longer needs must land before its shared memory is released
    for (int k = consumed; k <= consumed + 1; k++)
        if (k * BATCH < n_pad) wait_ids(k);

    if (inside) {
        const float bg0 = __ldg(vp.bg), bg1 = __ldg(vp.bg + 1), bg2 = __ldg(vp.bg + 2);
        out_color[pix_id] = C0 + T * bg0;
        out_color[N + pix_id] = C1 + T * bg1;
        out_color[2 * N + pix_id] = C2 + T * bg2;
        out_depth[pix_id] = depth_;
        out_hit_depth[pix_id] = hit_id;
        out_hit_color[pix_id] = hit_color_id;
        out_hcw[pix_id] = fmaxf(cw_max, 0.f);
        out_hdw[pix_id] = hit_dw;
        out_T[pix_id] = end_T;
        img.n_contrib[pix_id] = last_contributor;
    }
}

// ------------------------------------------------------------------ backward

// Sum 9 per-lane values across the warp with a transposing butterfly (12 shuffles instead of 45): at every step a
// lane keeps one half of its values and trades the other half with its partner. Afterwards value k's total sits in
// lane kLaneOfValue[k]; `slot_of_lane` returns the value index a lane ends up holding (or -1).
//   step xor 16: lanes with bit4 = 0 keep v0..v4, bit4 = 1 keep v5..v8            (5 shuffles)
//   step xor  8: of those, bit3 = 0 keeps the first ceil(half), bit3 = 1 the rest   (3 shuffles)
//   step xor  4: (2 shuffles), step xor 2: (1 shuffle), step xor 1: plain add        (1 shuffle)
__device__ __forceinline__ float warp_reduce9(const float v[9], const int lane) {
    const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4, b1 = lane & 2;
    // after xor 16: a[0..4]; lanes b4=0: sums of v0..v4, lanes b4=1: sums of v5..v8 (a[4] unused there)
    float a[5];
#pragma unroll
    for (int i = 0; i < 5; i++) {
        const float hi_val = (i < 4) ? v[5 + i] : 0.f;
        const float send = b4 ? v[i] : hi_val;
        const float keep = b4 ? hi_val : v[i];
        a[i] = keep + __shfl_xor_sync(FULL, send, 16);
    }
    // after xor 8: c[0..2]; b3=0 keeps a0..a2, b3=1 keeps a3..a4
    float c[3];
#pragma unroll
    for (int i = 0; i < 3; i++) {
        const float hi_val = (i < 2) ? a[3 + i] : 0.f;
        const float send = b3 ? a[i] : hi_val;
        const float keep = b3 ? hi_val : a[i];
        c[i] = keep + __shfl_xor_sync(FULL, send, 8);
    }
    // after xor 4: d[0..1]; b2=0 keeps c0..c1, b2=1 keeps c2
    float d[2];
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const float hi_val = (i < 1) ? c[2 + i] : 0.f;
        const float send = b2 ? c[i] : hi_val;
        const float keep = b2 ? hi_val : c[i];
        d[i] = keep + __shfl_xor_sync(FULL, send, 4);
    }
    // after xor 2: b1=0 keeps d0, b1=1 keeps d1
    float e;
    {
        const float send = b1 ? d[0] : d[1];
        const float keep = b1 ? d[1] : d[0];
        e = keep + __shfl_xor_sync(FULL, send, 2);
    }
    e += __shfl_xor_sync(FULL, e, 1);
    return e;
}

// value index held by a lane after warp_reduce9 (-1: padding)
__device__ __forceinline__ int reduce9_slot(const int lane) {
    const int b4 = (lane >> 4) & 1, b3 = (lane >> 3) & 1, b2 = (lane >> 2) & 1, b1 = (lane >> 1) & 1;
    // level sizes: 9 -> (5 | 4) -> (3 | 2) -> (2 | 1) -> (1 | 1)
    int base = b4 ? 5 : 0, cnt = b4 ? 4 : 5;           // values [base, base+cnt)
    {   // xor 8: first 3 stay with b3=0, rest with b3=1
        const int lo = 3;
        if (b3) { base += lo; cnt -= lo; } else { cnt = min(cnt, lo); }
    }
    {   // xor 4: first 2 stay with b2=0, rest with b2=1
        const int lo = 2;
        if (b2) { base += lo; cnt -= lo; } else { cnt = min(cnt, lo); }
    }
    {   // xor 2: first 1 stays with b1=0, rest with b1=1
        const int lo = 1;
        if (b1) { base += lo; cnt -= lo; } else { cnt = min(cnt, lo); }
    }
    return cnt > 0 ? base : -1;
}

// Depth-hit gradient of one pixel (backward.cu:997-1065): the first opaque Gaussian of the pixel receives the gradient
// of the rendered depth w.r.t. its centre and, on the plane branch, w.r.t. its surfel normal. The normal is a column of
// R(q): the chain to the quaternion (propagateRotationGrad, backward.cu:100-148) is linear in dL/dnormal, so the
// world-space dL/dnormal is what accumulates in the record and the per-Gaussian pass, which owns the quaternion, applies
// the chain once per Gaussian. This kernel therefore reads no parameter array, only the forward's records.
__device__ __forceinline__ void depth_hit_grad(const ViewParams &vp, const GeomState &g, const int *__restrict__ hit_image,
                                               const float *__restrict__ dL_ddepth, float *__restrict__ rec, const int px,
                                               const int py, const int pix_id, const bool inside) {
    if (inside) {
        const int gid = hit_image[pix_id];
        if (gid >= 0) {
            const float3 ray = pixel_ray(px, py, vp.focal_x, vp.focal_y, vp.cx, vp.cy);
            const float4 h0 = __ldg(g.hit + 2 * (size_t)gid), h1 = __ldg(g.hit + 2 * (size_t)gid + 1);
            const float3 nc = make_float3(h0.x, h0.y, h0.z);
            const float3 pc = make_float3(h1.x, h1.y, h1.z);
            // max(scales) without the scale modifier (backward.cu:1009); the record holds scale_max * scale_modifier
            // (exact for scale_modifier == 1, the only value the reference's callers pass, SLAM/render.py:41)
            const float scale_max = h0.w / vp.scale_modifier;
            const float num = pc.x * nc.x + pc.y * nc.y + pc.z * nc.z;
            const float ndotr = nc.x * ray.x + nc.y * ray.y + nc.z * ray.z;
            const float t = (float)((double)num / ((double)ndotr + 1e-8));
            const float hz = t * ray.z;
            const float angle_distance = fabsf(ndotr);
            const float depth_distance = fabsf(hz - pc.z);
            const float dL_ddi = dL_ddepth[pix_id];
            const float *vm = vp.view;
            float *r = rec + (size_t)gid * RTG_REC;
            if (depth_distance <= vp.depth_thr * scale_max && angle_distance >= vp.normal_thr) {
                const float nr = (float)((double)ndotr + 1e-8);
                const float inv_nr = 1.f / nr, inv_nr2 = inv_nr * inv_nr;
                const float np_ = num;
                const float dpx = ray.z * nc.x * inv_nr, dpy = ray.z * nc.y * inv_nr, dpz = ray.z * nc.z * inv_nr;
                const float v0 = __ldg(vm + 0), v1 = __ldg(vm + 1), v2 = __ldg(vm + 2), v4 = __ldg(vm + 4), v5 = __ldg(vm + 5),
                            v6 = __ldg(vm + 6), v8 = __ldg(vm + 8), v9 = __ldg(vm + 9), v10 = __ldg(vm + 10);
                atomicAdd(r + REC_DMEAN + 0, dL_ddi * (dpx * v0 + dpy * v1 + dpz * v2));
                atomicAdd(r + REC_DMEAN + 1, dL_ddi * (dpx * v4 + dpy * v5 + dpz * v6));
                atomicAdd(r + REC_DMEAN + 2, dL_ddi * (dpx * v8 + dpy * v9 + dpz * v10));
                const float n1 = ray.z * (nr * pc.x - np_ * ray.x) * inv_nr2;
                const float n2 = ray.z * (nr * pc.y - np_ * ray.y) * inv_nr2;
                const float n3 = ray.z * (nr * pc.z - np_ * ray.z) * inv_nr2;
                // view-space dL/dnormal -> world space
                atomicAdd(r + REC_DNORMAL + 0, dL_ddi * (n1 * v0 + n2 * v1 + n3 * v2));
                atomicAdd(r + REC_DNORMAL + 1, dL_ddi * (n1 * v4 + n2 * v5 + n3 * v6));
                atomicAdd(r + REC_DNORMAL + 2, dL_ddi * (n1 * v8 + n2 * v9 + n3 * v10));
            } else {
                atomicAdd(r + REC_DMEAN + 0, dL_ddi * __ldg(vm + 2));
                atomicAdd(r + REC_DMEAN + 1, dL_ddi * __ldg(vm + 6));
                atomicAdd(r + REC_DMEAN + 2, dL_ddi * __ldg(vm + 10));
            }
        }
    }
}

// Two entries at once: the xor-16 step hands entry 0's nine values to lanes 0-15 and entry 1's to lanes 16-31 (9
// shuffles), then each half-warp runs the transposing butterfly on its nine values (5 + 3 + 2 + 1): 20 shuffles for two
// entries instead of 24, and every total ends in exactly one lane (reduce18_slot).
__device__ __forceinline__ float warp_reduce18(const float v0[9], const float v1[9], const int lane) {
    const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4, b1 = lane & 2, b0 = lane & 1;
    float a[9];
#pragma unroll
    for (int i = 0; i < 9; i++) a[i] = (b4 ? v1[i] : v0[i]) + __shfl_xor_sync(FULL, b4 ? v0[i] : v1[i], 16);
    float c[5];  // b3 = 0 keeps a0..a4, b3 = 1 keeps a5..a8
#pragma unroll
    for (int i = 0; i < 5; i++) {
        const float hi_val = (i < 4) ? a[5 + i] : 0.f;
        c[i] = (b3 ? hi_val : a[i]) + __shfl_xor_sync(FULL, b3 ? a[i] : hi_val, 8);
    }
    float d[3];  // b2 = 0 keeps c0..c2, b2 = 1 keeps c3..c4
#pragma unroll
    for (int i = 0; i < 3; i++) {
        const float hi_val = (i < 2) ? c[3 + i] : 0.f;
        d[i] = (b2 ? hi_val : c[i]) + __shfl_xor_sync(FULL, b2 ? c[i] : hi_val, 4);
    }
    float e[2];  // b1 = 0 keeps d0..d1, b1 = 1 keeps d2
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const float hi_val = (i < 1) ? d[2 + i] : 0.f;
        e[i] = (b1 ? hi_val : d[i]) + __shfl_xor_sync(FULL, b1 ? d[i] : hi_val, 2);
    }
    return (b0 ? e[1] : e[0]) + __shfl_xor_sync(FULL, b0 ? e[0] : e[1], 1);  // b0 = 0 keeps e0, b0 = 1 keeps e1
}

// value index (of the lane's own entry, lane >> 4) held by a lane after warp_reduce18 (-1: padding)
__device__ __forceinline__ int reduce18_slot(const int lane) {
    int base = 0, cnt = 9;
    const int lo_of[4] = {5, 3, 2, 1};
#pragma unroll
    for (int s = 0; s < 4; s++) {
        const int lo = lo_of[s];
        if ((lane >> (3 - s)) & 1) { base += lo; cnt -= lo; } else { cnt = min(cnt, lo); }
    }
    return cnt > 0 ? base : -1;
}

// Per-pixel replay state of the backward. The reference keeps, per channel, the colour accumulated behind the current
// entry (accum_rec) and the previous entry's colour (backward.cu:947-958); both enter dL/dalpha only through their dot
// product with the pixel's dL/dC, so one scalar each is kept: A = accum_rec . dLp,  L = last_color . dLp.
struct BwdPix {
    float T, A, L, last_alpha, dLp0, dLp1, dLp2, bgw, pyf;
    uint32_t last_contributor;
};

// One (pixel, Gaussian) pair of the back-to-front replay (backward.cu:926-995), branch-free: a pair that does not blend
// is passed with alpha = au = 0, which leaves T (x 1/(1-0)), A (the recurrence's next step multiplies L by last_alpha = 0)
// and every sum bit-identical to skipping it. Adds the three colour terms and the six moments to v[].
__device__ __forceinline__ void bwd_blend(BwdPix &p, const float alpha, const float au, const float4 col, const float dx,
                                          const float dy, float v[9]) {
    float inv_1ma;  // 1 - alpha is in [0.01, 1]: the bare MUFU.RCP (no range fix-up code) is exact to 1 ulp there
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv_1ma) : "f"(1.f - alpha));
    p.T = p.T * inv_1ma;
    const float w = alpha * p.T;
    const float D = col.x * p.dLp0 + col.y * p.dLp1 + col.z * p.dLp2;
    p.A = fmaf(p.last_alpha, p.L - p.A, p.A);  // accum_rec = last_alpha * last_color + (1 - last_alpha) * accum_rec
    p.L = D;
    p.last_alpha = alpha;
    float dL_dalpha = (D - p.A) * p.T;
    dL_dalpha = fmaf(-p.bgw, inv_1ma, dL_dalpha);  // background term, bgw = T_final * (bg . dLp)  (backward.cu:976-981)
    v[REC_COLOR + 0] = fmaf(w, p.dLp0, v[REC_COLOR + 0]);
    v[REC_COLOR + 1] = fmaf(w, p.dLp1, v[REC_COLOR + 1]);
    v[REC_COLOR + 2] = fmaf(w, p.dLp2, v[REC_COLOR + 2]);
    const float u = au * dL_dalpha;
    const float ux = u * dx, uy = u * dy;
    v[REC_M0] += u;
    v[REC_MX] += ux;
    v[REC_MY] += uy;
    v[REC_MXX] = fmaf(ux, dx, v[REC_MXX]);
    v[REC_MXY] = fmaf(ux, dy, v[REC_MXY]);
    v[REC_MYY] = fmaf(uy, dy, v[REC_MYY]);
}

// Backward compositing. 128 threads per tile; a warp owns an 8x8 pixel patch and every lane two vertically adjacent
// pixels, so the per-entry costs that do not depend on the pixel (list walk, shared-memory fetch of the splat, the
// warp reduction and the atomic) are paid once per 64 pixels.
#define BWD_THREADS 128
// no minimum-blocks bound by default (BWD_MIN_BLOCKS selects one): the register cap a bound implies can cost more than
// the occupancy it buys
#ifndef BWD_MIN_BLOCKS
#define BWD_MIN_BLOCKS 0
#endif
#if BWD_MIN_BLOCKS > 0
#define BWD_BOUNDS __launch_bounds__(BWD_THREADS, BWD_MIN_BLOCKS)
#else
#define BWD_BOUNDS __launch_bounds__(BWD_THREADS)
#endif
// TGRAD: the pixel's dL/dT_map (`dL_dT`, (H, W)) is differentiated too. T_map = prod (1 - alpha) over the pairs the replay
// walks, so dT_map/dalpha = -T_map / (1 - alpha): the same form as the background term, to whose weight it is added
// (bgw = T_final * (bg . dLp + dL_dT)). A pixel is then skipped only if both its colour and its T gradient are zero.
template <bool TGRAD>
__global__ void BWD_BOUNDS render_bwd_kernel(const ViewParams vp, const GeomState g, const BinState b,
                                                               const ImgState img, const int *__restrict__ counters,
                                                               const float *__restrict__ final_T,
                                                               const int *__restrict__ hit_image, const float *__restrict__ dL_dcolor,
                                                               const float *__restrict__ dL_ddepth, float *__restrict__ rec,
                                                               const float *__restrict__ dL_dT) {
    __shared__ float4 s_s0[BATCH];
    __shared__ float4 s_s1[BATCH];
    __shared__ float4 s_rgb[BATCH];
    __shared__ int s_id[BATCH];
    __shared__ uint32_t s_mask[BATCH];
    __shared__ uint32_t s_max[4];
    // the blended prefix of the tile's id list arrives by TMA, back to front: one bulk copy per round of 256 ids (plus
    // up to 3 + 3 ids of alignment padding), issued by one thread two rounds ahead, completion on an mbarrier per buffer
    __shared__ __align__(16) int s_list[2 * (BATCH + 8)];
    __shared__ __align__(8) unsigned long long s_mbar[2];
#ifdef RTG_BWD_SMEM_REDUCE
    __shared__ float4 s_red[4][9 * 8];
    const uint32_t a_red = smem_addr(s_red[threadIdx.x >> 5]);
#endif

    if (counters[2]) return;
    if ((int)blockIdx.x >= counters[1]) return;  // empty tiles sit at the end of the launch order
    const int tile = (int)b.active[blockIdx.x];
    const uint32_t start = b.tile_offset[tile];  // multiple of RTG_LIST_ALIGN entries: 16-byte aligned list
    const int n = (int)b.tile_count[(size_t)tile * RTG_CNT_STRIDE];
    if (n == 0) return;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int tx = tile % vp.tiles_x, ty = tile / vp.tiles_x;
    // warp w: patch (w & 1, w >> 1) of 8x8 pixels; lane: column lane & 7, rows 2*(lane >> 3) and 2*(lane >> 3) + 1
    const int px = tx * RTG_TILE + (w & 1) * 8 + (lane & 7);
    const int pyA = ty * RTG_TILE + (w >> 1) * 8 + 2 * (lane >> 3), pyB = pyA + 1;
    const bool insA = px < vp.W && pyA < vp.H, insB = px < vp.W && pyB < vp.H;
    const int pidA = vp.W * pyA + px, pidB = vp.W * pyB + px;
    const int N = vp.H * vp.W;
    const float pxf = (float)px;
    const float tx0 = (float)(tx * RTG_TILE), ty0 = (float)(ty * RTG_TILE);
    const uint32_t a_s0 = smem_addr(s_s0), a_s1 = smem_addr(s_s1), a_rgb = smem_addr(s_rgb), a_id = smem_addr(s_id),
                   a_mask = smem_addr(s_mask);

    BwdPix A, B;
    {
        const float bg0 = __ldg(vp.bg), bg1 = __ldg(vp.bg + 1), bg2 = __ldg(vp.bg + 2);
        A.T = insA ? final_T[pidA] : 0.f; B.T = insB ? final_T[pidB] : 0.f;
        A.last_contributor = insA ? img.n_contrib[pidA] : 0u; B.last_contributor = insB ? img.n_contrib[pidB] : 0u;
        A.dLp0 = insA ? dL_dcolor[pidA] : 0.f; A.dLp1 = insA ? dL_dcolor[N + pidA] : 0.f; A.dLp2 = insA ? dL_dcolor[2 * N + pidA] : 0.f;
        B.dLp0 = insB ? dL_dcolor[pidB] : 0.f; B.dLp1 = insB ? dL_dcolor[N + pidB] : 0.f; B.dLp2 = insB ? dL_dcolor[2 * N + pidB] : 0.f;
        if constexpr (TGRAD) {
            const float dTA = insA ? dL_dT[pidA] : 0.f, dTB = insB ? dL_dT[pidB] : 0.f;
            A.bgw = A.T * ((bg0 * A.dLp0 + bg1 * A.dLp1 + bg2 * A.dLp2) + dTA);
            B.bgw = B.T * ((bg0 * B.dLp0 + bg1 * B.dLp1 + bg2 * B.dLp2) + dTB);
            // the replay of a pixel with a T gradient is kept (and so enters the tile's walked prefix m below)
            if (A.dLp0 == 0.f && A.dLp1 == 0.f && A.dLp2 == 0.f && dTA == 0.f) A.last_contributor = 0u;
            if (B.dLp0 == 0.f && B.dLp1 == 0.f && B.dLp2 == 0.f && dTB == 0.f) B.last_contributor = 0u;
        } else {
            A.bgw = A.T * (bg0 * A.dLp0 + bg1 * A.dLp1 + bg2 * A.dLp2); B.bgw = B.T * (bg0 * B.dLp0 + bg1 * B.dLp1 + bg2 * B.dLp2);
            // a pixel whose upstream colour gradient is exactly zero (outside the render mask of the mapping loss) adds
            // exact zeros to every colour-path term: skip its replay altogether
            if (A.dLp0 == 0.f && A.dLp1 == 0.f && A.dLp2 == 0.f) A.last_contributor = 0u;
            if (B.dLp0 == 0.f && B.dLp1 == 0.f && B.dLp2 == 0.f) B.last_contributor = 0u;
        }
        A.A = A.L = A.last_alpha = 0.f;
        B.A = B.L = B.last_alpha = 0.f;
        A.pyf = (float)pyA; B.pyf = (float)pyB;
    }

    // only the first `m` entries of the list were blended by some pixel of this tile
    uint32_t wmax = max(A.last_contributor, B.last_contributor);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(FULL, wmax, o));
    if (lane == 0) s_max[w] = wmax;
    __syncthreads();
    const uint32_t m = max(max(s_max[0], s_max[1]), max(s_max[2], s_max[3]));

#ifndef RTG_BWD_ILP1
    const int my_slot = reduce18_slot(lane);
#else
    const int my_slot = (lane & 1) ? -1 : reduce9_slot(lane);  // lanes 2k and 2k+1 hold the same total: one of them adds it
#endif

    const int rounds = ((int)m + BATCH - 1) / BATCH;
    const uint32_t a_list = smem_addr(s_list), a_mbar = smem_addr(s_mbar);
    // round k covers the list positions [lo, hi) = [max(0, m - (k+1)*256), m - k*256); the copy starts at lo rounded down to
    // a 16-byte boundary and ends at hi rounded up to one (the extra ids are never read)
    auto round_lo = [&](const int k) { return max(0, (int)m - (k + 1) * BATCH); };
    auto issue_ids = [&](const int k) {  // thread 0 only
        if (k < rounds) {
            const int lo = round_lo(k) & ~(RTG_LIST_ALIGN - 1), hi = ((int)m - k * BATCH + (RTG_LIST_ALIGN - 1)) & ~(RTG_LIST_ALIGN - 1);
            mbar_expect_tx(a_mbar + (k & 1) * 8, (uint32_t)(hi - lo) * 4u);
            bulk_g2s(a_list + (uint32_t)((k & 1) * (BATCH + 8)) * 4u, b.point_list + start + lo, (uint32_t)(hi - lo) * 4u, a_mbar + (k & 1) * 8);
        }
    };
    if (threadIdx.x == 0) {
        mbar_init(a_mbar, 1);
        mbar_init(a_mbar + 8, 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) { issue_ids(0); issue_ids(1); }
    for (int i = 0; i < rounds; i++) {
        __syncthreads();
        mbar_wait(a_mbar + (i & 1) * 8, (uint32_t)((i >> 1) & 1));
        const int lo_al = round_lo(i) & ~(RTG_LIST_ALIGN - 1);
        for (int q = threadIdx.x; q < BATCH; q += BWD_THREADS) {
            const int progress = i * BATCH + q;  // position from the back of the prefix
            if (progress < (int)m) {
                const int id = (int)lds32(a_list + (uint32_t)((i & 1) * (BATCH + 8) + ((int)m - 1 - progress - lo_al)) * 4u);
                const float4 s0 = __ldg(g.splat + 2 * (size_t)id), s1 = __ldg(g.splat + 2 * (size_t)id + 1);
                s_id[q] = id;
                s_s0[q] = s0;
                s_s1[q] = s1;
                s_rgb[q] = __ldg(g.rgb_flags + id);
                uint32_t mk = 0;
                const float2 nb = cut_slopes(s1.x, s1.y, s1.z);
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    const float x0 = tx0 + (float)((k & 1) * 8), y0 = ty0 + (float)((k >> 1) * 8);
                    if (!rect_below_cutoff(s0.x, s0.y, s1.x, s1.y, s1.z, s0.z, nb.x, nb.y, x0, x0 + 7.f, y0, y0 + 7.f)) mk |= (1u << k);
                }
                s_mask[q] = mk;
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) issue_ids(i + 2);  // buffer i & 1 has been read by everybody
        const int cnt = min(BATCH, (int)m - i * BATCH);
        const int chunks = (cnt + 31) >> 5;
        for (int c = 0; c < chunks; c++) {
            const int e = (c << 5) + lane;
            // list position of staged entry e (== the reference's `contributor`); entries at or beyond the warp's
            // deepest blended position are skipped by every lane
            const uint32_t pos_e = m - 1 - (uint32_t)(i * BATCH + e);
            const uint32_t mm = (e < cnt && pos_e < wmax) ? lds32(a_mask + e * 4) : 0u;
            uint32_t bits = __ballot_sync(FULL, (mm >> w) & 1u);
#ifndef RTG_BWD_ILP1  // -DRTG_BWD_ILP1: one entry per iteration (a longer dependent chain per entry)
            // two entries per iteration: the four alphas are independent, only the blends are sequential per pixel
            while (bits) {
                const int j0 = (c << 5) + __ffs(bits) - 1;
                bits &= bits - 1;
                const bool two = bits != 0u;  // warp-uniform
                const int j1 = two ? (c << 5) + __ffs(bits) - 1 : j0;
                if (two) bits &= bits - 1;
                const uint32_t pos0 = m - 1 - (uint32_t)(i * BATCH + j0), pos1 = m - 1 - (uint32_t)(i * BATCH + j1);
                const float4 s00 = lds128(a_s0 + j0 * 16), s10 = lds128(a_s1 + j0 * 16);
                const float4 s01 = lds128(a_s0 + j1 * 16), s11 = lds128(a_s1 + j1 * 16);
                const float dx0 = s00.x - pxf, dyA0 = s00.y - A.pyf, dyB0 = s00.y - B.pyf;
                const float dx1 = s01.x - pxf, dyA1 = s01.y - A.pyf, dyB1 = s01.y - B.pyf;
                const float pwA0 = pair_power(s10.x, s10.y, s10.z, dx0, dyA0), pwB0 = pair_power(s10.x, s10.y, s10.z, dx0, dyB0);
                const float pwA1 = pair_power(s11.x, s11.y, s11.z, dx1, dyA1), pwB1 = pair_power(s11.x, s11.y, s11.z, dx1, dyB1);
                float alA0, auA0, alB0, auB0, alA1, auA1, alB1, auB1;
                bool bA0, bB0, bA1, bB1;
                bool okA0 = pair_alpha_fast(pwA0, s10.w, alA0, auA0, bA0) && pos0 < A.last_contributor && RTG_FWD_PRETEST(pwA0, s00.z);
                bool okB0 = pair_alpha_fast(pwB0, s10.w, alB0, auB0, bB0) && pos0 < B.last_contributor && RTG_FWD_PRETEST(pwB0, s00.z);
                bool okA1 = pair_alpha_fast(pwA1, s11.w, alA1, auA1, bA1) && pos1 < A.last_contributor && RTG_FWD_PRETEST(pwA1, s01.z) && two;
                bool okB1 = pair_alpha_fast(pwB1, s11.w, alB1, auB1, bB1) && pos1 < B.last_contributor && RTG_FWD_PRETEST(pwB1, s01.z) && two;
                if ((bA0 && okA0) || (bB0 && okB0) || (bA1 && okA1) || (bB1 && okB1)) {  // a few pairs per frame
                    if (bA0 && okA0) okA0 = pair_alpha_exact(pwA0, s00.w, alA0, auA0);
                    if (bB0 && okB0) okB0 = pair_alpha_exact(pwB0, s00.w, alB0, auB0);
                    if (bA1 && okA1) okA1 = pair_alpha_exact(pwA1, s01.w, alA1, auA1);
                    if (bB1 && okB1) okB1 = pair_alpha_exact(pwB1, s01.w, alB1, auB1);
                }
                if (!__any_sync(FULL, okA0 || okB0 || okA1 || okB1)) continue;
                const float4 col0 = lds128(a_rgb + j0 * 16), col1 = lds128(a_rgb + j1 * 16);
                float v0[9], v1[9];
#pragma unroll
                for (int k = 0; k < 9; k++) v0[k] = v1[k] = 0.f;
                bwd_blend(A, okA0 ? alA0 : 0.f, okA0 ? auA0 : 0.f, col0, dx0, dyA0, v0);
                bwd_blend(B, okB0 ? alB0 : 0.f, okB0 ? auB0 : 0.f, col0, dx0, dyB0, v0);
                bwd_blend(A, okA1 ? alA1 : 0.f, okA1 ? auA1 : 0.f, col1, dx1, dyA1, v1);
                bwd_blend(B, okB1 ? alB1 : 0.f, okB1 ? auB1 : 0.f, col1, dx1, dyB1, v1);
                const float tot = warp_reduce18(v0, v1, lane);
                const int jm = (lane & 16) ? j1 : j0;
                if (my_slot >= 0 && (two || !(lane & 16))) atomicAdd(rec + (size_t)lds32(a_id + jm * 4) * RTG_REC + my_slot, tot);
            }
#else
            while (bits) {
                const int j = (c << 5) + __ffs(bits) - 1;
                bits &= bits - 1;
                const uint32_t pos = m - 1 - (uint32_t)(i * BATCH + j);
                const float4 s0 = lds128(a_s0 + j * 16), s1 = lds128(a_s1 + j * 16);
                const float dx = s0.x - pxf, dyA = s0.y - A.pyf, dyB = s0.y - B.pyf;
                const float pwA = pair_power(s1.x, s1.y, s1.z, dx, dyA), pwB = pair_power(s1.x, s1.y, s1.z, dx, dyB);
                float alA, auA, alB, auB;
                // same decisions as the forward: same power expression, same pretest, same alpha function
#ifdef RTG_BWD_BRANCHY_ALPHA
                const bool okA = pos < A.last_contributor && RTG_FWD_PRETEST(pwA, s0.z) && pair_alpha(pwA, s1.w, s0.w, alA, auA);
                const bool okB = pos < B.last_contributor && RTG_FWD_PRETEST(pwB, s0.z) && pair_alpha(pwB, s1.w, s0.w, alB, auB);
#else
                bool bandA, bandB;
                bool okA = pair_alpha_fast(pwA, s1.w, alA, auA, bandA) && pos < A.last_contributor && RTG_FWD_PRETEST(pwA, s0.z);
                bool okB = pair_alpha_fast(pwB, s1.w, alB, auB, bandB) && pos < B.last_contributor && RTG_FWD_PRETEST(pwB, s0.z);
                bandA = bandA && okA; bandB = bandB && okB;
                if (bandA || bandB) {  // a few pairs per frame
                    if (bandA) okA = pair_alpha_exact(pwA, s0.w, alA, auA);
                    if (bandB) okB = pair_alpha_exact(pwB, s0.w, alB, auB);
                }
#endif
                if (!__any_sync(FULL, okA || okB)) continue;
                const float4 col = lds128(a_rgb + j * 16);
                float v[9];
#pragma unroll
                for (int k = 0; k < 9; k++) v[k] = 0.f;
                bwd_blend(A, okA ? alA : 0.f, okA ? auA : 0.f, col, dx, dyA, v);
                bwd_blend(B, okB ? alB : 0.f, okB ? auB : 0.f, col, dx, dyB, v);
#ifdef RTG_BWD_SMEM_REDUCE
                // transposition through a warp-private [9][32] shared array: lane L < 18 sums 16 lanes of value L >> 1
                // (four 128-bit loads), lane pairs combine, even lanes add the total
                __syncwarp();
#pragma unroll
                for (int k = 0; k < 9; k++) sts32(a_red + (uint32_t)(k * 32 + lane) * 4, __float_as_uint(v[k]));
                __syncwarp();
                float tot = 0.f;
                if (lane < 18) {
                    const uint32_t a = a_red + (uint32_t)((lane >> 1) * 32 + (lane & 1) * 16) * 4;
                    const float4 q0 = lds128(a), q1 = lds128(a + 16), q2 = lds128(a + 32), q3 = lds128(a + 48);
                    tot = ((q0.x + q0.y) + (q0.z + q0.w)) + ((q1.x + q1.y) + (q1.z + q1.w)) +
                          (((q2.x + q2.y) + (q2.z + q2.w)) + ((q3.x + q3.y) + (q3.z + q3.w)));
                }
                tot += __shfl_xor_sync(FULL, tot, 1);
                if (lane < 18 && !(lane & 1)) atomicAdd(rec + (size_t)lds32(a_id + j * 4) * RTG_REC + (lane >> 1), tot);
#else
                const float tot = warp_reduce9(v, lane);
                if (my_slot >= 0) atomicAdd(rec + (size_t)lds32(a_id + j * 4) * RTG_REC + my_slot, tot);
#endif
            }
#endif
        }
    }

    depth_hit_grad(vp, g, hit_image, dL_ddepth, rec, px, pyA, pidA, insA);
    depth_hit_grad(vp, g, hit_image, dL_ddepth, rec, px, pyB, pidB, insB);
}

// ------------------------------------------------------------------ forward-mode pose tangents
// Tangent images of the forward's render along the six twist directions (preprocess_tangent_kernel holds the per-Gaussian
// tangents). One CTA per tile, in the forward's launch order, one pixel per thread on the forward's 8x4 warp patches. The
// tile's list is replayed front to back up to the longest prefix its pixels blended (max n_contrib), with the forward's
// decisions: the same patch masks, the same alpha function (pair_alpha: the exact expression inside the band around 1/255)
// and a pixel's own n_contrib. Per pixel: T, its 6 tangents and the 18 colour tangents of
//   C = sum c_i alpha_i T_i + T_final bg,   d alpha_i = au_i d power_i   (0 where alpha is clamped at 0.99),
// and the depth tangent of the hit Gaussian (hit_image), on the forward's plane / centre branch. No parameter array is read.
//   TAN_IMAGES:    J (6, 4, H, W): colour channels then depth, per direction; zeros where the tile is not rendered.
//   TAN_NORMAL_EQ: the residuals against the frame and the pixel selection of rtg_loss_l1, summed per tile into the
//                  RTG_GN_ALL Gauss-Newton terms (warp butterfly in double, warps in order, one row per TILE ID so that
//                  the launch order, which varies between runs, does not change any sum). No atomics.
//   TAN_NORMAL_EQ_ROBUST: the same rows for the Huber objective by iteratively reweighted least squares: each residual r
//                  (a colour channel, or the depth) gets the weight w = 1 for |r| <= delta, delta / |r| otherwise, in
//                  float from the float residual; the rows hold (w J_a) J_c and (w J_a) r, and the two residual-square
//                  terms hold sum 2 rho(r) (= sum r^2 while no |r| exceeds delta), so pose_gn_step_kernel is reused as is.
//   TAN_NORMAL_EQ_EXPOSURE[_ROBUST]: the frame's exposure (a, b) estimated with the pose: the colour residual is
//                  r = e^a C + b - C^ and its Jacobian row (e^a dC/dxi, e^a C, 1), eight columns; the depth rows keep six.
//                  RTG_GN_EXP_ALL terms per tile, reduced the same way; (e^a, b) is read from the device once per CTA.
enum { TAN_IMAGES = 0, TAN_NORMAL_EQ = 1, TAN_NORMAL_EQ_ROBUST = 2, TAN_NORMAL_EQ_EXPOSURE = 3, TAN_NORMAL_EQ_EXPOSURE_ROBUST = 4 };
constexpr bool tan_exposure(const int mode) { return mode == TAN_NORMAL_EQ_EXPOSURE || mode == TAN_NORMAL_EQ_EXPOSURE_ROBUST; }
constexpr bool tan_robust(const int mode) { return mode == TAN_NORMAL_EQ_ROBUST || mode == TAN_NORMAL_EQ_EXPOSURE_ROBUST; }
struct GnInputs {
    const float *render, *depth, *gt_color, *gt_depth;
    const uint8_t *mask;
    int channels_last;
    float depth_error_max;
    double *partial;  // [tiles][RTG_GN_ALL], or [tiles][RTG_GN_EXP_ALL] with exposure
};

// 2 rho(r) of the Huber loss: r^2 inside the threshold, delta (2 |r| - delta) outside
__device__ __forceinline__ float huber2(const float r, const float delta) {
    const float a = fabsf(r);
    return a <= delta ? r * r : delta * (2.f * a - delta);
}
__device__ __forceinline__ float huber_weight(const float r, const float delta) {
    const float a = fabsf(r);
    return a <= delta ? 1.f : delta / a;
}

// The body of the kernel signatures below; `huber` (colour, depth thresholds) is read by the robust modes only and `ab`
// (the device exposure) by the exposure modes only.
// ED (expected depth) replaces the hit depth by the alpha-blended depth of the same pairs: with w_i = alpha_i T_i and z_i
// the view-space z of Gaussian i's centre (hit record), m1 = sum w_i, m0 = sum w_i z_i, D = m0 / m1 (0 where m1 = 0) and
//   dz_i = (0, 0, 1, p_y, -p_x, 0),  dm1 = sum dw_i,  dm0 = sum (dw_i z_i + w_i dz_i),  dD = (dm0 - D dm1) / m1,
// carried in place of the hit-depth tangent. dT_{i+1} = dT_i - dw_i, so the sum telescopes to dm1 = -dT_final: the replay
// carries m0, m1 and dm0 only (m1 itself is summed, in render_feat_fwd_kernel's order, so that it is that map's coverage). TAN_IMAGES also writes (D, m1) to `expected` (2, H, W); the normal-equation
// modes take the depth residual D - D^ on S_e: in the mask, m1 >= min_cov, gt_depth > 0, D - gt_depth < depth_error_max.
template <int MODE, bool AA, bool ED = false>
__device__ __forceinline__ void render_tangent_body(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img,
                                                    const int *__restrict__ counters, const int *__restrict__ hit_image,
                                                    const float4 *__restrict__ tan, float *__restrict__ J, const GnInputs &in,
                                                    const float2 huber, const double *__restrict__ ab,
                                                    float *__restrict__ expected = nullptr, const float min_cov = 0.f) {
    constexpr bool EXPOSURE = tan_exposure(MODE);
    constexpr int NT = EXPOSURE ? RTG_GN_EXP_ALL : RTG_GN_ALL;
    __shared__ float4 s_s0[BATCH], s_s1[BATCH], s_rgb[BATCH];
    __shared__ int s_id[BATCH];
    __shared__ uint32_t s_mask[BATCH];
    __shared__ uint32_t s_max[8];
    __shared__ double s_red[MODE != TAN_IMAGES ? 8 : 1][NT];
    __shared__ float2 s_exp;  // (e^a, b)

    const int tile = (int)b.active[blockIdx.x];
    int px, py;
    bool inside;
    pixel_of(vp, tile, px, py, inside);
    const int pix = vp.W * py + px;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int n = counters[2] != 0 ? 0 : (int)b.tile_count[(size_t)tile * RTG_CNT_STRIDE];
    const uint32_t start = b.tile_offset[tile];
    const uint32_t last = (inside && n > 0) ? img.n_contrib[pix] : 0u;
    uint32_t wmax = last;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(FULL, wmax, o));
    if (lane == 0) s_max[w] = wmax;
    if constexpr (EXPOSURE)
        if (threadIdx.x == 0) s_exp = make_float2((float)exp(ab[0]), (float)ab[1]);
    __syncthreads();
    uint32_t m = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) m = max(m, s_max[k]);

    const float pxf = (float)px, pyf = (float)py;
    const float tx0 = (float)((tile % vp.tiles_x) * RTG_TILE), ty0 = (float)((tile / vp.tiles_x) * RTG_TILE);
    float T = 1.f, dT[6], dC[3][6];
#pragma unroll
    for (int k = 0; k < 6; k++) { dT[k] = 0.f; dC[0][k] = dC[1][k] = dC[2][k] = 0.f; }
    [[maybe_unused]] float m0 = 0.f, m1 = 0.f, dm0[6];
    if constexpr (ED)
#pragma unroll
        for (int k = 0; k < 6; k++) dm0[k] = 0.f;

    const int rounds = ((int)m + BATCH - 1) / BATCH;
    for (int i = 0; i < rounds; i++) {
        __syncthreads();  // the previous round has been consumed
        if (i * BATCH + (int)threadIdx.x < (int)m) {
            const int id = (int)b.point_list[start + (size_t)i * BATCH + threadIdx.x];
            const float4 s0 = __ldg(g.splat + 2 * (size_t)id), s1 = __ldg(g.splat + 2 * (size_t)id + 1);
            s_id[threadIdx.x] = id;
            s_s0[threadIdx.x] = s0;
            s_s1[threadIdx.x] = s1;
            s_rgb[threadIdx.x] = __ldg(g.rgb_flags + id);
            s_mask[threadIdx.x] = patch_mask(s0, s1, tx0, ty0);
        }
        __syncthreads();
        const int cnt = min(BATCH, (int)m - i * BATCH);
        for (int c = 0; c < ((cnt + 31) >> 5); c++) {
            const int e = (c << 5) + lane;
            const uint32_t mm = e < cnt ? s_mask[e] : 0u;
            uint32_t bits = __ballot_sync(FULL, (mm >> w) & 1u);
            while (bits) {
                const int j = (c << 5) + __ffs(bits) - 1;
                bits &= bits - 1;
                const uint32_t pos = (uint32_t)(i * BATCH + j);
                const float4 s0 = s_s0[j], s1 = s_s1[j];
                const float dx = s0.x - pxf, dy = s0.y - pyf;
                const float power = pair_power(s1.x, s1.y, s1.z, dx, dy);
                float alpha, au;
                // the backward's decisions: its own prefix, the same pretest, the same alpha function
                const bool ok = pos < last && RTG_FWD_PRETEST(power, s0.z) && pair_alpha(power, s1.w, s0.w, alpha, au);
                if (!__any_sync(FULL, ok)) continue;
                if (ok) {
                    const float4 *tr = tan + (size_t)s_id[j] * RTG_TAN_ROW;
                    const float4 col = s_rgb[j];
                    const float dadp = au <= 0.99f ? au : 0.f;  // d alpha / d power
                    const float gx = -(s1.x * dx + s1.y * dy), gy = -(s1.z * dy + s1.y * dx);  // d power / d centre
                    const float wgt = alpha * T;
                    // antialiased: alpha = o comp G, so d alpha = au (d power + d ln comp) below the clamp; d ln comp of the six
                    // directions sits in the colour slots of the rotation directions (preprocess_tangent_kernel)
                    float dlc[6];
                    if constexpr (AA) {
#pragma unroll
                        for (int k = 0; k < 3; k++) {
                            const float4 tr_k = __ldg(tr + 2 * (k + 3) + 1);
                            dlc[k] = tr_k.y; dlc[k + 3] = tr_k.z;
                        }
                    }
                    [[maybe_unused]] float4 pc;  // ED: the view-space centre (x, y, z) of the hit record
                    if constexpr (ED) pc = __ldg(g.hit + 2 * (size_t)s_id[j] + 1);
#pragma unroll
                    for (int k = 0; k < 6; k++) {
                        const float4 ta = __ldg(tr + 2 * k);
                        float4 tb = __ldg(tr + 2 * k + 1);
                        const float dpow = gx * ta.x + gy * ta.y - 0.5f * dx * dx * ta.z - dx * dy * ta.w - 0.5f * dy * dy * tb.x;
                        if (AA && k >= 3) tb.y = tb.z = tb.w = 0.f;  // a rotation does not move the colour
                        const float dal = AA ? dadp * (dpow + dlc[k]) : dadp * dpow;
                        const float dw = dal * T + alpha * dT[k];  // d (alpha T)
                        dC[0][k] += tb.y * wgt + col.x * dw;
                        dC[1][k] += tb.z * wgt + col.y * dw;
                        dC[2][k] += tb.w * wgt + col.z * dw;
                        if constexpr (ED) {
                            float dm = dw * pc.z;  // + w dz, dz = (0, 0, 1, p_y, -p_x, 0)
                            if (k == 2) dm += wgt;
                            if (k == 3) dm += wgt * pc.y;
                            if (k == 4) dm -= wgt * pc.x;
                            dm0[k] += dm;
                        }
                        dT[k] = dT[k] * (1.f - alpha) - T * dal;
                    }
                    if constexpr (ED) {  // in the order and form of render_feat_fwd_kernel's F = (z, 1) accumulators
                        m0 += wgt * pc.z;
                        m1 += wgt;
                    }
                    T = T * (1.f - alpha);
                }
            }
        }
    }

    // colour: the background term T_final bg; depth: the hit Gaussian's plane or centre depth
    const float bg0 = __ldg(vp.bg), bg1 = __ldg(vp.bg + 1), bg2 = __ldg(vp.bg + 2);
#pragma unroll
    for (int k = 0; k < 6; k++) { dC[0][k] += bg0 * dT[k]; dC[1][k] += bg1 * dT[k]; dC[2][k] += bg2 * dT[k]; }
    float dD[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    [[maybe_unused]] float D = 0.f;  // ED: the expected depth
    if constexpr (ED) {
        if (m1 > 0.f) {
            D = m0 / m1;
            const float inv = 1.f / m1;
#pragma unroll
            for (int k = 0; k < 6; k++) dD[k] = (dm0[k] + D * dT[k]) * inv;  // dm1 = -dT
        }
    }
    const int gid = (!ED && inside && n > 0) ? hit_image[pix] : -1;  // a never-rendered tile's hit map holds 0, not a hit
    if (gid >= 0) {
        const float3 ray = pixel_ray(px, py, vp.focal_x, vp.focal_y, vp.cx, vp.cy);
        const float4 h0 = __ldg(g.hit + 2 * (size_t)gid), h1 = __ldg(g.hit + 2 * (size_t)gid + 1);
        const float3 nc = make_float3(h0.x, h0.y, h0.z), pc = make_float3(h1.x, h1.y, h1.z);
        const float num = pc.x * nc.x + pc.y * nc.y + pc.z * nc.z;
        const float ndotr = nc.x * ray.x + nc.y * ray.y + nc.z * ray.z;
        const float tt = (float)((double)num / ((double)ndotr + 1e-8));
        // surfel_depth's decision
        if (fabsf(tt * ray.z - pc.z) <= h0.w * vp.depth_thr && fabsf(ndotr) >= vp.normal_thr) {
            // D = ray.z (n.p_c) / (n.ray + 1e-8): d(n.p_c) = n.rho (the rotation moves n and p_c alike), d(n.ray) = phi.(n x ray)
            const float inv_nr = 1.f / (float)((double)ndotr + 1e-8);
            const float s = -ray.z * num * inv_nr * inv_nr;
            dD[0] = ray.z * nc.x * inv_nr; dD[1] = ray.z * nc.y * inv_nr; dD[2] = ray.z * nc.z * inv_nr;
            dD[3] = s * (nc.y * ray.z - nc.z * ray.y); dD[4] = s * (nc.z * ray.x - nc.x * ray.z); dD[5] = s * (nc.x * ray.y - nc.y * ray.x);
        } else {  // centre depth: (rho + phi x p_c).z
            dD[2] = 1.f; dD[3] = pc.y; dD[4] = -pc.x;
        }
    }

    if constexpr (MODE == TAN_IMAGES) {
        if (inside) {
            const size_t HW = (size_t)vp.H * vp.W;
#pragma unroll
            for (int k = 0; k < 6; k++) {
                float *o = J + (size_t)(4 * k) * HW + pix;
                o[0] = dC[0][k]; o[HW] = dC[1][k]; o[2 * HW] = dC[2][k]; o[3 * HW] = dD[k];
            }
            if constexpr (ED) { expected[pix] = D; expected[HW + pix] = m1; }
        }
    } else {
        const int N = vp.H * vp.W;
        float rc[3] = {0.f, 0.f, 0.f}, rd = 0.f;
        [[maybe_unused]] float eC[3] = {0.f, 0.f, 0.f};  // e^a C, the colour row's exposure-gain column
        bool sc = inside && (in.mask == nullptr || in.mask[pix] != 0), sd = false;
        if (sc) {
#pragma unroll
            for (int ch = 0; ch < 3; ch++) {
                const float gt = frame_color(in.gt_color, in.channels_last, N, pix, ch);
                if constexpr (EXPOSURE) {
                    eC[ch] = s_exp.x * in.render[(size_t)ch * N + pix];
                    rc[ch] = (eC[ch] + s_exp.y) - gt;
                } else {
                    rc[ch] = in.render[(size_t)ch * N + pix] - gt;
                }
            }
            const float gd = in.gt_depth[pix];
            if constexpr (ED) {
                rd = D - gd;
                sd = m1 >= min_cov && gd > 0.f && rd < in.depth_error_max;  // S_e
            } else {
                rd = in.depth[pix] - gd;
                sd = frame_depth_pixel(hit_image[pix], gd, rd, in.depth_error_max);  // rtg_loss_l1's depth pixels
            }
        }
        if constexpr (EXPOSURE) {
            // Each term is reduced as soon as it is formed (double warp butterfly, lane 0 stores the warp's sum), the depth
            // set first: its tangents are then dead while the 46 colour terms are formed. The __syncwarp orders the
            // store before the next term; without it ptxas holds the lane-0 sums back and spills.
            auto put = [&](const int t, const float val) {
                double x = (double)val;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(FULL, x, o);
                if (lane == 0) s_red[w][t] = x;
                __syncwarp();
            };
            constexpr bool ROBUST = tan_robust(MODE);
            int q = RTG_GN_EXP_COLOR;
            {
                const float wd = ROBUST ? huber_weight(rd, huber.y) : 1.f;
#pragma unroll
                for (int a = 0; a < 6; a++) {
                    const float jd = wd * dD[a];
#pragma unroll
                    for (int c = a; c < 6; c++, q++) put(q, sd ? jd * dD[c] : 0.f);
                    put(RTG_GN_EXP_COLOR + 21 + a, sd ? jd * rd : 0.f);
                }
                if constexpr (ROBUST) put(RTG_GN_EXP_COLOR + 27, sd ? huber2(rd, huber.y) : 0.f);
                else put(RTG_GN_EXP_COLOR + 27, sd ? rd * rd : 0.f);
                put(RTG_GN_EXP_COLOR + 28, sd ? 1.f : 0.f);
            }
            const float ea = s_exp.x;
#pragma unroll
            for (int k = 0; k < 6; k++) { dC[0][k] *= ea; dC[1][k] *= ea; dC[2][k] *= ea; }
            // column k of channel ch's Jacobian row (e^a dC/dxi, e^a C, 1)
            auto jc = [&](const int ch, const int k) { return k < 6 ? dC[ch][k] : (k == 6 ? eC[ch] : 1.f); };
            const float w0 = ROBUST ? huber_weight(rc[0], huber.x) : 1.f, w1 = ROBUST ? huber_weight(rc[1], huber.x) : 1.f;
            const float w2 = ROBUST ? huber_weight(rc[2], huber.x) : 1.f;
            q = 0;
#pragma unroll
            for (int a = 0; a < 8; a++) {
                const float ja0 = w0 * jc(0, a), ja1 = w1 * jc(1, a), ja2 = w2 * jc(2, a);
#pragma unroll
                for (int c = a; c < 8; c++, q++) put(q, sc ? ja0 * jc(0, c) + ja1 * jc(1, c) + ja2 * jc(2, c) : 0.f);
                put(36 + a, sc ? ja0 * rc[0] + ja1 * rc[1] + ja2 * rc[2] : 0.f);
            }
            if constexpr (ROBUST) put(44, sc ? huber2(rc[0], huber.x) + huber2(rc[1], huber.x) + huber2(rc[2], huber.x) : 0.f);
            else put(44, sc ? rc[0] * rc[0] + rc[1] * rc[1] + rc[2] * rc[2] : 0.f);
            put(45, sc ? 1.f : 0.f);
        } else {
        float v[RTG_GN_ALL];
        int q = 0;
        if constexpr (MODE == TAN_NORMAL_EQ) {
#pragma unroll
            for (int a = 0; a < 6; a++)
#pragma unroll
                for (int c = a; c < 6; c++, q++) {
                    v[q] = sc ? dC[0][a] * dC[0][c] + dC[1][a] * dC[1][c] + dC[2][a] * dC[2][c] : 0.f;
                    v[RTG_GN_TERMS + q] = sd ? dD[a] * dD[c] : 0.f;
                }
#pragma unroll
            for (int a = 0; a < 6; a++) {
                v[21 + a] = sc ? dC[0][a] * rc[0] + dC[1][a] * rc[1] + dC[2][a] * rc[2] : 0.f;
                v[RTG_GN_TERMS + 21 + a] = sd ? dD[a] * rd : 0.f;
            }
            v[27] = sc ? rc[0] * rc[0] + rc[1] * rc[1] + rc[2] * rc[2] : 0.f;
            v[RTG_GN_TERMS + 27] = sd ? rd * rd : 0.f;
        } else {
            // a weight of 1 leaves w J_a bit-equal to J_a, so an unweighted pixel's terms are those of TAN_NORMAL_EQ
            const float w0 = huber_weight(rc[0], huber.x), w1 = huber_weight(rc[1], huber.x), w2 = huber_weight(rc[2], huber.x);
            const float wd = huber_weight(rd, huber.y);
#pragma unroll
            for (int a = 0; a < 6; a++) {
                const float ja0 = w0 * dC[0][a], ja1 = w1 * dC[1][a], ja2 = w2 * dC[2][a], jd = wd * dD[a];
#pragma unroll
                for (int c = a; c < 6; c++, q++) {
                    v[q] = sc ? ja0 * dC[0][c] + ja1 * dC[1][c] + ja2 * dC[2][c] : 0.f;
                    v[RTG_GN_TERMS + q] = sd ? jd * dD[c] : 0.f;
                }
                v[21 + a] = sc ? ja0 * rc[0] + ja1 * rc[1] + ja2 * rc[2] : 0.f;
                v[RTG_GN_TERMS + 21 + a] = sd ? jd * rd : 0.f;
            }
            v[27] = sc ? huber2(rc[0], huber.x) + huber2(rc[1], huber.x) + huber2(rc[2], huber.x) : 0.f;
            v[RTG_GN_TERMS + 27] = sd ? huber2(rd, huber.y) : 0.f;
        }
        v[28] = sc ? 1.f : 0.f;
        v[RTG_GN_TERMS + 28] = sd ? 1.f : 0.f;
#pragma unroll
        for (int t = 0; t < RTG_GN_ALL; t++) {
            double x = (double)v[t];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(FULL, x, o);
            if (lane == 0) s_red[w][t] = x;
        }
        }
        __syncthreads();
        if (threadIdx.x < NT) {
            double acc = 0.0;
#pragma unroll
            for (int k = 0; k < 8; k++) acc += s_red[k][threadIdx.x];
            in.partial[(size_t)tile * NT + threadIdx.x] = acc;
        }
    }
}

// Three signatures, so that TAN_IMAGES and TAN_NORMAL_EQ keep their parameter list (and their code), only the robust
// instantiation carries the Huber thresholds and only the exposure ones the pointer to the device exposure.
template <int MODE, bool AA>
__global__ void __launch_bounds__(256) render_tangent_kernel(const ViewParams vp, const GeomState g, const BinState b, const ImgState img,
                                                             const int *__restrict__ counters, const int *__restrict__ hit_image,
                                                             const float4 *__restrict__ tan, float *__restrict__ J, const GnInputs in) {
    static_assert(MODE == TAN_IMAGES || MODE == TAN_NORMAL_EQ, "the robust rows take the Huber thresholds");
    render_tangent_body<MODE, AA>(vp, g, b, img, counters, hit_image, tan, J, in, make_float2(0.f, 0.f), nullptr);
}
template <int MODE, bool AA>
__global__ void __launch_bounds__(256) render_tangent_kernel(const ViewParams vp, const GeomState g, const BinState b, const ImgState img,
                                                             const int *__restrict__ counters, const int *__restrict__ hit_image,
                                                             const float4 *__restrict__ tan, float *__restrict__ J, const GnInputs in,
                                                             const float2 huber) {
    static_assert(MODE == TAN_NORMAL_EQ_ROBUST, "only the robust rows take the Huber thresholds");
    render_tangent_body<MODE, AA>(vp, g, b, img, counters, hit_image, tan, J, in, huber, nullptr);
}
template <int MODE, bool AA>
__global__ void __launch_bounds__(256, 2) render_tangent_kernel(const ViewParams vp, const GeomState g, const BinState b, const ImgState img,
                                                             const int *__restrict__ counters, const int *__restrict__ hit_image,
                                                             const float4 *__restrict__ tan, float *__restrict__ J, const GnInputs in,
                                                             const float2 huber, const double *__restrict__ ab) {
    static_assert(tan_exposure(MODE), "only the exposure rows read the device exposure");
    render_tangent_body<MODE, AA>(vp, g, b, img, counters, hit_image, tan, J, in, huber, ab);
}
// Every mode with the expected depth in place of the hit depth (one signature: the unused arguments are not read), at two
// CTAs per SM: without the bound the normal-equation modes take 152 registers, one CTA.
template <int MODE, bool AA>
__global__ void __launch_bounds__(256, 2)
    render_tangent_expected_kernel(const ViewParams vp, const GeomState g, const BinState b, const ImgState img,
                                   const int *__restrict__ counters, const float4 *__restrict__ tan, float *__restrict__ J,
                                   const GnInputs in, const float2 huber, const double *__restrict__ ab,
                                   float *__restrict__ expected, const float min_cov) {
    render_tangent_body<MODE, AA, true>(vp, g, b, img, counters, nullptr, tan, J, in, huber, ab, expected, min_cov);
}

// One block: the fixed-order sum of the tiles' rows (one warp per term, fixed lane stride, fixed butterfly), then on one
// thread the weights and counts, the trace damping, solve6, exp(xi^) W2C and the three camera arrays. A singular system,
// an empty selection or an overflowed forward leaves the pose and the arrays unchanged and sets the status.
__global__ void __launch_bounds__(256) pose_gn_step_kernel(const int tiles, const double *__restrict__ partial,
                                                            const int *__restrict__ counters, const RtgPoseGN s) {
    __shared__ double s_tot[RTG_GN_ALL];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int term = w; term < RTG_GN_ALL; term += 8) {
        double acc = 0.0;
        for (int t = lane; t < tiles; t += 32) acc += partial[(size_t)t * RTG_GN_ALL + term];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(FULL, acc, o);
        if (lane == 0) s_tot[term] = acc;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    const double *cs = s_tot, *ds = s_tot + RTG_GN_TERMS;
    const double nc = 3.0 * cs[28], nd = ds[28];
    const double wc = nc > 0.0 ? (double)s.color_weight / nc : 0.0, wd = nd > 0.0 ? (double)s.depth_weight / nd : 0.0;
    double A[6][6], bvec[6], xi[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    int q = 0;
#pragma unroll
    for (int a = 0; a < 6; a++)
#pragma unroll
        for (int c = a; c < 6; c++, q++) { const double v = wc * cs[q] + wd * ds[q]; A[a][c] = v; A[c][a] = v; }
    double trace = 0.0;
#pragma unroll
    for (int a = 0; a < 6; a++) trace += A[a][a];
#pragma unroll
    for (int a = 0; a < 6; a++) { A[a][a] += trace * (double)s.damping; bvec[a] = -(wc * cs[21 + a] + wd * ds[21 + a]); }
    int status = RTG_POSE_GN_OK;
    if (counters[2] != 0) status = RTG_POSE_GN_OVERFLOW;
    else if (nc + nd == 0.0) status = RTG_POSE_GN_EMPTY;
    else if (!solve6(A, bvec, xi)) status = RTG_POSE_GN_SINGULAR;
    if (status == RTG_POSE_GN_OK) {
        double Tm[4][4], E[3][4];
#pragma unroll
        for (int i = 0; i < 16; i++) Tm[i / 4][i % 4] = s.pose[i];
        se3_exp_twist(xi, E);
        pose_left_update(E, Tm, s.pose, s.projection, s.viewmatrix, s.projmatrix, s.campos);
    } else {
#pragma unroll
        for (int a = 0; a < 6; a++) xi[a] = 0.0;
    }
    const double ec = 0.5 * wc * cs[27], ed = 0.5 * wd * ds[27];
    double *r = s.report;
    r[0] = ec + ed; r[1] = ec; r[2] = ed; r[3] = nc; r[4] = nd;
    r[5] = sqrt(xi[0] * xi[0] + xi[1] * xi[1] + xi[2] * xi[2]);
    r[6] = sqrt(xi[3] * xi[3] + xi[4] * xi[4] + xi[5] * xi[5]);
    r[7] = (double)status;
}

// pose_gn_step_kernel for the eight unknowns (rho, phi, a, b). The 8x8 system holds the depth block in its leading 6x6.
// Damping: the pose diagonals get damping * trace(H[0:6, 0:6]) as above, so that without the exposure columns the pose
// step is pose_gn_step_kernel's; the exposure diagonals are scaled by (1 + damping) instead, because the pose trace, of
// order (focal length * image gradient)^2, is many orders above H_bb = color_weight and would freeze (a, b). With no
// colour term (N_c = 0 or color_weight = 0) the exposure columns are empty: the 6x6 pose system is solved alone and
// (a, b) is kept. A singular system, an empty selection or an overflowed forward leaves pose and exposure unchanged.
__global__ void __launch_bounds__(256) pose_gn_exposure_step_kernel(const int tiles, const double *__restrict__ partial,
                                                                     const int *__restrict__ counters, const RtgPoseGN s,
                                                                     double *__restrict__ ab) {
    __shared__ double s_tot[RTG_GN_EXP_ALL];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int term = w; term < RTG_GN_EXP_ALL; term += 8) {
        double acc = 0.0;
        for (int t = lane; t < tiles; t += 32) acc += partial[(size_t)t * RTG_GN_EXP_ALL + term];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(FULL, acc, o);
        if (lane == 0) s_tot[term] = acc;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    const double *cs = s_tot, *ds = s_tot + RTG_GN_EXP_COLOR;
    const double nc = 3.0 * cs[45], nd = ds[28];
    const double wc = nc > 0.0 ? (double)s.color_weight / nc : 0.0, wd = nd > 0.0 ? (double)s.depth_weight / nd : 0.0;
    double A[8][8], bvec[8], x[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    int q = 0;
#pragma unroll
    for (int a = 0; a < 8; a++) {
#pragma unroll
        for (int c = a; c < 8; c++, q++) { const double v = wc * cs[q]; A[a][c] = v; A[c][a] = v; }
        bvec[a] = -(wc * cs[36 + a]);
    }
    q = 0;
#pragma unroll
    for (int a = 0; a < 6; a++) {
#pragma unroll
        for (int c = a; c < 6; c++, q++) { const double v = A[a][c] + wd * ds[q]; A[a][c] = v; A[c][a] = v; }
        bvec[a] -= wd * ds[21 + a];
    }
    double trace = 0.0;
#pragma unroll
    for (int a = 0; a < 6; a++) trace += A[a][a];
#pragma unroll
    for (int a = 0; a < 6; a++) A[a][a] += trace * (double)s.damping;
    A[6][6] *= 1.0 + (double)s.damping;
    A[7][7] *= 1.0 + (double)s.damping;
    const bool exposed = wc > 0.0;
    int status = RTG_POSE_GN_OK;
    if (counters[2] != 0) status = RTG_POSE_GN_OVERFLOW;
    else if (nc + nd == 0.0) status = RTG_POSE_GN_EMPTY;
    else if (exposed) {
        if (!solve_n<8>(A, bvec, x)) status = RTG_POSE_GN_SINGULAR;
    } else {
        double A6[6][6];
#pragma unroll
        for (int a = 0; a < 6; a++)
#pragma unroll
            for (int c = 0; c < 6; c++) A6[a][c] = A[a][c];
        if (!solve6(A6, bvec, x)) status = RTG_POSE_GN_SINGULAR;
    }
    if (status == RTG_POSE_GN_OK) {
        double Tm[4][4], E[3][4];
#pragma unroll
        for (int i = 0; i < 16; i++) Tm[i / 4][i % 4] = s.pose[i];
        se3_exp_twist(x, E);
        pose_left_update(E, Tm, s.pose, s.projection, s.viewmatrix, s.projmatrix, s.campos);
        if (exposed) { ab[0] += x[6]; ab[1] += x[7]; }
    } else {
#pragma unroll
        for (int a = 0; a < 6; a++) x[a] = 0.0;
    }
    const double ec = 0.5 * wc * cs[44], ed = 0.5 * wd * ds[27];
    double *r = s.report;
    r[0] = ec + ed; r[1] = ec; r[2] = ed; r[3] = nc; r[4] = nd;
    r[5] = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
    r[6] = sqrt(x[3] * x[3] + x[4] * x[4] + x[5] * x[5]);
    r[7] = (double)status;
}

size_t pose_gn_exposure_scratch_bytes(int P, int H, int W) {
    const size_t tiles = (size_t)((W + RTG_TILE - 1) / RTG_TILE) * ((H + RTG_TILE - 1) / RTG_TILE);
    return align_up((size_t)(P > 0 ? P : 0) * RTG_TAN_ROW * sizeof(float4), 256) + tiles * RTG_GN_EXP_ALL * sizeof(double);
}

size_t pose_gn_scratch_bytes(int P, int H, int W) {
    const size_t tiles = (size_t)((W + RTG_TILE - 1) / RTG_TILE) * ((H + RTG_TILE - 1) / RTG_TILE);
    return align_up((size_t)(P > 0 ? P : 0) * RTG_TAN_ROW * sizeof(float4), 256) + tiles * RTG_GN_ALL * sizeof(double);
}
static inline float4 *tan_rows(void *scratch) { return reinterpret_cast<float4 *>(scratch); }
static inline double *gn_partial(void *scratch, int P) {
    return reinterpret_cast<double *>(reinterpret_cast<char *>(scratch) + align_up((size_t)P * RTG_TAN_ROW * sizeof(float4), 256));
}

void launch_render_tangent_images(const ViewParams &vp, int P, const GeomState &g, const BinState &b, const ImgState &img,
                                  const int32_t *counters, const int *hit_image, void *scratch, float *J, cudaStream_t s) {
    const int T = vp.tiles_x * vp.tiles_y;
    if (vp.antialiased) render_tangent_kernel<TAN_IMAGES, true><<<T, 256, 0, s>>>(vp, g, b, img, counters, hit_image, tan_rows(scratch), J, GnInputs{});
    else render_tangent_kernel<TAN_IMAGES, false><<<T, 256, 0, s>>>(vp, g, b, img, counters, hit_image, tan_rows(scratch), J, GnInputs{});
}

void launch_pose_gn_normal_eq_step(const ViewParams &vp, int P, const GeomState &g, const BinState &b, const ImgState &img,
                                   const int32_t *counters, const RtgPoseGN &st, const RtgPoseRobust &robust, cudaStream_t s) {
    const int T = vp.tiles_x * vp.tiles_y;
    GnInputs in{st.render, st.depth, st.gt_color, st.gt_depth, st.render_mask, st.gt_channels_last, st.depth_error_max,
                gn_partial(st.scratch, P)};
    const float2 huber = make_float2(robust.color_delta, robust.depth_delta);
    const float4 *tan = tan_rows(st.scratch);
    if (robust.kernel == RTG_ROBUST_HUBER && vp.antialiased)
        render_tangent_kernel<TAN_NORMAL_EQ_ROBUST, true><<<T, 256, 0, s>>>(vp, g, b, img, counters, st.hit_depth, tan, nullptr, in, huber);
    else if (robust.kernel == RTG_ROBUST_HUBER)
        render_tangent_kernel<TAN_NORMAL_EQ_ROBUST, false><<<T, 256, 0, s>>>(vp, g, b, img, counters, st.hit_depth, tan, nullptr, in, huber);
    else if (vp.antialiased)
        render_tangent_kernel<TAN_NORMAL_EQ, true><<<T, 256, 0, s>>>(vp, g, b, img, counters, st.hit_depth, tan, nullptr, in);
    else
        render_tangent_kernel<TAN_NORMAL_EQ, false><<<T, 256, 0, s>>>(vp, g, b, img, counters, st.hit_depth, tan, nullptr, in);
    pose_gn_step_kernel<<<1, 256, 0, s>>>(T, in.partial, counters, st);
}

void launch_pose_gn_exposure_step(const ViewParams &vp, int P, const GeomState &g, const BinState &b, const ImgState &img,
                                  const int32_t *counters, const RtgPoseGN &st, const RtgPoseRobust &robust, double *ab,
                                  cudaStream_t s) {
    const int T = vp.tiles_x * vp.tiles_y;
    GnInputs in{st.render, st.depth, st.gt_color, st.gt_depth, st.render_mask, st.gt_channels_last, st.depth_error_max,
                gn_partial(st.scratch, P)};
    const float2 huber = make_float2(robust.color_delta, robust.depth_delta);
    const float4 *tan = tan_rows(st.scratch);
    if (robust.kernel == RTG_ROBUST_HUBER && vp.antialiased)
        render_tangent_kernel<TAN_NORMAL_EQ_EXPOSURE_ROBUST, true><<<T, 256, 0, s>>>(vp, g, b, img, counters, st.hit_depth, tan, nullptr, in, huber, ab);
    else if (robust.kernel == RTG_ROBUST_HUBER)
        render_tangent_kernel<TAN_NORMAL_EQ_EXPOSURE_ROBUST, false><<<T, 256, 0, s>>>(vp, g, b, img, counters, st.hit_depth, tan, nullptr, in, huber, ab);
    else if (vp.antialiased)
        render_tangent_kernel<TAN_NORMAL_EQ_EXPOSURE, true><<<T, 256, 0, s>>>(vp, g, b, img, counters, st.hit_depth, tan, nullptr, in, huber, ab);
    else
        render_tangent_kernel<TAN_NORMAL_EQ_EXPOSURE, false><<<T, 256, 0, s>>>(vp, g, b, img, counters, st.hit_depth, tan, nullptr, in, huber, ab);
    pose_gn_exposure_step_kernel<<<1, 256, 0, s>>>(T, in.partial, counters, st, ab);
}

void launch_render_tangent_expected_images(const ViewParams &vp, int P, const GeomState &g, const BinState &b, const ImgState &img,
                                           const int32_t *counters, void *scratch, float *J, float *expected, cudaStream_t s) {
    const int T = vp.tiles_x * vp.tiles_y;
    const float4 *tan = tan_rows(scratch);
    const float2 h = make_float2(0.f, 0.f);
    if (vp.antialiased)
        render_tangent_expected_kernel<TAN_IMAGES, true><<<T, 256, 0, s>>>(vp, g, b, img, counters, tan, J, GnInputs{}, h, nullptr, expected, 0.f);
    else
        render_tangent_expected_kernel<TAN_IMAGES, false><<<T, 256, 0, s>>>(vp, g, b, img, counters, tan, J, GnInputs{}, h, nullptr, expected, 0.f);
}

template <int MODE>
static void launch_tangent_expected_rows(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img,
                                         const int32_t *counters, const float4 *tan, const GnInputs &in, const float2 huber,
                                         const double *ab, const float min_cov, cudaStream_t s) {
    const int T = vp.tiles_x * vp.tiles_y;
    if (vp.antialiased)
        render_tangent_expected_kernel<MODE, true><<<T, 256, 0, s>>>(vp, g, b, img, counters, tan, nullptr, in, huber, ab, nullptr, min_cov);
    else
        render_tangent_expected_kernel<MODE, false><<<T, 256, 0, s>>>(vp, g, b, img, counters, tan, nullptr, in, huber, ab, nullptr, min_cov);
}

void launch_pose_gn_expected_step(const ViewParams &vp, int P, const GeomState &g, const BinState &b, const ImgState &img,
                                  const int32_t *counters, const RtgPoseGN &st, const RtgPoseRobust &robust, double *ab,
                                  float min_cov, cudaStream_t s) {
    const int T = vp.tiles_x * vp.tiles_y;
    GnInputs in{st.render, st.depth, st.gt_color, st.gt_depth, st.render_mask, st.gt_channels_last, st.depth_error_max,
                gn_partial(st.scratch, P)};
    const float2 huber = make_float2(robust.color_delta, robust.depth_delta);
    const float4 *tan = tan_rows(st.scratch);
    const bool hub = robust.kernel == RTG_ROBUST_HUBER;
    if (ab) {
        if (hub) launch_tangent_expected_rows<TAN_NORMAL_EQ_EXPOSURE_ROBUST>(vp, g, b, img, counters, tan, in, huber, ab, min_cov, s);
        else launch_tangent_expected_rows<TAN_NORMAL_EQ_EXPOSURE>(vp, g, b, img, counters, tan, in, huber, ab, min_cov, s);
        pose_gn_exposure_step_kernel<<<1, 256, 0, s>>>(T, in.partial, counters, st, ab);
    } else {
        if (hub) launch_tangent_expected_rows<TAN_NORMAL_EQ_ROBUST>(vp, g, b, img, counters, tan, in, huber, nullptr, min_cov, s);
        else launch_tangent_expected_rows<TAN_NORMAL_EQ>(vp, g, b, img, counters, tan, in, huber, nullptr, min_cov, s);
        pose_gn_step_kernel<<<1, 256, 0, s>>>(T, in.partial, counters, st);
    }
}

void launch_render_fwd(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img, const int32_t *counters,
                       float *out_color, float *out_depth, int *out_hit_color, int *out_hit_depth, float *out_hcw,
                       float *out_hdw, float *out_T, cudaStream_t s) {
    const int T = vp.tiles_x * vp.tiles_y;
    ProfScope ps(K_RENDER_FWD, s);
    render_fwd_kernel<<<T, 256, 0, s>>>(vp, g, b, img, counters, out_color, out_depth, out_hit_color, out_hit_depth, out_hcw,
                                        out_hdw, out_T);
}

void launch_render_bwd(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img, const int32_t *counters,
                       const float *final_T, const int *hit_image, const float *dL_dcolor, const float *dL_ddepth, float *rec,
                       cudaStream_t s, const float *dL_dT) {
    const int T = vp.tiles_x * vp.tiles_y;
    ProfScope ps(K_RENDER_BWD, s);
    if (dL_dT)
        render_bwd_kernel<true><<<T, BWD_THREADS, 0, s>>>(vp, g, b, img, counters, final_T, hit_image, dL_dcolor, dL_ddepth, rec, dL_dT);
    else
        render_bwd_kernel<false><<<T, BWD_THREADS, 0, s>>>(vp, g, b, img, counters, final_T, hit_image, dL_dcolor, dL_ddepth, rec, nullptr);
}

// ------------------------------------------------------------------ per-Gaussian contributions
// What each Gaussian adds to the forward's render, replayed from the forward's own decisions as in render_tangent_body:
// one CTA per tile in the forward's launch order, one pixel per thread on the forward's 8x4 warp patches, the tile's list
// walked front to back up to its longest blended prefix with the same patch masks, pretest and alpha function and a
// pixel's own n_contrib. A pixel carries only T: every pair it blends has the forward's colour weight w = alpha T, then
// T *= 1 - alpha, bit for bit as render_fwd_kernel. Per (warp, entry) with at least one blending lane, the count of those
// lanes goes to n_pixels and the warp sums of w (and, ERR, of w e with e the pixel's error) go to weight (and error):
// one butterfly for both sums (after the xor-16 step lanes 0-15 hold w, lanes 16-31 w e), lane 0 adds the count and
// sum w, lane 16 sum w e. The atomics' results are unused (RED). Reads no parameter array and no colour.
template <bool ERR>
__global__ void __launch_bounds__(256) render_contrib_kernel(const ViewParams vp, const GeomState g, const BinState b, const ImgState img,
                                                             const int *__restrict__ counters, const float *__restrict__ pixel_error,
                                                             int *__restrict__ n_pixels, float *__restrict__ weight,
                                                             float *__restrict__ error) {
    __shared__ float4 s_s0[BATCH], s_s1[BATCH];
    __shared__ int s_id[BATCH];
    __shared__ uint32_t s_mask[BATCH];
    __shared__ uint32_t s_max[8];

    if (counters[2] != 0) return;  // an overflowed forward rendered nothing
    const int tile = (int)b.active[blockIdx.x];
    const int n = (int)b.tile_count[(size_t)tile * RTG_CNT_STRIDE];
    if (n == 0) return;            // empty or masked-out tile
    int px, py;
    bool inside;
    pixel_of(vp, tile, px, py, inside);
    const int pix = vp.W * py + px;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const uint32_t start = b.tile_offset[tile];
    const uint32_t last = inside ? img.n_contrib[pix] : 0u;
    float e = 0.f;
    if constexpr (ERR) e = inside ? pixel_error[pix] : 0.f;
    uint32_t wmax = last;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(FULL, wmax, o));
    if (lane == 0) s_max[w] = wmax;
    __syncthreads();
    uint32_t m = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) m = max(m, s_max[k]);

    const float pxf = (float)px, pyf = (float)py;
    const float tx0 = (float)((tile % vp.tiles_x) * RTG_TILE), ty0 = (float)((tile / vp.tiles_x) * RTG_TILE);
    float T = 1.f;
    const int rounds = ((int)m + BATCH - 1) / BATCH;
    for (int i = 0; i < rounds; i++) {
        __syncthreads();  // the previous round has been consumed
        if (i * BATCH + (int)threadIdx.x < (int)m) {
            const int id = (int)b.point_list[start + (size_t)i * BATCH + threadIdx.x];
            const float4 s0 = __ldg(g.splat + 2 * (size_t)id), s1 = __ldg(g.splat + 2 * (size_t)id + 1);
            s_id[threadIdx.x] = id;
            s_s0[threadIdx.x] = s0;
            s_s1[threadIdx.x] = s1;
            s_mask[threadIdx.x] = patch_mask(s0, s1, tx0, ty0);
        }
        __syncthreads();
        const int cnt = min(BATCH, (int)m - i * BATCH);
        for (int c = 0; c < ((cnt + 31) >> 5); c++) {
            const int ej = (c << 5) + lane;
            const uint32_t mm = ej < cnt ? s_mask[ej] : 0u;
            uint32_t bits = __ballot_sync(FULL, (mm >> w) & 1u);
            while (bits) {
                const int j = (c << 5) + __ffs(bits) - 1;
                bits &= bits - 1;
                const uint32_t pos = (uint32_t)(i * BATCH + j);
                const float4 s0 = s_s0[j], s1 = s_s1[j];
                const float power = pair_power(s1.x, s1.y, s1.z, s0.x - pxf, s0.y - pyf);
                float alpha, au;
                const bool ok = pos < last && RTG_FWD_PRETEST(power, s0.z) && pair_alpha(power, s1.w, s0.w, alpha, au);
                const uint32_t who = __ballot_sync(FULL, ok);
                if (who == 0u) continue;
                float wt = 0.f;
                if (ok) {
                    wt = alpha * T;
                    T = T * (1.f - alpha);
                }
                float v;
                if constexpr (ERR) {
                    const float we = ok ? wt * e : 0.f;
                    const bool hi = lane & 16;
                    v = (hi ? we : wt) + __shfl_xor_sync(FULL, hi ? wt : we, 16);
                } else {
                    v = wt + __shfl_xor_sync(FULL, wt, 16);
                }
#pragma unroll
                for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
                if (lane == 0) {
                    const int id = s_id[j];
                    atomicAdd(n_pixels + id, __popc(who));
                    atomicAdd(weight + id, v);
                }
                if (ERR && lane == 16) atomicAdd(error + s_id[j], v);
            }
        }
    }
}

void launch_render_contributions(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img,
                                 const int32_t *counters, const float *pixel_error, int32_t *n_pixels, float *weight, float *error,
                                 cudaStream_t s) {
    const int T = vp.tiles_x * vp.tiles_y;
    if (pixel_error)
        render_contrib_kernel<true><<<T, 256, 0, s>>>(vp, g, b, img, counters, pixel_error, n_pixels, weight, error);
    else
        render_contrib_kernel<false><<<T, 256, 0, s>>>(vp, g, b, img, counters, nullptr, n_pixels, weight, nullptr);
}

// ------------------------------------------------------------------ per-Gaussian feature maps
// out[c, p] = sum_g w(p, g) F[g, c] and its transpose dL/dF[g, c] = sum_p w(p, g) G[c, p], with w = alpha T the forward's
// colour weight, replayed as render_contrib_kernel replays it. A CTA renders K channels [c0, c0 + K) of one tile; CTA
// b takes tile active[b / chunks] and chunk b % chunks, so the chunks of a heavy tile start together, early.

// Shared memory of one replay: the staged batch's splat records, ids and patch masks, and the warps' longest prefixes.
struct ReplaySmem {
    float4 s0[BATCH], s1[BATCH];
    int id[BATCH];
    uint32_t mask[BATCH];
    uint32_t wmax[8];
};

// The forward's colour blending of one tile, replayed front to back up to the longest prefix its pixels blended (max
// n_contrib), with the forward's patch masks, pretest and alpha function and the pixel's own n_contrib (`last`; 0 outside
// the image). Every thread of the CTA must call it. stage(slot, id) runs once per staged entry on its staging thread
// (before the batch's barrier); visit(slot, ok, wt) runs for every (warp, entry) the warp's patch mask lets through,
// warp-uniformly, with ok = the pair blends and wt = alpha T (0 when !ok); T then advances bit for bit as in
// render_fwd_kernel. Returns the pixel's final T.
template <typename Stage, typename Visit>
__device__ __forceinline__ float replay_blends(const ViewParams &vp, const GeomState &g, const BinState &b, const int tile,
                                               const uint32_t last, const float pxf, const float pyf, ReplaySmem &sm,
                                               Stage stage, Visit visit) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const uint32_t start = b.tile_offset[tile];
    uint32_t wmax = last;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(FULL, wmax, o));
    if (lane == 0) sm.wmax[w] = wmax;
    __syncthreads();
    uint32_t m = 0;
#pragma unroll
    for (int k = 0; k < 8; k++) m = max(m, sm.wmax[k]);

    const float tx0 = (float)((tile % vp.tiles_x) * RTG_TILE), ty0 = (float)((tile / vp.tiles_x) * RTG_TILE);
    float T = 1.f;
    const int rounds = ((int)m + BATCH - 1) / BATCH;
    for (int i = 0; i < rounds; i++) {
        __syncthreads();  // the previous round has been consumed
        if (i * BATCH + (int)threadIdx.x < (int)m) {
            const int id = (int)b.point_list[start + (size_t)i * BATCH + threadIdx.x];
            const float4 s0 = __ldg(g.splat + 2 * (size_t)id), s1 = __ldg(g.splat + 2 * (size_t)id + 1);
            sm.id[threadIdx.x] = id;
            sm.s0[threadIdx.x] = s0;
            sm.s1[threadIdx.x] = s1;
            sm.mask[threadIdx.x] = patch_mask(s0, s1, tx0, ty0);
            stage((int)threadIdx.x, id);
        }
        __syncthreads();
        const int cnt = min(BATCH, (int)m - i * BATCH);
        for (int c = 0; c < ((cnt + 31) >> 5); c++) {
            const int ej = (c << 5) + lane;
            const uint32_t mm = ej < cnt ? sm.mask[ej] : 0u;
            uint32_t bits = __ballot_sync(FULL, (mm >> w) & 1u);
            while (bits) {
                const int j = (c << 5) + __ffs(bits) - 1;
                bits &= bits - 1;
                const uint32_t pos = (uint32_t)(i * BATCH + j);
                const float4 s0 = sm.s0[j], s1 = sm.s1[j];
                const float power = pair_power(s1.x, s1.y, s1.z, s0.x - pxf, s0.y - pyf);
                float alpha, au;
                const bool ok = pos < last && RTG_FWD_PRETEST(power, s0.z) && pair_alpha(power, s1.w, s0.w, alpha, au);
                float wt = 0.f;
                if (ok) {
                    wt = alpha * T;
                    T = T * (1.f - alpha);
                }
                visit(j, ok, wt);
            }
        }
    }
    return T;
}

// Row stride (floats) of a staged feature chunk: 16-byte rows whose quarter-warp STS.128 fall into distinct banks.
template <int K>
constexpr int feat_stride() { return K == 4 ? 4 : K + 4; }

// Forward: each pixel keeps K accumulators; each staged entry's K features of the chunk sit in shared memory next to its
// splat record (channels >= C staged as 0). Every pixel of the image is written: 0 where the tile is empty, masked out or
// the forward overflowed (no background term: T_map holds the remainder).
template <int K>
__global__ void __launch_bounds__(256) render_feat_fwd_kernel(const ViewParams vp, const GeomState g, const BinState b,
                                                              const ImgState img, const int *__restrict__ counters,
                                                              const int C, const int chunks, const float *__restrict__ F,
                                                              float *__restrict__ out) {
    constexpr int FS = feat_stride<K>();
    __shared__ ReplaySmem sm;
    __shared__ __align__(16) float s_f[BATCH * FS];

    const int tile = (int)b.active[blockIdx.x / chunks];
    const int c0 = (int)(blockIdx.x % chunks) * K;
    const int kc = min(K, C - c0);
    int px, py;
    bool inside;
    pixel_of(vp, tile, px, py, inside);
    const int pix = vp.W * py + px;
    const size_t N = (size_t)vp.H * vp.W;
    float acc[K];
#pragma unroll
    for (int k = 0; k < K; k++) acc[k] = 0.f;
    const int n = counters[2] != 0 ? 0 : (int)b.tile_count[(size_t)tile * RTG_CNT_STRIDE];
    if (n > 0) {  // block-uniform
        const uint32_t last = inside ? img.n_contrib[pix] : 0u;
        auto stage = [&](const int slot, const int id) {
            const float *row = F + (size_t)id * C + c0;
            float v[K];
#pragma unroll
            for (int k = 0; k < K; k++) v[k] = k < kc ? __ldg(row + k) : 0.f;
            float4 *dst = reinterpret_cast<float4 *>(s_f + slot * FS);
#pragma unroll
            for (int q = 0; q < K / 4; q++) dst[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
        };
        auto visit = [&](const int j, const bool ok, const float wt) {
            if (!ok) return;
            const float4 *row = reinterpret_cast<const float4 *>(s_f + j * FS);
#pragma unroll
            for (int q = 0; q < K / 4; q++) {
                const float4 f = row[q];
                acc[4 * q] += wt * f.x;
                acc[4 * q + 1] += wt * f.y;
                acc[4 * q + 2] += wt * f.z;
                acc[4 * q + 3] += wt * f.w;
            }
        };
        replay_blends(vp, g, b, tile, last, (float)px, (float)py, sm, stage, visit);
    }
    if (inside) {
#pragma unroll
        for (int k = 0; k < K; k++)
            if (k < kc) out[(size_t)(c0 + k) * N + pix] = acc[k];
    }
}

template <int K>
constexpr int feat_log2() { return K == 16 ? 4 : (K == 8 ? 3 : 2); }

// Sum K per-lane values (K a power of two, 4..16) across the warp by recursive halving: at the step xor o (o = 16, 8, ...)
// a lane keeps one half of its values, the upper half if lane & o, and adds its partner's copy of that half (K/2, K/4, ...
// shuffles); once one value is left the remaining steps are plain butterfly adds. K - 1 + 5 - log2(K) shuffles in all
// (16 for K = 16, instead of 5 K). Afterwards lane l holds the total of value l >> (5 - log2 K) (feat_slot).
template <int K>
__device__ __forceinline__ float warp_reduce_halving(float v[K], const int lane) {
#pragma unroll
    for (int step = 0; step < feat_log2<K>(); step++) {
        const int h = K >> (step + 1), o = 16 >> step;
        // the halves are swapped with a bit mask, not a select: a select of two array elements becomes a select of their
        // addresses, which puts v in local memory
        const uint32_t hm = (lane & o) ? FULL : 0u;
#pragma unroll
        for (int k = 0; k < h; k++) {
            const uint32_t lo_bits = __float_as_uint(v[k]), hi_bits = __float_as_uint(v[h + k]);
            const float keep = __uint_as_float((hi_bits & hm) | (lo_bits & ~hm));
            const float send = __uint_as_float((lo_bits & hm) | (hi_bits & ~hm));
            v[k] = keep + __shfl_xor_sync(FULL, send, o);
        }
    }
    float s = v[0];
#pragma unroll
    for (int o = 32 / (2 * K); o > 0; o >>= 1) s += __shfl_xor_sync(FULL, s, o);
    return s;
}

// Backward: each pixel holds its K upstream values; per (warp, entry) with at least one blending lane the warp sums w G[c]
// of the K channels with warp_reduce_halving and adds them with one RED per channel, issued together by K lanes (K
// consecutive floats of the row). dL_dF must be zeroed by the caller: rows the frame never blends are left alone.
template <int K>
__global__ void __launch_bounds__(256) render_feat_bwd_kernel(const ViewParams vp, const GeomState g, const BinState b,
                                                              const ImgState img, const int *__restrict__ counters,
                                                              const int C, const int chunks, const float *__restrict__ dL_dout,
                                                              float *__restrict__ dL_dF) {
    __shared__ ReplaySmem sm;

    if (counters[2] != 0) return;  // an overflowed forward rendered nothing
    const int tile = (int)b.active[blockIdx.x / chunks];
    const int n = (int)b.tile_count[(size_t)tile * RTG_CNT_STRIDE];
    if (n == 0) return;            // empty or masked-out tile
    const int c0 = (int)(blockIdx.x % chunks) * K;
    const int kc = min(K, C - c0);
    int px, py;
    bool inside;
    pixel_of(vp, tile, px, py, inside);
    const int pix = vp.W * py + px;
    const size_t N = (size_t)vp.H * vp.W;
    const int lane = threadIdx.x & 31;
    const uint32_t last = inside ? img.n_contrib[pix] : 0u;
    float G[K];
#pragma unroll
    for (int k = 0; k < K; k++) G[k] = (inside && k < kc) ? __ldg(dL_dout + (size_t)(c0 + k) * N + pix) : 0.f;
    constexpr int SH = 5 - feat_log2<K>();
    const int slot = lane >> SH;                                       // the channel this lane holds after the reduction
    const bool writer = (lane & ((1 << SH) - 1)) == 0 && slot < kc;
    auto stage = [](const int, const int) {};
    auto visit = [&](const int j, const bool ok, const float wt) {
        if (__ballot_sync(FULL, ok) == 0u) return;
        float v[K];
#pragma unroll
        for (int k = 0; k < K; k++) v[k] = wt * G[k];  // wt = 0 on lanes that do not blend
        const float s = warp_reduce_halving<K>(v, lane);
        if (writer) atomicAdd(dL_dF + (size_t)sm.id[j] * C + c0 + slot, s);
    };
    replay_blends(vp, g, b, tile, last, (float)px, (float)py, sm, stage, visit);
}

// K channels per CTA: the smallest of 4, 8, 16 that holds C, 16 above that.
template <int K>
static void feat_launch(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img, const int32_t *counters,
                        int C, const float *in, float *out, bool bwd, cudaStream_t s) {
    const int chunks = (C + K - 1) / K;
    const int grid = vp.tiles_x * vp.tiles_y * chunks;
    if (bwd)
        render_feat_bwd_kernel<K><<<grid, 256, 0, s>>>(vp, g, b, img, counters, C, chunks, in, out);
    else
        render_feat_fwd_kernel<K><<<grid, 256, 0, s>>>(vp, g, b, img, counters, C, chunks, in, out);
}

static void feat_dispatch(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img,
                          const int32_t *counters, int C, const float *in, float *out, bool bwd, cudaStream_t s) {
    if (C <= 4) feat_launch<4>(vp, g, b, img, counters, C, in, out, bwd, s);
    else if (C <= 8) feat_launch<8>(vp, g, b, img, counters, C, in, out, bwd, s);
    else feat_launch<16>(vp, g, b, img, counters, C, in, out, bwd, s);
}

// Weight gradient: the feature map differentiated through its blend weights, with F and G = dL/dout held. For a pixel's
// blended entries i (front to back), h_i = sum_c G[c] F[i, c] and S_i = sum_{j > i} w_j h_j,
//   dL/dalpha_i = T_i h_i - S_i / (1 - alpha_i),
// render_bwd_kernel's dL/dalpha with the pair's colour term D replaced by h_i and no background term. u = au dL/dalpha
// feeds the six moments of the gradient record (REC_M0..REC_MYY), from where the per-Gaussian backward takes them to the
// geometry and the camera. The replay runs front to back, so S_i = a - sum_{j <= i} w_j h_j with a = sum_j w_j h_j: a comes
// from a first replay of the same tile in double, and the second replay subtracts the identical terms from it in the
// identical order, in double, so what is left is the suffix sum to double rounding however far it cancels. (The
// float map as a would carry an error of order 1e-7 |out| into every S_i, swamping the true S_i ~ T_i |h| of the entries
// deep in a saturated pixel.) dL/dalpha is linear in h: each K-channel chunk adds its partial moments. Per (warp, entry)
// with a blending lane the six sums go through warp_reduce_halving<8> and out as six REDs into the caller's zeroed record.
// A pixel whose chunk of G is all zero adds nothing and is not replayed.
template <int K>
__global__ void __launch_bounds__(256) render_feat_grad_kernel(const ViewParams vp, const GeomState g, const BinState b,
                                                               const ImgState img, const int *__restrict__ counters,
                                                               const int C, const int chunks, const float *__restrict__ F,
                                                               const float *__restrict__ dL_dout, float *__restrict__ rec) {
    constexpr int FS = feat_stride<K>();
    __shared__ ReplaySmem sm;
    __shared__ __align__(16) float s_f[BATCH * FS];

    if (counters[2] != 0) return;  // an overflowed forward rendered nothing
    const int tile = (int)b.active[blockIdx.x / chunks];
    const int n = (int)b.tile_count[(size_t)tile * RTG_CNT_STRIDE];
    if (n == 0) return;            // empty or masked-out tile
    const int c0 = (int)(blockIdx.x % chunks) * K;
    const int kc = min(K, C - c0);
    int px, py;
    bool inside;
    pixel_of(vp, tile, px, py, inside);
    const int pix = vp.W * py + px;
    const size_t N = (size_t)vp.H * vp.W;
    const int lane = threadIdx.x & 31;
    float G[K];
    bool any = false;
#pragma unroll
    for (int k = 0; k < K; k++) {
        G[k] = (inside && k < kc) ? __ldg(dL_dout + (size_t)(c0 + k) * N + pix) : 0.f;
        any |= G[k] != 0.f;
    }
    const uint32_t last = any ? img.n_contrib[pix] : 0u;
    const float pxf = (float)px, pyf = (float)py;
    auto stage = [&](const int slot, const int id) {
        const float *row = F + (size_t)id * C + c0;
        float v[K];
#pragma unroll
        for (int k = 0; k < K; k++) v[k] = k < kc ? __ldg(row + k) : 0.f;
        float4 *dst = reinterpret_cast<float4 *>(s_f + slot * FS);
#pragma unroll
        for (int q = 0; q < K / 4; q++) dst[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
    };
    auto h_of = [&](const int j) {
        const float4 *row = reinterpret_cast<const float4 *>(s_f + j * FS);
        float h = 0.f;
#pragma unroll
        for (int q = 0; q < K / 4; q++) {
            const float4 f = row[q];
            h = fmaf(G[4 * q], f.x, h);
            h = fmaf(G[4 * q + 1], f.y, h);
            h = fmaf(G[4 * q + 2], f.z, h);
            h = fmaf(G[4 * q + 3], f.w, h);
        }
        return h;
    };
    double a = 0.0;
    replay_blends(vp, g, b, tile, last, pxf, pyf, sm, stage, [&](const int j, const bool ok, const float wt) {
        if (ok) a += (double)wt * (double)h_of(j);
    });

    constexpr int SH = 5 - feat_log2<8>();
    const int slot = lane >> SH;                                   // the moment this lane holds after the reduction
    const bool writer = (lane & ((1 << SH) - 1)) == 0 && slot < 6;
    double rest = a;  // a - sum_{j <= i} w_j h_j = S_i, subtracted term by term in the order a was summed
    float T = 1.f;
    auto visit = [&](const int j, const bool ok, const float wt) {
        if (__ballot_sync(FULL, ok) == 0u) return;
        float v[8];
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = 0.f;
        if (ok) {  // the replay's own decision and weight; its alpha and au are recomputed from the same inputs
            const float4 s0 = sm.s0[j], s1 = sm.s1[j];
            const float dx = s0.x - pxf, dy = s0.y - pyf;
            float alpha, au;
            pair_alpha(pair_power(s1.x, s1.y, s1.z, dx, dy), s1.w, s0.w, alpha, au);
            const float h = h_of(j);
            rest -= (double)wt * (double)h;
            float inv_1ma;  // as in bwd_blend: 1 - alpha is in [0.01, 1], where the bare MUFU.RCP is exact to 1 ulp
            asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv_1ma) : "f"(1.f - alpha));
            const float dL_dalpha = T * h - (float)rest * inv_1ma;
            T = T * (1.f - alpha);
            const float u = au * dL_dalpha;
            const float ux = u * dx, uy = u * dy;
            v[0] = u;
            v[1] = ux;
            v[2] = uy;
            v[3] = ux * dx;
            v[4] = ux * dy;
            v[5] = uy * dy;
        }
        const float s = warp_reduce_halving<8>(v, lane);
        if (writer) atomicAdd(rec + (size_t)sm.id[j] * RTG_REC + REC_M0 + slot, s);
    };
    replay_blends(vp, g, b, tile, last, pxf, pyf, sm, stage, visit);
}

template <int K>
static void feat_grad_launch(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img,
                             const int32_t *counters, int C, const float *features, const float *dL_dout, float *rec,
                             cudaStream_t s) {
    const int chunks = (C + K - 1) / K;
    render_feat_grad_kernel<K><<<vp.tiles_x * vp.tiles_y * chunks, 256, 0, s>>>(vp, g, b, img, counters, C, chunks, features,
                                                                                dL_dout, rec);
}

void launch_render_features_grad(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img,
                                 const int32_t *counters, int C, const float *features, const float *dL_dout, float *rec,
                                 cudaStream_t s) {
    // chunks of at most 8 channels: with 16, ptxas holds the kernel to 80 registers around the staging's division call
    // (patch_mask) and spills
    if (C <= 4) feat_grad_launch<4>(vp, g, b, img, counters, C, features, dL_dout, rec, s);
    else feat_grad_launch<8>(vp, g, b, img, counters, C, features, dL_dout, rec, s);
}

void launch_render_features(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img,
                            const int32_t *counters, int C, const float *features, float *out, cudaStream_t s) {
    feat_dispatch(vp, g, b, img, counters, C, features, out, false, s);
}

void launch_render_features_bwd(const ViewParams &vp, const GeomState &g, const BinState &b, const ImgState &img,
                                const int32_t *counters, int C, const float *dL_dout, float *dL_dfeatures, cudaStream_t s) {
    feat_dispatch(vp, g, b, img, counters, C, dL_dout, dL_dfeatures, true, s);
}

}  // namespace rtg
