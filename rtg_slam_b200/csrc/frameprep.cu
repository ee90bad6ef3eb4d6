// Tracker-side preprocessing of an incoming depth frame (SURVEY.md section 8(f) #3): Tracker.map_preprocess,
// SLAM/multiprocess/tracker.py:97-132, i.e. bilateralFilter_torch (SLAM/utils.py:550-589, a Python double loop of up to
// 121 taps, each a handful of eager full-image kernels), the valid-range mask, compute_vertex_map / compute_normal_map
// (SLAM/utils.py:65-122; here: the ICP level builder at pool = 1), compute_confidence_map (SLAM/utils.py:125-138) and the
// invalid-confidence masking of depth / vertex / normal / confidence. Three launches in total, no host sync.
#include "common.cuh"
#include "kernels.h"
#include "prof.h"

namespace rtg {

// One thread per pixel; taps in the reference's order (row offset i outer, column offset j inner, both ascending), so
// the fp32 sums see the same sequence of additions. Zero padding: a padded (or zero) neighbour has weight 0.
__global__ void __launch_bounds__(256) bilateral_range_kernel(const float *__restrict__ depth, const int H, const int W,
                                                              const int filter, const int radius, const float two_sc2,
                                                              const float two_ss2, const float min_depth, const float max_depth,
                                                              float *__restrict__ out) {
    const int x = blockIdx.x * 16 + (threadIdx.x & 15), y = blockIdx.y * 16 + (threadIdx.x >> 4);
    if (x >= W || y >= H) return;
    const float d = depth[(size_t)y * W + x];
    float r = d;
    if (filter) {
        float wsum = 0.f, psum = 0.f;
        const int r2 = radius * radius;
        for (int i = -radius; i <= radius; i++) {
            const int yy = y + i;
            for (int j = -radius; j <= radius; j++) {
                if (i * i + j * j > r2) continue;
                const int xx = x + j;
                const float nb = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? depth[(size_t)yy * W + xx] : 0.f;
                const float sw = -(float)(i * i + j * j) / two_ss2;   // a Python double in the reference, rounded to fp32 there too
                const float diff = d - nb;
                const float cw = -(diff * diff) / two_sc2;
                const float w = (nb != 0.f) ? expf(sw + cw) : 0.f;
                wsum += w;
                psum += w * nb;
            }
        }
        r = (wsum == 0.f) ? 0.f : psum / wsum;
    }
    // tracker.py:112-113
    out[(size_t)y * W + x] = (r > min_depth && r < max_depth) ? r : 0.f;
}

// confidence = |cos(normal, pixel ray)| (utils.py:125-138); invalid = zero normal or low confidence (tracker.py:122-129)
__global__ void __launch_bounds__(256) confidence_mask_kernel(const int H, const int W, const float fx, const float fy, const float cx,
                                                              const float cy, const float thresh, float *__restrict__ depth,
                                                              float *__restrict__ vertex, float *__restrict__ normal,
                                                              float *__restrict__ confidence, uint8_t *__restrict__ invalid) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= H * W) return;
    const int y = idx / W, x = idx - y * W;
    float px = ((float)x - cx) / fx, py = ((float)y - cy) / fy, pz = 1.0f;
    const float mag = sqrtf(px * px + py * py + pz * pz);
    const float inv = 1.0f / (mag + 1e-8f);
    px *= inv; py *= inv; pz *= inv;
    float *n = normal + 3 * (size_t)idx;
    const float nx = n[0], ny = n[1], nz = n[2];
    // F.cosine_similarity(eps = 1e-8): both vectors divided by max(norm, eps) first
    const float nn = fmaxf(sqrtf(nx * nx + ny * ny + nz * nz), 1e-8f), pn = fmaxf(sqrtf(px * px + py * py + pz * pz), 1e-8f);
    const float c = fabsf((nx / nn) * (px / pn) + (ny / nn) * (py / pn) + (nz / nn) * (pz / pn));
    const bool bad = (nx == 0.f && ny == 0.f && nz == 0.f) || (c < thresh);
    if (bad) {
        depth[idx] = 0.f;
        n[0] = 0.f; n[1] = 0.f; n[2] = 0.f;
        float *v = vertex + 3 * (size_t)idx;
        v[0] = 0.f; v[1] = 0.f; v[2] = 0.f;
    }
    confidence[idx] = bad ? 0.f : c;
    if (invalid) invalid[idx] = bad ? 1 : 0;
}

// Level `scale` of a measured frame for coarse-to-fine tracking: coarse pixel (i, j) pools the fine block
// [s i, s i + s) x [s j, s j + s) (a trailing partial row / column is dropped). Colour: the block mean per channel; depth:
// the block mean when every depth is > 0, else 0; render mask: set when every pixel is set. Sums run over the block in row
// order. One thread per coarse pixel; there are never more coarse tiles than coarse pixels, so the first threads also pool
// one tile each: coarse tile (tx, ty) is set when any fine tile of [s tx, s tx + s) x [s ty, s ty + s) (clipped to the fine
// grid) is set -- a coarse 16x16 tile covers exactly those s x s fine tiles.
__global__ void __launch_bounds__(256) frame_downsample_kernel(const float *__restrict__ color, const float *__restrict__ depth,
                                                               const uint8_t *__restrict__ render_mask,
                                                               const int32_t *__restrict__ tile_mask, const int H, const int W,
                                                               const int s, const int channels_last, float *__restrict__ color_out,
                                                               float *__restrict__ depth_out, uint8_t *__restrict__ mask_out,
                                                               int32_t *__restrict__ tile_mask_out) {
    const int Hs = H / s, Ws = W / s;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= Hs * Ws) return;
    const int i = idx % Ws, j = idx / Ws;
    const float n_block = (float)(s * s);
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, d = 0.f;
    bool all_depth = true, all_mask = true;
    for (int dy = 0; dy < s; dy++) {
        const size_t row = (size_t)(s * j + dy) * W + (size_t)s * i;
        for (int dx = 0; dx < s; dx++) {
            const size_t p = row + dx;
            if (channels_last) {
                c0 += color[3 * p]; c1 += color[3 * p + 1]; c2 += color[3 * p + 2];
            } else {
                c0 += color[p]; c1 += color[(size_t)H * W + p]; c2 += color[2 * (size_t)H * W + p];
            }
            const float dv = depth[p];
            all_depth &= dv > 0.f;
            d += dv;
            if (render_mask) all_mask &= render_mask[p] != 0;
        }
    }
    const size_t HWs = (size_t)Hs * Ws;
    color_out[idx] = c0 / n_block;
    color_out[HWs + idx] = c1 / n_block;
    color_out[2 * HWs + idx] = c2 / n_block;
    depth_out[idx] = all_depth ? d / n_block : 0.f;
    if (render_mask) mask_out[idx] = all_mask ? 1 : 0;
    if (tile_mask) {
        const int ftx = (W + RTG_TILE - 1) / RTG_TILE, fty = (H + RTG_TILE - 1) / RTG_TILE;
        const int ctx = (Ws + RTG_TILE - 1) / RTG_TILE, cty = (Hs + RTG_TILE - 1) / RTG_TILE;
        if (idx < ctx * cty) {
            const int tx = idx % ctx, ty = idx / ctx;
            int any = 0;
            for (int y = s * ty; y < min(s * ty + s, fty); y++)
                for (int x = s * tx; x < min(s * tx + s, ftx); x++) any |= tile_mask[(size_t)y * ftx + x] != 0;
            tile_mask_out[idx] = any;
        }
    }
}

void launch_frame_downsample(const float *color, const float *depth, const uint8_t *render_mask, const int32_t *tile_mask, int H,
                             int W, int scale, int channels_last, float *color_out, float *depth_out, uint8_t *mask_out,
                             int32_t *tile_mask_out, cudaStream_t s) {
    const int n = (H / scale) * (W / scale);
    frame_downsample_kernel<<<(n + 255) / 256, 256, 0, s>>>(color, depth, render_mask, tile_mask, H, W, scale, channels_last,
                                                            color_out, depth_out, mask_out, tile_mask_out);
}

void launch_icp_build_level(const float *depth, int H, int W, int pool, float fx, float fy, float cx, float cy, float *vertex,
                            float *normal, void *ws_, cudaStream_t s);  // icp.cu

void launch_frame_preprocess(const float *depth_in, int H, int W, int filter, int radius, float sigma_color, float sigma_space,
                             float min_depth, float max_depth, float fx, float fy, float cx, float cy, float conf_thresh,
                             float *depth_out, float *vertex, float *normal, float *confidence, uint8_t *invalid, void *ws,
                             cudaStream_t s) {
    {
        ProfScope ps(K_ICP_MISC, s);
        dim3 grid((W + 15) / 16, (H + 15) / 16);
        bilateral_range_kernel<<<grid, 256, 0, s>>>(depth_in, H, W, filter, radius, 2.0f * sigma_color * sigma_color,
                                                    2.0f * sigma_space * sigma_space, min_depth, max_depth, depth_out);
    }
    if (!vertex) return;  // filter + range mask only
    launch_icp_build_level(depth_out, H, W, 1, fx, fy, cx, cy, vertex, normal, ws, s);
    {
        ProfScope ps(K_ICP_MISC, s);
        confidence_mask_kernel<<<(H * W + 255) / 256, 256, 0, s>>>(H, W, fx, fy, cx, cy, conf_thresh, depth_out, vertex, normal,
                                                                  confidence, invalid);
    }
}

}  // namespace rtg
