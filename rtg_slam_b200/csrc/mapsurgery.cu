// Map surgery on the Gaussian SoA and nearest-neighbour queries (SURVEY.md section 8(f) #4).
//
//  * soa_compact: GaussianPointCloud.delete / remove (SLAM/gaussian_pointcloud.py:195-235) index every attribute tensor
//    with a boolean mask, i.e. eleven nonzero + gather passes and eleven host synchronisations. Here ONE scan of the mask
//    yields the list of kept rows and one gather launch moves every attribute (rows of 1..45 words, coalesced word-wise).
//  * knn: the 3-NN mean squared distance + indices of simple-knn's distCUDA2 (submodules/simple-knn/simple_knn.cu:169-251,
//    used by GaussianPointCloud.update_geometry, gaussian_pointcloud.py:376) and the K-NN of pytorch3d's knn_points as
//    Mapping.temp_points_filter / gaussians_isolated call it (SLAM/multiprocess/mapper.py:812-819,903-910). The reference
//    sorts Morton codes with a device radix sort and prunes 1024-point boxes; here the reference points are counting-sorted
//    into a uniform grid sized on the device from their bounding box (histogram, scan, scatter: no comparison sort, no host
//    round trip) and every query walks cubic shells of cells around its own cell until the K-th best distance is provably
//    final. Exact, like the reference's search; ties between equidistant neighbours may resolve to a different index.
#include "common.cuh"
#include "kernels.h"
#include "prof.h"

namespace rtg {

// ------------------------------------------------------------------ exclusive scan of uint32 (three small launches)
#define SCAN_BLOCK 1024
__global__ void __launch_bounds__(SCAN_BLOCK) scan_block_sums_kernel(const uint32_t *__restrict__ in, uint32_t n, uint32_t *__restrict__ sums) {
    __shared__ uint32_t s_w[32];
    const uint32_t i = blockIdx.x * SCAN_BLOCK + threadIdx.x;
    uint32_t v = i < n ? in[i] : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
        uint32_t t = s_w[threadIdx.x];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (threadIdx.x == 0) sums[blockIdx.x] = t;
    }
}

// inclusive scan of one block's values in shared memory order; returns this thread's exclusive prefix inside the block
__device__ __forceinline__ uint32_t block_exclusive(uint32_t v, uint32_t *s_w, uint32_t &block_total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_w[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        uint32_t t = s_w[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t u = __shfl_up_sync(0xffffffffu, t, o);
            if (lane >= o) t += u;
        }
        s_w[lane] = t;
    }
    __syncthreads();
    block_total = s_w[31];
    const uint32_t before = wid > 0 ? s_w[wid - 1] : 0u;
    __syncthreads();
    return before + incl - v;
}

__global__ void __launch_bounds__(SCAN_BLOCK) scan_sums_kernel(uint32_t *__restrict__ sums, uint32_t nb, uint32_t *__restrict__ total,
                                                               uint32_t *__restrict__ total_host) {
    __shared__ uint32_t s_w[32];
    uint32_t carry = 0;
    for (uint32_t base = 0; base < nb; base += SCAN_BLOCK) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t v = i < nb ? sums[i] : 0u;
        uint32_t bt;
        const uint32_t ex = block_exclusive(v, s_w, bt);
        if (i < nb) sums[i] = carry + ex;
        carry += bt;
    }
    if (threadIdx.x == 0) {
        if (total) *total = carry;
        if (total_host) *total_host = carry;
    }
}

__global__ void __launch_bounds__(SCAN_BLOCK) scan_apply_kernel(const uint32_t *__restrict__ in, uint32_t n, const uint32_t *__restrict__ sums,
                                                                uint32_t *__restrict__ out) {
    __shared__ uint32_t s_w[32];
    const uint32_t i = blockIdx.x * SCAN_BLOCK + threadIdx.x;
    const uint32_t v = i < n ? in[i] : 0u;
    uint32_t bt;
    const uint32_t ex = block_exclusive(v, s_w, bt);
    if (i < n) out[i] = sums[blockIdx.x] + ex;
}

size_t exclusive_scan_sums_words(uint32_t n) { return (n + SCAN_BLOCK - 1) / SCAN_BLOCK; }

// out[i] = sum of in[0..i); sums: scratch of ceil(n / 1024) words; total (device) / total_host (mapped) may be NULL
void exclusive_scan_u32(const uint32_t *in, uint32_t n, uint32_t *out, uint32_t *sums, uint32_t *total, uint32_t *total_host,
                        cudaStream_t s) {
    const uint32_t nb = (n + SCAN_BLOCK - 1) / SCAN_BLOCK;
    scan_block_sums_kernel<<<nb, SCAN_BLOCK, 0, s>>>(in, n, sums);
    scan_sums_kernel<<<1, SCAN_BLOCK, 0, s>>>(sums, nb, total, total_host);
    scan_apply_kernel<<<nb, SCAN_BLOCK, 0, s>>>(in, n, sums, out);
}

// ------------------------------------------------------------------ compaction of the SoA by a keep mask
__global__ void __launch_bounds__(256) mask_to_u32_kernel(const uint8_t *__restrict__ mask, int invert, uint32_t n, uint32_t *__restrict__ flag) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flag[i] = ((mask[i] != 0) != (invert != 0)) ? 1u : 0u;
}

__global__ void __launch_bounds__(256) kept_rows_kernel(const uint32_t *__restrict__ flag, const uint32_t *__restrict__ excl, uint32_t n,
                                                        uint32_t *__restrict__ src_row) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && flag[i]) src_row[excl[i]] = i;
}

struct SoaArrays {
    const uint32_t *in[RTG_SOA_MAX_ARRAYS];
    uint32_t *out[RTG_SOA_MAX_ARRAYS];
    uint32_t words[RTG_SOA_MAX_ARRAYS];
    int n;
};

// blockIdx.y = attribute; thread -> (kept row, word) so that writes are contiguous and reads contiguous inside a row
__global__ void __launch_bounds__(256) soa_gather_kernel(const SoaArrays a, const uint32_t *__restrict__ src_row,
                                                         const uint32_t *__restrict__ n_kept) {
    const int arr = blockIdx.y;
    const uint32_t w = a.words[arr];
    const uint64_t total = (uint64_t)(*n_kept) * w;
    const uint32_t *__restrict__ in = a.in[arr];
    uint32_t *__restrict__ out = a.out[arr];
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t row = (uint32_t)(i / w), word = (uint32_t)(i - (uint64_t)row * w);
        out[i] = in[(size_t)src_row[row] * w + word];
    }
}

size_t soa_compact_ws_bytes(int64_t P) {
    const size_t n = (size_t)P;
    return 3 * align_up(n * 4, 256) + align_up(((n + SCAN_BLOCK - 1) / SCAN_BLOCK) * 4, 256) + 512;
}

void launch_soa_compact(const uint8_t *mask, int invert, int64_t P, int n_arrays, const void *const *in, void *const *out,
                        const int32_t *words_per_row, uint32_t *n_kept, uint32_t *n_kept_host, void *ws, cudaStream_t s) {
    char *p = reinterpret_cast<char *>(ws);
    uint32_t *flag = carve<uint32_t>(p, (size_t)P), *excl = carve<uint32_t>(p, (size_t)P), *src_row = carve<uint32_t>(p, (size_t)P);
    uint32_t *sums = carve<uint32_t>(p, ((size_t)P + SCAN_BLOCK - 1) / SCAN_BLOCK);
    const uint32_t n = (uint32_t)P;
    mask_to_u32_kernel<<<(n + 255) / 256, 256, 0, s>>>(mask, invert, n, flag);
    exclusive_scan_u32(flag, n, excl, sums, n_kept, n_kept_host, s);
    kept_rows_kernel<<<(n + 255) / 256, 256, 0, s>>>(flag, excl, n, src_row);
    SoaArrays a;
    a.n = n_arrays;
    for (int i = 0; i < n_arrays; i++) {
        a.in[i] = reinterpret_cast<const uint32_t *>(in[i]);
        a.out[i] = reinterpret_cast<uint32_t *>(out[i]);
        a.words[i] = (uint32_t)words_per_row[i];
    }
    if (n_arrays > 0) soa_gather_kernel<<<dim3(RTG_NUM_SMS * 4, n_arrays), 256, 0, s>>>(a, src_row, n_kept);
}

// ------------------------------------------------------------------ uniform grid over the reference points
struct KnnGrid {
    float minx, miny, minz, inv_cs, cs;
    int nx, ny, nz, ncell;
};

__device__ __forceinline__ int float_to_ordered_i(float f) {
    const int i = __float_as_int(f);
    return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float ordered_to_float_i(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

__global__ void knn_init_kernel(int *__restrict__ bbox) {
    if (threadIdx.x < 3) bbox[threadIdx.x] = 0x7fffffff;
    else if (threadIdx.x < 6) bbox[threadIdx.x] = (int)0x80000000;
}

__global__ void __launch_bounds__(256) knn_bbox_kernel(const float *__restrict__ pts, uint32_t n, int *__restrict__ bbox) {
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const float v = pts[3 * (size_t)i + c];
            mn[c] = fminf(mn[c], v); mx[c] = fmaxf(mx[c], v);
        }
    }
#pragma unroll
    for (int c = 0; c < 3; c++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[c] = fminf(mn[c], __shfl_xor_sync(0xffffffffu, mn[c], o));
            mx[c] = fmaxf(mx[c], __shfl_xor_sync(0xffffffffu, mx[c], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int c = 0; c < 3; c++) {
            if (mn[c] <= mx[c]) {
                atomicMin(bbox + c, float_to_ordered_i(mn[c]));
                atomicMax(bbox + 3 + c, float_to_ordered_i(mx[c]));
            }
        }
    }
}

// cell size so that the grid has at most `max_cells` cells and about `per_cell` points per cell of the occupied volume
__global__ void knn_grid_kernel(const int *__restrict__ bbox, uint32_t n, int max_cells, float per_cell, KnnGrid *__restrict__ grid) {
    if (threadIdx.x != 0) return;
    float mn[3], ext[3];
    for (int c = 0; c < 3; c++) {
        mn[c] = ordered_to_float_i(bbox[c]);
        ext[c] = fmaxf(ordered_to_float_i(bbox[3 + c]) - mn[c], 0.f);
    }
    const float longest = fmaxf(fmaxf(ext[0], ext[1]), fmaxf(ext[2], 1e-6f));
    const float target = fminf((float)max_cells, fmaxf((float)n / per_cell, 1.f));
    // start from the cube-root rule on the non-degenerate extents, then grow the cell until the grid fits
    float vol = 1.f;
    int dims = 0;
    for (int c = 0; c < 3; c++)
        if (ext[c] > 1e-4f * longest) { vol *= ext[c]; dims++; }
    float cs = dims > 0 ? powf(vol / target, 1.f / (float)dims) : longest;
    cs = fmaxf(cs, longest / 1000.f);
    int nx, ny, nz;
    for (int it = 0; it < 64; it++) {
        nx = (int)(ext[0] / cs) + 1; ny = (int)(ext[1] / cs) + 1; nz = (int)(ext[2] / cs) + 1;
        if ((long long)nx * ny * nz <= (long long)max_cells) break;
        cs *= 1.15f;
    }
    if ((long long)nx * ny * nz > (long long)max_cells) { nx = ny = nz = 1; cs = longest * 1.01f + 1e-6f; }
    grid->minx = mn[0]; grid->miny = mn[1]; grid->minz = mn[2];
    grid->cs = cs; grid->inv_cs = 1.f / cs;
    grid->nx = nx; grid->ny = ny; grid->nz = nz; grid->ncell = nx * ny * nz;
}

__device__ __forceinline__ int3 knn_cell_of(const KnnGrid &g, float x, float y, float z) {
    int cx = (int)floorf((x - g.minx) * g.inv_cs), cy = (int)floorf((y - g.miny) * g.inv_cs), cz = (int)floorf((z - g.minz) * g.inv_cs);
    cx = min(g.nx - 1, max(0, cx)); cy = min(g.ny - 1, max(0, cy)); cz = min(g.nz - 1, max(0, cz));
    return make_int3(cx, cy, cz);
}

__global__ void __launch_bounds__(256) knn_count_kernel(const float *__restrict__ pts, uint32_t n, const KnnGrid *__restrict__ grid,
                                                        uint32_t *__restrict__ cell_count, uint32_t *__restrict__ cell_of) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const KnnGrid g = *grid;
    const int3 c = knn_cell_of(g, pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2]);
    const uint32_t cell = (uint32_t)((c.z * g.ny + c.y) * g.nx + c.x);
    cell_of[i] = cell;
    atomicAdd(cell_count + cell, 1u);
}

__global__ void __launch_bounds__(256) knn_scatter_kernel(const float *__restrict__ pts, uint32_t n, const uint32_t *__restrict__ cell_of,
                                                          const uint32_t *__restrict__ cell_start, uint32_t *__restrict__ cell_fill,
                                                          float4 *__restrict__ sorted) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t cell = cell_of[i];
    const uint32_t pos = cell_start[cell] + atomicAdd(cell_fill + cell, 1u);
    sorted[pos] = make_float4(pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2], __uint_as_float(i));
}

// K best (ascending) squared distances + indices in registers; same insertion as simple_knn.cu:147-167
template <int K>
__device__ __forceinline__ void knn_insert(float dist, uint32_t idx, float (&best)[K], uint32_t (&best_i)[K]) {
#pragma unroll
    for (int j = 0; j < K; j++) {
        if (best[j] > dist) {
            const float t = best[j]; best[j] = dist; dist = t;
            const uint32_t u = best_i[j]; best_i[j] = idx; idx = u;
        }
    }
}

// One thread per query. Shell R = cells at Chebyshev distance exactly R from the query's (clamped) cell. After shells
// 0..R every reference point whose distance to the query is below R * cell_size has been seen (moving a query into the
// bounding box moves it towards every reference point on each axis), so the search stops once best[K-1] <= (R * cs)^2
// or the shells cover the grid. `skip_self`: query i ignores reference point i (distCUDA2 semantics).
template <int K>
__global__ void __launch_bounds__(128) knn_query_kernel(const float *__restrict__ q, uint32_t nq, const KnnGrid *__restrict__ grid,
                                                        const uint32_t *__restrict__ cell_start, const float4 *__restrict__ sorted,
                                                        uint32_t n_ref, int skip_self, float *__restrict__ out_d2,
                                                        int32_t *__restrict__ out_idx, float *__restrict__ out_mean) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    const KnnGrid g = *grid;
    const float qx = q[3 * (size_t)i], qy = q[3 * (size_t)i + 1], qz = q[3 * (size_t)i + 2];
    const int3 c = knn_cell_of(g, qx, qy, qz);
    float best[K];
    uint32_t best_i[K];
#pragma unroll
    for (int j = 0; j < K; j++) { best[j] = 3.402823466e+38f; best_i[j] = 0x7fffffffu; }
    const int Rmax = max(max(c.x, g.nx - 1 - c.x), max(max(c.y, g.ny - 1 - c.y), max(c.z, g.nz - 1 - c.z)));
    for (int R = 0; R <= Rmax; R++) {
        const int z0 = max(0, c.z - R), z1 = min(g.nz - 1, c.z + R);
        const int y0 = max(0, c.y - R), y1 = min(g.ny - 1, c.y + R);
        const int x0 = max(0, c.x - R), x1 = min(g.nx - 1, c.x + R);
        for (int z = z0; z <= z1; z++) {
            const bool fz = (z == c.z - R) || (z == c.z + R);
            for (int y = y0; y <= y1; y++) {
                const bool fy = fz || (y == c.y - R) || (y == c.y + R);
                // on a face in z or y the whole x range belongs to the shell; otherwise only its two end cells
                for (int x = x0; x <= x1; x += (fy ? 1 : max(1, x1 - x0))) {
                    if (!fy && x != c.x - R && x != c.x + R) continue;
                    const uint32_t cell = (uint32_t)((z * g.ny + y) * g.nx + x);
                    const uint32_t b = cell_start[cell], e = cell_start[cell + 1];
                    for (uint32_t k = b; k < e; k++) {
                        const float4 p = __ldg(sorted + k);
                        const uint32_t pid = __float_as_uint(p.w);
                        if (skip_self && pid == i) continue;
                        const float dx = p.x - qx, dy = p.y - qy, dz = p.z - qz;
                        knn_insert<K>(dx * dx + dy * dy + dz * dz, pid, best, best_i);
                    }
                }
            }
        }
        const float reach = (float)R * g.cs;
        if (best[K - 1] <= reach * reach) break;
    }
    if (out_d2) {
#pragma unroll
        for (int j = 0; j < K; j++) out_d2[(size_t)i * K + j] = best[j];
    }
    if (out_idx) {
#pragma unroll
        for (int j = 0; j < K; j++) out_idx[(size_t)i * K + j] = (int32_t)best_i[j];
    }
    if (out_mean) {
        float sacc = 0.f;
#pragma unroll
        for (int j = 0; j < K; j++) sacc += best[j];
        out_mean[i] = sacc / (float)K;  // (best[0] + best[1] + best[2]) / 3.0f for K = 3 (simple_knn.cu:213)
    }
}

__global__ void knn_empty_kernel(uint32_t nq, int K, float *__restrict__ out_d2, int32_t *__restrict__ out_idx, float *__restrict__ out_mean) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    for (int j = 0; j < K; j++) {
        if (out_d2) out_d2[(size_t)i * K + j] = 3.402823466e+38f;
        if (out_idx) out_idx[(size_t)i * K + j] = 0x7fffffff;
    }
    if (out_mean) out_mean[i] = 3.402823466e+38f;
}

static int knn_max_cells(int64_t n_ref) {
    long long c = (long long)n_ref / 2;
    if (c < 4096) c = 4096;
    if (c > (1 << 21)) c = 1 << 21;
    return (int)c;
}

size_t knn_ws_bytes(int64_t n_ref) {
    const size_t n = (size_t)n_ref, nc = (size_t)knn_max_cells(n_ref) + 1;
    return 512 + align_up(n * 4, 256) + 3 * align_up(nc * 4, 256) + align_up(((nc + SCAN_BLOCK - 1) / SCAN_BLOCK) * 4, 256) +
           align_up(n * 16, 256) + 512;
}

int launch_knn(const float *query, int64_t n_query, const float *ref, int64_t n_ref, int K, int skip_self, float *out_d2, int32_t *out_idx,
               float *out_mean, void *ws, cudaStream_t s) {
    if (K < 1 || K > 8) return -1;
    if (n_ref == 0) {
        knn_empty_kernel<<<(unsigned)((n_query + 255) / 256), 256, 0, s>>>((uint32_t)n_query, K, out_d2, out_idx, out_mean);
        return 0;
    }
    char *p = reinterpret_cast<char *>(ws);
    int *bbox = carve<int>(p, 8);
    KnnGrid *grid = carve<KnnGrid>(p, 1);
    const uint32_t n = (uint32_t)n_ref, nq = (uint32_t)n_query;
    const int max_cells = knn_max_cells(n_ref);
    uint32_t *cell_of = carve<uint32_t>(p, n);
    uint32_t *cell_count = carve<uint32_t>(p, (size_t)max_cells + 1);
    uint32_t *cell_start = carve<uint32_t>(p, (size_t)max_cells + 1);
    uint32_t *cell_fill = carve<uint32_t>(p, (size_t)max_cells + 1);
    uint32_t *sums = carve<uint32_t>(p, ((size_t)max_cells + 1 + SCAN_BLOCK - 1) / SCAN_BLOCK);
    float4 *sorted = carve<float4>(p, n);
    cudaMemsetAsync(cell_count, 0, ((size_t)max_cells + 1) * 4, s);
    cudaMemsetAsync(cell_fill, 0, ((size_t)max_cells + 1) * 4, s);
    knn_init_kernel<<<1, 32, 0, s>>>(bbox);
    knn_bbox_kernel<<<RTG_NUM_SMS * 2, 256, 0, s>>>(ref, n, bbox);
    knn_grid_kernel<<<1, 32, 0, s>>>(bbox, n, max_cells, 4.f, grid);
    knn_count_kernel<<<(n + 255) / 256, 256, 0, s>>>(ref, n, grid, cell_count, cell_of);
    exclusive_scan_u32(cell_count, (uint32_t)max_cells + 1, cell_start, sums, nullptr, nullptr, s);
    knn_scatter_kernel<<<(n + 255) / 256, 256, 0, s>>>(ref, n, cell_of, cell_start, cell_fill, sorted);
    const int nb = (int)((nq + 127) / 128);
#define KNN_CASE(KK)                                                                                                      \
    case KK:                                                                                                             \
        knn_query_kernel<KK><<<nb, 128, 0, s>>>(query, nq, grid, cell_start, sorted, n, skip_self, out_d2, out_idx, out_mean); \
        break;
    switch (K) {
        KNN_CASE(1) KNN_CASE(2) KNN_CASE(3) KNN_CASE(4) KNN_CASE(5) KNN_CASE(6) KNN_CASE(7) KNN_CASE(8)
        default: return -1;
    }
#undef KNN_CASE
    return 0;
}

}  // namespace rtg
