// Optional per-kernel timing with CUDA events on the launching stream (used by bench.py for the roofline line).
// Off by default; when off a ProfScope costs one branch.
#pragma once
#include <cuda_runtime.h>

namespace rtg {

enum KernelId {
    K_PREPROCESS_FWD = 0, K_TILE_SCAN, K_SCATTER, K_TILE_SORT, K_RENDER_FWD, K_RENDER_BWD, K_PREPROCESS_BWD, K_ADAM,
    K_ICP_BUILD, K_ICP_ITER, K_ICP_MISC, K_BWD_ZERO, K_TSDF_INTEGRATE, K_TSDF_EXTRACT, K_TSDF_RAYCAST, K_COUNT
};

void prof_begin(int id, cudaStream_t s);
void prof_end(int id, cudaStream_t s);

struct ProfScope {
    int id;
    cudaStream_t s;
    ProfScope(int id_, cudaStream_t s_) : id(id_), s(s_) { prof_begin(id, s); }
    ~ProfScope() { prof_end(id, s); }
};

}  // namespace rtg
