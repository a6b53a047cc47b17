// lod_size.cuh -- the size of a hierarchy node's box seen from the viewpoint, the one quantity the LOD cut
// (hierarchy.cu) and the budget's threshold selection (lod_budget.cu) compare against a threshold.  Both files are
// compiled with -fmad=false, so this expression rounds the same way in each, operation by operation.  Also the count
// both take of a node's rows under the view cull's row mask (lod_cull.cu).
#pragma once
#include <float.h>
#include <stdint.h>

namespace h3dgs {

// min.w / distance from the viewpoint to the box, FLT_MAX when the viewpoint is inside (faces included)
__device__ __forceinline__ float box_size(const float4 mn, const float4 mx, float vx, float vy, float vz) {
    const bool inside = vx >= mn.x && vx <= mx.x && vy >= mn.y && vy <= mx.y && vz >= mn.z && vz <= mx.z;
    if (inside) return FLT_MAX;
    const float cx = fmaxf(mn.x, fminf(mx.x, vx)) - vx;
    const float cy = fmaxf(mn.y, fminf(mx.y, vy)) - vy;
    const float cz = fmaxf(mn.z, fminf(mx.z, vz)) - vz;
    const float dist = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(cx, cx), __fmul_rn(cy, cy)), __fmul_rn(cz, cz)));
    return mn.w / dist;
}

// rows of [begin, begin + n) whose mask byte is set (the mask holds 0 or 1)
__device__ __forceinline__ int masked_rows(const uint8_t* __restrict__ mask, int begin, int n) {
    int c = 0;
    for (int q = 0; q < n; q++) c += __ldg(mask + begin + q);
    return c;
}

}  // namespace h3dgs
