// float_key.cuh -- the bounding-box reduction shared by knn.cu and hier_build.cu: order-preserving uint keys of floats
// (every word of a box {~key(min), key(max)} is then reduced with atomicMax from 0) and the warp min / max.
#pragma once
#include <stdint.h>
#include <string.h>

namespace h3dgs {

__host__ __device__ __forceinline__ uint32_t f2key(float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float key2f(uint32_t k) {
    const uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    float f;
    memcpy(&f, &u, 4);
    return f;
}
__device__ __forceinline__ float warp_min(float v) {
    for (int o = 16; o; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

}  // namespace h3dgs
