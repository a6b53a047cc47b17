// eval_pixel.cuh -- render_hierarchy.py:82-113's preprocessing of one evaluated pixel, shared by the metrics pass
// (metrics.cu) and the LPIPS input pass (lpips.cu) so that both see the same pair.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace h3dgs {

__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

// The image's channel c at pixel p of a [3,H,W] frame (plane = H*W): exposed when exposure ([3][4]) is given, clamped
// to [0,1].  image.permute(1,2,0) @ E[:3,:3] + E[:3,3]: the matrix acts from the right, out[c] = sum_k img[k] E[k][c] + E[c][3].
// Without an exposure this is also the target's value, clamp(gt, 0, 1).  The alpha mask multiplies the result.
__device__ __forceinline__ float eval_value(const float* __restrict__ img, const float* __restrict__ exposure, size_t plane,
                                            size_t p, int c) {
    float a;
    if (exposure)
        a = img[p] * exposure[c] + img[plane + p] * exposure[4 + c] + img[2 * plane + p] * exposure[8 + c] + exposure[4 * c + 3];
    else
        a = img[(size_t)c * plane + p];
    return clamp01(a);
}

}  // namespace h3dgs
