// loss.cu -- fused L1 + SSIM loss, forward and backward (SURVEY.md 8f-2: the step either side of the
// rasterizer in train_post.py:134-142 / train_single.py:101-117).  Semantics = the reference's
// utils/loss_utils.py:17-63 (11x11 Gaussian window, sigma 1.5, zero padding, groups = channels,
// C1 = 0.01^2, C2 = 0.03^2), pinned by golden fixtures generated from that file (tests/golden/loss_*.npz).
//
// The reference runs 5 grouped conv2d (121 taps) + ~20 elementwise kernels forward and their autograd
// backward.  Here: ONE kernel forward (separable 11+11 taps in shared memory, 16x16 output tiles with a
// 5-pixel halo, all five moments at once, SSIM + L1 partial sums, and the three derivative maps the
// backward needs) and ONE kernel backward (the three maps convolved with the same window and combined
// with img / gt per pixel).  The 11 window weights travel as a by-value kernel argument, as in metrics.cu: no
// __constant__ upload, so the first call needs no host synchronisation and may happen inside a CUDA graph capture.
// With mu = G*x etc.:
//   s = A1 A2 / (B1 B2),  A1 = 2 mu1 mu2 + C1, A2 = 2 s12 + C2, B1 = mu1^2 + mu2^2 + C1, B2 = s1 + s2 + C2
//   d(sum s)/d img1 = G*(ds/dmu1) + 2 img1 (G*(ds/dE11)) + img2 (G*(ds/dE12))
//   ds/dmu1 = 2 mu2 (A2 - A1)/(B1 B2) - s (2 mu1/B1 - 2 mu1/B2),  ds/dE11 = -s/B2,  ds/dE12 = 2 A1/(B1 B2)
#include "common.cuh"

namespace h3dgs {

constexpr int kR = 5, kTS = 16, kHalo = kTS + 2 * kR;      // 26
struct LossWindow { float w[11]; };

__device__ __forceinline__ float block_sum_256(float v, float* s_red) {
    v += __shfl_down_sync(0xffffffffu, v, 16); v += __shfl_down_sync(0xffffffffu, v, 8);
    v += __shfl_down_sync(0xffffffffu, v, 4);  v += __shfl_down_sync(0xffffffffu, v, 2);
    v += __shfl_down_sync(0xffffffffu, v, 1);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x < 8) t = s_red[threadIdx.x];
    if (warp == 0) { t += __shfl_down_sync(0xffffffffu, t, 4); t += __shfl_down_sync(0xffffffffu, t, 2); t += __shfl_down_sync(0xffffffffu, t, 1); }
    __syncthreads();
    return t;      // valid in thread 0
}

__global__ void __launch_bounds__(256)
l1_ssim_forward_kernel(int H, int W, const float* __restrict__ img, const float* __restrict__ gt,
                       double* __restrict__ sums, float* __restrict__ maps, size_t map_stride, const LossWindow win)
{
    __shared__ float sa[kHalo][kHalo + 1], sb[kHalo][kHalo + 1];
    __shared__ float hz[5][kHalo][kTS];
    __shared__ float s_red[8];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int bx = blockIdx.x * kTS, by = blockIdx.y * kTS, c = blockIdx.z;
    const size_t plane = (size_t)H * W;
    const float* ia = img + (size_t)c * plane;
    const float* ib = gt + (size_t)c * plane;
    for (int i = tid; i < kHalo * kHalo; i += 256) {
        const int ly = i / kHalo, lx = i - ly * kHalo;
        const int gy = by + ly - kR, gx = bx + lx - kR;
        const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
        sa[ly][lx] = in ? ia[(size_t)gy * W + gx] : 0.f;        // zero padding (conv2d padding=5)
        sb[ly][lx] = in ? ib[(size_t)gy * W + gx] : 0.f;
    }
    __syncthreads();
    for (int i = tid; i < kHalo * kTS; i += 256) {
        const int r = i / kTS, x = i - r * kTS;
        float m1 = 0.f, m2 = 0.f, e11 = 0.f, e22 = 0.f, e12 = 0.f;
#pragma unroll
        for (int k = 0; k < 11; k++) {
            const float w = win.w[k], a = sa[r][x + k], b = sb[r][x + k];
            m1 += w * a; m2 += w * b; e11 += w * a * a; e22 += w * b * b; e12 += w * a * b;
        }
        hz[0][r][x] = m1; hz[1][r][x] = m2; hz[2][r][x] = e11; hz[3][r][x] = e22; hz[4][r][x] = e12;
    }
    __syncthreads();
    float mu1 = 0.f, mu2 = 0.f, e11 = 0.f, e22 = 0.f, e12 = 0.f;
#pragma unroll
    for (int k = 0; k < 11; k++) {
        const float w = win.w[k];
        mu1 += w * hz[0][ty + k][tx]; mu2 += w * hz[1][ty + k][tx];
        e11 += w * hz[2][ty + k][tx]; e22 += w * hz[3][ty + k][tx]; e12 += w * hz[4][ty + k][tx];
    }
    const int px = bx + tx, py = by + ty;
    float ssim_v = 0.f, l1_v = 0.f;
    if (px < W && py < H) {
        const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
        const float s1 = e11 - mu1 * mu1, s2 = e22 - mu2 * mu2, s12 = e12 - mu1 * mu2;
        const float A1 = 2.f * mu1 * mu2 + C1, A2 = 2.f * s12 + C2;
        const float B1 = mu1 * mu1 + mu2 * mu2 + C1, B2 = s1 + s2 + C2;
        const float iB1 = 1.f / B1, iB2 = 1.f / B2;
        const float s = A1 * A2 * iB1 * iB2;
        ssim_v = s;
        l1_v = fabsf(sa[ty + kR][tx + kR] - sb[ty + kR][tx + kR]);
        if (maps) {
            const size_t o = (size_t)c * plane + (size_t)py * W + px;
            maps[o] = 2.f * mu2 * (A2 - A1) * iB1 * iB2 - s * (2.f * mu1 * iB1 - 2.f * mu1 * iB2);   // ds/dmu1
            maps[map_stride + o] = -s * iB2;                                                       // ds/dE11
            maps[2 * map_stride + o] = 2.f * A1 * iB1 * iB2;                                       // ds/dE12
        }
    }
    const float l1_sum = block_sum_256(l1_v, s_red);
    const float ss_sum = block_sum_256(ssim_v, s_red);
    if (tid == 0) { atomicAdd(sums, (double)l1_sum); atomicAdd(sums + 1, (double)ss_sum); }
}

__global__ void __launch_bounds__(256)
l1_ssim_backward_kernel(int H, int W, const float* __restrict__ img, const float* __restrict__ gt,
                        const float* __restrict__ maps, size_t map_stride, const float* __restrict__ coeffs,
                        float* __restrict__ dL_dimg, const LossWindow win)
{
    __shared__ float sm[3][kHalo][kHalo + 1];
    __shared__ float hz[3][kHalo][kTS];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int bx = blockIdx.x * kTS, by = blockIdx.y * kTS, c = blockIdx.z;
    const size_t plane = (size_t)H * W;
    for (int i = tid; i < kHalo * kHalo; i += 256) {
        const int ly = i / kHalo, lx = i - ly * kHalo;
        const int gy = by + ly - kR, gx = bx + lx - kR;
        const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
        const size_t o = (size_t)c * plane + (size_t)gy * W + gx;
        sm[0][ly][lx] = in ? maps[o] : 0.f;
        sm[1][ly][lx] = in ? maps[map_stride + o] : 0.f;
        sm[2][ly][lx] = in ? maps[2 * map_stride + o] : 0.f;
    }
    __syncthreads();
    for (int i = tid; i < kHalo * kTS; i += 256) {
        const int r = i / kTS, x = i - r * kTS;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll
        for (int k = 0; k < 11; k++) {
            const float w = win.w[k];
            a0 += w * sm[0][r][x + k]; a1 += w * sm[1][r][x + k]; a2 += w * sm[2][r][x + k];
        }
        hz[0][r][x] = a0; hz[1][r][x] = a1; hz[2][r][x] = a2;
    }
    __syncthreads();
    float c0 = 0.f, c1 = 0.f, c2 = 0.f;
#pragma unroll
    for (int k = 0; k < 11; k++) {
        const float w = win.w[k];
        c0 += w * hz[0][ty + k][tx]; c1 += w * hz[1][ty + k][tx]; c2 += w * hz[2][ty + k][tx];
    }
    const int px = bx + tx, py = by + ty;
    if (px < W && py < H) {
        const size_t o = (size_t)c * plane + (size_t)py * W + px;
        const float a = img[o], b = gt[o];
        const float sgn = (a > b) ? 1.f : ((a < b) ? -1.f : 0.f);
        dL_dimg[o] = coeffs[0] * sgn + coeffs[1] * (c0 + 2.f * a * c1 + b * c2);
    }
}

static LossWindow make_loss_window() {
    // utils/loss_utils.py:23-25: exp(-(x - 5)^2 / (2 * 1.5^2)), normalised in fp32 (the weights of metrics.cu)
    LossWindow w; float sum = 0.f;
    for (int x = 0; x < 11; x++) { w.w[x] = (float)exp(-(double)((x - 5) * (x - 5)) / (2.0 * 1.5 * 1.5)); sum += w.w[x]; }
    for (int x = 0; x < 11; x++) w.w[x] /= sum;
    return w;
}

}  // namespace h3dgs

using namespace h3dgs;

extern "C" int h3dgs_l1_ssim_forward(int32_t C, int32_t H, int32_t W, const float* img, const float* gt, double* sums,
                                     float* maps, void* stream)
{
    if (C <= 0 || H <= 0 || W <= 0 || !img || !gt || !sums) { set_error("l1_ssim_forward: bad arguments"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    H3_CUDA(cudaMemsetAsync(sums, 0, 2 * sizeof(double), s));
    const dim3 grid((W + kTS - 1) / kTS, (H + kTS - 1) / kTS, C);
    l1_ssim_forward_kernel<<<grid, 256, 0, s>>>(H, W, img, gt, sums, maps, (size_t)C * H * W, make_loss_window());
    H3_LAUNCHED("l1_ssim_forward", 0, s);
    return H3DGS_OK;
}

extern "C" int h3dgs_l1_ssim_backward(int32_t C, int32_t H, int32_t W, const float* img, const float* gt,
                                      const float* maps, const float* coeffs, float* dL_dimg, void* stream)
{
    if (C <= 0 || H <= 0 || W <= 0 || !img || !gt || !maps || !coeffs || !dL_dimg) { set_error("l1_ssim_backward: bad arguments"); return H3DGS_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    const dim3 grid((W + kTS - 1) / kTS, (H + kTS - 1) / kTS, C);
    l1_ssim_backward_kernel<<<grid, 256, 0, s>>>(H, W, img, gt, maps, (size_t)C * H * W, coeffs, dL_dimg, make_loss_window());
    H3_LAUNCHED("l1_ssim_backward", 0, s);
    return H3DGS_OK;
}
